/*
 * frcnn_b200.h -- C ABI of libfrcnn_b200.so: the Hopper (sm_90a) Faster R-CNN forward
 * detection path, a from-scratch replacement for the hot path of mitmul/chainer-faster-rcnn.
 *
 * Conventions (differences from the reference's only FFI, models/gpu_nms.hpp:9-10, are deliberate):
 *   * every pointer is a DEVICE pointer unless the name ends in `_host`;
 *   * every call is stream-ordered on `stream` (a cudaStream_t passed as void*), never
 *     synchronises and never allocates: scratch comes from the caller (`ws`, sized by the
 *     matching *_workspace_bytes query);
 *   * every call returns an int status: 0 = FRCNN_OK, negative = error; the message is available
 *     from frcnn_last_error().  (The reference prints CUDA errors and continues,
 *     models/nms_kernel.cu:12-19; this library never does.)
 *   * data-dependent result counts (SURVEY.md Q11) are written to device ints; result buffers have
 *     a fixed capacity and rows past the count are zero-filled.
 *   * the library is re-entrant; the caller owns all buffers.
 *
 * Dense operands are NHWC bf16.  "bf16x3" precision: a tensor is a pair of bf16 planes (hi, lo)
 * with value = hi + lo (16 significant bits); the contraction computes hi*hi + lo*hi + hi*lo
 * with fp32 accumulation in registers.  Passing NULL for the lo planes selects single-pass bf16.
 */
#ifndef FRCNN_B200_H_
#define FRCNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FRCNN_OK 0
#define FRCNN_ERR_ARG (-1)        /* invalid argument / unsupported size */
#define FRCNN_ERR_CUDA (-2)       /* a CUDA runtime / driver call failed */
#define FRCNN_ERR_WORKSPACE (-3)  /* workspace too small */

/* NMS comparison semantics. */
#define FRCNN_NMS_GE_DOUBLE 0 /* suppress if (double)iou_f32 >= thresh  -- models/cpu_nms.pyx:66 (live path) */
#define FRCNN_NMS_GT_FLOAT 1  /* suppress if iou_f32 > (float)thresh     -- models/nms_kernel.cu:71          */

int frcnn_version(void);
const char* frcnn_last_error(void);

/* ---------------------------------------------------------------------------------------------
 * Reference ABI, kept verbatim: models/gpu_nms.hpp:9-10 (`_nms`), bound by models/gpu_nms.pyx:13-14.
 * HOST pointers; boxes row-major [boxes_num, boxes_dim>=4], pre-sorted by descending score;
 * keep_out sized boxes_num; blocking; `>` comparison as models/nms_kernel.cu:71.
 * Unlike the reference, a CUDA failure sets *num_out = -1 (and frcnn_last_error()).
 */
void _nms(int* keep_out, int* num_out, const float* boxes_host, int boxes_num, int boxes_dim,
          float nms_overlap_thresh, int device_id);

/* Host-pointer greedy NMS with models/cpu_nms.pyx:18-69 semantics (internal descending sort with
 * ties -> lower index first, +1 pixel convention, (double)iou >= thresh).  dets_host [n,5].
 * Returns the number kept (>= 0) or a negative status.  Blocking.  device_id < 0: the calling thread's current device
 * (cpu_nms has no device argument); an explicit id is used and the caller's current device restored.  n <= 2048 runs as ONE
 * kernel on mapped pinned memory held per calling thread (no allocation, no cudaMemcpy, no stream synchronise per call);
 * n <= 16384 through the chip-wide pipeline of frcnn_nms. */
int frcnn_cpu_nms_host(const float* dets_host, int n, double thresh, int* keep_out_host, int device_id);
/* Diagnostics (no reference counterpart) of the calling thread's last small-n host NMS call: out8[0..5] = SM clock stamps --
 * kernel entry, rows read from the mapped host block, ranked, diagonal blocks built, greedy chain resolved, keep list
 * written; out8[6] = host ns inside the kernel-launch call, out8[7] = host ns polling the completion flag.  Returns 1 if
 * out8 was filled, 0 if this thread has not made such a call yet. */
int frcnn_host_nms_phase_cycles(long long* out8);
/* Host-side helper (no CUDA call, no reference counterpart) of the in-graph per-class NMS hand-off: forward.py:48-57 builds
 * dets = hstack(boxes[:, 4c:4c+4], prob[:, c]) per class and calls cpu_nms(dets, 0.3); the model call already ran that NMS
 * for every class inside its graph (frcnn_detect).  Returns the class c (1 .. num_classes-1) whose rows of the result
 * block equal `dets` [R,5] BIT FOR BIT (tries `hint` first), or 0 -- then the caller runs frcnn_cpu_nms_host. */
int frcnn_match_class_dets(const float* dets, int R, const float* boxes, int ld_boxes, const float* prob, int ld_prob,
                           int num_classes, int hint);

/* ---------------------------------------------------------------------------------------------
 * Device NMS on UNSORTED dets [n,5] (x1,y1,x2,y2,score): replaces models/cpu_nms.pyx:18-69.
 * keep_out (capacity n) receives original indices in descending-score order, *num_out the count;
 * max_keep > 0 stops after that many survivors (the reference's `keep[:post_nms_top_n]`,
 * models/proposal_layer.py:189-190), <= 0 keeps all.  n <= 16384.
 */
size_t frcnn_nms_workspace_bytes(int n);
int frcnn_nms(const float* dets, int n, double thresh, int mode, int max_keep, int* keep_out, int* num_out,
              void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ProposalLayer.__call__ (models/proposal_layer.py:102-198) fused on device: all-anchor grid
 * (:207-221), bbox_transform_inv + clip_boxes + filter_boxes (models/bbox_transform.py:41-109),
 * fg-score slice (:152-154), descending sort + top pre_nms_top_n (:158-170), greedy NMS
 * (models/cpu_nms.pyx) and top post_nms_top_n (:189-193).
 *
 * cls / bbox element (channel c, pixel p=h*W+w) is read at base[c*chan_stride + p*pix_stride]:
 *   reference layout (1,2A,H,W)/(1,4A,H,W): chan_stride=H*W, pix_stride=1;  NHWC rows of ld floats:
 *   chan_stride=1, pix_stride=ld.
 * cls_is_logits != 0: `cls` holds the 2A RPN logits and the 2A-way channel softmax of
 *   models/region_proposal_network.py:119 (SURVEY.md Q1) is computed here; else `cls` is rpn_cls_prob.
 * anchors: [A,4] float64 (models/generate_anchors.py:47-55 output), device memory.
 * out_rois [post_nms_top_n,4], out_scores [post_nms_top_n], *out_count = R; rows >= R are zero.
 * Optional debug outputs (may be NULL): dbg_sorted_dets [pre_nms_top_n,5] (the dets handed to NMS),
 *   dbg_sorted_anchor_idx [pre_nms_top_n], dbg_num_sorted (int).
 * Limits: pre_nms_top_n <= 16384 (and > 0), A <= 32.
 */
size_t frcnn_proposals_workspace_bytes(int A, int H, int W, int pre_nms_top_n);
int frcnn_proposals(const float* cls, long cls_chan_stride, long cls_pix_stride, int cls_is_logits,
                    const float* bbox, long bbox_chan_stride, long bbox_pix_stride, const double* anchors,
                    int A, int H, int W, int feat_stride, int im_h, int im_w, int min_size,
                    int pre_nms_top_n, int post_nms_top_n, double nms_thresh, float* out_rois,
                    float* out_scores, int* out_count, float* dbg_sorted_dets, int* dbg_sorted_anchor_idx,
                    int* dbg_num_sorted, void* ws, size_t ws_bytes, void* stream);
/* frcnn_proposals over N same-size images in one launch per kernel (five launches for the whole batch).  Image n reads
 * cls + n*cls_image_stride and bbox + n*bbox_image_stride (floats) and writes out_rois + n*rois_image_stride,
 * out_scores + n*scores_image_stride, out_count + n*count_image_stride and the optional debug outputs at their image
 * strides (elements): dense [N][post][4] arrays and result blocks some words apart both fit.  The anchors and the clip
 * bounds (im_h, im_w) are shared by all images.  Each image's scratch is its own slice of `ws`
 * (frcnn_proposals_batch_workspace_bytes = N slices at a 256-byte-aligned stride).  Every image's outputs are
 * bit-identical to frcnn_proposals on that image.  frcnn_debug_sort_clocks records image 0 only.
 * Errors: N outside [1,65535], a NULL required pointer, or (N > 1) an output stride smaller than one image's output
 * (rois: 4*post_nms_top_n, a multiple of 4; scores: post_nms_top_n; count: 1; dbg dets: 5*k, dbg index: k with
 * k = min(pre_nms_top_n, A*H*W)) -> FRCNN_ERR_ARG; a workspace below the query -> FRCNN_ERR_WORKSPACE. */
size_t frcnn_proposals_batch_workspace_bytes(int N, int A, int H, int W, int pre_nms_top_n);
int frcnn_proposals_batch(int N, const float* cls, long cls_chan_stride, long cls_pix_stride, long cls_image_stride,
                          int cls_is_logits, const float* bbox, long bbox_chan_stride, long bbox_pix_stride,
                          long bbox_image_stride, const double* anchors, int A, int H, int W, int feat_stride, int im_h,
                          int im_w, int min_size, int pre_nms_top_n, int post_nms_top_n, double nms_thresh,
                          float* out_rois, long rois_image_stride, float* out_scores, long scores_image_stride,
                          int* out_count, long count_image_stride, float* dbg_sorted_dets, long dbg_dets_image_stride,
                          int* dbg_sorted_anchor_idx, long dbg_idx_image_stride, int* dbg_num_sorted,
                          long dbg_num_image_stride, void* ws, size_t ws_bytes, void* stream);
/* frcnn_proposals_batch over a CANVAS batch: N images of different sizes, each at the top-left of its H x W slot of the
 * feature map.  extents (device, int32 [N][2]): image n's size (height, width) in INPUT pixels; its feature-map extent is
 * ceil(extent / 2^halvings) (4 for VGG16), clamped to [0, H] x [0, W].  Cells outside it propose nothing.  im_info (device,
 * int32 [N][2]): image n's clip bounds (im_h, im_w).  Both are read at run time, so a captured graph serves any mix of
 * sizes.  Image n's rois, scores and count are bit-identical to frcnn_proposals on its own extent-sized map with its own
 * clip bounds.  Other arguments as frcnn_proposals_batch (workspace: frcnn_proposals_batch_workspace_bytes of the canvas);
 * no debug outputs.  Errors: NULL extents / im_info, N outside [1,65535], halvings outside [0,30] -> FRCNN_ERR_ARG. */
int frcnn_proposals_batch_ext(int N, const float* cls, long cls_chan_stride, long cls_pix_stride, long cls_image_stride,
                              int cls_is_logits, const float* bbox, long bbox_chan_stride, long bbox_pix_stride,
                              long bbox_image_stride, const double* anchors, int A, int H, int W, int feat_stride,
                              const int* extents, int halvings, const int* im_info, int min_size, int pre_nms_top_n,
                              int post_nms_top_n, double nms_thresh, float* out_rois, long rois_image_stride, float* out_scores,
                              long scores_image_stride, int* out_count, long count_image_stride, void* ws, size_t ws_bytes,
                              void* stream);

/* ---------------------------------------------------------------------------------------------
 * Dense contraction on Hopper tensor cores (TMA -> smem -> wgmma -> register accumulators -> epilogue):
 * 3x3 stride-1 pad-1 convolution or 1x1 convolution / GEMM over NHWC bf16, fused bias (+ReLU).
 * Replaces L.Convolution2D (models/vgg16.py:39-67, models/region_proposal_network.py:53-57) and
 * L.Linear (models/faster_rcnn.py:33-36; a Linear over R rows is the 1x1 case with H=1, W=R).
 *   x_hi/x_lo : [H,W,Cin] bf16 (x_lo NULL -> single-pass bf16), Cin % 8 == 0
 *   w_hi/w_lo : [ksize*ksize, Cout, Cin] bf16 (tap-major, K-major rows), see frcnn_pack_conv_weights
 *   bias      : [>= round_up(max(Cout, ld_f32), 32)] fp32 (zero padded past Cout)
 *   y_hi/y_lo : [H,W,Cout] bf16 outputs (may be NULL), Cout % 32 == 0 when used
 *   y_f32     : [H*W, ld_f32] fp32 output (may be NULL), ld_f32 % 32 == 0, ld_f32 >= Cout;
 *               padded columns receive 0 (+bias pad)
 *   fuse_pool2x2 : != 0 fuses F.MaxPooling2D(2,2) (ceil mode, models/vgg16.py:43,48,55,62) into the
 *               epilogue: y_hi/y_lo are then [ceil(H/2), ceil(W/2), Cout] and the un-pooled map is never
 *               written (needs relu != 0, bf16 output only)
 *   m_valid   : optional device int: rows (pixels) >= *m_valid are written as zeros (GEMM over a
 *               data-dependent number of RoIs); NULL = all valid.
 */
int frcnn_conv2d(const void* x_hi, const void* x_lo, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                 const float* bias, int Cout, int ksize, int relu, int fuse_pool2x2, void* y_hi, void* y_lo, float* y_f32,
                 int ld_f32, const int* m_valid, void* stream);
/* frcnn_conv2d over a batch of N >= 1 images of one shape in one launch: x [N,H,W,Cin], y [N,H,W,Cout] (pooled:
 * [N,ceil(H/2),ceil(W/2),Cout]), y_f32 [N*H*W, ld_f32].  The input is read through a 4-D tensor map, so each image is
 * zero-padded on its own; the tile shape and N tile are the one-image plan, so every image's output is bit-identical to
 * frcnn_conv2d on that image.  No m_valid. */
int frcnn_conv2d_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                       const float* bias, int Cout, int ksize, int relu, int fuse_pool2x2, void* y_hi, void* y_lo, float* y_f32,
                       int ld_f32, void* stream);
/* frcnn_conv2d_batch over a CANVAS batch: image n sits at the top-left of its H x W slot and is extents[2n] x extents[2n+1]
 * input pixels (device int32 [N][2], read at run time), i.e. ceil(extent / 2^halvings) pixels at this layer's input
 * resolution, clamped to [0, H] x [0, W].  Every output pixel outside that extent (bf16 hi / lo, pooled, fp32) is written
 * as 0 -- the zero padding the next 3x3 convolution then reads, as the one-image launch gets it from the TMA
 * out-of-bounds fill -- so each image's pixels equal frcnn_conv2d on the image alone.  The input outside the extent must be
 * zero (what this entry writes).  extents NULL, N < 1 or halvings outside [0,30] -> FRCNN_ERR_ARG. */
int frcnn_conv2d_batch_ext(const void* x_hi, const void* x_lo, int N, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                           const float* bias, int Cout, int ksize, int relu, int fuse_pool2x2, void* y_hi, void* y_lo,
                           float* y_f32, int ld_f32, const int* extents, int halvings, void* stream);
/* Tuning override for tests / benchmarks: force the N tile (64/128/256) and the pixel tile
 * (tile_h*tile_w == 128); 0 = automatic. Process-wide. */
void frcnn_conv2d_set_tile(int block_n, int tile_h, int tile_w);
/* 0 = automatic (single CTAs, the faster choice measured on an H100), 1 = single CTAs, 2 = CTA pairs where the layer
 * allows it (64-channel K blocks).  A pair is a cluster of 2 CTAs on neighbouring pixel tiles of the same N tile:
 * each loads half of the weight tile and multicasts it to both.  Per calling thread; for tests and A/B timing. */
void frcnn_conv2d_set_cta_group(int cta_group);
/* Host staging for callers that hold HOST arrays (forward.py:88-99 uploads a float32 image and reads the results back):
 * pinned blocks owned by the library and explicit asynchronous copies on the caller's stream.  frcnn_host_alloc returns
 * NULL on failure (see frcnn_last_error). */
void* frcnn_host_alloc(size_t bytes);
int frcnn_host_free(void* p);
int frcnn_memcpy_h2d_async(void* dst_device, const void* src_host, size_t bytes, void* stream);
int frcnn_memcpy_d2h_async(void* dst_host, const void* src_device, size_t bytes, void* stream);
int frcnn_stream_synchronize(void* stream);
/* Upload of a pageable host buffer through a pinned staging block of the same size, 1 MB chunks: the host copy of chunk k
 * overlaps the DMA of chunk k-1 on `stream`.  Returns when the last chunk is enqueued (the staging block is busy until the
 * stream reaches that point). */
int frcnn_upload_pageable(void* dst_device, const void* src_host, void* staging_pinned, size_t bytes, void* stream);
/* Host memcpy (pageable -> pinned staging) on a small pool of sleeping worker threads; dst and src must not overlap. */
int frcnn_host_copy(void* dst, const void* src, size_t bytes);

/* Programmatic dependent launch for the forward-path kernels (per calling thread; default OFF -- it measured no gain on the
 * replayed graph, DESIGN.md 4 -- or the FRCNN_PDL environment variable "0"/"1"): a kernel's CTAs may become resident and run their prologue while the previous kernel of
 * the stream drains; every such kernel waits (griddepcontrol.wait) before it touches global memory.  on < 0 restores the
 * environment default.  Read when a launch is enqueued, i.e. fixed inside a captured graph. */
void frcnn_set_programmatic_launch(int on);

/* Cap on the persistent grid of subsequent frcnn_conv2d launches (0 = all SMs).  With several independent images in
 * flight on different streams, launches that each take a share of the SMs run side by side instead of queueing behind
 * each other's one-CTA-per-SM grids, and a smaller grid quantises a layer's tile count into fuller waves.  The value is baked
 * into a CUDA graph at capture time. */
void frcnn_conv2d_set_max_ctas(int max_ctas);
/* Shared memory (bytes, 0..96 KB) that subsequent frcnn_conv2d launches of the calling thread leave unused on every SM
 * (fewer pipeline stages), so that small kernels of other streams can be resident beside the persistent convolution CTAs.
 * Where fewer than two stages of the planned N tile would fit, a narrower N tile is used.
 * Read at launch time (fixed inside a captured graph). */
void frcnn_conv2d_set_smem_reserve(int bytes);
/* The plan of the calling thread's last frcnn_conv2d / frcnn_conv2d_res / frcnn_conv3x3_c8 / frcnn_gemm_nt_splitk /
 * frcnn_linear GEMM launch (or their _batch forms): copies min(n, 12) ints to out in the order BN, BK, x3, promote (long-K
 * partial sums), CTA group, tile_h, tile_w, pipeline stages, grid (CTAs), tiles (pair-tiles for CTA pairs, all split-K
 * parts and all images of a batch included),
 * split-K parts, splits; all zero when the last call launched nothing.  Returns the number of fields (12). */
int frcnn_conv2d_last_plan(int* out, int n);

/* OIHW fp32 weights (Chainer layout, e.g. trunk/conv1_1/W) -> [kh*kw, Cout, Cin_pad] bf16 hi/lo.
 * For Linear weights (Cout, K) pass kh=kw=1.  `perm_chw_to_hwc` != 0 with (c,h,w) = (pc,ph,pw)
 * additionally permutes the K axis from (c,h,w) order (fc6/W over a (C,7,7) pool, models/faster_rcnn.py:127)
 * to the (h,w,c) order frcnn_roi_pool emits.  w_lo may be NULL. */
int frcnn_pack_conv_weights(const float* w_oihw, int Cout, int Cin, int kh, int kw, int Cin_pad, void* w_hi,
                            void* w_lo, int perm_chw_to_hwc, int pc, int ph, int pw, void* stream);
/* (C,H,W) fp32 image (the reference's input layout, forward.py:45) -> [H,W,C_pad] bf16 hi/lo. */
int frcnn_pack_image(const float* x_chw, int C, int H, int W, int C_pad, void* y_hi, void* y_lo, void* stream);
/* Caller-side preprocessing on the device ("next" row, SURVEY.md 8f rank 4): forward.py:34-45 img_preprocessing.
 * img_hwc: uint8 [h0,w0,3] BGR (what cv.imread returns); out_chw: float32 [3,H,W] =
 * cv.resize(float32(img) - (mean_b,mean_g,mean_r), fx=fy=im_scale, INTER_LINEAR) transposed to CHW -- the tensor
 * forward.py:90-92 uploads.  H, W = round-half-even(h0*im_scale), round-half-even(w0*im_scale) (caller computes,
 * forward.py:38-41).  Uploading the raw uint8 image cuts the H2D bytes 4x or more. */
int frcnn_preprocess_bgr8(const unsigned char* img_hwc, int h0, int w0, double mean_b, double mean_g, double mean_r,
                          double im_scale, int H, int W, float* out_chw, void* stream);

/* First layer as a GEMM: (C<=3,H,W) fp32 image -> [H,W,32] bf16 hi/lo whose 32 "channels" are the pixel's
 * zero-padded 3x3xC neighbourhood (k = (r*3+s)*C + c, zeros for k >= 9C), and the matching weight pack
 * OIHW (Cout,Cin<=3,3,3) -> [1,Cout,32].  conv1_1 (models/vgg16.py:39) is then frcnn_conv2d with ksize = 1,
 * Cin = 32: one 64-byte-row k-block per pixel tile instead of nine 32-byte-row blocks. */
int frcnn_pack_image_im2col3x3(const float* x_chw, int C, int H, int W, void* y_hi, void* y_lo, void* stream);
/* The compact first-layer path (what the whole-graph entry and the engine use): frcnn_pack_image_c8 writes the image as
 * [H][W+2][8] bf16 planes (3 of 8 channels used, one zero pixel left and right of every row; frcnn_image_c8_elems elements
 * per plane incl. a few zeroed slack pixels), source element (c,h,w) = x[c*stride_c + h*stride_h + w*stride_w];
 * frcnn_pack_conv_weights_c8 packs OIHW (Cout, Cin<=3, 3, 3) as [3][Cout][32]; frcnn_conv3x3_c8 is conv1_1
 * (models/vgg16.py:39-40: 3x3, pad 1, + bias, ReLU) as a K = 3 x 32 GEMM whose A operand is read through a sliding-window
 * tensor map (pixel stride 16 B, 64-byte rows): the 4x larger im2col copy of frcnn_pack_image_im2col3x3 is never written. */
size_t frcnn_image_c8_elems(int H, int W);
int frcnn_pack_image_c8(const float* x, int C, int H, int W, long stride_c, long stride_h, long stride_w, void* y_hi, void* y_lo,
                        void* stream);
int frcnn_pack_conv_weights_c8(const float* w_oihw, int Cout, int Cin, void* w_hi, void* w_lo, void* stream);
int frcnn_conv3x3_c8(const void* x_hi, const void* x_lo, int H, int W, const void* w_hi, const void* w_lo, const float* bias,
                     int Cout, int relu, void* y_hi, void* y_lo, void* stream);
/* The same for a batch of N images of one shape: image n's source is x + n*stride_n, its compact planes start
 * n * frcnn_image_c8_elems(H, W) elements into y_hi / y_lo, and frcnn_conv3x3_c8_batch writes y [N,H,W,Cout], each image
 * bit-identical to frcnn_conv3x3_c8 on it. */
int frcnn_pack_image_c8_batch(const float* x, int N, int C, int H, int W, long stride_n, long stride_c, long stride_h,
                              long stride_w, void* y_hi, void* y_lo, void* stream);
int frcnn_conv3x3_c8_batch(const void* x_hi, const void* x_lo, int N, int H, int W, const void* w_hi, const void* w_lo,
                           const float* bias, int Cout, int relu, void* y_hi, void* y_lo, void* stream);
/* The same over a CANVAS batch of N H x W slots, image n of extents[2n] x extents[2n+1] pixels at the top-left of its slot
 * (device int32 [N][2], clamped to [0, H] x [0, W]).  frcnn_pack_image_c8_batch_ext reads only the image's own pixels and
 * writes zeros everywhere else in its plane; frcnn_conv3x3_c8_batch_ext writes 0 at every output pixel outside the extent
 * (frcnn_conv2d_batch_ext with halvings 0).  NULL extents -> FRCNN_ERR_ARG. */
int frcnn_pack_image_c8_batch_ext(const float* x, int N, int C, int H, int W, long stride_n, long stride_c, long stride_h,
                                  long stride_w, const int* extents, void* y_hi, void* y_lo, void* stream);
int frcnn_conv3x3_c8_batch_ext(const void* x_hi, const void* x_lo, int N, int H, int W, const void* w_hi, const void* w_lo,
                               const float* bias, int Cout, int relu, const int* extents, void* y_hi, void* y_lo, void* stream);
/* Raw photos into a canvas batch in ONE launch: frcnn_preprocess_bgr8 + frcnn_pack_image_c8_batch_ext for all N slots,
 * without the float32 image in between.  Image n is the dense uint8 [h0,w0,3] BGR block at arena + src_off[n]; the planes
 * y_hi / y_lo (frcnn_image_c8_elems(Hc, Wc) elements per slot, y_lo may be NULL) receive, inside the image's resized extent,
 * bit for bit what frcnn_preprocess_bgr8 followed by the pack writes, and 0 at every other stored pixel (pad columns and
 * slack included).  Everything per image is DEVICE memory read when the kernel runs, so a launch captured in a CUDA graph
 * serves any mix of sizes:
 *   src_off   int64  [N]     byte offset of the image inside the arena
 *   src_hw    int32  [N][2]  (h0, w0); a component <= 0 marks an empty slot
 *   inv_scale double [N]     1.0 / im_scale, divided on the host in double as frcnn_preprocess_bgr8 does
 *   extents   int32  [N][2]  the resized (H, W), the array the other *_batch_ext entries read, clamped to the canvas
 * A slot whose source does not lie inside [0, arena_bytes) (negative offset, offset + 3*h0*w0 > arena_bytes in 64-bit
 * arithmetic) is treated as empty, and a clamped extent only shrinks what is written: no value of these arrays moves an
 * access outside the arena or the planes.  NULL pointers, N outside 1..65535 or a non-positive canvas -> FRCNN_ERR_ARG. */
int frcnn_preprocess_bgr8_canvas(const unsigned char* arena, long long arena_bytes, const long long* src_off, const int* src_hw,
                                 const double* inv_scale, const int* extents, int N, int Hc, int Wc, double mean_b,
                                 double mean_g, double mean_r, void* y_hi, void* y_lo, void* stream);

/* Same with an explicit source layout: element (c, h, w) is x[c*stride_c + h*stride_h + w*stride_w] (in floats).
 * (H*W, W, 1) = dense (C,H,W); (1, W*C, C) = dense (H,W,C) memory, which is what forward.py:45's
 * `img.transpose([2, 0, 1]).astype(np.float32)` hands to the model (astype keeps the transposed strides). */
int frcnn_pack_image_im2col3x3_strided(const float* x, int C, int H, int W, long stride_c, long stride_h, long stride_w,
                                       void* y_hi, void* y_lo, void* stream);
int frcnn_pack_conv_weights_im2col3x3(const float* w_oihw, int Cout, int Cin, void* w_hi, void* w_lo, void* stream);
/* [H,W,C] bf16 hi(/lo) -> (C,H,W) fp32 (the reference's feature-map layout); for inspection/tests. */
int frcnn_unpack_nhwc(const void* x_hi, const void* x_lo, int H, int W, int C, float* y_chw, void* stream);

/* F.MaxPooling2D(2,2), Chainer cover_all=True == ceil mode (models/vgg16.py:43,48,55,62; SURVEY Q8).
 * [H,W,C] -> [ceil(H/2),ceil(W/2),C], C % 8 == 0. */
int frcnn_maxpool2x2_ceil(const void* x_hi, const void* x_lo, int H, int W, int C, void* y_hi, void* y_lo,
                          void* stream);
/* The same over a batch in one launch: [N,H,W,C] -> [N,ceil(H/2),ceil(W/2),C], 1 <= N <= 65535. */
int frcnn_maxpool2x2_ceil_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int C, void* y_hi, void* y_lo,
                                void* stream);

/* F.roi_pooling_2d(feature_map, [0|rois], outh, outw, scale) (models/faster_rcnn.py:123-126), Caffe
 * semantics.  feat [H,W,C] bf16 hi(/lo); rois [R_cap,4] fp32; *count valid rows (NULL = R_cap).
 * out_hi/out_lo: [R_cap, outh*outw, C] bf16 (row = one RoI, K order (ph,pw,c)); rows >= count are 0.
 * out_f32 (optional): same layout in fp32.  outh, outw < 32; C a multiple of 8. */
int frcnn_roi_pool(const void* feat_hi, const void* feat_lo, int H, int W, int C, const float* rois,
                   const int* count, int R_cap, int outh, int outw, float scale, void* out_hi, void* out_lo,
                   float* out_f32, void* stream);
/* frcnn_roi_pool over N images in one launch: feat [N,H,W,C]; image n's RoIs at rois + n*rois_stride (floats, a multiple
 * of 4), its count at counts[n*count_stride] (counts NULL = R_cap each), its output rows at n*out_stride elements into
 * out_hi / out_lo / out_f32 (out_stride >= R_cap*outh*outw*C and a multiple of 8 when N > 1).  Each image's rows are
 * bit-identical to frcnn_roi_pool on it. */
int frcnn_roi_pool_batch(const void* feat_hi, const void* feat_lo, int N, int H, int W, int C, const float* rois,
                         long rois_stride, const int* counts, long count_stride, int R_cap, int outh, int outw, float scale,
                         void* out_hi, void* out_lo, float* out_f32, long out_stride, void* stream);
/* frcnn_roi_pool_batch over a CANVAS batch: image n's map is the top-left ceil(extent / 2^halvings) pixels of its H x W slot
 * (extents: device int32 [N][2] in input pixels, clamped to [0, H] x [0, W]), and its bins are clamped to that map, not to
 * the slot.  Each image's rows are bit-identical to frcnn_roi_pool on its own map.  NULL extents, halvings outside [0,30]
 * -> FRCNN_ERR_ARG. */
int frcnn_roi_pool_batch_ext(const void* feat_hi, const void* feat_lo, int N, int H, int W, int C, const float* rois,
                             long rois_stride, const int* counts, long count_stride, int R_cap, int outh, int outw, float scale,
                             const int* extents, int halvings, void* out_hi, void* out_lo, float* out_f32, long out_stride,
                             void* stream);

/* L.Linear (+ F.relu) for a small number of rows: fc6 / fc7 / cls_score|bbox_pred over the R <= post_nms_top_n RoIs
 * (models/faster_rcnn.py:33-36,127-134).  y[r, c] = act(sum_k x[r,k] * w[c,k] + bias[c]) for r < R_cap, c < Cout.
 * Operands swapped on the tensor cores (weight rows = the M side, RoIs = the N side) and K split over the SMs; the
 * fp32 partial slabs live in `workspace` (frcnn_linear_workspace_bytes) and are summed in fixed order (deterministic).
 *   x_hi/x_lo [R_cap, K] bf16 planes (x_lo NULL = single-pass bf16), K % 64 == 0; w_hi/w_lo [Cout, K] as
 *   frcnn_pack_conv_weights produces them (taps = 1); bias [Cout] fp32; m_valid (optional, device): rows >= *m_valid are 0.
 *   y_hi/y_lo [R_cap, Cout] bf16 planes and/or y_f32 [R_cap, ld_f32] fp32 (columns [Cout, ld_f32) are written as 0). */
size_t frcnn_linear_workspace_bytes(int R_cap, int K, int Cout);
int frcnn_linear(const void* x_hi, const void* x_lo, int R_cap, int K, const void* w_hi, const void* w_lo,
                 const float* bias, int Cout, int relu, const int* m_valid, void* y_hi, void* y_lo, float* y_f32,
                 int ld_f32, void* workspace, size_t workspace_bytes, void* stream);
/* frcnn_linear over the RoIs of N images in one GEMM.  Every image owns a segment of ld1 = round_up(R_cap, 32) rows:
 * x [N][ld1][K] (rows past R_cap should be zero; they only reach their own, discarded, output rows), y_hi/y_lo
 * [N][ld1][Cout] and y_f32 [N][ld1][ld_f32], rows >= image n's count written as 0.  counts (optional, device): image n
 * has min(counts[n * count_stride], R_cap) RoIs.  The N tile, split count and partial-sum promotion are those
 * frcnn_linear picks for one image, so each image's rows are bit-identical to frcnn_linear on that image. */
size_t frcnn_linear_batch_workspace_bytes(int N, int R_cap, int K, int Cout);
int frcnn_linear_batch(const void* x_hi, const void* x_lo, int N, int R_cap, int K, const void* w_hi, const void* w_lo,
                       const float* bias, int Cout, int relu, const int* counts, int count_stride, void* y_hi, void* y_lo,
                       float* y_f32, int ld_f32, void* workspace, size_t workspace_bytes, void* stream);

/* Head tail (models/faster_rcnn.py:175-178): softmax over num_classes scores + per-class
 * bbox_transform_inv + clip_boxes.  scores element (r,c) at scores[r*ld + c], deltas (r,j) at
 * deltas[r*ld + j] (same ld).  out_prob [R_cap,num_classes], out_boxes [R_cap,4*num_classes];
 * rows >= *count are zero. */
int frcnn_head_decode(const float* scores, const float* deltas, int ld, const float* rois, const int* count,
                      int R_cap, int num_classes, int im_h, int im_w, float* out_prob, float* out_boxes,
                      void* stream);
/* frcnn_head_decode over N images in one launch.  Image n: scores / deltas rows at n*in_stride floats on, rois at
 * n*rois_stride (a multiple of 4), count at counts[n*count_stride] (NULL = R_cap), out_prob at n*prob_stride
 * (>= R_cap*num_classes), out_boxes at n*boxes_stride (>= 4*R_cap*num_classes, a multiple of 4).  One clip bound for all.
 * Each image's outputs are bit-identical to frcnn_head_decode on it. */
int frcnn_head_decode_batch(int N, const float* scores, const float* deltas, int ld, long in_stride, const float* rois,
                            long rois_stride, const int* counts, long count_stride, int R_cap, int num_classes, int im_h,
                            int im_w, float* out_prob, long prob_stride, float* out_boxes, long boxes_stride, void* stream);
/* frcnn_head_decode_batch with a clip bound per image: im_info (device int32 [N][2]) holds image n's (im_h, im_w), read at
 * run time.  NULL im_info -> FRCNN_ERR_ARG. */
int frcnn_head_decode_batch_ext(int N, const float* scores, const float* deltas, int ld, long in_stride, const float* rois,
                                long rois_stride, const int* counts, long count_stride, int R_cap, int num_classes,
                                const int* im_info, float* out_prob, long prob_stride, float* out_boxes, long boxes_stride,
                                void* stream);

/* Stand-alone box algebra, the array-level helpers of models/bbox_transform.py:
 *   out[n, 4k..4k+3] = bbox_transform_inv(boxes[n], trans[n, 4k..4k+3])   (:41-76), k < K
 *   clip != 0 additionally applies clip_boxes(out, (im_h, im_w))          (:79-99)
 *   ok_flags (optional, K == 1): 1 where both sides >= min_size           (filter_boxes, :102-109)
 * boxes [N,4], trans [N,4K], out [N,4K] fp32; bit-identical to the fused kernels.
 * trans == NULL: `boxes` is [N,4K] and only the clip / filter steps are applied. */
int frcnn_bbox_decode(const float* boxes, const float* trans, int N, int K, int clip, int im_h, int im_w,
                      int min_size, float* out, unsigned char* ok_flags, void* stream);

/* Per-class detection (forward.py:48-57): for cls 1..num_classes-1 greedy NMS (cpu_nms semantics,
 * thresh) over (boxes[:,4c:4c+4], prob[:,c]), then score >= conf.
 * keep_idx [num_classes-1, R_cap] (RoI indices, descending score), keep_count [num_classes-1] =
 * survivors of the NMS, conf_count [num_classes-1] = how many of those (a prefix) have score >= conf.
 * R_cap <= 2048. */
int frcnn_detect(const float* prob, const float* boxes, const int* count, int R_cap, int num_classes,
                 double nms_thresh, float conf, int* keep_idx, int* keep_count, int* conf_count, void* stream);
/* frcnn_detect over N images in one launch (grid: num_classes-1 CTAs per image).  Image n reads prob / boxes at
 * n*prob_stride / n*boxes_stride floats on (boxes: a multiple of 4) and its count at counts[n*count_stride] (NULL = R_cap),
 * and writes keep_idx, keep_count, conf_count at their image strides (>= (num_classes-1)*R_cap, num_classes-1,
 * num_classes-1 when N > 1).  Each image's outputs are bit-identical to frcnn_detect on it. */
int frcnn_detect_batch(int N, const float* prob, long prob_stride, const float* boxes, long boxes_stride, const int* counts,
                       long count_stride, int R_cap, int num_classes, double nms_thresh, float conf, int* keep_idx,
                       long keep_idx_stride, int* keep_count, long keep_count_stride, int* conf_count,
                       long conf_count_stride, void* stream);
/* The detection list forward.py:50-59 draws, on the device (one CTA per image): for class c = 1 .. num_classes-1 in order and
 * the first conf_count[c-1] entries r of its keep_idx row (frcnn_detect_batch's outputs, read at their image strides, as are
 * prob and boxes), the row out_dets = (c, x1, y1, x2, y2) int32 and out_scores = prob[r][c].  Each coordinate is
 * `int(boxes[r][4c+j] / im_scale[n])` as NumPy >= 2 computes it: the float32 quotient by (float)im_scale[n], truncated toward
 * zero.  Where Python's int() would raise or leave the int32 range, the quotient converts as cvt.rzi.s32.f32 does: NaN -> 0,
 * saturation to [INT32_MIN, INT32_MAX].  Image n's list is at out_dets + n*cap*5 / out_scores + n*cap, cap =
 * (num_classes-1) * R_cap (enough for every list), its length at out_det_count[n]; rows past it are NOT written.  conf_count
 * is clamped to [0, R_cap]; a keep_idx entry outside [0, R_cap) gives the row (c, 0, 0, 0, 0), score 0, and reads nothing.
 * NULL pointers, N outside [1,65535], R_cap < 1, num_classes < 2 or a negative stride -> FRCNN_ERR_ARG. */
int frcnn_detection_lists_batch(int N, const float* prob, long prob_stride, const float* boxes, long boxes_stride,
                                const int* keep_idx, long keep_idx_stride, const int* conf_count, long conf_count_stride,
                                const double* im_scale, int R_cap, int num_classes, int* out_dets, float* out_scores,
                                int* out_det_count, void* stream);

/* PASCAL VOC detection metric on the device (voc_eval.cu): per-class average precision over a dataset of images, from
 * frcnn_detect_batch's keep lists, appended batch by batch into a workspace and evaluated against the ground truth in one
 * static launch sequence.  Neither entry synchronises or allocates.
 *
 * The workspace (frcnn_voc_eval_workspace_bytes; 0 on bad sizes) holds the dataset's detections, at most `capacity` of them
 * over all classes, and the evaluation's scratch; it must be zeroed (cudaMemsetAsync) before the first append of a dataset,
 * and each image index appended once.  Its first bytes are the curves of the last frcnn_voc_eval: int32 tp_cum[capacity] at
 * byte 0 and fp_cum[capacity] at byte align256(4 * capacity), class c's n_det[c] points in rank order starting at the sum of
 * n_det over the classes before it.  capacity in [1, 2^30]; num_classes in [2, 65536]. */
size_t frcnn_voc_eval_workspace_bytes(int num_classes, int capacity, int max_images, int max_gt);
/* Appends images image_base .. image_base+N-1 of the dataset: for class c = 1 .. num_classes-1 the first conf_count[c-1] entries
 * r of its keep_idx row, score prob[r][c] and box boxes[r][4c..4c+3] / (float)im_scale[n] as a float32 quotient (the division
 * of frcnn_detection_lists_batch without its truncation).  Inputs and strides as frcnn_detection_lists_batch; im_scale: device
 * double [N], this batch's scales.  conf_count is clamped to [0, R_cap]; a keep_idx entry outside [0, R_cap) appends a zero box
 * of score 0.  A detection counter keeps counting past `capacity`, but nothing is written past it (frcnn_voc_eval then reports
 * the overflow).  NULL pointers, N outside [1,65535], R_cap < 1, bad sizes, a negative stride or image_base + N > max_images
 * -> FRCNN_ERR_ARG; a workspace below frcnn_voc_eval_workspace_bytes(num_classes, capacity, max_images, 0) ->
 * FRCNN_ERR_WORKSPACE. */
int frcnn_voc_eval_append_batch(int N, const float* prob, long prob_stride, const float* boxes, long boxes_stride,
                                const int* keep_idx, long keep_idx_stride, const int* conf_count, long conf_count_stride,
                                const double* im_scale, int R_cap, int num_classes, int image_base, int capacity, int max_images,
                                void* ws, size_t ws_bytes, void* stream);
/* The VOC devkit's metric over the appended detections.  Ground truth as a device CSR over n_images images: gt_offsets int32
 * [n_images+1], image n's boxes rows [gt_offsets[n], gt_offsets[n+1]) of gt_boxes float32 [n_gt][4] (x1, y1, x2, y2 in
 * source-photo coordinates), gt_labels int32 [n_gt] (1 .. num_classes-1), gt_difficult uint8 [n_gt].  Per class, the
 * detections in rank order (score descending in the score order of DESIGN §2, then image, then keep-list position) are
 * matched greedily per image: float64 +1 IoU with every GT box of the class (difficult included), the first maximum; above
 * iou_thresh (strictly) a difficult GT ignores the detection, an unclaimed GT makes it a TP and is claimed, a claimed GT makes
 * it an FP; otherwise (a NaN overlap included) it is an FP.  AP: the VOC07 11-point and the area (VOC2010+) variants.
 * out: device double [3 + 6*(num_classes-1)]: out[0] the status (0, or 1: more than `capacity` detections were appended, and
 * nothing else is meaningful), out[1] mAP07, out[2] mAP (means over the classes with npos > 0, NaN if none), then per class
 * c = 1 .. num_classes-1 at out[3 + 6*(c-1)]: npos (non-difficult GT), n_det, tp, fp, ap07, ap (NaN when npos == 0).  Counts
 * are exact in a double.  The evaluation leaves the appended detections as they are (it may be repeated).  NULL pointers,
 * bad sizes, n_images outside [0, max_images], n_gt outside [0, max_gt] or a non-finite iou_thresh -> FRCNN_ERR_ARG; a short
 * workspace -> FRCNN_ERR_WORKSPACE. */
int frcnn_voc_eval(int num_classes, int capacity, int max_images, int max_gt, int n_images, const int* gt_offsets,
                   const float* gt_boxes, const int* gt_labels, const unsigned char* gt_difficult, int n_gt, double iou_thresh,
                   double* out, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The whole forward path behind one call (forward_graph.cu): FasterRCNN.__call__, inference branch
 * (models/faster_rcnn.py:92-134,175-178) with the VGG16 trunk -- host orchestration only: it carves the caller's
 * workspace and enqueues, on `stream`, the same kernels in the same order as the entry points above (static launch
 * sequence: capturable into a CUDA graph).  No allocation, no synchronisation.
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
    int H, W;                               /* image size (the trunk needs H, W >= 16) */
    int num_classes, n_anchors, feat_stride; /* 21, 9, 16 */
    int pre_nms_top_n, post_nms_top_n, min_size; /* ProposalLayer limits (models/proposal_layer.py:51-56) */
    double nms_thresh;                       /* RPN_NMS_THRESH 0.7 */
    int x3;                                  /* 1: bf16 hi+lo planes ("bf16x3"), 0: hi planes only */
} frcnn_forward_config;

typedef struct {                             /* one layer as frcnn_pack_conv_weights* / a padded fp32 bias produce it */
    const void* hi; const void* lo; const float* bias;
} frcnn_packed_layer;

typedef struct {
    frcnn_packed_layer conv[13];             /* conv1_1 (frcnn_pack_conv_weights_c8) ... conv5_3 */
    frcnn_packed_layer rpn3;                 /* RPN/rpn_conv_3x3 */
    frcnn_packed_layer rpn_heads;            /* rpn_cls_score | rpn_bbox_pred rows concatenated: [1, 6A, 512] */
    frcnn_packed_layer fc6;                  /* K axis permuted (c,h,w) -> (h,w,c) (perm_chw_to_hwc) */
    frcnn_packed_layer fc7;
    frcnn_packed_layer head;                 /* cls_score | bbox_pred rows concatenated: [1, 5*num_classes, 4096] */
    const double* anchors;                   /* [n_anchors, 4] float64 (generate_anchors) */
} frcnn_vgg16_weights;

size_t frcnn_forward_workspace_bytes(const frcnn_forward_config* config);      /* 0 on a bad config (see frcnn_last_error) */
/* image_chw: (3,H,W) float32 device image (mean-subtracted, as forward.py:45 builds it); im_h/im_w: the clip bounds the
 * caller passes as img_info (forward.py:93 passes (H, H), Q7).  Outputs (device): out_prob [post_nms_top_n, num_classes]
 * softmax, out_boxes [post_nms_top_n, 4*num_classes] decoded + clipped, *out_count valid rows (rows past it are zero). */
int frcnn_forward_vgg16(const frcnn_forward_config* config, const frcnn_vgg16_weights* weights, const float* image_chw,
                        int im_h, int im_w, void* workspace, size_t workspace_bytes, float* out_prob, float* out_boxes,
                        int* out_count, void* stream);
/* The same forward path over N images of config->H x config->W in one call: every stage is one launch sequence for the
 * whole batch (frcnn_forward_vgg16 is the case N = 1).  images_nchw: (N,3,H,W) float32 device images; one clip bound
 * (im_h, im_w) for all.  Outputs: out_prob [N][post_nms_top_n][num_classes], out_boxes [N][post_nms_top_n][4*num_classes],
 * out_count [N].  Image n's outputs are bit-identical to frcnn_forward_vgg16 on image n.  N outside [1,65535] ->
 * FRCNN_ERR_ARG (and frcnn_forward_batch_workspace_bytes returns 0); a workspace below
 * frcnn_forward_batch_workspace_bytes(config, N) -> FRCNN_ERR_WORKSPACE.  Static launch sequence: capturable. */
size_t frcnn_forward_batch_workspace_bytes(const frcnn_forward_config* config, int N);
int frcnn_forward_vgg16_batch(const frcnn_forward_config* config, const frcnn_vgg16_weights* weights, int N,
                              const float* images_nchw, int im_h, int im_w, void* workspace, size_t workspace_bytes,
                              float* out_prob, float* out_boxes, int* out_count, void* stream);
/* The same forward path over a CANVAS batch: N images of DIFFERENT sizes, each at the top-left of its config->H x config->W
 * slot (the canvas Hc x Wc).  images_nchw: (N,3,Hc,Wc) float32 device images (pixels outside an image are never read);
 * extents: device int32 [N][2], image n's (height, width), (0, 0) = an empty slot; im_info: device int32 [N][2], image n's
 * clip bounds (im_h, im_w).  Both are read when the kernels run, so the static launch sequence, captured once into a CUDA
 * graph, serves any mix of sizes.  The launches are those of the *_batch_ext entries, in the order of
 * frcnn_forward_vgg16_batch; image n's outputs are bit-identical to frcnn_forward_vgg16 on that image alone.  Outputs as
 * frcnn_forward_vgg16_batch.  The workspace (frcnn_forward_vgg16_canvas_workspace_bytes, 0 on a bad config or N) also serves
 * frcnn_detect_vgg16_raw.  NULL pointers or N outside [1,65535] -> FRCNN_ERR_ARG; a short workspace -> FRCNN_ERR_WORKSPACE. */
size_t frcnn_forward_vgg16_canvas_workspace_bytes(const frcnn_forward_config* config, int N);
int frcnn_forward_vgg16_canvas(const frcnn_forward_config* config, const frcnn_vgg16_weights* weights, int N,
                               const float* images_nchw, const int* extents, const int* im_info, void* workspace,
                               size_t workspace_bytes, float* out_prob, float* out_boxes, int* out_count, void* stream);

/* The device block [header | pixels] of raw photos (frcnn_detect_vgg16_raw, frcnn_b200.preprocess.raw_header_layout).  The
 * header holds FRCNN_RAW_FIELDS arrays of 8 * N bytes each; array f starts at byte 8 * N * f:
 *   FRCNN_RAW_EXTENTS   int32  [N][2]  the resized (H, W) of image n, (0, 0) = an empty slot
 *   FRCNN_RAW_IM_INFO   int32  [N][2]  its clip bounds (im_h, im_w) (forward.py passes (H, H))
 *   FRCNN_RAW_SRC_HW    int32  [N][2]  its source size (h0, w0)
 *   FRCNN_RAW_SRC_OFF   int64  [N]     byte offset of its uint8 (h0, w0, 3) BGR pixels in the pixel area
 *   FRCNN_RAW_INV_SCALE double [N]     1.0 / im_scale
 * (see frcnn_preprocess_bgr8_canvas).  The pixel area starts at frcnn_raw_header_bytes(N), a multiple of 256 (0 for N outside
 * [1,65535]). */
#define FRCNN_RAW_EXTENTS 0
#define FRCNN_RAW_IM_INFO 1
#define FRCNN_RAW_SRC_HW 2
#define FRCNN_RAW_SRC_OFF 3
#define FRCNN_RAW_INV_SCALE 4
#define FRCNN_RAW_FIELDS 5
size_t frcnn_raw_header_bytes(int N);

/* forward.py's whole loop on RAW photos of different sizes behind one call: frcnn_preprocess_bgr8_canvas (resize, mean
 * subtraction (mean_b, mean_g, mean_r) and first-layer pack of every slot), the launch sequence of frcnn_forward_vgg16_canvas,
 * frcnn_detect_batch (per-class NMS det_nms_thresh, score >= det_conf; forward.py uses 0.3 and 0.8) and
 * frcnn_detection_lists_batch.  block: the device block [header | arena_bytes bytes of pixels] (8-byte aligned); im_scale:
 * device double [N], image n's im_scale (the divisor of its boxes).  Outputs: out_prob / out_boxes / out_count as
 * frcnn_forward_vgg16_canvas, and image n's detection list at out_dets + n*cap*5 / out_scores + n*cap, its length in
 * out_det_count[n], cap = (num_classes-1) * post_nms_top_n.  Workspace: frcnn_forward_vgg16_canvas_workspace_bytes.  Static
 * launch sequence: captured once, it serves any batch that fits the canvas and the arena.  Errors as
 * frcnn_forward_vgg16_canvas, and a non-positive arena_bytes -> FRCNN_ERR_ARG. */
int frcnn_detect_vgg16_raw(const frcnn_forward_config* config, const frcnn_vgg16_weights* weights, int N, const void* block,
                           long long arena_bytes, double mean_b, double mean_g, double mean_r, const double* im_scale,
                           double det_nms_thresh, float det_conf, void* workspace, size_t workspace_bytes, float* out_prob,
                           float* out_boxes, int* out_count, int* out_dets, float* out_scores, int* out_det_count, void* stream);

/* ------------------------------------------------------------------------------------------------
 * ResNet trunk support (SURVEY.md 8f rank 2; chainer ResNetLayers as used by models/resnet.py:11-45).
 * ------------------------------------------------------------------------------------------------ */

/* frcnn_conv2d with a residual input: y = act(conv(x) + bias + (res_hi + res_lo)), res [H][W][Cout] bf16 planes
 * (res_lo may be NULL) -- the "h + shortcut, then ReLU" tail of a bottleneck block in one epilogue.  bf16 output only. */
int frcnn_conv2d_res(const void* x_hi, const void* x_lo, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                     const float* bias, int Cout, int ksize, int relu, const void* res_hi, const void* res_lo, void* y_hi,
                     void* y_lo, void* stream);

/* General first-layer im2col: (C,H,W) fp32 -> [Ho][Wo][K_pad] bf16 hi/lo, K index (r*ksize+s)*C + c, zero padding,
 * Ho = (H + 2*pad - ksize)/stride + 1 (conv1 of ResNet: ksize 7, stride 2, pad 3, K = 147 -> K_pad 160), and the matching
 * weight packing [1][Cout][K_pad] (scale: optional per-output-channel factor, e.g. a folded BatchNorm). */
int frcnn_pack_image_im2col(const float* x_chw, int C, int H, int W, int ksize, int stride, int pad, int K_pad, void* y_hi,
                            void* y_lo, void* stream);
int frcnn_pack_conv_weights_im2col(const float* w_oihw, const float* scale, int Cout, int Cin, int ksize, int K_pad, void* w_hi,
                                   void* w_lo, void* stream);

/* F.max_pooling_2d(x, 3, stride=2), Chainer defaults pad=0 / cover_all=True: [H][W][C] -> [ceil((H-3)/2)+1][...][C]. */
int frcnn_maxpool3x3s2_ceil(const void* x_hi, const void* x_lo, int H, int W, int C, void* y_hi, void* y_lo, void* stream);

/* Pixels (2h, 2w) of an NHWC map: the input of a stride-2 1x1 convolution.  [H][W][C] -> [ceil(H/2)][ceil(W/2)][C]. */
int frcnn_subsample2x(const void* x_hi, const void* x_lo, int H, int W, int C, void* y_hi, void* y_lo, void* stream);

/* The same kernels over a batch of N images of one shape in one launch (1 <= N <= 65535; image n's planes n image sizes
 * into every buffer), each image bit-identical to the one-image entry on it:
 *   frcnn_pack_image_im2col_batch    (N,C,H,W) fp32 -> [N][Ho][Wo][K_pad]
 *   frcnn_maxpool3x3s2_ceil_batch    [N][H][W][C] -> [N][ceil((H-3)/2)+1][...][C]
 *   frcnn_subsample2x_batch          [N][H][W][C] -> [N][ceil(H/2)][ceil(W/2)][C]
 *   frcnn_conv2d_res_batch           frcnn_conv2d_res with x [N,H,W,Cin] and res, y [N,H,W,Cout] (frcnn_conv2d_batch's plan)
 * The caller passes the residual planes of the output's shape; they are read at each output pixel's own image offset. */
int frcnn_pack_image_im2col_batch(const float* x_nchw, int N, int C, int H, int W, int ksize, int stride, int pad, int K_pad,
                                  void* y_hi, void* y_lo, void* stream);
int frcnn_maxpool3x3s2_ceil_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int C, void* y_hi, void* y_lo, void* stream);
int frcnn_subsample2x_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int C, void* y_hi, void* y_lo, void* stream);
int frcnn_conv2d_res_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                           const float* bias, int Cout, int ksize, int relu, const void* res_hi, const void* res_lo, void* y_hi,
                           void* y_lo, void* stream);
/* A ResNet trunk over a CANVAS batch: image n sits at the top-left of its slot and its true size is extents[2n] x
 * extents[2n+1] (device int32 [N][2], read at run time, clamped to the slot) at the resolution of the entry's INPUT.
 *   frcnn_pack_image_im2col_batch_ext   extents in input pixels: a tap outside the image reads as the zero padding (whatever
 *                                       the canvas holds there) and every output pixel outside the image's own output size
 *                                       ((e + 2*pad - ksize) / stride + 1, 0 when negative) is written as 0.
 *   frcnn_maxpool3x3s2_ceil_batch_ext   extents of the pooled map: each window is clipped at the image's border as the
 *                                       one-image kernel clips it at the map's, so no pixel outside the image is read; every
 *                                       output pixel outside (e - 2) / 2 + 1 (0 for e <= 1) is written as 0.
 *   frcnn_conv2d_res_batch_ext          frcnn_conv2d_batch_ext with the residual add: every output pixel outside
 *                                       ceil(extent / 2^halvings) is written as 0 after the add, whatever the residual holds
 *                                       there.
 * frcnn_subsample2x_batch needs no extents: an output pixel inside ceil(e / 2) reads an input pixel inside e, and one
 * outside reads an input pixel outside e -- so its input must be 0 outside every image (what the entries above write),
 * and the output then is too.  Each image's pixels equal the one-image entry on the image alone.  NULL extents or N outside
 * [1, 65535] (frcnn_conv2d_res_batch_ext: N < 1, halvings outside [0,30]) -> FRCNN_ERR_ARG. */
int frcnn_pack_image_im2col_batch_ext(const float* x_nchw, int N, int C, int H, int W, int ksize, int stride, int pad, int K_pad,
                                      const int* extents, void* y_hi, void* y_lo, void* stream);
int frcnn_maxpool3x3s2_ceil_batch_ext(const void* x_hi, const void* x_lo, int N, int H, int W, int C, const int* extents, void* y_hi,
                                      void* y_lo, void* stream);
int frcnn_conv2d_res_batch_ext(const void* x_hi, const void* x_lo, int N, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                               const float* bias, int Cout, int ksize, int relu, const void* res_hi, const void* res_lo, void* y_hi,
                               void* y_lo, const int* extents, int halvings, void* stream);
/* The per-level extents of a ResNet canvas batch of N Hc x Wc slots, in one launch (the first of the plan, so that every
 * later launch reads its level's [N][2] slice with halvings 0): out (device int32 [5][N][2]) receives, per image and axis,
 * from its extent e (extents [N][2], input pixels):
 *   level 0  conv1 7x7/2 pad 3      c  = (e - 1) / 2 + 1               (0 for e = 0)
 *   level 1  pool1 3x3/2 cover_all  p  = (c - 2) / 2 + 1               (0 for c <= 1)
 *   level 2..4  res3, res4, res5    r' = (r + 1) / 2                   (res2 keeps level 1)
 * each clamped to that level's canvas size (the same rules applied to Hc and Wc).  NULL pointers, N outside [1, 65535] or a
 * non-positive canvas -> FRCNN_ERR_ARG. */
int frcnn_resnet_level_extents(const int* extents, int N, int Hc, int Wc, int* out, void* stream);
/* Raw photos into the first-layer im2col planes of a ResNet canvas batch in ONE launch: frcnn_preprocess_bgr8, a copy into
 * the top-left of a zeroed Hc x Wc slot and frcnn_pack_image_im2col_batch_ext for all N slots, without the float32 images
 * in between.  The descriptors (arena, src_off, src_hw, inv_scale, extents) and the empty-slot rule are those of
 * frcnn_preprocess_bgr8_canvas; ksize / stride / pad / K_pad those of frcnn_pack_image_im2col_batch_ext with C = 3.
 * y_hi / y_lo (y_lo may be NULL) receive the whole [N][Ho][Wo][K_pad], Ho = (Hc + 2*pad - ksize) / stride + 1 (Wo alike):
 * inside each image's conv_out(extent), bit for bit what those three steps write (a tap outside the resized image reads as
 * the zero padding), and 0 at every other output pixel and at every k >= 3*ksize^2.  NULL pointers, N outside 1..65535, a
 * non-positive canvas, ksize outside 1..45, stride < 1, pad < 0 or 2*pad + max(Hc, Wc) > 2^30, K_pad not a multiple of 8
 * in [3*ksize^2, 65536] or a canvas smaller than the filter -> FRCNN_ERR_ARG. */
int frcnn_preprocess_bgr8_canvas_im2col(const unsigned char* arena, long long arena_bytes, const long long* src_off,
                                        const int* src_hw, const double* inv_scale, const int* extents, int N, int Hc, int Wc,
                                        double mean_b, double mean_g, double mean_r, int ksize, int stride, int pad, int K_pad,
                                        void* y_hi, void* y_lo, void* stream);
/* The VOC training dataset's transform (datasets/pascal_voc_dataset.py get_example: float32 mean subtraction, then
 * cv.resize(..., INTER_CUBIC)) on raw photos, straight into the first-layer im2col planes of a canvas batch in ONE launch.
 * Arguments, descriptors, output layout, empty-slot rule and errors are those of frcnn_preprocess_bgr8_canvas_im2col; only the
 * resize differs: OpenCV's generic float bicubic (A = -0.75, float coordinate, replicate borders, no clamping of the
 * result), restated bit for bit -- what cv2.resize computes on a float32 image with IPP off.  Each tap's pixel is
 * float(double(u8) - mean_c).  A descriptor whose inv_scale is 0, negative, infinite or NaN moves no access outside the
 * arena or the slot and gives finite values.  The training canvas uses ksize 3, stride 1, pad 1, K_pad 32. */
int frcnn_preprocess_voc_canvas_im2col(const unsigned char* arena, long long arena_bytes, const long long* src_off,
                                       const int* src_hw, const double* inv_scale, const int* extents, int N, int Hc, int Wc,
                                       double mean_b, double mean_g, double mean_r, int ksize, int stride, int pad, int K_pad,
                                       void* y_hi, void* y_lo, void* stream);
/* The VOC dataset's box scaling (`bbox *= im_scale` on float32 boxes) for N canvas slots, into a trainer's ground truth:
 * gt [N][max_gt][5] (device float32) row g of slot n = (f32(box) * f32(im_scale) for x1, y1, x2, y2, the label copied) for
 * g < c = clamp(count[n], 0, max_gt), and 0 for g >= c; gt_counts[n] (device int32 [N]) = c.  scale (device float32 [N]):
 * im_scale rounded to float32; count (device int32 [N]); raw_gt (device float32 [N][max_gt][5]): the boxes in source-photo
 * coordinates and the labels.  NULL pointers, N outside [1, 65535] or max_gt outside [1, 2^20] -> FRCNN_ERR_ARG. */
int frcnn_voc_scale_gt_batch(const float* scale, const int* count, const float* raw_gt, int N, int max_gt, float* gt, int* gt_counts,
                             void* stream);
/* Training-time augmentation on raw photos (py-faster-rcnn's TRAIN.USE_FLIPPED and TRAIN.SCALES), drawn per slot on the
 * device so that a captured step augments afresh on every replay.  The host computes S candidates per slot (1 <= S <= 8,
 * frcnn_b200.preprocess.voc_aug_candidates, from plan_size at every scale): cand_hw int32 [N][S][2] the resized (H, W),
 * cand_inv float64 [N][S] 1.0 / im_scale, cand_scale float32 [N][S] im_scale rounded to float32.  The device only selects
 * among them.
 *
 * frcnn_voc_augment_batch: one thread per slot, the first launch of an augmenting step.
 *   draw 1: choice[n] (int32 [N][2]: flip, scale index) <- the draw of seeds[n] (uint64 [N]), with s = seeds[n] ^ mix64(3):
 *             flip  = sample_key(s, 0) >> 63
 *             index = ((sample_key(s, 1) >> 32) * S) >> 32
 *           mix64 is the splitmix64 finaliser and sample_key(seed, i) = (mix64(seed ^ i * 0xD6E8FEB86659FD93) &
 *           0xFFFFFFFF00000000) | i, the hash and key of the device subsampling (frcnn_anchor_targets_batch mode 1) and the
 *           dropout masks (salts 1 and 2).
 *   draw 2: the same draw with the flip written as 0 (scale jitter only).
 *   draw 0: choice is read as the host wrote it (seeds may be NULL).
 * Then, in every mode, with k = clamp(choice[n][1], 0, S - 1): extents[n] and im_info[n] (int32 [N][2], the raw header's
 * FRCNN_RAW_EXTENTS / FRCNN_RAW_IM_INFO) <- cand_hw[n][k], inv_scale[n] (FRCNN_RAW_INV_SCALE) <- cand_inv[n][k], scale[n] (the
 * ground-truth section's float32 im_scale) <- cand_scale[n][k] and flip[n] (int32 [N]) <- (choice[n][0] != 0).  A slot whose
 * src_hw[n] (int32 [N][2]) is not positive stays empty: extents and im_info 0 x 0, inv_scale, scale and flip 0.  NULL
 * pointers (seeds only when draw != 0), draw outside 0..2, N outside [1, 65535] or S outside [1, 8] -> FRCNN_ERR_ARG. */
int frcnn_voc_augment_batch(const unsigned long long* seeds, int N, int S, const int* cand_hw, const double* cand_inv,
                            const float* cand_scale, const int* src_hw, int draw, int* choice, int* flip, int* extents, int* im_info,
                            double* inv_scale, float* scale, void* stream);
/* frcnn_preprocess_voc_canvas_im2col with a per-slot horizontal flip: flip (device int32 [N]) nonzero resizes slot n from its
 * mirrored photo p[:, ::-1], bit for bit cubic_resize(mean_subtract(p)[:, ::-1]) -- each horizontal tap's column i is read as
 * w0 - 1 - i, and the weights, the border rule and the summation order are those of the mirrored image's own columns.  A
 * slot whose flip is 0 equals frcnn_preprocess_voc_canvas_im2col bit for bit.  Every other argument and error as
 * frcnn_preprocess_voc_canvas_im2col; a NULL flip -> FRCNN_ERR_ARG. */
int frcnn_preprocess_voc_canvas_im2col_flip(const unsigned char* arena, long long arena_bytes, const long long* src_off,
                                            const int* src_hw, const double* inv_scale, const int* extents, const int* flip, int N,
                                            int Hc, int Wc, double mean_b, double mean_g, double mean_r, int ksize, int stride,
                                            int pad, int K_pad, void* y_hi, void* y_lo, void* stream);
/* frcnn_voc_scale_gt_batch with a per-slot horizontal flip: where flip[n] (device int32 [N]) is nonzero, the rows g < c of
 * slot n are first mirrored in its photo's w0 = src_hw[2n+1] columns (py-faster-rcnn's inclusive-pixel flip, float32):
 * x1' = (f32(w0) - x2) - 1, x2' = (f32(w0) - x1) - 1, y1 and y2 unchanged; then every coordinate times f32(im_scale).  The
 * same kernel as frcnn_voc_scale_gt_batch (counts clamped, rows past the count zeroed).  NULL pointers, N outside
 * [1, 65535] or max_gt outside [1, 2^20] -> FRCNN_ERR_ARG. */
int frcnn_voc_flip_scale_gt_batch(const float* scale, const int* count, const float* raw_gt, const int* src_hw, const int* flip,
                                  int N, int max_gt, float* gt, int* gt_counts, void* stream);

/* ------------------------------------------------------------------------------------------------
 * RPN training targets and losses (SURVEY.md 8f rank 1, the train_rpn.py step).  Box arithmetic is
 * float64 in the reference's operation order: labels and indices are bit-identical to the reference.
 * ------------------------------------------------------------------------------------------------ */

/* models/bbox.pyx:16-56 bbox_overlaps.  boxes [n,4], query [k,4], out [n,k], all float64 device
 * memory.  (The reference runs this on the host even in GPU mode, anchor_target_layer.py:179-187.) */
int frcnn_bbox_overlaps(const double* boxes, int n, const double* query, int k, double* out, void* stream);

/* AnchorTargetLayer.__call__ (models/anchor_target_layer.py:66-198).
 *   anchors [A,4] float64 base anchors; all anchors = base + (w,h,w,h)*feat_stride, row (h*W+w)*A+a,
 *   kept in float64 (:108); gt_boxes [n_gt,5] float32 (x1,y1,x2,y2,cls), n_gt >= 1.
 *   neg_thr / pos_thr / batch / num_fg: RPN_NEGATIVE_OVERLAP 0.3, RPN_POSITIVE_OVERLAP 0.7,
 *   RPN_BATCHSIZE 256, int(RPN_FG_FRACTION*RPN_BATCHSIZE) = 128 (:44-47,149).
 *   subsample_mode 0: labels BEFORE subsampling (:131-146);
 *                  1: device subsampling (:148-168) by a counter hash of (seed, anchor index) -- the
 *                     reference draws from NumPy's global RNG on the host, which cannot be matched
 *                     bit-for-bit without that host state; no host sync.  Requires 0 <= num_fg <= batch.
 *                     Rule: with key(s, i) = (mix64(s ^ i*0xD6E8FEB86659FD93) & 0xFFFFFFFF00000000) | i
 *                     in uint64 (mix64 = one splitmix64 step: add 0x9E3779B97F4A7C15, then its
 *                     finaliser; i = anchor index in [0, n_all)), if n_fg > num_fg the
 *                     n_fg - num_fg positives with the smallest key(seed, i) become -1; then, with
 *                     num_bg = batch - (positives left), if n_bg > num_bg the n_bg - num_bg negatives with
 *                     the smallest key(seed ^ 0xA5A5A5A5DEADBEEF, i) become -1 (the top 32 bits of the
 *                     key decide, the lower index goes first on a tie);
 *                  2: disable_pos[n_disable] = positions in the inside-compact arrays to set to -1
 *                     (exactly what the reference's np.random.choice calls return).
 * Outputs (device): labels_full int32 [n_all] in {-1,0,1}, -1 for anchors outside the image
 *   (= bbox_labels_mapped of region_proposal_network.py:164-165); targets_full float32 [n_all,4]
 *   (16-byte aligned; zeros outside); inds_inside int32 [n_all capacity] (ascending);
 *   counts int32 [8] = {n_inside, n_fg, n_bg, n_fg before subsampling, n_bg before, n_all, 0, 0}.
 * The reference's compact outputs are labels_full[inds_inside], targets_full[inds_inside].
 * No anchor inside the image (the reference raises on its empty arg-max): counts = {0, 0, 0, 0, 0, n_all, 0, 0},
 * every label -1, every target 0, and frcnn_rpn_loss then returns four zero losses and zero gradients. */
size_t frcnn_anchor_targets_workspace_bytes(int n_all, int n_gt);
int frcnn_anchor_targets(const double* anchors, int A, int feat_h, int feat_w, int feat_stride, const float* gt_boxes,
                         int n_gt, int im_h, int im_w, double neg_thr, double pos_thr, int batch, int num_fg,
                         int subsample_mode, unsigned long long seed, const int* disable_pos, int n_disable,
                         int* labels_full, float* targets_full, int* inds_inside, int* counts, void* workspace,
                         size_t workspace_bytes, void* stream);

/* RegionProposalNetwork._calc_rpn_loss_cls / _calc_rpn_loss_bbox (models/region_proposal_network.py
 * :160-204) and, in the same pass, d(rpn_loss)/d(score) and d(rpn_loss)/d(bbox_pred).
 *   score: channel c of pixel k at score[c*score_cs + k*score_ps] (2A channels; 2-way softmax between
 *   channel a and A+a, ignore label -1, normalised by max(#valid,1)); bbox likewise (4A channels;
 *   channel j*A+a = coordinate j of anchor a, :186-191; Huber `delta`, summed over every INSIDE anchor,
 *   divided by the number of ALL anchors).  labels_full / targets_full / counts from
 *   frcnn_anchor_targets.  losses float32 [4] = {rpn_loss_cls, rpn_loss_bbox, rpn_cls_accuracy,
 *   rpn_loss = cls + loss_lambda*bbox}.  dscore / dbbox (optional, same addressing as score / bbox)
 *   receive grad_scale * d(rpn_loss)/d(.), zeros where no loss term applies. */
size_t frcnn_rpn_loss_workspace_bytes(int n_all);
int frcnn_rpn_loss(const float* score, long score_cs, long score_ps, const float* bbox, long bbox_cs, long bbox_ps,
                   const double* anchors, int A, int feat_h, int feat_w, int feat_stride, int im_h, int im_w,
                   const int* labels_full, const float* targets_full, const int* counts, double delta, double loss_lambda,
                   double grad_scale, float* losses, float* dscore, float* dbbox, void* workspace, size_t workspace_bytes,
                   void* stream);

/* frcnn_anchor_targets over the N slots of a canvas whose feature map is fhc x fwc (one launch per kernel, the slot is a
 * grid dimension; frcnn_anchor_targets launches the same kernels with N = 1).
 *   extents int32 [N][2]: each image's (height, width) in input pixels; its feature map is fh_n x fw_n =
 *   ceil(extent / 2^halvings) (clamped to fhc x fwc; halvings = 4 for VGG16).  im_info int32 [N][2]: the clip bounds of
 *   the inside test.  gt float32 [N][max_gt][5]: slot n's gt_counts[n] boxes (clamped to max_gt) in its first rows.
 *   subsample_mode 0: none; 1: the rule of frcnn_anchor_targets with slot n's seed seeds[n] (uint64 device memory, read
 *   when the kernel runs); 2: slot n disables the inside positions disable_pos[disable_offsets[n] .. disable_offsets[n+1])
 *   (offsets int32 [N+1] device memory, clamped to [0, n_disable)).
 * Outputs: slot n's labels_full / targets_full / inds_inside start at n*cap, cap = A*fhc*fwc, and its counts at 8n.
 * Anchors are numbered in the image's own frame, (y*fw_n + x)*A + a, and the device-subsample key hashes that index, so
 * slot n's first A*fh_n*fw_n entries (and its first counts[0] inside indices) equal what frcnn_anchor_targets returns for
 * that image alone, bit for bit; entries past them are not written.  A slot with a 0 x 0 extent or gt_counts[n] < 1 is
 * empty: its counts are all zero.  Workspace: frcnn_anchor_targets_batch_workspace_bytes(N, cap, max_gt). */
size_t frcnn_anchor_targets_batch_workspace_bytes(int N, int n_cap, int max_gt);
int frcnn_anchor_targets_batch(const double* anchors, int A, int fhc, int fwc, int feat_stride, int N, const int* extents,
                               int halvings, const int* im_info, const float* gt, int max_gt, const int* gt_counts, double neg_thr,
                               double pos_thr, int batch, int num_fg, int subsample_mode, const unsigned long long* seeds,
                               const int* disable_pos, int n_disable, const int* disable_offsets, int* labels_full,
                               float* targets_full, int* inds_inside, int* counts, void* workspace, size_t workspace_bytes,
                               void* stream);

/* frcnn_rpn_loss over the N slots of frcnn_anchor_targets_batch (same canvas, extents, halvings and im_info), on the NHWC
 * head matrix head [N*fhc*fwc][ld] (slot n's pixel (y, x) in row n*fhc*fwc + y*fwc + x; scores in columns [0, 2A), deltas
 * in [2A, 6A), ld >= 6A).  losses float32 [N][4] as frcnn_rpn_loss's.  dhead (optional) [N*fhc*fwc][ld]: EVERY element is
 * written -- slot n's anchors get grad_scale * d(rpn_loss_n)/d(.), every other row and the columns >= 6A get 0 -- so it
 * needs no zeroing.  Each slot is normalised by its own counts and its own A*fh_n*fw_n, like the reference's per-device
 * loss: slot n's losses and gradient rows equal frcnn_rpn_loss on that image alone, bit for bit.  An empty slot (counts[5]
 * == 0) gets zero losses and a zero gradient.  Workspace: frcnn_rpn_loss_batch_workspace_bytes(N, A*fhc*fwc). */
size_t frcnn_rpn_loss_batch_workspace_bytes(int N, int n_cap);
int frcnn_rpn_loss_batch(const float* head, int ld, const double* anchors, int A, int fhc, int fwc, int feat_stride, int N,
                         const int* extents, int halvings, const int* im_info, const int* labels_full, const float* targets_full,
                         const int* counts, double delta, double loss_lambda, double grad_scale, float* losses, float* dhead,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ---- RCNN-head training (rcnn_train.cu; train_rcnn.py, models/faster_rcnn.py:136-173) ---- */

/* ProposalTargetLayer, part 1 (proposal_target_layer.py:91-96): best ground-truth overlap of every proposal, float64 in
 * bbox.pyx order.  rois [R_cap,4] fp32 (*count valid, NULL = R_cap), gt_boxes [n_gt,5]; max_overlaps double [R_cap]
 * (-1 for rows >= count), argmax int32 [R_cap].  The fg/bg sampling (:99-129) draws from NumPy's RNG on the host in the
 * reference; the caller does the same (or any other rule) on these two small arrays and passes keep_inds to part 2. */
int frcnn_roi_overlaps(const float* rois, const int* count, int R_cap, const float* gt_boxes, int n_gt, double* max_overlaps,
                       int* argmax, void* stream);
/* part 2 (:138-147): use_gt_boxes [n,5] = gt[argmax[keep]], labels int32 [n] = use_gt_boxes[:,4] (faster_rcnn.py:154),
 * bbox_reg_targets [n, 4*num_classes] = float32 bbox_transform of the kept proposal scattered to its class's 4 columns
 * (rows whose class is 0 stay zero).  A kept row with argmax -1 (no overlap above -1) takes gt row 0. */
int frcnn_roi_targets(const float* rois, const float* gt_boxes, const int* argmax, const int* keep_inds, int n, int num_classes,
                      float* use_gt_boxes, float* bbox_reg_targets, int* labels, void* stream);
/* Array-level helpers of models/bbox_transform.py used by the training code: bbox_transform (:18-38) on float32 rows
 * (ex_rois [n,4], gt rows gt_stride >= 4 floats apart) -> out [n,4] (dx, dy, dw, dh); keep_inside (:112-130) as a 0/1 flag
 * per box: x1 >= 0, y1 >= 0, x2 < im_w, y2 < im_h. */
int frcnn_bbox_transform(const float* ex_rois, const float* gt_rois, int gt_stride, int n, float* out, void* stream);
int frcnn_keep_inside(const float* boxes, int n, int im_h, int im_w, unsigned char* flags, void* stream);
/* faster_rcnn.py:151-165 on the merged head output head_out [R_cap][ld] (columns [0,num_classes) scores, then
 * 4*num_classes deltas): losses float32 [4] = {loss_cls, loss_bbox, cls_accuracy, loss_rcnn}; dhead (optional, same shape)
 * = grad_scale * d(loss_rcnn)/d(head_out), zero on rows not kept and on columns >= 5*num_classes.  1 <= n <= 128,
 * num_classes >= 1, ld >= 5*num_classes.  keep_inds must not repeat a row (the reference's sampling never does): a repeated
 * row's gradient is written, not summed.  A label outside [0, num_classes) makes loss_cls NaN; loss_bbox stays finite. */
int frcnn_rcnn_loss(const float* head_out, int ld, int R_cap, const int* keep_inds, int n, const int* labels,
                    const float* bbox_reg_targets, int num_classes, double delta, double grad_scale, float* losses, float* dhead,
                    void* stream);
/* F.dropout with an explicit mask: x = mask ? x*scale : 0 in place on the bf16 hi(/lo) planes (scale = 1/(1-ratio)). */
int frcnn_dropout(void* x_hi, void* x_lo, const unsigned char* mask, long n, float scale, void* stream);
/* F.roi_pooling_2d backward: dfeat [H*W][C] fp32 = sum over (roi, bin) of the bin's gradient g [R_cap][outh*outw][C]
 * (bf16 hi/lo) at the bin's first maximum of feat; order-independent 64-bit fixed-point accumulation (bit-reproducible). */
size_t frcnn_roi_pool_backward_workspace_bytes(int H, int W, int C);
int frcnn_roi_pool_backward(const void* feat_hi, const void* feat_lo, int H, int W, int C, const float* rois, const int* count,
                            int R_cap, int outh, int outw, float scale, const void* g_hi, const void* g_lo, float* dfeat,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ---- the RCNN step over the N slots of a canvas (rcnn_train.cu).  The slot is a grid dimension and every per-slot count,
 * extent and seed is device memory read when the kernel runs, so one launch sequence (and one captured graph) serves any
 * mix of sizes.  frcnn_rcnn_loss and frcnn_roi_pool_backward launch the kernels of their _batch forms with N = 1; the
 * one-image overlaps / targets and the batched proposal targets share their per-row device code. */

/* ProposalTargetLayer (proposal_target_layer.py:76-150) over N slots, one CTA per slot.
 *   rois: slot n's proposals [R_cap][4] fp32 at rois + n*rois_stride (16-byte aligned), the first counts[n*count_stride] of
 *   them valid (counts NULL: R_cap) -- the rois / count outputs of frcnn_proposals_batch_ext as they are.  1 <= R_cap <= 4096.
 *   gt [N][max_gt][5] fp32 with gt_counts[n] (clamped to max_gt) rows in slot n.
 *   Part 1: max_overlaps double [N][R_cap] and argmax int32 [N][R_cap] as frcnn_roi_overlaps computes them.
 *   Part 2, the kept set (at most 128 rows):
 *     mode 1 (device): fg = {r < R_n : max_ov >= 0.5}, bg = {r < R_n : 0.1 <= max_ov < 0.5} (a row without an overlap,
 *       max_ov = -1, is in neither); the min(32, |fg|) fg rows with the smallest key(seeds[n], r), then the
 *       min(128 - n_fg, |bg|) bg rows with the smallest key(seeds[n] ^ 0xA5A5A5A5DEADBEEF, r), key as in
 *       frcnn_anchor_targets mode 1 (seeds uint64 [N] device memory).  The kept list is the kept fg rows in ascending r,
 *       then the kept bg rows in ascending r.
 *     mode 2 (list): slot n keeps keep_list[list_offsets[n] .. list_offsets[n+1]) in that order (offsets int32 [N+1],
 *       clamped to [0, n_list)); entries outside [0, R_n), and entries past the 128th kept one, are skipped and counted.
 *       The list must not repeat a row (see frcnn_rcnn_loss).
 *   Part 3: keep int32 [N][128], labels int32 [N][128] (= use_gt_boxes[:, 4], background rows included, faster_rcnn.py:154),
 *   use_gt_boxes [N][128][5], bbox_reg_targets [N][128][4*num_classes] as frcnn_roi_targets computes them; rows past
 *   n_keep hold keep -1 and zeros.
 *   out_counts int32 [N][8] = {n_keep, kept rows with max_ov >= 0.5, |fg|, |bg|, list entries skipped, R_n, 0, 0}.
 * A slot with no ground truth or no RoIs has all-zero counts.  In list mode each slot's outputs equal frcnn_roi_overlaps +
 * frcnn_roi_targets on that slot, bit for bit (both give a kept row with argmax -1 gt row 0). */
int frcnn_proposal_targets_batch(int N, const float* rois, long rois_stride, const int* counts, long count_stride, int R_cap,
                                 const float* gt, int max_gt, const int* gt_counts, int num_classes, int mode,
                                 const unsigned long long* seeds, const int* keep_list, int n_list, const int* list_offsets,
                                 int* keep, int* labels, float* use_gt_boxes, float* bbox_reg_targets, double* max_overlaps,
                                 int* argmax, int* out_counts, void* stream);

/* frcnn_rcnn_loss over the N slots of frcnn_proposal_targets_batch: head [N*R_cap][ld] with slot n's row r at n*R_cap + r;
 * keep / labels / bbox_reg_targets [N][128][...] and counts [N][8] as that entry writes them (slot n reads its n_keep =
 * counts[8n] on the device).  losses float32 [N][4].  dhead (optional, [N*R_cap][ld]) is written in EVERY element: kept rows
 * get grad_scale * d(loss_rcnn_n)/d(.), everything else 0, so it needs no zeroing.  Each slot is normalised by its own
 * n_keep, like the reference's per-device loss (ParallelUpdater sums the gradients); its losses and gradient rows equal
 * frcnn_rcnn_loss on it, bit for bit.  A slot with n_keep = 0 gets zero losses and a zero gradient (counts shows which). */
int frcnn_rcnn_loss_batch(int N, const float* head, int ld, int R_cap, const int* keep, const int* labels,
                          const float* bbox_reg_targets, const int* counts, int num_classes, double delta, double grad_scale,
                          float* losses, float* dhead, void* stream);

/* frcnn_roi_pool_backward on an N-slot canvas feature map feat [N][H][W][C] (bf16 hi/lo): slot n's RoIs at
 * rois + n*rois_stride, its count at counts[n*count_stride] (NULL: R_cap), its gradient rows g [N][R_cap][outh*outw][C].
 * Bins are clamped to the slot's own ceil(extents[n] / 2^halvings) map, exactly as frcnn_roi_pool_batch_ext clamps them,
 * and each slot has its own fixed-point accumulator, so dfeat [N*H*W][C] fp32 is 0 outside each image and slot n's map
 * equals frcnn_roi_pool_backward on that image's own map, bit for bit.
 * Workspace: frcnn_roi_pool_backward_batch_workspace_bytes(N, H, W, C). */
size_t frcnn_roi_pool_backward_batch_workspace_bytes(int N, int H, int W, int C);
int frcnn_roi_pool_backward_batch_ext(const void* feat_hi, const void* feat_lo, int N, int H, int W, int C, const float* rois,
                                      long rois_stride, const int* counts, long count_stride, int R_cap, int outh, int outw,
                                      float scale, const int* extents, int halvings, const void* g_hi, const void* g_lo,
                                      float* dfeat, void* workspace, size_t workspace_bytes, void* stream);

/* Ratio-0.5 F.dropout keep masks for N slots: masks uint8 [N][rows][cols], element (r, c) of slot n =
 *     key(seeds[n] ^ mix64(salt), r*cols + c) >> 63
 * with key and mix64 as in frcnn_anchor_targets mode 1 (seeds uint64 [N] device memory; salt tells the layers apart).
 * frcnn_dropout applies them to the flat [N*rows][cols] activations. */
int frcnn_dropout_masks_batch(int N, int rows, int cols, const unsigned long long* seeds, unsigned long long salt,
                              unsigned char* masks, void* stream);

/* ---- the backward pass of the reference's training steps.  In the reference it is `loss.backward()` inside Chainer's
 * updater (train_rpn.py:169-174 / train_rcnn.py with StandardUpdater or ParallelUpdater; the graph is the one
 * models/vgg16.py:38-82, models/region_proposal_network.py:117-120 and models/faster_rcnn.py:123-134 build) followed by
 * MomentumSGD + WeightDecay (train_rpn.py:165-167).  Chainer's per-function backward code is un-vendored; these entry
 * points are its replacement: L.Convolution2D / L.Linear backward-data = frcnn_conv2d on frcnn_pack_conv_weights_dgrad,
 * backward-filter = frcnn_gemm_nt_splitk (+ frcnn_wgrad_reduce, frcnn_bias_grad), F.relu / F.max_pooling_2d / F.dropout
 * backward = frcnn_grad_prepare, F.roi_pooling_2d backward = frcnn_roi_pool_backward, the optimizer = frcnn_optimizer_update. */

/* Split-K "NT" GEMM on the tensor-core kernel of frcnn_conv2d (same bf16 hi/lo operand planes), the engine of the
 * weight-gradient pass (conv backward-filter as a GEMM over the pixel axis):
 *     parts[g][s][m][n] = sum over k in split s of  A[m][k] * B_g[n][k + off(g)]        (fp32, row stride ld)
 *   A [M][K], B [N][K]: bf16 hi (+ lo, both or neither) planes, K contiguous, K % 64 == 0; reads outside [0,K) are 0.
 *   groups = 1: B_g = B, off = 0.  groups = 9 (the 3x3 taps when K is a zero-padded pixel axis of row pitch
 *   row_stride, row_stride % 8 == 0): B is THREE planes [3][N][K] holding the operand pre-shifted by -1 / 0 / +1
 *   pixel (plane j at k = the unshifted operand at k + j - 1; a TMA box must start 16-byte aligned, so the column
 *   shift cannot be a coordinate), B_g = plane g%3 and off(g) = (g/3 - 1)*row_stride.
 *   splits: requested K splits (the effective number is frcnn_gemm_nt_splitk_splits(K, splits)); parts holds
 *   groups*effective_splits slabs of M*ld floats, ld % 32 == 0, ld >= N.  zero_bias: ld zeros in device memory (the
 *   kernel's bias input).  The caller reduces over s. */
int frcnn_gemm_nt_splitk_splits(int K, int splits);
int frcnn_gemm_nt_splitk(const void* a_hi, const void* a_lo, int M, int K, const void* b_hi, const void* b_lo, int N,
                         int groups, int row_stride, int splits, const float* zero_bias, float* parts, int ld,
                         void* stream);

/* ---- conv backward, memory-bound parts (train_backward.cu).  The "transposed padded" layout used by the weight-
 * gradient GEMM: a [C][Kp] bf16 plane per hi/lo where pixel (h,w) of an H x W map sits at k = (h+1)*Wp + 8 + w
 * (8 zero columns on the left keep every 8-pixel group 16-byte aligned), Wp = W+9 rounded up to 8, Kp = (H+2)*Wp rounded up
 * to 64, everything else zero (the buffer must be zeroed once; the kernels only write the interior and zeros into the
 * padding).  frcnn_padded_pixels returns Kp and the row pitch Wp. */
long frcnn_padded_pixels(int H, int W, int* row_pitch);

/* Gradient / activation re-layout with the element-wise backward ops fused:
 *   source  : bf16 hi(/lo) NHWC planes g [H][W][C] -- or [ceil(H/2)][ceil(W/2)][C] when p_hi is given -- or fp32 [H*W][ld_f32]
 *   y (opt) : the forward post-ReLU activation [H][W][C]: value *= (y > 0), false for NaN  (F.relu backward)
 *   p (opt) : the 2x2/2 ceil-mode max-pooled y: the source is routed to the FIRST maximum of each window in scan order
 *             (F.max_pooling_2d backward), zero elsewhere
 *   outputs : o (opt) NHWC hi/lo [H][W][C]; t (opt) transposed padded planes [planes][C][Kp], planes = 1 (at k) or 3
 *             (plane j at k holds pixel k + j - 1: the pre-shifted B operand of frcnn_gemm_nt_splitk groups = 9).
 * With y = p = NULL and planes = 3 this is the plain activation transposer.  times2 != 0 (bf16 source only) doubles each
 * plane as bf16(2 x), exact for finite values, +-inf on overflow, NaN stays NaN: the backward factor 1/(1-ratio) of a
 * ratio-0.5 F.dropout whose kept set is {y > 0}. */
int frcnn_grad_prepare(const void* g_hi, const void* g_lo, const float* g_f32, int ld_f32, const void* y_hi, const void* y_lo,
                       const void* p_hi, const void* p_lo, int H, int W, int C, void* o_hi, void* o_lo, void* t_hi, void* t_lo,
                       int planes, int times2, void* stream);

/* frcnn_grad_prepare over N images in one launch (frcnn_grad_prepare is this with N = 1): every NHWC source, mask and
 * output is [N][H][W][C] (the pooled ones [N][ceil(H/2)][ceil(W/2)][C], the fp32 source [N*H*W][ld_f32]), and the
 * transposed planes are [planes][C][N*Kp] with image n's padded block in columns [n*Kp, (n+1)*Kp).  Image n's results
 * equal frcnn_grad_prepare on it, bit for bit.
 * Each Kp block keeps its own zero halo (rows 0 and H+1, the 8 left columns, the columns past W, the tail past
 * (H+2)*Wp), so frcnn_gemm_nt_splitk with K = N*Kp, unchanged, sums the weight gradient over the N images, the 9-tap
 * groups included: an A column k is nonzero only at a pixel row 1..H of its block, and the B read at k +- Wp (and the
 * +-1 pixel plane shift) then stays inside that block's halo.  This needs the buffer zeroed once, as for one image.
 * On a canvas no extents are needed: every forward launch is an _ext entry, so each stored post-ReLU activation is exactly
 * 0 outside its image and the ReLU mask zeroes every incoming gradient there -- including what the ceil-mode pool routes
 * to a window element past an odd edge -- and the data-gradient convolutions are _ext launches too. */
int frcnn_grad_prepare_batch(const void* g_hi, const void* g_lo, const float* g_f32, int ld_f32, const void* y_hi,
                             const void* y_lo, const void* p_hi, const void* p_lo, int N, int H, int W, int C, void* o_hi,
                             void* o_lo, void* t_hi, void* t_lo, int planes, int times2, void* stream);

/* The two re-layouts the ResNet trunk's backward adds (frcnn_grad_prepare's outputs, N = 1, bit-exact rules restated by
 * tests/resnet_train_ref.py):
 *   frcnn_maxpool3x3s2_backward  F.max_pooling_2d(3, stride=2, pad=0, cover_all=True) backward fused with the ReLU mask of
 *       its input: g and p [pool3s2_out(H)][pool3s2_out(W)][C] (the pooled gradient and the pooled map), y [H][W][C] the
 *       post-ReLU pool input, H, W >= 2.  Window (i, j) covers rows [2i, min(2i+3, H)) x columns [2j, min(2j+3, W)) and sends
 *       g[i][j] to the FIRST element in scan order whose value equals p[i][j]; pairs are read as DESIGN §2 reads them (an
 *       infinite hi stands alone) and compared as floats (+0 == -0, NaN equals nothing).  A pixel sums what its (up to four)
 *       windows send, in fp32 in ascending (i, j) order from +0; the sum is kept where y > 0 (hi read as int16 in
 *       (0, +inf]), +0 elsewhere, and re-split into hi/lo.  Transposed output: planes = 1.
 *   frcnn_grad_prepare_stride2   the backward of frcnn_subsample2x: the source g [ceil(H/2)][ceil(W/2)][C] at pixels (2i, 2j)
 *       of the H x W map and 0 everywhere else, then the optional y > 0 mask as in frcnn_grad_prepare (kept pairs keep their
 *       words); transposed output with planes = 1 or 3.
 * Their _batch forms run N images in one launch (the one-image entries are these with N = 1): every NHWC plane is [N][...]
 * of the one-image shape (g and p of frcnn_maxpool3x3s2_backward_batch [N][pool3s2_out(H)][pool3s2_out(W)][C], g of
 * frcnn_grad_prepare_stride2_batch [N][ceil(H/2)][ceil(W/2)][C]), and the transposed planes are [planes][C][N*Kp] with image
 * n's padded block in columns [n*Kp, (n+1)*Kp), as frcnn_grad_prepare_batch writes them.  Image n's results equal the
 * one-image entry on it, bit for bit.  N < 1, N * ceil(C/64) > 65535 and the one-image entry's errors -> FRCNN_ERR_ARG.
 * On a canvas no extents are needed, for the reason frcnn_grad_prepare_batch gives, and:
 *   - pool backward: y (conv1's output) is 0 outside each image, and so are p and g, which frcnn_maxpool3x3s2_ceil_batch_ext
 *     and the _ext data-gradient convolutions write as 0 outside the image's pooled extent.  A window that runs past the
 *     image's border, which the one-image entry on the cropped image clips, only adds elements of value 0.  Where p > 0
 *     they never match; where p == 0 the element chosen may differ, but the pixel it leaves or takes has y == 0 in both
 *     cases, so the y > 0 mask zeroes it.  A window that exists on the canvas and not on the cropped image has g == 0, and
 *     the fp32 sums start from +0, so one more +0 term changes no sum (a sum from +0 is never -0).
 *   - stride-2 scatter: inside the image, pixel (2i, 2j) reads g[i][j] inside the subsampled extent, as on the cropped
 *     image; outside it, y == 0 (and g == 0) give 0. */
int frcnn_maxpool3x3s2_backward(const void* g_hi, const void* g_lo, const void* y_hi, const void* y_lo, const void* p_hi,
                                const void* p_lo, int H, int W, int C, void* o_hi, void* o_lo, void* t_hi, void* t_lo, void* stream);
int frcnn_grad_prepare_stride2(const void* g_hi, const void* g_lo, const void* y_hi, const void* y_lo, int H, int W, int C,
                               void* o_hi, void* o_lo, void* t_hi, void* t_lo, int planes, void* stream);
int frcnn_maxpool3x3s2_backward_batch(const void* g_hi, const void* g_lo, const void* y_hi, const void* y_lo, const void* p_hi,
                                      const void* p_lo, int N, int H, int W, int C, void* o_hi, void* o_lo, void* t_hi, void* t_lo,
                                      void* stream);
int frcnn_grad_prepare_stride2_batch(const void* g_hi, const void* g_lo, const void* y_hi, const void* y_lo, int N, int H, int W,
                                     int C, void* o_hi, void* o_lo, void* t_hi, void* t_lo, int planes, void* stream);

/* ---- frozen BatchNorm in training (resnet_train.cu).  A convolution and its frozen BN are the folded convolution
 * Wf = W*s, bf = beta + (b - mean)*s, s = gamma/sqrt(var + eps) (float64, per output channel).
 *   frcnn_fold_batchnorm       wf[i] = f32(f64(w[i]) * s[i / per_out]) for Cout*per_out weights; bf (optional) [Cout] =
 *                              f32(f64(beta) + (f64(b) - f64(mean)) * s), b = 0 when NULL -- resnet_engine.fold_batchnorm's
 *                              arithmetic, bit for bit.
 *   frcnn_wgrad_reduce_scaled  frcnn_wgrad_reduce with a per-output-channel float64 scale instead of the scalar one:
 *                              dw[m][n][g] = f32(f64(s[m]) * f64(fp32 sum over splits s = 0, 1, ... of parts[g][s][m][n])).
 *                              With groups = splits = N = ld = 1 and parts = a bias sum [M] it scales a bias gradient. */
int frcnn_fold_batchnorm(const float* w, const double* s, int Cout, long per_out, const float* b, const float* beta,
                         const float* mean, float* wf, float* bf, void* stream);
int frcnn_wgrad_reduce_scaled(const float* parts, int groups, int splits, int M_parts, int M, int ld, int N, const double* s,
                              float* dw, void* stream);

/* dw[m][n][g] (the reference's OIHW float32, g = r*3+s or 1) = scale * sum over splits of parts[g][s][m][n], m < M;
 * parts slabs have M_parts >= M rows of ld floats. */
int frcnn_wgrad_reduce(const float* parts, int groups, int splits, int M_parts, int M, int ld, int N, float scale, float* dw,
                       void* stream);

/* db[c] = scale * sum over k of (t_hi + t_lo)[c][k] -- the bias gradient from the transposed dY. */
int frcnn_bias_grad(const void* t_hi, const void* t_lo, int C, long Kp, float scale, float* db, void* stream);

/* chainer.optimizer.WeightDecay(rate) hook + optimizers.MomentumSGD(lr, momentum) (train_rpn.py:165-167) on float32
 * master weights: g' = fma(rate, w, g); v = momentum*v - lr*g'; w += v.  frcnn_optimizer_update's MomentumSGD rule with
 * the hyper-parameters passed by value (the same kernel). */
int frcnn_sgd_momentum(float* w, float* v, const float* g, long n, float lr, float momentum, float weight_decay, void* stream);

/* bf16 gradient bucket for the multi-GPU step (train_rpn.py:169-174 ParallelUpdater; BASELINE config #5 "bf16, NCCL grad
 * allreduce"): frcnn_cast_f32_bf16 rounds a bucket of fp32 gradients to bf16 for the all-reduce (src 16-byte, dst 8-byte
 * aligned), frcnn_sgd_momentum_bf16g is frcnn_sgd_momentum reading the reduced bf16 gradient (fp32 masters / momentum). */
int frcnn_cast_f32_bf16(const float* src, void* dst_bf16, long n, void* stream);
int frcnn_sgd_momentum_bf16g(float* w, float* v, const void* g_bf16, long n, float lr, float momentum, float weight_decay,
                             void* stream);

/* The optimizer step of every trainer: chainer.optimizer.WeightDecay(rate) hook + one of Chainer v1's rules, on n float32
 * master weights w with the rule's float32 state s0 (and s1), each element on its own.  g: n float32 gradients, or
 * (g_bf16 = 1) the bf16 bucket of the multi-GPU exchange, widened exactly.  hyper: FRCNN_OPT_HYPER_LEN float32 values in
 * DEVICE memory, read when the kernel runs -- so a launch captured into a CUDA graph uses whatever was written there
 * before each replay.  The arithmetic is update_one_cpu of Chainer 1.22 in float32, every operation correctly rounded on
 * its own in the order written (no contraction), after g' = fma(rate, w, g):
 *   FRCNN_OPT_MOMENTUM_SGD  s0 = v              hyper {rate, lr, momentum}
 *       v = momentum*v - lr*g';  w = w + v                         (frcnn_sgd_momentum, bit for bit)
 *   FRCNN_OPT_ADAM          s0 = m, s1 = v      hyper {rate, lr_t, 1-beta1, 1-beta2, eps}
 *       m = m + (1-beta1)*(g' - m);  v = v + (1-beta2)*(g'*g' - v);  w = w - (lr_t*m) / (sqrt(v) + eps)
 *       lr_t = alpha * sqrt(1 - beta2^t) / (1 - beta1^t) for update t = 1, 2, ... (Chainer's Adam.lr), in float64 on the
 *       host and rounded once to float32
 *   FRCNN_OPT_ADAGRAD       s0 = h              hyper {rate, lr, eps}
 *       h = h + g'*g';  w = w - (lr*g') / (sqrt(h) + eps)
 *   FRCNN_OPT_RMSPROP       s0 = ms             hyper {rate, lr, alpha, 1-alpha, eps}
 *       ms = ms*alpha;  ms = ms + ((1-alpha)*g')*g';  w = w - (lr*g') / (sqrt(ms) + eps)
 * Constants such as 1-beta1 are computed in float64 and rounded to float32 by the caller, as NumPy rounds a Python float
 * that meets a float32 array; entries past the rule's list are not read.  s1 must be NULL for the one-state rules.
 * Memory traffic: 20 bytes per element (Adam 28; 2 fewer with a bf16 gradient).  An unknown rule, a NULL pointer, s1
 * given or missing against the rule, g_bf16 outside {0, 1} or n < 0 -> FRCNN_ERR_ARG; n = 0 launches nothing. */
#define FRCNN_OPT_MOMENTUM_SGD 0
#define FRCNN_OPT_ADAM 1
#define FRCNN_OPT_ADAGRAD 2
#define FRCNN_OPT_RMSPROP 3
#define FRCNN_OPT_HYPER_LEN 5
int frcnn_optimizer_update(int rule, float* w, float* s0, float* s1, const void* g, int g_bf16, long n, const float* hyper,
                           void* stream);

/* Weights of the data-gradient convolution: out[t][ci][co] = W[co][ci][kh-1-r][kw-1-s] (t = r*kw+s), bf16 hi/lo, co
 * zero-padded to Cout_pad -- feed to frcnn_conv2d with Cin := Cout_pad, Cout := Cin. */
int frcnn_pack_conv_weights_dgrad(const float* w_oihw, int Cout, int Cin, int kh, int kw, int Cout_pad, void* w_hi, void* w_lo,
                                  void* stream);

/* Profiling hook (not part of the drop-in surface): a device buffer of 8 int64 that receives the
 * per-phase clock64() stamps of subsequent top-k sort launches; NULL disables.  A batched launch
 * (frcnn_proposals_batch) records image 0 only. */
void frcnn_debug_sort_clocks(long long* dev_buf);

#ifdef __cplusplus
}
#endif
#endif /* FRCNN_B200_H_ */
