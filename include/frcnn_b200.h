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
 * frcnn_linear GEMM launch: copies min(n, 12) ints to out in the order BN, BK, x3, promote (long-K partial sums), CTA
 * group, tile_h, tile_w, pipeline stages, grid (CTAs), tiles (pair-tiles for CTA pairs, all split-K parts included),
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

/* F.roi_pooling_2d(feature_map, [0|rois], outh, outw, scale) (models/faster_rcnn.py:123-126), Caffe
 * semantics.  feat [H,W,C] bf16 hi(/lo); rois [R_cap,4] fp32; *count valid rows (NULL = R_cap).
 * out_hi/out_lo: [R_cap, outh*outw, C] bf16 (row = one RoI, K order (ph,pw,c)); rows >= count are 0.
 * out_f32 (optional): same layout in fp32.  outh, outw < 32; C a multiple of 8. */
int frcnn_roi_pool(const void* feat_hi, const void* feat_lo, int H, int W, int C, const float* rois,
                   const int* count, int R_cap, int outh, int outw, float scale, void* out_hi, void* out_lo,
                   float* out_f32, void* stream);

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

/* Head tail (models/faster_rcnn.py:175-178): softmax over num_classes scores + per-class
 * bbox_transform_inv + clip_boxes.  scores element (r,c) at scores[r*ld + c], deltas (r,j) at
 * deltas[r*ld + j] (same ld).  out_prob [R_cap,num_classes], out_boxes [R_cap,4*num_classes];
 * rows >= *count are zero. */
int frcnn_head_decode(const float* scores, const float* deltas, int ld, const float* rois, const int* count,
                      int R_cap, int num_classes, int im_h, int im_w, float* out_prob, float* out_boxes,
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
 *                     bit-for-bit without that host state; no host sync;
 *                  2: disable_pos[n_disable] = positions in the inside-compact arrays to set to -1
 *                     (exactly what the reference's np.random.choice calls return).
 * Outputs (device): labels_full int32 [n_all] in {-1,0,1}, -1 for anchors outside the image
 *   (= bbox_labels_mapped of region_proposal_network.py:164-165); targets_full float32 [n_all,4]
 *   (16-byte aligned; zeros outside); inds_inside int32 [n_all capacity] (ascending);
 *   counts int32 [8] = {n_inside, n_fg, n_bg, n_fg before subsampling, n_bg before, n_all, 0, 0}.
 * The reference's compact outputs are labels_full[inds_inside], targets_full[inds_inside]. */
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

/* ---- RCNN-head training (rcnn_train.cu; train_rcnn.py, models/faster_rcnn.py:136-173) ---- */

/* ProposalTargetLayer, part 1 (proposal_target_layer.py:91-96): best ground-truth overlap of every proposal, float64 in
 * bbox.pyx order.  rois [R_cap,4] fp32 (*count valid, NULL = R_cap), gt_boxes [n_gt,5]; max_overlaps double [R_cap]
 * (-1 for rows >= count), argmax int32 [R_cap].  The fg/bg sampling (:99-129) draws from NumPy's RNG on the host in the
 * reference; the caller does the same (or any other rule) on these two small arrays and passes keep_inds to part 2. */
int frcnn_roi_overlaps(const float* rois, const int* count, int R_cap, const float* gt_boxes, int n_gt, double* max_overlaps,
                       int* argmax, void* stream);
/* part 2 (:138-147): use_gt_boxes [n,5] = gt[argmax[keep]], labels int32 [n] = use_gt_boxes[:,4] (faster_rcnn.py:154),
 * bbox_reg_targets [n, 4*num_classes] = float32 bbox_transform of the kept proposal scattered to its class's 4 columns
 * (rows whose class is 0 stay zero). */
int frcnn_roi_targets(const float* rois, const float* gt_boxes, const int* argmax, const int* keep_inds, int n, int num_classes,
                      float* use_gt_boxes, float* bbox_reg_targets, int* labels, void* stream);
/* Array-level helpers of models/bbox_transform.py used by the training code: bbox_transform (:18-38) on float32 rows
 * (ex_rois [n,4], gt rows gt_stride >= 4 floats apart) -> out [n,4] (dx, dy, dw, dh); keep_inside (:112-130) as a 0/1 flag
 * per box: x1 >= 0, y1 >= 0, x2 < im_w, y2 < im_h. */
int frcnn_bbox_transform(const float* ex_rois, const float* gt_rois, int gt_stride, int n, float* out, void* stream);
int frcnn_keep_inside(const float* boxes, int n, int im_h, int im_w, unsigned char* flags, void* stream);
/* faster_rcnn.py:151-165 on the merged head output head_out [R_cap][ld] (columns [0,num_classes) scores, then
 * 4*num_classes deltas): losses float32 [4] = {loss_cls, loss_bbox, cls_accuracy, loss_rcnn}; dhead (optional, same shape)
 * = grad_scale * d(loss_rcnn)/d(head_out), zero on rows not kept.  1 <= n <= 128. */
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

/* ---- the backward pass of the reference's training steps.  In the reference it is `loss.backward()` inside Chainer's
 * updater (train_rpn.py:169-174 / train_rcnn.py with StandardUpdater or ParallelUpdater; the graph is the one
 * models/vgg16.py:38-82, models/region_proposal_network.py:117-120 and models/faster_rcnn.py:123-134 build) followed by
 * MomentumSGD + WeightDecay (train_rpn.py:165-167).  Chainer's per-function backward code is un-vendored; these entry
 * points are its replacement: L.Convolution2D / L.Linear backward-data = frcnn_conv2d on frcnn_pack_conv_weights_dgrad,
 * backward-filter = frcnn_gemm_nt_splitk (+ frcnn_wgrad_reduce, frcnn_bias_grad), F.relu / F.max_pooling_2d / F.dropout
 * backward = frcnn_grad_prepare, F.roi_pooling_2d backward = frcnn_roi_pool_backward, the optimizer = frcnn_sgd_momentum. */

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

/* dw[m][n][g] (the reference's OIHW float32, g = r*3+s or 1) = scale * sum over splits of parts[g][s][m][n], m < M;
 * parts slabs have M_parts >= M rows of ld floats. */
int frcnn_wgrad_reduce(const float* parts, int groups, int splits, int M_parts, int M, int ld, int N, float scale, float* dw,
                       void* stream);

/* db[c] = scale * sum over k of (t_hi + t_lo)[c][k] -- the bias gradient from the transposed dY. */
int frcnn_bias_grad(const void* t_hi, const void* t_lo, int C, long Kp, float scale, float* db, void* stream);

/* chainer.optimizer.WeightDecay(rate) hook + optimizers.MomentumSGD(lr, momentum) (train_rpn.py:165-167) on float32
 * master weights: g' = g + rate*w; v = momentum*v - lr*g'; w += v. */
int frcnn_sgd_momentum(float* w, float* v, const float* g, long n, float lr, float momentum, float weight_decay, void* stream);

/* bf16 gradient bucket for the multi-GPU step (train_rpn.py:169-174 ParallelUpdater; BASELINE config #5 "bf16, NCCL grad
 * allreduce"): frcnn_cast_f32_bf16 rounds a bucket of fp32 gradients to bf16 for the all-reduce (src 16-byte, dst 8-byte
 * aligned), frcnn_sgd_momentum_bf16g is frcnn_sgd_momentum reading the reduced bf16 gradient (fp32 masters / momentum). */
int frcnn_cast_f32_bf16(const float* src, void* dst_bf16, long n, void* stream);
int frcnn_sgd_momentum_bf16g(float* w, float* v, const void* g_bf16, long n, float lr, float momentum, float weight_decay,
                             void* stream);

/* Weights of the data-gradient convolution: out[t][ci][co] = W[co][ci][kh-1-r][kw-1-s] (t = r*kw+s), bf16 hi/lo, co
 * zero-padded to Cout_pad -- feed to frcnn_conv2d with Cin := Cout_pad, Cout := Cin. */
int frcnn_pack_conv_weights_dgrad(const float* w_oihw, int Cout, int Cin, int kh, int kw, int Cout_pad, void* w_hi, void* w_lo,
                                  void* stream);

/* Profiling hook (not part of the drop-in surface): a device buffer of 8 int64 that receives the
 * per-phase clock64() stamps of subsequent top-k sort launches; NULL disables. */
void frcnn_debug_sort_clocks(long long* dev_buf);

#ifdef __cplusplus
}
#endif
#endif /* FRCNN_B200_H_ */
