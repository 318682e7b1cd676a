// rcnn_train.cu -- the RCNN-head training step on device (SURVEY.md 8f rank 4, train_rcnn.py / models/faster_rcnn.py:136-173).
//
// Replaces (all under /root/reference):
//   models/proposal_target_layer.py:76-150  ProposalTargetLayer: IoU of every proposal with the ground truth (float64,
//                                           bbox.pyx order -- the reference copies proposals to the HOST for it), matched
//                                           gt rows, float32 bbox_transform, class-wise regression targets
//   models/faster_rcnn.py:151-165           the two RCNN losses on the kept rows (21-way softmax cross entropy against
//                                           use_gt_boxes[:, 4]; Huber delta, per-row sums averaged over the rows) and, in the
//                                           same pass, d(loss_rcnn)/d(cls_score | bbox_pred)
//   F.dropout (faster_rcnn.py:127-128)      y = x * mask / (1 - ratio) with an explicit mask (the reference draws it from
//                                           Chainer's RNG: unpinnable; the mask is an input here)
//   F.roi_pooling_2d backward               the gradient of each pooled bin goes to the bin's first maximum; summed with
//                                           64-bit fixed-point atomics (order independent: bit-reproducible), then converted
// Small latency-bound kernels (<= 300 RoIs): no tensor cores by design.
#include "common.cuh"
#include "nms_math.cuh"

namespace frcnn {

__global__ void roi_overlaps_kernel(const float* __restrict__ rois, const int* __restrict__ count, int R_cap,
                                    const float* __restrict__ gt, int n_gt, double* __restrict__ max_ov, int* __restrict__ argmax) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R_cap) return;
    const int R = count ? min(*count, R_cap) : R_cap;
    double best = -1.0;
    int bi = -1;
    if (r < R) {
        const float4 rb = reinterpret_cast<const float4*>(rois)[r];
        const double b[4] = {rb.x, rb.y, rb.z, rb.w};
        for (int g = 0; g < n_gt; ++g) {
            const float* gr = gt + (size_t)g * 5;
            const double q[4] = {gr[0], gr[1], gr[2], gr[3]};
            const double ov = iou_f64(b, q, box_area_f64(q[0], q[1], q[2], q[3]));   // bbox.pyx on (double)proposal x (double)gt row
            if (ov > best) { best = ov; bi = g; }          // first maximum (numpy argmax)
        }
    }
    max_ov[r] = best;
    argmax[r] = bi;
}

// float32 bbox_transform (bbox_transform.py:18-38 with float32 operands) + class-wise scatter (proposal_target_layer.py:138-147)
__global__ void roi_targets_kernel(const float* __restrict__ rois, const float* __restrict__ gt, const int* __restrict__ argmax,
                                   const int* __restrict__ keep, int n, int num_classes, float* __restrict__ use_gt,
                                   float* __restrict__ ext, int* __restrict__ labels) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = keep[i];
    const float4 e = reinterpret_cast<const float4*>(rois)[r];
    const float* q = gt + (size_t)argmax[r] * 5;
    for (int j = 0; j < 5; ++j) use_gt[i * 5 + j] = q[j];
    const float ew = __fadd_rn(__fsub_rn(e.z, e.x), 1.0f), eh = __fadd_rn(__fsub_rn(e.w, e.y), 1.0f);
    const float ecx = __fadd_rn(e.x, __fmul_rn(0.5f, ew)), ecy = __fadd_rn(e.y, __fmul_rn(0.5f, eh));
    const float gw = __fadd_rn(__fsub_rn(q[2], q[0]), 1.0f), gh = __fadd_rn(__fsub_rn(q[3], q[1]), 1.0f);
    const float gcx = __fadd_rn(q[0], __fmul_rn(0.5f, gw)), gcy = __fadd_rn(q[1], __fmul_rn(0.5f, gh));
    const float t[4] = {__fdiv_rn(__fsub_rn(gcx, ecx), ew), __fdiv_rn(__fsub_rn(gcy, ecy), eh),
                        logf(__fdiv_rn(gw, ew)), logf(__fdiv_rn(gh, eh))};
    const int cls = (int)q[4];
    labels[i] = cls;                                        // faster_rcnn.py:154: use_gt_boxes[:, -1]
    float* row = ext + (size_t)i * 4 * num_classes;
    for (int j = 0; j < 4 * num_classes; ++j) row[j] = 0.f;
    if (q[4] > 0.f && cls < num_classes)
        for (int j = 0; j < 4; ++j) row[4 * cls + j] = t[j];
}

// Stand-alone array helpers of models/bbox_transform.py (training side): bbox_transform (:18-38) on float32 rows and the
// keep_inside predicate (:112-130).  gt rows may be wider than 4 (gt_stride floats per row).
__global__ void bbox_transform_kernel(const float* __restrict__ ex, const float* __restrict__ gt, int gt_stride, int n,
                                      float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 e = reinterpret_cast<const float4*>(ex)[i];
    const float* q = gt + (size_t)i * gt_stride;
    const float ew = __fadd_rn(__fsub_rn(e.z, e.x), 1.0f), eh = __fadd_rn(__fsub_rn(e.w, e.y), 1.0f);
    const float ecx = __fadd_rn(e.x, __fmul_rn(0.5f, ew)), ecy = __fadd_rn(e.y, __fmul_rn(0.5f, eh));
    const float gw = __fadd_rn(__fsub_rn(q[2], q[0]), 1.0f), gh = __fadd_rn(__fsub_rn(q[3], q[1]), 1.0f);
    const float gcx = __fadd_rn(q[0], __fmul_rn(0.5f, gw)), gcy = __fadd_rn(q[1], __fmul_rn(0.5f, gh));
    reinterpret_cast<float4*>(out)[i] = make_float4(__fdiv_rn(__fsub_rn(gcx, ecx), ew), __fdiv_rn(__fsub_rn(gcy, ecy), eh),
                                                   logf(__fdiv_rn(gw, ew)), logf(__fdiv_rn(gh, eh)));
}

__global__ void keep_inside_kernel(const float* __restrict__ boxes, int n, float im_h, float im_w, unsigned char* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 b = reinterpret_cast<const float4*>(boxes)[i];
    flags[i] = (b.x >= 0.f && b.y >= 0.f && b.z < im_w && b.w < im_h) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------ losses + head gradient
// One warp per kept row; per-row results go to shared memory and thread 0 adds them in row order (deterministic).
__global__ void __launch_bounds__(1024) rcnn_loss_kernel(const float* __restrict__ head, int ld, int R_cap, const int* __restrict__ keep,
                                                        int n, const int* __restrict__ labels, const float* __restrict__ ext,
                                                        int num_classes, double delta, double grad_scale,
                                                        float* __restrict__ losses, float* __restrict__ dhead) {
    __shared__ double s_ce[128], s_hub[128], s_ok[128];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    if (dhead != nullptr)
        for (long i = threadIdx.x; i < (long)R_cap * ld; i += blockDim.x) dhead[i] = 0.f;
    __syncthreads();
    for (int i = warp; i < n; i += nwarp) {
        const int r = keep[i];
        const float* z = head + (size_t)r * ld;
        const int t = labels[i];
        // 21-way log-softmax in double
        double m = -1e300;
        for (int c = lane; c < num_classes; c += 32) m = fmax(m, (double)z[c]);
        for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
        double se = 0.0;
        for (int c = lane; c < num_classes; c += 32) se += exp((double)z[c] - m);
        for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
        const double lse = m + log(se);
        // arg-max (first maximum) for the accuracy
        int am = 0;
        double av = -1e300;
        for (int c = 0; c < num_classes; ++c) { const double v = z[c]; if (v > av) { av = v; am = c; } }
        double hub = 0.0;
        const int nb = 4 * num_classes;
        for (int j = lane; j < nb; j += 32) {
            const double d = (double)z[num_classes + j] - (double)ext[(size_t)i * nb + j];
            const double ad = fabs(d);
            hub += ad < delta ? 0.5 * d * d : delta * (ad - 0.5 * delta);
            if (dhead) dhead[(size_t)r * ld + num_classes + j] = (float)((ad < delta ? d : (d > 0 ? delta : -delta)) * grad_scale / n);
        }
        for (int o = 16; o > 0; o >>= 1) hub += __shfl_xor_sync(0xffffffffu, hub, o);
        // softmax as exp(z - m) / se, not exp(z - lse): at |m| beyond ~2^29 lse = m + log(se) rounds log(se) away and
        // classes tied at the maximum would each get probability 1
        if (dhead)
            for (int c = lane; c < num_classes; c += 32)
                dhead[(size_t)r * ld + c] = (float)((exp((double)z[c] - m) / se - (c == t ? 1.0 : 0.0)) * grad_scale / n);
        // a ground-truth class outside [0, num_classes) (a dataset with another class count, a NaN label) must not index the
        // score row: its loss becomes NaN -- loud in the reported loss, the caller's check -- instead of a silently wrong value
        const bool t_ok = t >= 0 && t < num_classes;
        if (lane == 0) { s_ce[i] = t_ok ? lse - (double)z[t] : nan(""); s_hub[i] = hub; s_ok[i] = am == t ? 1.0 : 0.0; }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ce = 0, hub = 0, ok = 0;
        for (int i = 0; i < n; ++i) { ce += s_ce[i]; hub += s_hub[i]; ok += s_ok[i]; }
        const double dn = n > 0 ? (double)n : 1.0;
        losses[0] = (float)(ce / dn);
        losses[1] = (float)(hub / dn);
        losses[2] = (float)(ok / dn);
        losses[3] = (float)(ce / dn + hub / dn);
    }
}

// ------------------------------------------------------------------------------------------ dropout with an explicit mask
__global__ void dropout_kernel(__nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, const unsigned char* __restrict__ mask,
                               long n, float scale) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float k = mask[i] ? scale : 0.f;                  // scale = 1/(1-ratio) = 2: exact on both planes
    hi[i] = __float2bfloat16_rn(__bfloat162float(hi[i]) * k);
    if (lo) lo[i] = __float2bfloat16_rn(__bfloat162float(lo[i]) * k);
}

// ------------------------------------------------------------------------------------------ RoI pooling backward
constexpr double FIX_SCALE = 17592186044416.0;              // 2^44: sums of |g| up to 2^19 with a 5.7e-14 quantum

// One thread per (roi, bin, 8 channels): rescans its window with the forward kernel's bins (roi_bin) and pair values
// (pool_pair_value), from -inf with a strict '>' (the first maximum in (y, x) order; a window with no number above -inf
// routes nothing) and adds the bin's gradient to the arg-max position of a 64-bit fixed-point map (integer atomics commute:
// the result does not depend on the order of arrival).
__global__ void roi_pool_backward_kernel(const __nv_bfloat16* __restrict__ fh, const __nv_bfloat16* __restrict__ fl, int H, int W,
                                         int C, const float* __restrict__ rois, const int* __restrict__ count, int R_cap, int PH,
                                         int PW, float scale, const __nv_bfloat16* __restrict__ gh, const __nv_bfloat16* __restrict__ gl,
                                         long long* __restrict__ dfix) {
    const int C8 = C / 8;
    const long total = (long)R_cap * PH * PW * C8;
    const int R = count ? min(*count, R_cap) : R_cap;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        long t = i / C8;
        const int pw = (int)(t % PW); t /= PW;
        const int ph = (int)(t % PH);
        const int r = (int)(t / PH);
        if (r >= R) continue;
        const float4 roi = reinterpret_cast<const float4*>(rois)[r];
        const int2 bh = roi_bin(roi_coord(roi.y, scale), roi_coord(roi.w, scale), PH, ph, H);
        const int2 bw = roi_bin(roi_coord(roi.x, scale), roi_coord(roi.z, scale), PW, pw, W);
        const int hs = bh.x, he = bh.y, ws = bw.x, we = bw.y;
        if (!(he > hs && we > ws)) continue;
        float m[8];
        int am[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { m[j] = -INFINITY; am[j] = -1; }       // NaN and -inf never win: no gradient
        for (int y = hs; y < he; ++y)
            for (int x = ws; x < we; ++x) {
                const long off = ((long)y * W + x) * C + 8 * c8;
                const uint4 h4 = *reinterpret_cast<const uint4*>(fh + off);
                const __nv_bfloat16* hb = reinterpret_cast<const __nv_bfloat16*>(&h4);
                uint4 l4 = make_uint4(0, 0, 0, 0);
                if (fl) l4 = *reinterpret_cast<const uint4*>(fl + off);
                const __nv_bfloat16* lb = reinterpret_cast<const __nv_bfloat16*>(&l4);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float v = pool_pair_value(__bfloat162float(hb[j]), __bfloat162float(lb[j]));
                    if (v > m[j]) { m[j] = v; am[j] = y * W + x; }
                }
            }
        const long goff = (((long)r * PH + ph) * PW + pw) * C + 8 * c8;
        const uint4 g4 = *reinterpret_cast<const uint4*>(gh + goff);
        const __nv_bfloat16* ghb = reinterpret_cast<const __nv_bfloat16*>(&g4);
        uint4 gl4 = make_uint4(0, 0, 0, 0);
        if (gl) gl4 = *reinterpret_cast<const uint4*>(gl + goff);
        const __nv_bfloat16* glb = reinterpret_cast<const __nv_bfloat16*>(&gl4);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const double g = (double)__bfloat162float(ghb[j]) + (double)__bfloat162float(glb[j]);
            if (am[j] >= 0 && g != 0.0)
                atomicAdd(reinterpret_cast<unsigned long long*>(dfix + (long)am[j] * C + 8 * c8 + j),
                          (unsigned long long)__double2ll_rn(g * FIX_SCALE));
        }
    }
}

__global__ void fixed_to_float_kernel(const long long* __restrict__ dfix, long n, float* __restrict__ out) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)((double)dfix[i] / FIX_SCALE);
}

}  // namespace frcnn

using namespace frcnn;

extern "C" {

int frcnn_roi_overlaps(const float* rois, const int* count, int R_cap, const float* gt_boxes, int n_gt, double* max_overlaps,
                       int* argmax, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(rois && gt_boxes && max_overlaps && argmax && R_cap > 0 && n_gt > 0, "roi_overlaps: bad arguments");
    roi_overlaps_kernel<<<cdiv(R_cap, 128), 128, 0, (cudaStream_t)stream>>>(rois, count, R_cap, gt_boxes, n_gt, max_overlaps, argmax);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_roi_targets(const float* rois, const float* gt_boxes, const int* argmax, const int* keep_inds, int n, int num_classes,
                      float* use_gt_boxes, float* bbox_reg_targets, int* labels, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(rois && gt_boxes && argmax && keep_inds && use_gt_boxes && bbox_reg_targets && labels && n >= 0 && num_classes > 0,
                  "roi_targets: bad arguments");
    if (n == 0) return FRCNN_OK;
    roi_targets_kernel<<<cdiv(n, 128), 128, 0, (cudaStream_t)stream>>>(rois, gt_boxes, argmax, keep_inds, n, num_classes,
                                                                     use_gt_boxes, bbox_reg_targets, labels);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_bbox_transform(const float* ex_rois, const float* gt_rois, int gt_stride, int n, float* out, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(n >= 0 && gt_stride >= 4, "bbox_transform: bad arguments");
    if (n == 0) return FRCNN_OK;
    FRCNN_REQUIRE(ex_rois && gt_rois && out, "bbox_transform: null pointer");
    bbox_transform_kernel<<<cdiv(n, 128), 128, 0, (cudaStream_t)stream>>>(ex_rois, gt_rois, gt_stride, n, out);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_keep_inside(const float* boxes, int n, int im_h, int im_w, unsigned char* flags, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(n >= 0, "keep_inside: bad arguments");
    if (n == 0) return FRCNN_OK;
    FRCNN_REQUIRE(boxes && flags, "keep_inside: null pointer");
    keep_inside_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(boxes, n, (float)im_h, (float)im_w, flags);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_rcnn_loss(const float* head_out, int ld, int R_cap, const int* keep_inds, int n, const int* labels,
                    const float* bbox_reg_targets, int num_classes, double delta, double grad_scale, float* losses, float* dhead,
                    void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(head_out && keep_inds && labels && bbox_reg_targets && losses && R_cap > 0 && num_classes >= 1 &&
                  ld / 5 >= num_classes, "rcnn_loss: bad arguments");                   // ld >= 5*num_classes, no overflow
    FRCNN_REQUIRE(n >= 1 && n <= 128, "rcnn_loss: 1 <= kept rows <= 128 (ROIS_PER_IMAGE), got %d", n);
    FRCNN_REQUIRE(delta > 0, "rcnn_loss: delta must be positive");
    rcnn_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(head_out, ld, R_cap, keep_inds, n, labels, bbox_reg_targets, num_classes,
                                                          delta, grad_scale, losses, dhead);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_dropout(void* x_hi, void* x_lo, const unsigned char* mask, long n, float scale, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(x_hi && mask && n >= 0, "dropout: bad arguments");
    if (n == 0) return FRCNN_OK;
    dropout_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)x_hi, (__nv_bfloat16*)x_lo, mask, n, scale);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

size_t frcnn_roi_pool_backward_workspace_bytes(int H, int W, int C) { return (size_t)H * W * C * sizeof(long long); }

int frcnn_roi_pool_backward(const void* feat_hi, const void* feat_lo, int H, int W, int C, const float* rois, const int* count,
                            int R_cap, int outh, int outw, float scale, const void* g_hi, const void* g_lo, float* dfeat,
                            void* workspace, size_t workspace_bytes, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(feat_hi && rois && g_hi && dfeat && workspace && H > 0 && W > 0 && C > 0 && C % 8 == 0 && R_cap > 0,
                  "roi_pool_backward: bad arguments");
    if (workspace_bytes < frcnn_roi_pool_backward_workspace_bytes(H, W, C)) {
        set_error("roi_pool_backward: workspace %zu < %zu bytes", workspace_bytes, frcnn_roi_pool_backward_workspace_bytes(H, W, C));
        return FRCNN_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const long n = (long)H * W * C;
    FRCNN_CUDA_OK(cudaMemsetAsync(workspace, 0, n * sizeof(long long), st));
    const long total = (long)R_cap * outh * outw * (C / 8);
    long grid = (total + 255) / 256;
    if (grid > 132l * 16) grid = 132l * 16;
    roi_pool_backward_kernel<<<(unsigned)grid, 256, 0, st>>>((const __nv_bfloat16*)feat_hi, (const __nv_bfloat16*)feat_lo, H, W, C, rois,
                                                            count, R_cap, outh, outw, scale, (const __nv_bfloat16*)g_hi,
                                                            (const __nv_bfloat16*)g_lo, (long long*)workspace);
    FRCNN_LAUNCH_OK();
    fixed_to_float_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const long long*)workspace, n, dfeat);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

}  // extern "C"
