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

// Best ground-truth overlap of one proposal (bbox.pyx on (double)proposal x (double)gt row); -1 / -1 when no overlap is
// above -1 (no gt row, or every IoU NaN)
__device__ __forceinline__ double roi_best_overlap(float4 rb, const float* __restrict__ gt, int n_gt, int& bi) {
    const double b[4] = {rb.x, rb.y, rb.z, rb.w};
    double best = -1.0;
    bi = -1;
    for (int g = 0; g < n_gt; ++g) {
        const float* gr = gt + (size_t)g * 5;
        const double q[4] = {gr[0], gr[1], gr[2], gr[3]};
        const double ov = iou_f64(b, q, box_area_f64(q[0], q[1], q[2], q[3]));
        if (ov > best) { best = ov; bi = g; }              // first maximum (numpy argmax)
    }
    return best;
}

__global__ void roi_overlaps_kernel(const float* __restrict__ rois, const int* __restrict__ count, int R_cap,
                                    const float* __restrict__ gt, int n_gt, double* __restrict__ max_ov, int* __restrict__ argmax) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R_cap) return;
    const int R = count ? min(*count, R_cap) : R_cap;
    double best = -1.0;
    int bi = -1;
    if (r < R) best = roi_best_overlap(reinterpret_cast<const float4*>(rois)[r], gt, n_gt, bi);
    max_ov[r] = best;
    argmax[r] = bi;
}

// One kept row of part 3: float32 bbox_transform (bbox_transform.py:18-38 with float32 operands) of proposal e against its
// matched gt row gt[am], scattered to the class's 4 columns (proposal_target_layer.py:138-147).  A row without an overlap
// (am = -1: no gt row, or every IoU NaN) takes gt row 0, as NumPy's argmax of an all-NaN row does.
__device__ __forceinline__ void roi_target_row(float4 e, const float* __restrict__ gt, int am, int num_classes,
                                               float* __restrict__ use_gt, float* __restrict__ row, int* __restrict__ label) {
    const float* q = gt + (size_t)max(am, 0) * 5;
    for (int j = 0; j < 5; ++j) use_gt[j] = q[j];
    const float ew = __fadd_rn(__fsub_rn(e.z, e.x), 1.0f), eh = __fadd_rn(__fsub_rn(e.w, e.y), 1.0f);
    const float ecx = __fadd_rn(e.x, __fmul_rn(0.5f, ew)), ecy = __fadd_rn(e.y, __fmul_rn(0.5f, eh));
    const float gw = __fadd_rn(__fsub_rn(q[2], q[0]), 1.0f), gh = __fadd_rn(__fsub_rn(q[3], q[1]), 1.0f);
    const float gcx = __fadd_rn(q[0], __fmul_rn(0.5f, gw)), gcy = __fadd_rn(q[1], __fmul_rn(0.5f, gh));
    const float t[4] = {__fdiv_rn(__fsub_rn(gcx, ecx), ew), __fdiv_rn(__fsub_rn(gcy, ecy), eh),
                        logf(__fdiv_rn(gw, ew)), logf(__fdiv_rn(gh, eh))};
    const int cls = (int)q[4];
    *label = cls;                                           // faster_rcnn.py:154: use_gt_boxes[:, -1]
    for (int j = 0; j < 4 * num_classes; ++j) row[j] = 0.f;
    if (q[4] > 0.f && cls < num_classes)
        for (int j = 0; j < 4; ++j) row[4 * cls + j] = t[j];
}

__global__ void roi_targets_kernel(const float* __restrict__ rois, const float* __restrict__ gt, const int* __restrict__ argmax,
                                   const int* __restrict__ keep, int n, int num_classes, float* __restrict__ use_gt,
                                   float* __restrict__ ext, int* __restrict__ labels) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = keep[i];
    roi_target_row(reinterpret_cast<const float4*>(rois)[r], gt, argmax[r], num_classes, use_gt + i * 5,
                   ext + (size_t)i * 4 * num_classes, labels + i);
}

// ------------------------------------------------------------------------------------------ ProposalTargetLayer over N slots
constexpr int PT_ROWS_MAX = 4096, PT_KEEP = 128, PT_FG = 32, PT_THREADS = 512;   // ROIS_PER_IMAGE, FG_FRACTION * 128

struct PropTargetArgs {
    const float* rois; long rois_stride; const int* count; long count_stride; int R_cap;
    const float* gt; int max_gt; const int* gt_counts; int num_classes;
    int mode; const unsigned long long* seeds; const int* keep_list; int n_list; const int* list_offsets;
    int* keep; int* labels; float* use_gt; float* targets; double* max_ov; int* argmax; int* counts;
};

// Appends, in ascending r, every r < R with pred(r) to out[base ...]; returns the new base.  Block-uniform.
template <typename Pred>
__device__ int block_append(int R, Pred pred, int* out, int base, int* s_warp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    for (int r0 = 0; r0 < R; r0 += blockDim.x) {
        const int r = r0 + threadIdx.x;
        const bool f = r < R && pred(r);
        const unsigned m = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < nwarp; ++w) { before += w < warp ? s_warp[w] : 0; total += s_warp[w]; }
        if (f) out[base + before + __popc(m & ((1u << lane) - 1u))] = r;
        base += total;
        __syncthreads();
    }
    return base;
}

// One CTA per slot: part 1 (overlaps), part 2 (the kept set), part 3 (the targets of the kept rows)
__global__ void __launch_bounds__(PT_THREADS) proposal_targets_kernel(PropTargetArgs a) {
    __shared__ unsigned long long s_key[PT_ROWS_MAX];
    __shared__ unsigned char s_cls[PT_ROWS_MAX];            // 1: fg, 2: bg, 0: neither
    __shared__ unsigned char s_kept[PT_ROWS_MAX];
    __shared__ int s_keep[PT_KEEP];
    __shared__ int s_warp[32];
    __shared__ int s_n[2];
    const int n = blockIdx.x, R_cap = a.R_cap;
    const float* __restrict__ rois = a.rois + (long)n * a.rois_stride;
    const float* __restrict__ gt = a.gt + (size_t)n * a.max_gt * 5;
    const int n_gt = min(max(__ldg(a.gt_counts + n), 0), a.max_gt);
    int R = a.count ? min(max(__ldg(a.count + (long)n * a.count_stride), 0), R_cap) : R_cap;
    if (n_gt < 1) R = 0;                                    // no ground truth: an empty slot
    double* __restrict__ max_ov = a.max_ov + (long)n * R_cap;
    int* __restrict__ argmax = a.argmax + (long)n * R_cap;
    const unsigned long long seed = a.mode == 1 ? __ldg(a.seeds + n) : 0ull;
    // ---- part 1 + the fg / bg sets (:99, :113-114); -1 (no overlap, NaN IoUs) is in neither
    int fg = 0, bg = 0;
    for (int r0 = 0; r0 < R_cap; r0 += blockDim.x) {
        const int r = r0 + threadIdx.x;
        unsigned char c = 0;
        if (r < R_cap) {
            double best = -1.0;
            int bi = -1;
            if (r < R) best = roi_best_overlap(reinterpret_cast<const float4*>(rois)[r], gt, n_gt, bi);
            max_ov[r] = best;
            argmax[r] = bi;
            if (r < R) {
                c = best >= 0.5 ? 1 : (best < 0.5 && best >= 0.1 ? 2 : 0);
                s_cls[r] = c;
                s_key[r] = sample_key(c == 1 ? seed : seed ^ BG_SEED_XOR, r);
            }
        }
        fg += __syncthreads_count(c == 1);
        bg += __syncthreads_count(c == 2);
    }
    int n_keep = 0, skipped = 0;
    if (a.mode == 1) {
        // min(32, |fg|) fg rows, then min(128 - n_fg, |bg|) bg rows, each the smallest keys of its set
        const int q_fg = min(PT_FG, fg), q_bg = min(PT_KEEP - q_fg, bg);
        for (int r = threadIdx.x; r < R; r += blockDim.x) {
            const unsigned char c = s_cls[r];
            int rank = 0;
            if (c != 0) {
                const unsigned long long k = s_key[r];
                for (int q = 0; q < R; ++q) rank += (s_cls[q] == c && s_key[q] < k) ? 1 : 0;
            }
            s_kept[r] = c != 0 && rank < (c == 1 ? q_fg : q_bg);
        }
        __syncthreads();
        n_keep = block_append(R, [&](int r) { return s_kept[r] && s_cls[r] == 1; }, s_keep, 0, s_warp);
        n_keep = block_append(R, [&](int r) { return s_kept[r] && s_cls[r] == 2; }, s_keep, n_keep, s_warp);
    } else {
        // the caller's list in its order; entries outside [0, R) and entries past the 128th kept one are skipped
        const int lo = min(max(__ldg(a.list_offsets + n), 0), a.n_list);
        const int hi = min(max(__ldg(a.list_offsets + n + 1), lo), a.n_list);
        if (threadIdx.x == 0) {
            int k = 0;
            for (int t = lo; t < hi; ++t) {
                const int r = __ldg(a.keep_list + t);
                if (r >= 0 && r < R && k < PT_KEEP) s_keep[k++] = r;
            }
            s_n[0] = k;
            s_n[1] = R > 0 ? (hi - lo) - k : 0;
        }
        __syncthreads();
        n_keep = s_n[0];
        skipped = s_n[1];
    }
    // ---- part 3 on the kept rows; rows past n_keep are filled with keep -1 and zeros
    int fg_kept = 0;
    for (int i0 = 0; i0 < PT_KEEP; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        bool f = false;
        if (i < PT_KEEP) {
            const long o = (long)n * PT_KEEP + i;
            const int nb = 4 * a.num_classes;
            if (i < n_keep) {
                const int r = s_keep[i];
                f = max_ov[r] >= 0.5;
                roi_target_row(reinterpret_cast<const float4*>(rois)[r], gt, argmax[r], a.num_classes, a.use_gt + o * 5,
                               a.targets + o * nb, a.labels + o);
                a.keep[o] = r;
            } else {
                for (int j = 0; j < 5; ++j) a.use_gt[o * 5 + j] = 0.f;
                for (int j = 0; j < nb; ++j) a.targets[o * nb + j] = 0.f;
                a.labels[o] = 0;
                a.keep[o] = -1;
            }
        }
        fg_kept += __syncthreads_count(f);
    }
    if (threadIdx.x == 0) {
        int* c = a.counts + 8 * n;
        c[0] = n_keep; c[1] = fg_kept; c[2] = fg; c[3] = bg; c[4] = skipped; c[5] = R; c[6] = 0; c[7] = 0;
    }
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
// One CTA per slot (blockIdx.x), one warp per kept row; per-row results go to shared memory and thread 0 adds them in row
// order (deterministic).  Slot n's head rows start at n*R_cap, its keep / labels / targets rows at n*keep_stride and its
// row count is counts[8n] when counts != NULL (else n_fixed).  One image: N = 1, counts = NULL.
__global__ void __launch_bounds__(1024) rcnn_loss_kernel(const float* __restrict__ head, int ld, int R_cap, const int* __restrict__ keep,
                                                        int n_fixed, const int* __restrict__ counts, int keep_stride,
                                                        const int* __restrict__ labels, const float* __restrict__ ext,
                                                        int num_classes, double delta, double grad_scale,
                                                        float* __restrict__ losses, float* __restrict__ dhead) {
    __shared__ double s_ce[128], s_hub[128], s_ok[128];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    const int slot = blockIdx.x;
    const int n = counts ? min(max(__ldg(counts + 8 * slot), 0), 128) : n_fixed;
    head += (size_t)slot * R_cap * ld;
    if (dhead != nullptr) dhead += (size_t)slot * R_cap * ld;
    keep += (size_t)slot * keep_stride;
    labels += (size_t)slot * keep_stride;
    ext += (size_t)slot * keep_stride * 4 * num_classes;
    losses += 4 * slot;
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

// ratio-0.5 keep masks: mask[n][i] = top bit of sample_key(seeds[n] ^ mix64(salt), i), i = r*cols + c (include/frcnn_b200.h)
__global__ void dropout_masks_kernel(const unsigned long long* __restrict__ seeds, unsigned long long salt, int per_slot,
                                     unsigned char* __restrict__ mask) {
    const unsigned long long s = __ldg(seeds + blockIdx.y) ^ mix64(salt);
    unsigned char* m = mask + (size_t)blockIdx.y * per_slot;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_slot; i += gridDim.x * blockDim.x)
        m[i] = (unsigned char)(sample_key(s, i) >> 63);
}

// ------------------------------------------------------------------------------------------ RoI pooling backward
constexpr double FIX_SCALE = 17592186044416.0;              // 2^44: sums of |g| up to 2^19 with a 5.7e-14 quantum

// One thread per (slot, roi, bin, 8 channels): rescans its window with the forward kernel's bins (roi_bin) and pair values
// (pool_pair_value), from -inf with a strict '>' (the first maximum in (y, x) order; a window with no number above -inf
// routes nothing) and adds the bin's gradient to the arg-max position of a 64-bit fixed-point map (integer atomics commute:
// the result does not depend on the order of arrival).  Slot n's map is [H][W][C] n*H*W*C elements in (its accumulator
// likewise), its RoIs sit n*rois_is floats in, its count n*count_is ints in, and its gradient rows start at row n*R_cap; on
// a canvas (extents != NULL) its bins are clamped to ceil(extent / 2^halvings), as the forward clamps them.
__global__ void roi_pool_backward_kernel(const __nv_bfloat16* __restrict__ fh, const __nv_bfloat16* __restrict__ fl, int N, int H, int W,
                                         int C, const float* __restrict__ rois, long rois_is, const int* __restrict__ count,
                                         long count_is, int R_cap, int PH, int PW, float scale, const int* __restrict__ extents,
                                         int halvings, const __nv_bfloat16* __restrict__ gh, const __nv_bfloat16* __restrict__ gl,
                                         long long* __restrict__ dfix) {
    const int C8 = C / 8;
    const long total = (long)N * R_cap * PH * PW * C8;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        long t = i / C8;
        const int pw = (int)(t % PW); t /= PW;
        const int ph = (int)(t % PH); t /= PH;
        const int r = (int)(t % R_cap);
        const int n = (int)(t / R_cap);
        const int R = count ? min(count[n * count_is], R_cap) : R_cap;
        if (r >= R) continue;
        const int lim_h = extents ? canvas_extent(extents, n, 0, halvings, H) : H;
        const int lim_w = extents ? canvas_extent(extents, n, 1, halvings, W) : W;
        const long fo = (long)n * H * W * C;
        const float4 roi = reinterpret_cast<const float4*>(rois + n * rois_is)[r];
        const int2 bh = roi_bin(roi_coord(roi.y, scale), roi_coord(roi.w, scale), PH, ph, lim_h);
        const int2 bw = roi_bin(roi_coord(roi.x, scale), roi_coord(roi.z, scale), PW, pw, lim_w);
        const int hs = bh.x, he = bh.y, ws = bw.x, we = bw.y;
        if (!(he > hs && we > ws)) continue;
        float m[8];
        int am[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { m[j] = -INFINITY; am[j] = -1; }       // NaN and -inf never win: no gradient
        for (int y = hs; y < he; ++y)
            for (int x = ws; x < we; ++x) {
                const long off = fo + ((long)y * W + x) * C + 8 * c8;
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
        const long goff = ((((long)n * R_cap + r) * PH + ph) * PW + pw) * C + 8 * c8;
        const uint4 g4 = *reinterpret_cast<const uint4*>(gh + goff);
        const __nv_bfloat16* ghb = reinterpret_cast<const __nv_bfloat16*>(&g4);
        uint4 gl4 = make_uint4(0, 0, 0, 0);
        if (gl) gl4 = *reinterpret_cast<const uint4*>(gl + goff);
        const __nv_bfloat16* glb = reinterpret_cast<const __nv_bfloat16*>(&gl4);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const double g = (double)__bfloat162float(ghb[j]) + (double)__bfloat162float(glb[j]);
            if (am[j] >= 0 && g != 0.0)
                atomicAdd(reinterpret_cast<unsigned long long*>(dfix + fo + (long)am[j] * C + 8 * c8 + j),
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
    rcnn_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(head_out, ld, R_cap, keep_inds, n, nullptr, 0, labels, bbox_reg_targets,
                                                          num_classes, delta, grad_scale, losses, dhead);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_rcnn_loss_batch(int N, const float* head, int ld, int R_cap, const int* keep, const int* labels,
                          const float* bbox_reg_targets, const int* counts, int num_classes, double delta, double grad_scale,
                          float* losses, float* dhead, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "rcnn_loss_batch: N = %d not in [1, 65535]", N);
    FRCNN_REQUIRE(head && keep && labels && bbox_reg_targets && counts && losses, "rcnn_loss_batch: null pointer");
    FRCNN_REQUIRE(R_cap > 0 && num_classes >= 1 && ld / 5 >= num_classes, "rcnn_loss_batch: bad shape R_cap=%d ld=%d num_classes=%d",
                  R_cap, ld, num_classes);
    FRCNN_REQUIRE((long)N * R_cap * ld < (1l << 40), "rcnn_loss_batch: head matrix too large");
    FRCNN_REQUIRE(delta > 0, "rcnn_loss_batch: delta must be positive");
    rcnn_loss_kernel<<<N, 1024, 0, (cudaStream_t)stream>>>(head, ld, R_cap, keep, 0, counts, 128, labels, bbox_reg_targets, num_classes,
                                                          delta, grad_scale, losses, dhead);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_dropout_masks_batch(int N, int rows, int cols, const unsigned long long* seeds, unsigned long long salt,
                              unsigned char* masks, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "dropout_masks_batch: N = %d not in [1, 65535]", N);
    FRCNN_REQUIRE(rows > 0 && cols > 0 && (long)rows * cols < (1l << 31), "dropout_masks_batch: bad shape rows=%d cols=%d", rows, cols);
    FRCNN_REQUIRE(seeds && masks, "dropout_masks_batch: null pointer");
    const int per = rows * cols;
    const int grid = min(cdiv(per, 256), 1024);
    dropout_masks_kernel<<<dim3(grid, N), 256, 0, (cudaStream_t)stream>>>(seeds, salt, per, masks);
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

size_t frcnn_roi_pool_backward_batch_workspace_bytes(int N, int H, int W, int C) {
    if (N < 1 || H < 0 || W < 0 || C < 0) return 0;
    return (size_t)N * H * W * C * sizeof(long long);
}

// zero the accumulator, route every slot's bins, convert
static int roi_pool_backward_n(const void* feat_hi, const void* feat_lo, int N, int H, int W, int C, const float* rois, long rois_is,
                               const int* count, long count_is, int R_cap, int outh, int outw, float scale, const int* extents,
                               int halvings, const void* g_hi, const void* g_lo, float* dfeat, void* workspace, cudaStream_t st) {
    const long n = (long)N * H * W * C;
    FRCNN_CUDA_OK(cudaMemsetAsync(workspace, 0, n * sizeof(long long), st));
    const long total = (long)N * R_cap * outh * outw * (C / 8);
    long grid = (total + 255) / 256;
    if (grid > 132l * 16) grid = 132l * 16;
    roi_pool_backward_kernel<<<(unsigned)grid, 256, 0, st>>>((const __nv_bfloat16*)feat_hi, (const __nv_bfloat16*)feat_lo, N, H, W, C,
                                                            rois, rois_is, count, count_is, R_cap, outh, outw, scale, extents, halvings,
                                                            (const __nv_bfloat16*)g_hi, (const __nv_bfloat16*)g_lo, (long long*)workspace);
    FRCNN_LAUNCH_OK();
    fixed_to_float_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const long long*)workspace, n, dfeat);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

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
    return roi_pool_backward_n(feat_hi, feat_lo, 1, H, W, C, rois, 0, count, 0, R_cap, outh, outw, scale, nullptr, 0, g_hi, g_lo, dfeat,
                               workspace, (cudaStream_t)stream);
}

int frcnn_roi_pool_backward_batch_ext(const void* feat_hi, const void* feat_lo, int N, int H, int W, int C, const float* rois,
                                      long rois_stride, const int* counts, long count_stride, int R_cap, int outh, int outw,
                                      float scale, const int* extents, int halvings, const void* g_hi, const void* g_lo,
                                      float* dfeat, void* workspace, size_t workspace_bytes, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "roi_pool_backward_batch_ext: N = %d not in [1, 65535]", N);
    FRCNN_REQUIRE(H > 0 && W > 0 && C > 0 && C % 8 == 0 && R_cap > 0 && outh > 0 && outw > 0,
                  "roi_pool_backward_batch_ext: bad shape H=%d W=%d C=%d R_cap=%d", H, W, C, R_cap);
    FRCNN_REQUIRE(halvings >= 0 && halvings <= 30, "roi_pool_backward_batch_ext: halvings must be in [0,30] (got %d)", halvings);
    FRCNN_REQUIRE(feat_hi && rois && g_hi && dfeat && extents, "roi_pool_backward_batch_ext: null pointer");
    FRCNN_REQUIRE(rois_stride >= 4l * R_cap && rois_stride % 4 == 0,
                  "roi_pool_backward_batch_ext: rois image stride %ld must be a multiple of 4 and >= 4*R_cap", rois_stride);
    FRCNN_REQUIRE(!counts || count_stride >= 0, "roi_pool_backward_batch_ext: count image stride must be >= 0");
    FRCNN_REQUIRE((long)N * H * W * C < (1l << 40) && (long)N * R_cap * outh * outw * C < (1l << 40),
                  "roi_pool_backward_batch_ext: too large");
    const size_t need = frcnn_roi_pool_backward_batch_workspace_bytes(N, H, W, C);
    if (!workspace || workspace_bytes < need) {
        set_error("roi_pool_backward_batch_ext: workspace %zu < %zu bytes", workspace ? workspace_bytes : 0, need);
        return FRCNN_ERR_WORKSPACE;
    }
    return roi_pool_backward_n(feat_hi, feat_lo, N, H, W, C, rois, rois_stride, counts, count_stride, R_cap, outh, outw, scale, extents,
                               halvings, g_hi, g_lo, dfeat, workspace, (cudaStream_t)stream);
}

int frcnn_proposal_targets_batch(int N, const float* rois, long rois_stride, const int* counts, long count_stride, int R_cap,
                                 const float* gt, int max_gt, const int* gt_counts, int num_classes, int mode,
                                 const unsigned long long* seeds, const int* keep_list, int n_list, const int* list_offsets,
                                 int* keep, int* labels, float* use_gt_boxes, float* bbox_reg_targets, double* max_overlaps,
                                 int* argmax, int* out_counts, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "proposal_targets_batch: N = %d not in [1, 65535]", N);
    FRCNN_REQUIRE(R_cap >= 1 && R_cap <= PT_ROWS_MAX, "proposal_targets_batch: R_cap = %d not in [1, %d]", R_cap, PT_ROWS_MAX);
    FRCNN_REQUIRE(max_gt >= 1, "proposal_targets_batch: max_gt must be at least 1 (got %d)", max_gt);
    FRCNN_REQUIRE((long)N * max_gt < (1l << 31), "proposal_targets_batch: N * max_gt = %ld ground-truth rows, must be < 2^31",
                  (long)N * max_gt);
    FRCNN_REQUIRE(num_classes >= 1 && num_classes <= 4096, "proposal_targets_batch: num_classes = %d not in [1, 4096]", num_classes);
    FRCNN_REQUIRE(rois && gt && gt_counts && keep && labels && use_gt_boxes && bbox_reg_targets && max_overlaps && argmax && out_counts,
                  "proposal_targets_batch: null pointer");
    FRCNN_REQUIRE(reinterpret_cast<uintptr_t>(rois) % 16 == 0, "proposal_targets_batch: rois must be 16-byte aligned");
    FRCNN_REQUIRE(N == 1 || (rois_stride >= 4l * R_cap && rois_stride % 4 == 0),
                  "proposal_targets_batch: rois image stride %ld must be a multiple of 4 and >= 4*R_cap", rois_stride);
    FRCNN_REQUIRE(!counts || count_stride >= 0, "proposal_targets_batch: count image stride must be >= 0");
    FRCNN_REQUIRE(mode == 1 || mode == 2, "proposal_targets_batch: mode %d not in {1 (device), 2 (list)}", mode);
    FRCNN_REQUIRE(mode != 1 || seeds, "proposal_targets_batch: mode 1 without per-slot seeds");
    FRCNN_REQUIRE(mode != 2 || (list_offsets && n_list >= 0 && (n_list == 0 || keep_list)),
                  "proposal_targets_batch: mode 2 needs the offsets [N+1] and a list of n_list >= 0 entries");
    const PropTargetArgs a{rois, rois_stride, counts, count_stride, R_cap, gt, max_gt, gt_counts, num_classes, mode, seeds,
                           keep_list, mode == 2 ? n_list : 0, list_offsets, keep, labels, use_gt_boxes, bbox_reg_targets,
                           max_overlaps, argmax, out_counts};
    proposal_targets_kernel<<<N, PT_THREADS, 0, (cudaStream_t)stream>>>(a);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

}  // extern "C"
