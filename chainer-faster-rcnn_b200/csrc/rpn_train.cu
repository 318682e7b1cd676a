// rpn_train.cu -- RPN training targets and losses on device (SURVEY.md 8f rank 1: the train_rpn.py step).
//
// Replaces (all under /root/reference):
//   models/bbox.pyx:16-56                      bbox_overlaps (float64 IoU matrix; the reference runs it on the HOST even in
//                                              GPU mode: anchor_target_layer.py:179-187 "TODO: Use bbox_overlaps for GPU")
//   models/anchor_target_layer.py:66-198       AnchorTargetLayer.__call__: all anchors (float64, no float32 cast), inside
//                                              filter (bbox_transform.py:112-130), IoU, labelling rules :131-146 (bg < 0.3,
//                                              every per-gt arg-max row = 1, >= 0.7 = 1, bg rule applied LAST so it clobbers
//                                              positives), subsampling :148-168, regression targets (bbox_transform.py:18-38)
//   models/region_proposal_network.py:160-204  the two losses (2-way softmax cross entropy with ignore -1 normalised by the
//                                              valid count; Huber delta summed over every INSIDE anchor / number of ALL anchors)
//                                              and, in the same pass, their gradients w.r.t. the RPN head outputs.
//
// All box arithmetic is float64 with one rounding per operation in the reference's order (explicit __d*_rn intrinsics, no
// FMA contraction), so labels / indices are bit-identical to the CPU oracle.  These are small latency-bound integer/float64
// kernels -- no tensor cores by design.  Subsampling: the reference draws from NumPy's global Mersenne Twister on the host;
// the device offers (0) none, (1) a counter-hash selection (deterministic in (seed, anchor index), no host sync), and
// (2) explicit index sets (how parity with a recorded reference run is pinned).
#include "common.cuh"
#include "nms_math.cuh"

namespace frcnn {

struct AnchorGeom {
    const double* anchors;   // [A,4]
    int A, H, W, stride, im_h, im_w;
};

__device__ __forceinline__ bool anchor_box(const AnchorGeom& g, int i, double b[4]) {
    int a = i % g.A, k = i / g.A;
    double sx = (double)((k % g.W) * g.stride), sy = (double)((k / g.W) * g.stride);
    b[0] = __dadd_rn(g.anchors[a * 4 + 0], sx);
    b[1] = __dadd_rn(g.anchors[a * 4 + 1], sy);
    b[2] = __dadd_rn(g.anchors[a * 4 + 2], sx);
    b[3] = __dadd_rn(g.anchors[a * 4 + 3], sy);
    // keep_inside (bbox_transform.py:124-129): x1 >= 0, y1 >= 0, x2 < width, y2 < height
    return b[0] >= 0.0 && b[1] >= 0.0 && b[2] < (double)g.im_w && b[3] < (double)g.im_h;
}

// ------------------------------------------------------------------------------------------ bbox_overlaps (generic)
__global__ void bbox_overlaps_kernel(const double* __restrict__ boxes, int N, const double* __restrict__ query, int K,
                                     double* __restrict__ out) {
    long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)N * K) return;
    int n = (int)(t / K), k = (int)(t % K);
    double b[4] = {boxes[n * 4], boxes[n * 4 + 1], boxes[n * 4 + 2], boxes[n * 4 + 3]};
    double q[4] = {query[k * 4], query[k * 4 + 1], query[k * 4 + 2], query[k * 4 + 3]};
    out[t] = iou_f64(b, q, box_area_f64(q[0], q[1], q[2], q[3]));
}

// ------------------------------------------------------------------------------------------ 1. overlaps: row max / arg-max, column max
constexpr int GT_CHUNK = 256;

__global__ void __launch_bounds__(256) anchor_overlap_kernel(AnchorGeom g, int n_all, const float* __restrict__ gt, int n_gt,
                                                            double* __restrict__ max_ov, int* __restrict__ argmax,
                                                            unsigned long long* __restrict__ gt_max_bits) {
    __shared__ float s_gt[GT_CHUNK * 4];
    __shared__ double s_area[GT_CHUNK];
    __shared__ unsigned long long s_max[GT_CHUNK];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double b[4];
    bool inside = i < n_all && anchor_box(g, i, b);
    double best = -1.0;
    int best_g = 0;
    for (int g0 = 0; g0 < n_gt; g0 += GT_CHUNK) {
        int gc = min(GT_CHUNK, n_gt - g0);
        __syncthreads();
        for (int t = threadIdx.x; t < gc; t += blockDim.x) {
            const float* q = gt + (size_t)(g0 + t) * 5;
            s_gt[t * 4 + 0] = q[0]; s_gt[t * 4 + 1] = q[1]; s_gt[t * 4 + 2] = q[2]; s_gt[t * 4 + 3] = q[3];
            s_area[t] = box_area_f64(q[0], q[1], q[2], q[3]);
            s_max[t] = 0ull;
        }
        __syncthreads();
        if (inside) {
            for (int t = 0; t < gc; ++t) {
                const double q[4] = {s_gt[t * 4], s_gt[t * 4 + 1], s_gt[t * 4 + 2], s_gt[t * 4 + 3]};
                double ov = iou_f64(b, q, s_area[t]);
                if (ov > best) { best = ov; best_g = g0 + t; }          // strict: first maximum wins (numpy argmax)
                unsigned long long bits = (unsigned long long)__double_as_longlong(ov);   // ov >= 0: bit order == value order
                if (bits > s_max[t]) atomicMax(&s_max[t], bits);
            }
        }
        __syncthreads();
        for (int t = threadIdx.x; t < gc; t += blockDim.x)
            if (s_max[t] != 0ull) atomicMax(&gt_max_bits[g0 + t], s_max[t]);
    }
    if (i < n_all) {
        max_ov[i] = inside ? best : -1.0;
        argmax[i] = inside ? best_g : -1;
    }
}

// ------------------------------------------------------------------------------------------ 2. labels (before subsampling) + targets
__global__ void __launch_bounds__(256) anchor_label_kernel(AnchorGeom g, int n_all, const float* __restrict__ gt, int n_gt,
                                                          const double* __restrict__ max_ov, const int* __restrict__ argmax,
                                                          const unsigned long long* __restrict__ gt_max_bits,
                                                          double neg_thr, double pos_thr,
                                                          int* __restrict__ labels_full, float* __restrict__ targets_full) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_all) return;
    double b[4];
    bool inside = anchor_box(g, i, b);
    float4 tgt = make_float4(0.f, 0.f, 0.f, 0.f);
    int label = -1;
    if (inside) {
        double mo = max_ov[i];
        bool is_gt_best = false;                       // np.where(overlaps == gt_max_overlaps)[0]: every tie, any gt (:196)
        for (int t = 0; t < n_gt && !is_gt_best; ++t) {
            const float* gr = gt + (size_t)t * 5;
            const double q[4] = {gr[0], gr[1], gr[2], gr[3]};
            double ov = iou_f64(b, q, box_area_f64(q[0], q[1], q[2], q[3]));
            is_gt_best = (unsigned long long)__double_as_longlong(ov) == gt_max_bits[t];
        }
        // :137-146 in order: bg, per-gt best, >= pos_thr, bg again (clobbers)
        if (mo < neg_thr) label = 0;
        if (is_gt_best) label = 1;
        if (mo >= pos_thr) label = 1;
        if (mo < neg_thr) label = 0;
        // bbox_transform (bbox_transform.py:18-38) in float64 on (float64 anchor, float32 gt row), cast to float32 (:117)
        const float* q = gt + (size_t)argmax[i] * 5;
        double ew = __dadd_rn(__dsub_rn(b[2], b[0]), 1.0), eh = __dadd_rn(__dsub_rn(b[3], b[1]), 1.0);
        double ecx = __dadd_rn(b[0], __dmul_rn(0.5, ew)), ecy = __dadd_rn(b[1], __dmul_rn(0.5, eh));
        // the gt row is float32: "gt[:,2] - gt[:,0] + 1.0" and "gt[:,0] + 0.5*w" stay float32 in NumPy (python scalars do not
        // upcast); the mix with the float64 anchor terms happens at the subtraction / division
        float gwf = __fadd_rn(__fsub_rn(q[2], q[0]), 1.0f), ghf = __fadd_rn(__fsub_rn(q[3], q[1]), 1.0f);
        float gcxf = __fadd_rn(q[0], __fmul_rn(0.5f, gwf)), gcyf = __fadd_rn(q[1], __fmul_rn(0.5f, ghf));
        tgt.x = (float)__ddiv_rn(__dsub_rn((double)gcxf, ecx), ew);
        tgt.y = (float)__ddiv_rn(__dsub_rn((double)gcyf, ecy), eh);
        tgt.z = (float)log(__ddiv_rn((double)gwf, ew));
        tgt.w = (float)log(__ddiv_rn((double)ghf, eh));
    }
    labels_full[i] = label;
    reinterpret_cast<float4*>(targets_full)[i] = tgt;
}

// ------------------------------------------------------------------------------------------ 3. compaction + subsampling (one CTA)
__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {       // splitmix64 finaliser
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

__device__ __forceinline__ unsigned long long sample_key(unsigned long long seed, int i) {
    return (mix64(seed ^ ((unsigned long long)(unsigned)i * 0xD6E8FEB86659FD93ull)) & 0xFFFFFFFF00000000ull) | (unsigned)i;
}

__device__ int block_sum(int v, int* s_warp) {           // all threads get the total; blockDim.x == 1024
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    int t = s_warp[threadIdx.x & 31];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    return t;
}

// Disable (label := -1) the n_dis entries with label == which that have the smallest sample_key (hash, then index).
// Every thread caches the 32-bit hashes of the (at most KEYS_PER_THREAD) anchors it owns in registers, so the threshold
// search touches no memory: 32 steps on the hash, then -- only among hash ties at the threshold -- 32 steps on the index.
constexpr int KEYS_PER_THREAD = 40;          // 1024 threads x 40 = 40,960 anchors (an 800x1333 map has 37,800)

__device__ __forceinline__ uint32_t sample_hash(unsigned long long seed, int i) { return (uint32_t)(sample_key(seed, i) >> 32); }

__device__ void disable_smallest(int* labels, int n_all, int which, int n_dis, unsigned long long seed, int* s_warp) {
    if (n_dis <= 0) return;
    const bool cached = n_all <= KEYS_PER_THREAD * (int)blockDim.x;
    uint32_t hs[KEYS_PER_THREAD];
    unsigned long long valid = 0;             // bit j: owned element j is a candidate (label == which)
    if (cached) {
#pragma unroll
        for (int j = 0; j < KEYS_PER_THREAD; ++j) {
            const int i = threadIdx.x + j * blockDim.x;
            const bool c = i < n_all && labels[i] == which;
            hs[j] = c ? sample_hash(seed, i) : 0u;
            valid |= (unsigned long long)(c ? 1 : 0) << j;
        }
    }
    // T = largest x in [0, 2^32] with |{hash < x}| <= n_dis
    unsigned long long T = 0;
    for (int bit = 32; bit >= 0; --bit) {
        const unsigned long long cand = T | (1ull << bit);
        if (cand > 0x100000000ull) continue;
        int c = 0;
        if (cached) {
#pragma unroll
            for (int j = 0; j < KEYS_PER_THREAD; ++j) c += (((valid >> j) & 1ull) != 0 && (unsigned long long)hs[j] < cand) ? 1 : 0;
        } else {
            for (int i = threadIdx.x; i < n_all; i += blockDim.x)
                c += (labels[i] == which && (unsigned long long)sample_hash(seed, i) < cand) ? 1 : 0;
        }
        if (block_sum(c, s_warp) <= n_dis) T = cand;
    }
    // everything with hash < T goes; r more among hash == T (almost always a single element), lowest indices first
    int c = 0;
    for (int i = threadIdx.x; i < n_all; i += blockDim.x)
        c += (labels[i] == which && (unsigned long long)sample_hash(seed, i) < T) ? 1 : 0;
    const int r = n_dis - block_sum(c, s_warp);
    unsigned long long Y = 0;                 // largest y with |{hash == T, index < y}| <= r
    if (r > 0) {
        for (int bit = 31; bit >= 0; --bit) {
            const unsigned long long cand = Y | (1ull << bit);
            int e = 0;
            for (int i = threadIdx.x; i < n_all; i += blockDim.x)
                e += (labels[i] == which && (unsigned long long)sample_hash(seed, i) == T && (unsigned long long)i < cand) ? 1 : 0;
            if (block_sum(e, s_warp) <= r) Y = cand;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_all; i += blockDim.x) {
        if (labels[i] != which) continue;
        const unsigned long long h = sample_hash(seed, i);
        if (h < T || (h == T && (unsigned long long)i < Y)) labels[i] = -1;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(1024) anchor_subsample_kernel(AnchorGeom g, int n_all, int mode, unsigned long long seed,
                                                               const int* __restrict__ disable_pos, int n_disable,
                                                               int batch, int num_fg, int* __restrict__ labels_full,
                                                               int* __restrict__ inds_inside, int* __restrict__ counts) {
    __shared__ int s_warp[32];
    __shared__ int s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    // ordered compaction of the inside indices (np.where order)
    for (int i0 = 0; i0 < n_all; i0 += blockDim.x) {
        int i = i0 + threadIdx.x;
        double b[4];
        bool in = i < n_all && anchor_box(g, i, b);
        unsigned m = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < 32; ++w) {
            int c = s_warp[w];
            before += w < warp ? c : 0;
            total += c;
        }
        int base = s_base;
        if (in) inds_inside[base + before + __popc(m & ((1u << lane) - 1u))] = i;
        __syncthreads();
        if (threadIdx.x == 0) s_base = base + total;
        __syncthreads();
    }
    const int n_inside = s_base;
    int fg = 0, bg = 0;
    for (int i = threadIdx.x; i < n_all; i += blockDim.x) {
        int l = labels_full[i];
        fg += l == 1;
        bg += l == 0;
    }
    const int fg_before = block_sum(fg, s_warp), bg_before = block_sum(bg, s_warp);
    int fg_after = fg_before, bg_after = bg_before;
    if (mode == 1) {
        // anchor_target_layer.py:148-168: at most num_fg positives, then at most batch - (#positives) negatives
        if (fg_before > num_fg) { disable_smallest(labels_full, n_all, 1, fg_before - num_fg, seed, s_warp); fg_after = num_fg; }
        int num_bg = batch - fg_after;
        if (bg_before > num_bg) {
            disable_smallest(labels_full, n_all, 0, bg_before - num_bg, seed ^ 0xA5A5A5A5DEADBEEFull, s_warp);
            bg_after = num_bg;
        }
    } else if (mode == 2) {
        __syncthreads();
        for (int t = threadIdx.x; t < n_disable; t += blockDim.x) {
            int p = disable_pos[t];
            if (p >= 0 && p < n_inside) labels_full[inds_inside[p]] = -1;      // positions in the inside-compact arrays
        }
        __syncthreads();
        fg = bg = 0;
        for (int i = threadIdx.x; i < n_all; i += blockDim.x) {
            int l = labels_full[i];
            fg += l == 1;
            bg += l == 0;
        }
        fg_after = block_sum(fg, s_warp);
        bg_after = block_sum(bg, s_warp);
    }
    if (threadIdx.x == 0) {
        counts[0] = n_inside; counts[1] = fg_after; counts[2] = bg_after; counts[3] = fg_before; counts[4] = bg_before;
        counts[5] = n_all; counts[6] = 0; counts[7] = 0;
    }
}

// ------------------------------------------------------------------------------------------ 4. losses + their gradients
struct LossArgs {
    const float* score; long score_cs, score_ps;
    const float* bbox; long bbox_cs, bbox_ps;
    const int* labels_full; const float* targets_full; const int* counts;
    float* dscore; float* dbbox;
    double delta, lambda, grad_scale;
    double* partials;        // [grid][4]: sum ce, sum huber, #correct, unused
};

__global__ void __launch_bounds__(256) rpn_loss_kernel(AnchorGeom g, int n_all, LossArgs p) {
    __shared__ double s_red[8][3];
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double ce = 0.0, hub = 0.0, correct = 0.0;
    if (i < n_all) {
        const int a = i % g.A;
        const long k = i / g.A;                                   // pixel index h*W + w
        double b[4];
        const bool inside = anchor_box(g, i, b);
        const int valid_n = max(p.counts[1] + p.counts[2], 1);     // softmax_cross_entropy normalize=True: 1/max(count,1)
        // ---- classification: 2-way softmax between channel a (bg) and A+a (fg)  (rpn.py:174-177)
        const long o0 = (long)a * p.score_cs + k * p.score_ps, o1 = (long)(g.A + a) * p.score_cs + k * p.score_ps;
        const int label = p.labels_full[i];
        float g0 = 0.f, g1 = 0.f;
        if (label >= 0) {
            double z0 = (double)p.score[o0], z1 = (double)p.score[o1];
            double m = fmax(z0, z1);
            double e0 = exp(z0 - m), e1 = exp(z1 - m);
            double lse = m + log(e0 + e1);
            ce = lse - (label == 1 ? z1 : z0);
            correct = ((z1 > z0) ? 1 : 0) == label ? 1.0 : 0.0;   // argmax: first maximum on a tie
            double p1 = e1 / (e0 + e1), p0 = e0 / (e0 + e1);
            double s = p.grad_scale / (double)valid_n;
            g0 = (float)((p0 - (label == 0 ? 1.0 : 0.0)) * s);
            g1 = (float)((p1 - (label == 1 ? 1.0 : 0.0)) * s);
        }
        if (p.dscore != nullptr) { p.dscore[o0] = g0; p.dscore[o1] = g1; }
        // ---- regression: channel j*A + a holds coordinate j of anchor a (rpn.py:186-191); every INSIDE anchor counts
        const float4 t = reinterpret_cast<const float4*>(p.targets_full)[i];
        const float tv[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const long o = (long)(j * g.A + a) * p.bbox_cs + k * p.bbox_ps;
            float gd = 0.f;
            if (inside) {
                double d = (double)p.bbox[o] - (double)tv[j];
                double ad = fabs(d);
                hub += ad < p.delta ? 0.5 * d * d : p.delta * (ad - 0.5 * p.delta);
                double dd = ad < p.delta ? d : (d > 0 ? p.delta : -p.delta);
                gd = (float)(dd * p.lambda * p.grad_scale / (double)n_all);
            }
            if (p.dbbox != nullptr) p.dbbox[o] = gd;
        }
    }
    // fixed-order block reduction (shuffle tree, then warp 0 over the 8 warp sums): deterministic
    for (int o = 16; o > 0; o >>= 1) {
        ce += __shfl_xor_sync(0xffffffffu, ce, o);
        hub += __shfl_xor_sync(0xffffffffu, hub, o);
        correct += __shfl_xor_sync(0xffffffffu, correct, o);
    }
    if ((threadIdx.x & 31) == 0) { s_red[threadIdx.x >> 5][0] = ce; s_red[threadIdx.x >> 5][1] = hub; s_red[threadIdx.x >> 5][2] = correct; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a0 = 0, a1 = 0, a2 = 0;
        for (int w = 0; w < 8; ++w) { a0 += s_red[w][0]; a1 += s_red[w][1]; a2 += s_red[w][2]; }
        p.partials[blockIdx.x * 4 + 0] = a0; p.partials[blockIdx.x * 4 + 1] = a1; p.partials[blockIdx.x * 4 + 2] = a2;
    }
}

__global__ void rpn_loss_finish_kernel(const double* __restrict__ partials, int n_blocks, const int* __restrict__ counts,
                                       int n_all, double lambda, float* __restrict__ losses) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double ce = 0, hub = 0, ok = 0;
    for (int b = 0; b < n_blocks; ++b) { ce += partials[b * 4]; hub += partials[b * 4 + 1]; ok += partials[b * 4 + 2]; }
    int valid = counts[1] + counts[2];
    double lc = ce / (double)max(valid, 1), lb = hub / (double)n_all;
    losses[0] = (float)lc;                                       // rpn_loss_cls
    losses[1] = (float)lb;                                       // rpn_loss_bbox
    losses[2] = valid > 0 ? (float)(ok / (double)valid) : 0.f;   // rpn_cls_accuracy
    losses[3] = (float)(lc + lambda * lb);                       // rpn_loss (rpn.py:144)
}

static bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

}  // namespace frcnn

using namespace frcnn;

extern "C" {

int frcnn_bbox_overlaps(const double* boxes, int n, const double* query, int k, double* out, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(n >= 0 && k >= 0, "bbox_overlaps: negative size");
    if (n == 0 || k == 0) return FRCNN_OK;
    FRCNN_REQUIRE(boxes && query && out, "bbox_overlaps: null pointer");
    long total = (long)n * k;
    bbox_overlaps_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(boxes, n, query, k, out);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

size_t frcnn_anchor_targets_workspace_bytes(int n_all, int n_gt) {
    FRCNN_ENTRY();
    if (n_all < 0 || n_gt < 0) return 0;
    return align_up((size_t)n_all * sizeof(double), 256) + align_up((size_t)n_all * sizeof(int), 256) +
           align_up((size_t)(n_gt > 0 ? n_gt : 1) * sizeof(unsigned long long), 256);
}

int frcnn_anchor_targets(const double* anchors, int A, int feat_h, int feat_w, int feat_stride, const float* gt_boxes,
                         int n_gt, int im_h, int im_w, double neg_thr, double pos_thr, int batch, int num_fg,
                         int subsample_mode, unsigned long long seed, const int* disable_pos, int n_disable,
                         int* labels_full, float* targets_full, int* inds_inside, int* counts, void* workspace,
                         size_t workspace_bytes, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(A > 0 && feat_h > 0 && feat_w > 0 && feat_stride > 0, "anchor_targets: bad geometry A=%d H=%d W=%d", A, feat_h, feat_w);
    FRCNN_REQUIRE(n_gt > 0, "anchor_targets: needs at least one ground-truth box (the reference's argmax over an empty axis raises)");
    FRCNN_REQUIRE(anchors && gt_boxes && labels_full && targets_full && inds_inside && counts && workspace, "anchor_targets: null pointer");
    FRCNN_REQUIRE(subsample_mode >= 0 && subsample_mode <= 2, "anchor_targets: subsample_mode %d not in {0,1,2}", subsample_mode);
    FRCNN_REQUIRE(subsample_mode != 2 || n_disable == 0 || disable_pos, "anchor_targets: mode 2 without an index list");
    // the reference's np.random.choice raises when asked for more negatives than exist; here num_bg = batch - n_fg would
    // go negative and the normaliser counts[1] + counts[2] with it
    FRCNN_REQUIRE(subsample_mode != 1 || (num_fg >= 0 && num_fg <= batch),
                  "anchor_targets: mode 1 needs 0 <= num_fg <= batch, got num_fg=%d batch=%d", num_fg, batch);
    FRCNN_REQUIRE(aligned(targets_full, 16), "anchor_targets: targets_full must be 16-byte aligned");
    const long n_all_l = (long)A * feat_h * feat_w;
    FRCNN_REQUIRE(n_all_l < (1l << 30), "anchor_targets: too many anchors");
    const int n_all = (int)n_all_l;
    if (workspace_bytes < frcnn_anchor_targets_workspace_bytes(n_all, n_gt)) {
        set_error("anchor_targets: workspace %zu < %zu bytes", workspace_bytes, frcnn_anchor_targets_workspace_bytes(n_all, n_gt));
        return FRCNN_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    double* max_ov = (double*)w;                w += align_up((size_t)n_all * sizeof(double), 256);
    int* argmax = (int*)w;                      w += align_up((size_t)n_all * sizeof(int), 256);
    unsigned long long* gt_max = (unsigned long long*)w;
    AnchorGeom g{anchors, A, feat_h, feat_w, feat_stride, im_h, im_w};
    FRCNN_CUDA_OK(cudaMemsetAsync(gt_max, 0, (size_t)n_gt * sizeof(unsigned long long), st));
    const int grid = cdiv(n_all, 256);
    anchor_overlap_kernel<<<grid, 256, 0, st>>>(g, n_all, gt_boxes, n_gt, max_ov, argmax, gt_max);
    FRCNN_LAUNCH_OK();
    anchor_label_kernel<<<grid, 256, 0, st>>>(g, n_all, gt_boxes, n_gt, max_ov, argmax, gt_max, neg_thr, pos_thr, labels_full, targets_full);
    FRCNN_LAUNCH_OK();
    anchor_subsample_kernel<<<1, 1024, 0, st>>>(g, n_all, subsample_mode, seed, disable_pos, n_disable, batch, num_fg,
                                                 labels_full, inds_inside, counts);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

size_t frcnn_rpn_loss_workspace_bytes(int n_all) {
    FRCNN_ENTRY();
    if (n_all < 0) return 0;
    return (size_t)cdiv(n_all > 0 ? n_all : 1, 256) * 4 * sizeof(double);
}

int frcnn_rpn_loss(const float* score, long score_cs, long score_ps, const float* bbox, long bbox_cs, long bbox_ps,
                   const double* anchors, int A, int feat_h, int feat_w, int feat_stride, int im_h, int im_w,
                   const int* labels_full, const float* targets_full, const int* counts, double delta, double loss_lambda,
                   double grad_scale, float* losses, float* dscore, float* dbbox, void* workspace, size_t workspace_bytes,
                   void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(A > 0 && feat_h > 0 && feat_w > 0 && feat_stride > 0, "rpn_loss: bad geometry");
    FRCNN_REQUIRE(score && bbox && anchors && labels_full && targets_full && counts && losses && workspace, "rpn_loss: null pointer");
    FRCNN_REQUIRE(aligned(targets_full, 16), "rpn_loss: targets_full must be 16-byte aligned");
    FRCNN_REQUIRE(delta > 0, "rpn_loss: delta must be positive");
    const long n_all_l = (long)A * feat_h * feat_w;
    FRCNN_REQUIRE(n_all_l < (1l << 30), "rpn_loss: too many anchors");
    const int n_all = (int)n_all_l;
    if (workspace_bytes < frcnn_rpn_loss_workspace_bytes(n_all)) {
        set_error("rpn_loss: workspace %zu < %zu bytes", workspace_bytes, frcnn_rpn_loss_workspace_bytes(n_all));
        return FRCNN_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    AnchorGeom g{anchors, A, feat_h, feat_w, feat_stride, im_h, im_w};
    LossArgs p{score, score_cs, score_ps, bbox, bbox_cs, bbox_ps, labels_full, targets_full, counts, dscore, dbbox,
               delta, loss_lambda, grad_scale, (double*)workspace};
    const int grid = cdiv(n_all, 256);
    rpn_loss_kernel<<<grid, 256, 0, st>>>(g, n_all, p);
    FRCNN_LAUNCH_OK();
    rpn_loss_finish_kernel<<<1, 32, 0, st>>>((const double*)workspace, grid, counts, n_all, loss_lambda, losses);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

}  // extern "C"
