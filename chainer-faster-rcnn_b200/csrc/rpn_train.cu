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

// The anchors of N slots.  One image (extents == NULL): H x W is its feature map and (im_h, im_w) its clip bounds.  A canvas:
// H x W is the canvas feature map, slot n's map is ceil(extents[n] / 2^halvings) (canvas_extent) and its clip bounds are
// im_info[n].  Every per-slot anchor array is `cap` = A*H*W entries long, and anchor (y*fw_n + x)*A + a is numbered in the
// slot's own frame, so a slot's arrays are those of its image alone.
struct AnchorSlots {
    AnchorGeom geo;
    const int* extents; int halvings; const int* im_info;
    long cap;
};

__device__ __forceinline__ AnchorGeom slot_geom(const AnchorSlots& s, int n) {
    AnchorGeom g = s.geo;
    if (s.extents != nullptr) {
        g.H = canvas_extent(s.extents, n, 0, s.halvings, s.geo.H);
        g.W = canvas_extent(s.extents, n, 1, s.halvings, s.geo.W);
        g.im_h = __ldg(s.im_info + 2 * n);
        g.im_w = __ldg(s.im_info + 2 * n + 1);
    }
    return g;
}

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

// Everything the three target kernels read and write, for N slots (blockIdx.y = slot).  Slot n's ground truth is
// gt_counts[n] (clamped to max_gt; NULL: n_gt) rows at gt + n*max_gt*5; its arrays and workspace sit n*cap (n*max_gt for
// gt_max, n*8 for counts) entries in.  A slot with no ground-truth row is empty, like one with a 0 x 0 extent.
struct TargetArgs {
    AnchorSlots s;
    const float* gt; int max_gt; const int* gt_counts; int n_gt;
    double* max_ov; int* argmax; unsigned long long* gt_max;
    int* labels_full; float* targets_full; int* inds_inside; int* counts;
};

struct TargetSlot {
    AnchorGeom g;
    int n_all, n_gt;
    const float* gt;
    long base;                       // offset of the slot's anchor arrays
};

__device__ __forceinline__ TargetSlot target_slot(const TargetArgs& t, int n) {
    TargetSlot r;
    r.g = slot_geom(t.s, n);
    r.n_gt = t.gt_counts != nullptr ? min(__ldg(t.gt_counts + n), t.max_gt) : t.n_gt;
    if (r.n_gt < 1) r.g.H = r.g.W = 0;
    r.n_all = r.g.A * r.g.H * r.g.W;
    r.gt = t.gt + (size_t)n * t.max_gt * 5;
    r.base = (long)n * t.s.cap;
    return r;
}

__global__ void __launch_bounds__(256) anchor_overlap_kernel(TargetArgs ta) {
    __shared__ float s_gt[GT_CHUNK * 4];
    __shared__ double s_area[GT_CHUNK];
    __shared__ unsigned long long s_max[GT_CHUNK];
    const TargetSlot sl = target_slot(ta, blockIdx.y);
    if ((long)blockIdx.x * blockDim.x >= sl.n_all) return;             // whole block past the slot's anchors
    const AnchorGeom g = sl.g;
    const int n_all = sl.n_all, n_gt = sl.n_gt;
    const float* __restrict__ gt = sl.gt;
    double* __restrict__ max_ov = ta.max_ov + sl.base;
    int* __restrict__ argmax = ta.argmax + sl.base;
    unsigned long long* __restrict__ gt_max_bits = ta.gt_max + (size_t)blockIdx.y * ta.max_gt;
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
__global__ void __launch_bounds__(256) anchor_label_kernel(TargetArgs t, double neg_thr, double pos_thr) {
    const TargetSlot sl = target_slot(t, blockIdx.y);
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sl.n_all) return;
    const AnchorGeom g = sl.g;
    const int n_gt = sl.n_gt;
    const float* __restrict__ gt = sl.gt;
    const double* __restrict__ max_ov = t.max_ov + sl.base;
    const int* __restrict__ argmax = t.argmax + sl.base;
    const unsigned long long* __restrict__ gt_max_bits = t.gt_max + (size_t)blockIdx.y * t.max_gt;
    int* __restrict__ labels_full = t.labels_full + sl.base;
    float* __restrict__ targets_full = t.targets_full + 4 * sl.base;
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
// (mix64 / sample_key: common.cuh)
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

// Subsampling of one slot per CTA.  Mode 1 draws with seeds[n] (NULL: seed); mode 2 disables slot n's list
// disable_pos[disable_offsets[n] .. disable_offsets[n+1]) (NULL offsets: the whole list), clamped to [0, n_disable).
struct SubsampleArgs {
    int mode; unsigned long long seed; const unsigned long long* seeds;
    const int* disable_pos; int n_disable; const int* disable_offsets;
    int batch, num_fg;
};

__global__ void __launch_bounds__(1024) anchor_subsample_kernel(TargetArgs t, SubsampleArgs sa) {
    __shared__ int s_warp[32];
    __shared__ int s_base;
    const TargetSlot sl = target_slot(t, blockIdx.y);
    const AnchorGeom g = sl.g;
    const int n_all = sl.n_all, mode = sa.mode;
    int* __restrict__ labels_full = t.labels_full + sl.base;
    int* __restrict__ inds_inside = t.inds_inside + sl.base;
    int* __restrict__ counts = t.counts + 8 * blockIdx.y;
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
        const int batch = sa.batch, num_fg = sa.num_fg;
        const unsigned long long seed = sa.seeds != nullptr ? sa.seeds[blockIdx.y] : sa.seed;
        // anchor_target_layer.py:148-168: at most num_fg positives, then at most batch - (#positives) negatives
        if (fg_before > num_fg) { disable_smallest(labels_full, n_all, 1, fg_before - num_fg, seed, s_warp); fg_after = num_fg; }
        int num_bg = batch - fg_after;
        if (bg_before > num_bg) {
            disable_smallest(labels_full, n_all, 0, bg_before - num_bg, seed ^ BG_SEED_XOR, s_warp);
            bg_after = num_bg;
        }
    } else if (mode == 2) {
        const int* disable_pos = sa.disable_pos;
        int n_disable = sa.n_disable;
        if (sa.disable_offsets != nullptr) {
            const int lo = min(max(sa.disable_offsets[blockIdx.y], 0), sa.n_disable);
            const int hi = min(max(sa.disable_offsets[blockIdx.y + 1], lo), sa.n_disable);
            disable_pos += lo;
            n_disable = hi - lo;
        }
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
    double* partials;        // [N][gridDim.x][4]: sum ce, sum huber, #correct, unused
    // canvas (s.extents != NULL): slot n's pixel (y, x) is row n*H*W + y*W + x of the score / bbox addressing, and when
    // zero_ld > 0 the gradient is an NHWC matrix [N*H*W][zero_ld] whose every element outside the slots' anchor entries
    // (other rows, columns >= 6A) is written as 0 by the same launch
    int zero_ld;
};

__device__ __forceinline__ AnchorGeom loss_slot(const AnchorSlots& s, const LossArgs& p, int n, int& n_all) {
    AnchorGeom g = slot_geom(s, n);
    if (s.extents != nullptr && p.counts[8 * n + 5] == 0) g.H = g.W = 0;      // a slot frcnn_anchor_targets_batch left empty
    n_all = g.A * g.H * g.W;
    return g;
}

__global__ void __launch_bounds__(256) rpn_loss_kernel(AnchorSlots s, LossArgs p) {
    __shared__ double s_red[8][3];
    const int slot = blockIdx.y;
    int n_all;
    const AnchorGeom g = loss_slot(s, p, slot, n_all);
    p.labels_full += (long)slot * s.cap;
    p.targets_full += 4 * (long)slot * s.cap;
    p.counts += 8 * slot;
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double ce = 0.0, hub = 0.0, correct = 0.0;
    if (p.zero_ld > 0) {
        const long px = (long)s.geo.H * s.geo.W, total = px * p.zero_ld, c6 = 6l * g.A;
        float* dst = p.dscore + slot * px * p.zero_ld;
        for (long e = i; e < total; e += (long)gridDim.x * blockDim.x) {
            const long r = e / p.zero_ld, c = e - r * p.zero_ld;
            if (c >= c6 || r / s.geo.W >= g.H || r % s.geo.W >= g.W) dst[e] = 0.f;
        }
    }
    if (i < n_all) {
        const int a = i % g.A;
        const int kk = i / g.A;                                   // pixel index h*W + w in the slot's own frame
        const long k = (long)slot * s.geo.H * s.geo.W + (long)(kk / g.W) * s.geo.W + kk % g.W;
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
        double* part = p.partials + ((long)slot * gridDim.x + blockIdx.x) * 4;
        part[0] = a0; part[1] = a1; part[2] = a2;
    }
}

// one CTA per slot: the slot's first cdiv(n_all, 256) block partials in order; an empty slot gets four zeros
__global__ void rpn_loss_finish_kernel(AnchorSlots s, LossArgs p, int grid_x, float* __restrict__ losses) {
    if (threadIdx.x != 0) return;
    const int slot = blockIdx.x;
    int n_all;
    loss_slot(s, p, slot, n_all);
    const double* partials = p.partials + (long)slot * grid_x * 4;
    const int* counts = p.counts + 8 * slot;
    const double lambda = p.lambda;
    losses += 4 * slot;
    if (n_all == 0) {
        losses[0] = losses[1] = losses[2] = losses[3] = 0.f;
        return;
    }
    const int n_blocks = (n_all + 255) / 256;
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

size_t frcnn_anchor_targets_batch_workspace_bytes(int N, int n_cap, int max_gt) {
    FRCNN_ENTRY();
    if (N < 1 || n_cap < 0 || max_gt < 0) return 0;
    const size_t n = (size_t)N * n_cap;
    return align_up(n * sizeof(double), 256) + align_up(n * sizeof(int), 256) +
           align_up((size_t)N * (max_gt > 0 ? max_gt : 1) * sizeof(unsigned long long), 256);
}

// overlaps, labels + targets, then one subsampling CTA per slot; the workspace holds max_ov [N*cap], argmax [N*cap] and
// gt_max [N*max_gt]
static int launch_targets(TargetArgs t, const SubsampleArgs& sa, int N, double neg_thr, double pos_thr, void* workspace,
                          cudaStream_t st) {
    const size_t n = (size_t)N * t.s.cap;
    char* w = (char*)workspace;
    t.max_ov = (double*)w;                      w += align_up(n * sizeof(double), 256);
    t.argmax = (int*)w;                         w += align_up(n * sizeof(int), 256);
    t.gt_max = (unsigned long long*)w;
    FRCNN_CUDA_OK(cudaMemsetAsync(t.gt_max, 0, (size_t)N * t.max_gt * sizeof(unsigned long long), st));
    const dim3 grid(cdiv((int)t.s.cap, 256), N);
    anchor_overlap_kernel<<<grid, 256, 0, st>>>(t);
    FRCNN_LAUNCH_OK();
    anchor_label_kernel<<<grid, 256, 0, st>>>(t, neg_thr, pos_thr);
    FRCNN_LAUNCH_OK();
    anchor_subsample_kernel<<<dim3(1, N), 1024, 0, st>>>(t, sa);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
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
    TargetArgs t{};
    t.s = AnchorSlots{AnchorGeom{anchors, A, feat_h, feat_w, feat_stride, im_h, im_w}, nullptr, 0, nullptr, n_all};
    t.gt = gt_boxes; t.max_gt = n_gt; t.gt_counts = nullptr; t.n_gt = n_gt;
    t.labels_full = labels_full; t.targets_full = targets_full; t.inds_inside = inds_inside; t.counts = counts;
    const SubsampleArgs sa{subsample_mode, seed, nullptr, disable_pos, n_disable, nullptr, batch, num_fg};
    return launch_targets(t, sa, 1, neg_thr, pos_thr, workspace, (cudaStream_t)stream);
}

int frcnn_anchor_targets_batch(const double* anchors, int A, int fhc, int fwc, int feat_stride, int N, const int* extents,
                               int halvings, const int* im_info, const float* gt, int max_gt, const int* gt_counts, double neg_thr,
                               double pos_thr, int batch, int num_fg, int subsample_mode, const unsigned long long* seeds,
                               const int* disable_pos, int n_disable, const int* disable_offsets, int* labels_full,
                               float* targets_full, int* inds_inside, int* counts, void* workspace, size_t workspace_bytes,
                               void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "anchor_targets_batch: N = %d not in [1, 65535]", N);
    FRCNN_REQUIRE(A > 0 && fhc > 0 && fwc > 0 && feat_stride > 0, "anchor_targets_batch: bad geometry A=%d H=%d W=%d", A, fhc, fwc);
    FRCNN_REQUIRE(halvings >= 0 && halvings <= 30, "anchor_targets_batch: halvings must be in [0,30] (got %d)", halvings);
    FRCNN_REQUIRE(max_gt >= 1, "anchor_targets_batch: max_gt must be at least 1 (got %d)", max_gt);
    FRCNN_REQUIRE(extents && im_info && gt_counts, "anchor_targets_batch: null extents / im_info / gt_counts");
    FRCNN_REQUIRE(anchors && gt && labels_full && targets_full && inds_inside && counts, "anchor_targets_batch: null pointer");
    FRCNN_REQUIRE(subsample_mode >= 0 && subsample_mode <= 2, "anchor_targets_batch: subsample_mode %d not in {0,1,2}", subsample_mode);
    FRCNN_REQUIRE(subsample_mode != 1 || seeds, "anchor_targets_batch: mode 1 without per-slot seeds");
    FRCNN_REQUIRE(subsample_mode != 1 || (num_fg >= 0 && num_fg <= batch),
                  "anchor_targets_batch: mode 1 needs 0 <= num_fg <= batch, got num_fg=%d batch=%d", num_fg, batch);
    FRCNN_REQUIRE(subsample_mode != 2 || (disable_offsets && n_disable >= 0 && (n_disable == 0 || disable_pos)),
                  "anchor_targets_batch: mode 2 needs the offsets [N+1] and an index list of n_disable >= 0 entries");
    FRCNN_REQUIRE(aligned(targets_full, 16), "anchor_targets_batch: targets_full must be 16-byte aligned");
    const long cap = (long)A * fhc * fwc;
    FRCNN_REQUIRE(cap < (1l << 30) && (long)N * cap < (1l << 31) && (long)N * max_gt < (1l << 31),
                  "anchor_targets_batch: too many anchors or ground-truth rows");
    if (!workspace) {
        set_error("anchor_targets_batch: no workspace");
        return FRCNN_ERR_WORKSPACE;
    }
    const size_t need = frcnn_anchor_targets_batch_workspace_bytes(N, (int)cap, max_gt);
    if (workspace_bytes < need) {
        set_error("anchor_targets_batch: workspace %zu < %zu bytes", workspace_bytes, need);
        return FRCNN_ERR_WORKSPACE;
    }
    TargetArgs t{};
    t.s = AnchorSlots{AnchorGeom{anchors, A, fhc, fwc, feat_stride, 0, 0}, extents, halvings, im_info, cap};
    t.gt = gt; t.max_gt = max_gt; t.gt_counts = gt_counts; t.n_gt = max_gt;
    t.labels_full = labels_full; t.targets_full = targets_full; t.inds_inside = inds_inside; t.counts = counts;
    const SubsampleArgs sa{subsample_mode, 0ull, subsample_mode == 1 ? seeds : nullptr, disable_pos, subsample_mode == 2 ? n_disable : 0,
                           subsample_mode == 2 ? disable_offsets : nullptr, batch, num_fg};
    return launch_targets(t, sa, N, neg_thr, pos_thr, workspace, (cudaStream_t)stream);
}

size_t frcnn_rpn_loss_workspace_bytes(int n_all) {
    FRCNN_ENTRY();
    if (n_all < 0) return 0;
    return (size_t)cdiv(n_all > 0 ? n_all : 1, 256) * 4 * sizeof(double);
}

size_t frcnn_rpn_loss_batch_workspace_bytes(int N, int n_cap) {
    FRCNN_ENTRY();
    if (N < 1 || n_cap < 0) return 0;
    return (size_t)N * frcnn_rpn_loss_workspace_bytes(n_cap);
}

// the loss kernel over cdiv(cap, 256) x N blocks, then one finishing CTA per slot
static int launch_loss(const AnchorSlots& s, const LossArgs& p, int N, float* losses, cudaStream_t st) {
    const int grid_x = cdiv((int)(s.cap > 0 ? s.cap : 1), 256);
    rpn_loss_kernel<<<dim3(grid_x, N), 256, 0, st>>>(s, p);
    FRCNN_LAUNCH_OK();
    rpn_loss_finish_kernel<<<N, 32, 0, st>>>(s, p, grid_x, losses);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
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
    const AnchorSlots s{AnchorGeom{anchors, A, feat_h, feat_w, feat_stride, im_h, im_w}, nullptr, 0, nullptr, n_all};
    const LossArgs p{score, score_cs, score_ps, bbox, bbox_cs, bbox_ps, labels_full, targets_full, counts, dscore, dbbox,
                     delta, loss_lambda, grad_scale, (double*)workspace, 0};
    return launch_loss(s, p, 1, losses, (cudaStream_t)stream);
}

int frcnn_rpn_loss_batch(const float* head, int ld, const double* anchors, int A, int fhc, int fwc, int feat_stride, int N,
                         const int* extents, int halvings, const int* im_info, const int* labels_full, const float* targets_full,
                         const int* counts, double delta, double loss_lambda, double grad_scale, float* losses, float* dhead,
                         void* workspace, size_t workspace_bytes, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "rpn_loss_batch: N = %d not in [1, 65535]", N);
    FRCNN_REQUIRE(A > 0 && fhc > 0 && fwc > 0 && feat_stride > 0, "rpn_loss_batch: bad geometry A=%d H=%d W=%d", A, fhc, fwc);
    FRCNN_REQUIRE(ld >= 6 * A, "rpn_loss_batch: ld = %d < 6A = %d", ld, 6 * A);
    FRCNN_REQUIRE(halvings >= 0 && halvings <= 30, "rpn_loss_batch: halvings must be in [0,30] (got %d)", halvings);
    FRCNN_REQUIRE(extents && im_info, "rpn_loss_batch: null extents / im_info");
    FRCNN_REQUIRE(head && anchors && labels_full && targets_full && counts && losses, "rpn_loss_batch: null pointer");
    FRCNN_REQUIRE(aligned(targets_full, 16), "rpn_loss_batch: targets_full must be 16-byte aligned");
    FRCNN_REQUIRE(delta > 0, "rpn_loss_batch: delta must be positive");
    const long cap = (long)A * fhc * fwc;
    FRCNN_REQUIRE(cap < (1l << 30) && (long)N * fhc * fwc * ld < (1l << 40), "rpn_loss_batch: too many anchors");
    if (!workspace) {
        set_error("rpn_loss_batch: no workspace");
        return FRCNN_ERR_WORKSPACE;
    }
    if (workspace_bytes < frcnn_rpn_loss_batch_workspace_bytes(N, (int)cap)) {
        set_error("rpn_loss_batch: workspace %zu < %zu bytes", workspace_bytes, frcnn_rpn_loss_batch_workspace_bytes(N, (int)cap));
        return FRCNN_ERR_WORKSPACE;
    }
    const AnchorSlots s{AnchorGeom{anchors, A, fhc, fwc, feat_stride, 0, 0}, extents, halvings, im_info, cap};
    const LossArgs p{head, 1, ld, head + 2 * A, 1, ld, labels_full, targets_full, counts, dhead, dhead ? dhead + 2 * A : nullptr,
                     delta, loss_lambda, grad_scale, (double*)workspace, dhead ? ld : 0};
    return launch_loss(s, p, N, losses, (cudaStream_t)stream);
}

}  // extern "C"
