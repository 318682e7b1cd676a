// voc_eval.cu -- the PASCAL VOC detection metric on the device (frcnn_voc_eval_append_batch, frcnn_voc_eval): per-class
// average precision, 11-point (VOC07) and area (VOC2010+), and their means over a dataset, from frcnn_detect_batch's keep
// lists, without downloading a detection.
//
// Append: one warp per (image, class) reserves the class's conf_count slots of the dataset-wide pool with ONE atomicAdd and
// records (first slot, count) in the segment table [NC-1][max_images]; the boxes are divided by (float)im_scale exactly as
// frcnn_detection_lists_batch divides them, without its truncation to int.
//
// Evaluate (a static launch sequence):
//   1. class_offsets: per class, an exclusive scan of the segment counts over images -> the class-major, image-major,
//      keep-list-ordered position of every detection, and each class's detection count;
//   2. match: one warp per (class, image) segment ranks its detections by (score desc, keep-list position) with nms_math's
//      score order, then greedily matches them in that order against the image's GT boxes of the class (float64 +1 IoU,
//      first maximum in GT order) and writes TP / FP / ignored per detection, and the rank-sort key per detection;
//   3. a stable LSD radix sort (8-bit digits: tile histograms, per-digit scan over tiles, stable scatter) of the class-major
//      positions by (class, score descending): since the input is in (image, keep-list position) order within a class, the
//      output is the class's rank order -- score descending, then image, then position;
//   4. curve: one CTA per class: int32 prefix sums of TP / FP in rank order (the curves, kept at the start of the workspace),
//      precision, its reverse running maximum, the 11-point AP and a fixed-order reduction of the area AP;
//   5. finish: the status word and the means.
// Every float64 operation is an explicit __d*_rn (no FMA contraction), so the decisions equal NumPy's bit for bit.
#include <float.h>
#include <limits.h>

#include "common.cuh"
#include "nms_math.cuh"

namespace frcnn {
namespace {

constexpr int kAppendWarps = 8;
constexpr int kMatchWarps = 8;
constexpr int kSortThreads = 256, kSortRounds = 8, kSortTile = kSortThreads * kSortRounds;
constexpr int kRadix = 256;
constexpr int kScanThreads = 1024;
constexpr int kCapacityMax = 1 << 30;

enum { FLAG_IGNORED = 0, FLAG_TP = 1, FLAG_FP = 2 };

struct EvalStrides { long prob, boxes, keep_idx, conf_count; };

// Byte offsets of the workspace.  The curves come first (documented in the header); the GT claim flags last, so the append
// entry needs no max_gt.
struct VocLayout {
    size_t tp_cum, fp_cum, total, seg, pool_box, pool_score, seg_off, class_count, flags, keys[2], vals[2], hist, row_total,
        env, claimed, bytes;
};

VocLayout voc_layout(int NC, int cap, int max_images, int max_gt) {
    VocLayout L;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        const size_t o = off;
        off = align_up(off + bytes, 256);
        return o;
    };
    const size_t C = (size_t)cap, S = (size_t)(NC - 1) * max_images, tiles = (size_t)cdiv(cap, kSortTile);
    L.tp_cum = take(4 * C);
    L.fp_cum = take(4 * C);
    L.total = take(8);
    L.seg = take(8 * S);
    L.pool_box = take(16 * C);
    L.pool_score = take(4 * C);
    L.seg_off = take(4 * S);
    L.class_count = take(4 * (size_t)(NC - 1));
    L.flags = take(C);
    L.keys[0] = take(8 * C);
    L.keys[1] = take(8 * C);
    L.vals[0] = take(4 * C);
    L.vals[1] = take(4 * C);
    L.hist = take(4 * kRadix * tiles);
    L.row_total = take(4 * kRadix);
    L.env = take(8 * C);
    L.claimed = take((size_t)max_gt);
    L.bytes = off;
    return L;
}

template <typename T>
T* at(void* ws, size_t off) { return reinterpret_cast<T*>(static_cast<char*>(ws) + off); }

// detections held by the pool: all of them, or none once more were appended than it holds (the status word says so)
__device__ __forceinline__ int stored(const unsigned long long* total, int cap) {
    const unsigned long long t = *total;
    return t <= (unsigned long long)cap ? (int)t : 0;
}

// ------------------------------------------------------------------------------------------ block scans (kScanThreads)
// inclusive scan of v over the block in thread order; *total gets the block's sum.  s: kScanThreads/32 ints.
__device__ __forceinline__ int block_incl_sum(int v, int* s, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += u;
    }
    if (lane == 31) s[warp] = v;
    __syncthreads();
    if (warp == 0) {
        int w = lane < kScanThreads / 32 ? s[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += u;
        }
        if (lane < kScanThreads / 32) s[lane] = w;
    }
    __syncthreads();
    v += warp > 0 ? s[warp - 1] : 0;
    *total = s[kScanThreads / 32 - 1];
    __syncthreads();
    return v;
}

// inclusive running maximum of v (>= 0, never NaN) in thread order; *total gets the block's maximum.  s: kScanThreads/32.
__device__ __forceinline__ double block_incl_max(double v, double* s, double* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const double u = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v = fmax(v, u);
    }
    if (lane == 31) s[warp] = v;
    __syncthreads();
    if (warp == 0) {
        double w = lane < kScanThreads / 32 ? s[lane] : 0.0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const double u = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w = fmax(w, u);
        }
        if (lane < kScanThreads / 32) s[lane] = w;
    }
    __syncthreads();
    v = warp > 0 ? fmax(v, s[warp - 1]) : v;
    *total = s[kScanThreads / 32 - 1];
    __syncthreads();
    return v;
}

// ------------------------------------------------------------------------------------------ append
// grid (N, ceil((NC-1)/kAppendWarps)); one warp per (image, class).
__global__ void __launch_bounds__(kAppendWarps * 32) voc_append_kernel(const float* prob, const float* boxes, const int* keep_idx,
                                                                      const int* conf_count, const double* im_scale, int R_cap,
                                                                      int NC, EvalStrides is, int image_base, int cap,
                                                                      int max_images, unsigned long long* total, int2* seg,
                                                                      float4* pool_box, float* pool_score) {
    const int lane = threadIdx.x & 31;
    const int c = blockIdx.y * kAppendWarps + (threadIdx.x >> 5) + 1;
    if (c >= NC) return;
    const long img = blockIdx.x;
    prob += img * is.prob;
    boxes += img * is.boxes;
    keep_idx += img * is.keep_idx + (long)(c - 1) * R_cap;
    const int n = min(max(conf_count[img * is.conf_count + c - 1], 0), R_cap);
    unsigned long long slot = 0;
    if (lane == 0 && n > 0) slot = atomicAdd(total, (unsigned long long)n);
    slot = __shfl_sync(0xffffffffu, slot, 0);
    if (lane == 0)
        seg[(long)(c - 1) * max_images + image_base + img] = make_int2((int)min(slot, (unsigned long long)cap), n);
    const float s = __double2float_rn(im_scale[img]);
    for (int j = lane; j < n && slot + j < (unsigned long long)cap; j += 32) {
        const int r = keep_idx[j];
        float4 b = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        float sc = 0.0f;
        if (r >= 0 && r < R_cap) {              // not an index frcnn_detect writes: a zero box of score 0, nothing read
            const float* q = boxes + (long)r * 4 * NC + 4 * c;
            b = make_float4(__fdiv_rn(q[0], s), __fdiv_rn(q[1], s), __fdiv_rn(q[2], s), __fdiv_rn(q[3], s));
            sc = prob[(long)r * NC + c];
        }
        pool_box[slot + j] = b;
        pool_score[slot + j] = sc;
    }
}

// ------------------------------------------------------------------------------------------ 1. class offsets
// one CTA per class: seg_off[c][n] = detections of class c in images < n; class_count[c] = all of them
__global__ void __launch_bounds__(kScanThreads) voc_class_offsets_kernel(const int2* seg, int max_images, int* seg_off,
                                                                        int* class_count) {
    __shared__ int s[kScanThreads / 32];
    const long row = (long)blockIdx.x * max_images;
    int carry = 0;
    for (int n0 = 0; n0 < max_images; n0 += kScanThreads) {
        const int n = n0 + threadIdx.x;
        const int v = n < max_images ? seg[row + n].y : 0;
        int tot;
        const int incl = block_incl_sum(v, s, &tot);
        if (n < max_images) seg_off[row + n] = carry + incl - v;
        carry += tot;
    }
    if (threadIdx.x == 0) class_count[blockIdx.x] = carry;
}

// ------------------------------------------------------------------------------------------ 2. matching
// float64 min / max that propagate NaN as np.minimum / np.maximum do (fmin / fmax return the other operand)
__device__ __forceinline__ double nan_max(double a, double b) { return (a != a || b != b) ? __longlong_as_double(0x7ff8000000000000ll) : fmax(a, b); }
__device__ __forceinline__ double nan_min(double a, double b) { return (a != a || b != b) ? __longlong_as_double(0x7ff8000000000000ll) : fmin(a, b); }

// The devkit's overlap of detection box b with GT box g, in its operation order.
__device__ __forceinline__ double voc_overlap(const double b[4], double b_area, const float* g4) {
    const double g0 = g4[0], g1 = g4[1], g2 = g4[2], g3 = g4[3];
    const double iw = nan_max(__dadd_rn(__dsub_rn(nan_min(g2, b[2]), nan_max(g0, b[0])), 1.0), 0.0);
    const double ih = nan_max(__dadd_rn(__dsub_rn(nan_min(g3, b[3]), nan_max(g1, b[1])), 1.0), 0.0);
    const double inters = __dmul_rn(iw, ih);
    const double g_area = __dmul_rn(__dadd_rn(__dsub_rn(g2, g0), 1.0), __dadd_rn(__dsub_rn(g3, g1), 1.0));
    return __ddiv_rn(inters, __dsub_rn(__dadd_rn(b_area, g_area), inters));
}

// One warp per (class, image) segment, grid over (NC-1) * max_images segments.
__global__ void __launch_bounds__(kMatchWarps * 32) voc_match_kernel(
    int NC, int max_images, int n_images, int n_gt, const int* gt_offsets, const float* gt_boxes, const int* gt_labels,
    const unsigned char* gt_difficult, double thr, const unsigned long long* total, int cap, const int2* seg,
    const float4* pool_box, const float* pool_score, const int* seg_off, const int* class_count, unsigned char* flags,
    unsigned long long* keys, int* vals, int* order, unsigned char* claimed) {
    const int lane = threadIdx.x & 31;
    const long sidx = (long)blockIdx.x * kMatchWarps + (threadIdx.x >> 5);
    if (sidx >= (long)(NC - 1) * max_images || stored(total, cap) == 0) return;
    const int k = (int)(sidx / max_images), img = (int)(sidx % max_images), c = k + 1;
    const int2 sg = seg[sidx];
    const int cnt = sg.y;
    if (cnt == 0) return;
    int dst = seg_off[sidx];
    for (int q = 0; q < k; ++q) dst += class_count[q];
    const float* score = pool_score + sg.x;
    // the sort key (class, score descending) and the rank of each detection within the segment: score order, then position
    for (int j = lane; j < cnt; j += 32) {
        const uint32_t kj = float_to_ordered(score[j]);
        keys[dst + j] = ((unsigned long long)k << 32) | (unsigned long long)(~kj);
        vals[dst + j] = dst + j;
        int rank = 0;
        for (int q = 0; q < cnt; ++q) rank += ahead(float_to_ordered(score[q]), q, kj, j);
        order[dst + rank] = j;
    }
    __syncwarp();
    int g0 = 0, g1 = 0;
    if (img < n_images) {
        g0 = min(max(gt_offsets[img], 0), n_gt);
        g1 = min(max(gt_offsets[img + 1], g0), n_gt);
    }
    for (int r = 0; r < cnt; ++r) {
        const int j = order[dst + r];
        const float4 bf = pool_box[sg.x + j];
        const double b[4] = {bf.x, bf.y, bf.z, bf.w};
        const double b_area = __dmul_rn(__dadd_rn(__dsub_rn(b[2], b[0]), 1.0), __dadd_rn(__dsub_rn(b[3], b[1]), 1.0));
        // first maximum in GT order; any NaN overlap makes the maximum NaN (np.max), and a NaN is never > thr
        double best = 0.0;
        int arg = INT_MAX, nan_seen = 0;
        for (int g = g0 + lane; g < g1; g += 32) {
            if (gt_labels[g] != c) continue;
            const double ov = voc_overlap(b, b_area, gt_boxes + 4l * g);
            if (ov != ov) nan_seen = 1;
            else if (arg == INT_MAX || ov > best) { best = ov; arg = g; }
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, d);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, d);
            if (oa != INT_MAX && (arg == INT_MAX || ob > best || (ob == best && oa < arg))) { best = ob; arg = oa; }
        }
        nan_seen = __any_sync(0xffffffffu, nan_seen);
        if (lane == 0) {
            unsigned char f = FLAG_FP;
            if (!nan_seen && arg != INT_MAX && best > thr) {
                if (gt_difficult[arg]) f = FLAG_IGNORED;
                else if (!claimed[arg]) { f = FLAG_TP; claimed[arg] = 1; }
            }
            flags[dst + j] = f;
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------ 3. stable LSD radix sort
// tile histograms of digit (key >> shift) & 255, digit-major: hist[d * tiles + tile]
__global__ void __launch_bounds__(kSortThreads) voc_radix_hist_kernel(const unsigned long long* keys, const unsigned long long* total,
                                                                     int cap, int shift, int tiles, int* hist) {
    __shared__ int h[kRadix];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int n = stored(total, cap);
    const long start = (long)blockIdx.x * kSortTile;
    const long end = min(start + kSortTile, (long)n);
    for (long i = start + threadIdx.x; i < end; i += kSortThreads) atomicAdd(&h[(keys[i] >> shift) & (kRadix - 1)], 1);
    __syncthreads();
    hist[(long)threadIdx.x * tiles + blockIdx.x] = h[threadIdx.x];
}

// one CTA per digit: exclusive scan of its row over the tiles, in place; row_total[d] = the row's sum
__global__ void __launch_bounds__(kScanThreads) voc_radix_rows_kernel(int* hist, int tiles, int* row_total) {
    __shared__ int s[kScanThreads / 32];
    int* row = hist + (long)blockIdx.x * tiles;
    int carry = 0;
    for (int t0 = 0; t0 < tiles; t0 += kScanThreads) {
        const int t = t0 + threadIdx.x;
        const int v = t < tiles ? row[t] : 0;
        int tot;
        const int incl = block_incl_sum(v, s, &tot);
        if (t < tiles) row[t] = carry + incl - v;
        carry += tot;
    }
    if (threadIdx.x == 0) row_total[blockIdx.x] = carry;
}

// stable scatter of one tile: kSortRounds rounds of kSortThreads consecutive items; within a round the rank among equal
// digits comes from __match_any_sync (lanes) and per-warp digit counts (warps); across rounds from a running count
__global__ void __launch_bounds__(kSortThreads) voc_radix_scatter_kernel(const unsigned long long* keys_in, const int* vals_in,
                                                                        const unsigned long long* total, int cap, int shift,
                                                                        int tiles, const int* hist, const int* row_total,
                                                                        unsigned long long* keys_out, int* vals_out) {
    constexpr int W = kSortThreads / 32;
    __shared__ int s_base[kRadix];
    __shared__ int s_cnt[W][kRadix];
    __shared__ int s_scan[W];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = stored(total, cap);
    const long start = (long)blockIdx.x * kSortTile;
    if (start >= n) return;
    // digit base: exclusive scan of the 256 row totals (one digit per thread), plus this tile's row prefix
    {
        const int v = row_total[tid];
        int incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += u;
        }
        if (lane == 31) s_scan[warp] = incl;
        __syncthreads();
        int before = 0;
#pragma unroll
        for (int w = 0; w < W; ++w) before += w < warp ? s_scan[w] : 0;
        s_base[tid] = before + incl - v + hist[(long)tid * tiles + blockIdx.x];
#pragma unroll
        for (int w = 0; w < W; ++w) s_cnt[w][tid] = 0;
    }
    __syncthreads();
    const unsigned lt = (1u << lane) - 1u;
    for (int round = 0; round < kSortRounds; ++round) {
        const long i = start + (long)round * kSortThreads + tid;
        const bool valid = i < n;
        unsigned long long key = 0;
        int val = 0, d = kRadix + lane;                 // an invalid lane matches no other lane
        if (valid) {
            key = keys_in[i];
            val = vals_in[i];
            d = (int)((key >> shift) & (kRadix - 1));
        }
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int pre = __popc(peers & lt);
        if (valid && pre == 0) s_cnt[warp][d] = __popc(peers);
        __syncthreads();
        if (valid) {
            int off = s_base[d] + pre;
            for (int w = 0; w < warp; ++w) off += s_cnt[w][d];
            keys_out[off] = key;
            vals_out[off] = val;
        }
        __syncthreads();
        int sum = 0;
#pragma unroll
        for (int w = 0; w < W; ++w) {
            sum += s_cnt[w][tid];
            s_cnt[w][tid] = 0;
        }
        s_base[tid] += sum;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------ 4. curves and APs
// One CTA per class; its detections are rank positions [base, base + n) of the sorted values.
// out row k (class k+1): npos, n_det, tp, fp, ap07, ap
__global__ void __launch_bounds__(kScanThreads) voc_curve_kernel(const int* class_count, const unsigned long long* total, int cap,
                                                                const int* rank_pos, const unsigned char* flags, int n_gt,
                                                                const int* gt_labels,
                                                                const unsigned char* gt_difficult, int* tp_cum, int* fp_cum,
                                                                double* env, double* out) {
    __shared__ int s_i[kScanThreads / 32];
    __shared__ double s_d[kScanThreads / 32];
    __shared__ double s_p[11];
    const int k = blockIdx.x, c = k + 1, tid = threadIdx.x;
    const bool any = stored(total, cap) > 0;
    int base = 0;
    for (int q = 0; q < k && any; ++q) base += class_count[q];
    const int n = any ? class_count[k] : 0;
    int npos = 0;
    for (int g0 = 0; g0 < n_gt; g0 += kScanThreads) {
        const int g = g0 + tid;
        int tot;
        block_incl_sum(g < n_gt && gt_labels[g] == c && !gt_difficult[g], s_i, &tot);
        npos += tot;
    }
    tp_cum += base;
    fp_cum += base;
    env += base;
    rank_pos += base;
    // forward: TP / FP prefix sums (a chunk holds at most kScanThreads of each: 16 bits apiece) and the precision
    int tp = 0, fp = 0;
    for (int s0 = 0; s0 < n; s0 += kScanThreads) {
        const int i = s0 + tid;
        const int p = i < n ? rank_pos[i] : -1;   // a position outside the pool only if an image index was appended twice
        const int f = p < 0 ? FLAG_IGNORED : (p < cap ? flags[p] : FLAG_FP);
        int tot;
        const int incl = block_incl_sum((f == FLAG_TP ? 1 << 16 : 0) | (f == FLAG_FP ? 1 : 0), s_i, &tot);
        if (i < n) {
            const int t = tp + (incl >> 16), u = fp + (incl & 0xffff);
            tp_cum[i] = t;
            fp_cum[i] = u;
            env[i] = __ddiv_rn((double)t, fmax(__dadd_rn((double)t, (double)u), DBL_EPSILON));
        }
        tp += tot >> 16;
        fp += tot & 0xffff;
    }
    __syncthreads();
    // backward: the precision envelope (running maximum from the end; mpre's trailing 0 changes nothing) and, at every
    // position where recall changes, the area term (rec[i] - rec[i-1]) * env[i]; each thread sums its positions in order
    const double dn = (double)npos;
    double carry = 0.0, acc = 0.0;
    for (int e = n; e > 0; e -= kScanThreads) {
        const int i = e - 1 - tid;
        const double p = i >= 0 ? env[i] : 0.0;
        double tot;
        const double v = fmax(block_incl_max(p, s_d, &tot), carry);
        if (i >= 0) {
            env[i] = v;
            const int t = tp_cum[i], t_prev = i > 0 ? tp_cum[i - 1] : 0;
            if (t != t_prev) acc = __dadd_rn(acc, __dmul_rn(__dsub_rn(__ddiv_rn((double)t, dn), __ddiv_rn((double)t_prev, dn)), v));
        }
        carry = fmax(carry, tot);
    }
    // fixed-order reduction of the per-thread sums: warps by shuffle tree, then the warp sums in order
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, d));
    if ((tid & 31) == 0) s_d[tid >> 5] = acc;
    __syncthreads();
    // 11-point: p(t) = max(prec[rec >= t]) = env[first i with rec[i] >= t] (rec never decreases), 0 if there is none
    if (tid < 11) {
        const double t = __dmul_rn((double)tid, 0.1);
        int lo = 0, hi = n;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (__ddiv_rn((double)tp_cum[mid], dn) >= t) hi = mid; else lo = mid + 1;
        }
        s_p[tid] = lo < n ? env[lo] : 0.0;
    }
    __syncthreads();
    if (tid == 0) {
        double ap = 0.0, ap07 = 0.0;
        for (int w = 0; w < kScanThreads / 32; ++w) ap = __dadd_rn(ap, s_d[w]);
        for (int q = 0; q < 11; ++q) ap07 = __dadd_rn(ap07, __ddiv_rn(s_p[q], 11.0));
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        double* o = out + 3 + 6 * k;
        o[0] = npos;
        o[1] = n;
        o[2] = tp;
        o[3] = fp;
        o[4] = npos > 0 ? ap07 : nan;
        o[5] = npos > 0 ? ap : nan;
    }
}

// ------------------------------------------------------------------------------------------ 5. status and means
__global__ void voc_finish_kernel(int NC, const unsigned long long* total, int cap, double* out) {
    double s07 = 0.0, s = 0.0;
    int m = 0;
    for (int k = 0; k < NC - 1; ++k) {
        const double* o = out + 3 + 6 * k;
        if (o[0] > 0.0) {
            s07 = __dadd_rn(s07, o[4]);
            s = __dadd_rn(s, o[5]);
            ++m;
        }
    }
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    out[0] = *total > (unsigned long long)cap ? 1.0 : 0.0;
    out[1] = m > 0 ? __ddiv_rn(s07, (double)m) : nan;
    out[2] = m > 0 ? __ddiv_rn(s, (double)m) : nan;
}

int class_bits(int NC) { return NC - 2 > 0 ? 32 - __builtin_clz((unsigned)(NC - 2)) : 0; }

}  // namespace
}  // namespace frcnn

using namespace frcnn;

#define VOC_REQUIRE_SHAPE(fn, NC, cap, max_images)                                                                            \
    do {                                                                                                                      \
        FRCNN_REQUIRE((NC) >= 2 && (NC) <= 65536, "%s: num_classes must be in [2,65536] (got %d)", fn, (int)(NC));             \
        FRCNN_REQUIRE((cap) >= 1 && (cap) <= kCapacityMax, "%s: capacity must be in [1,%d] (got %d)", fn, kCapacityMax,          \
                      (int)(cap));                                                                                            \
        FRCNN_REQUIRE((max_images) >= 1, "%s: max_images must be >= 1 (got %d)", fn, (int)(max_images));                      \
        FRCNN_REQUIRE((long long)((NC) - 1) * (max_images) <= 0x7fffffffll, "%s: (num_classes-1) * max_images is too large",  \
                      fn);                                                                                                    \
    } while (0)

extern "C" size_t frcnn_voc_eval_workspace_bytes(int num_classes, int capacity, int max_images, int max_gt) {
    if (num_classes < 2 || num_classes > 65536 || capacity < 1 || capacity > kCapacityMax || max_images < 1 || max_gt < 0 ||
        (long long)(num_classes - 1) * max_images > 0x7fffffffll) {
        set_error("frcnn_voc_eval_workspace_bytes: bad sizes (num_classes=%d capacity=%d max_images=%d max_gt=%d)", num_classes,
                  capacity, max_images, max_gt);
        return 0;
    }
    return voc_layout(num_classes, capacity, max_images, max_gt).bytes;
}

extern "C" int frcnn_voc_eval_append_batch(int N, const float* prob, long prob_stride, const float* boxes, long boxes_stride,
                                           const int* keep_idx, long keep_idx_stride, const int* conf_count, long conf_count_stride,
                                           const double* im_scale, int R_cap, int num_classes, int image_base, int capacity,
                                           int max_images, void* ws, size_t ws_bytes, void* stream) {
    FRCNN_ENTRY();
    const char* fn = "frcnn_voc_eval_append_batch";
    FRCNN_REQUIRE(prob, "%s: prob is NULL", fn);
    FRCNN_REQUIRE(boxes, "%s: boxes is NULL", fn);
    FRCNN_REQUIRE(keep_idx, "%s: keep_idx is NULL", fn);
    FRCNN_REQUIRE(conf_count, "%s: conf_count is NULL", fn);
    FRCNN_REQUIRE(im_scale, "%s: im_scale is NULL", fn);
    FRCNN_REQUIRE(ws, "%s: ws is NULL", fn);
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "%s: N must be in [1,65535] (got N=%d)", fn, N);
    FRCNN_REQUIRE(R_cap >= 1, "%s: R_cap must be >= 1 (got R_cap=%d)", fn, R_cap);
    VOC_REQUIRE_SHAPE(fn, num_classes, capacity, max_images);
    FRCNN_REQUIRE((long)(num_classes - 1) * R_cap <= 0x7fffffffl, "%s: (num_classes-1) * R_cap is too large", fn);
    FRCNN_REQUIRE(prob_stride >= 0 && boxes_stride >= 0 && keep_idx_stride >= 0 && conf_count_stride >= 0,
                  "%s: image strides must be >= 0", fn);
    FRCNN_REQUIRE(image_base >= 0 && (long)image_base + N <= max_images,
                  "%s: images [%d, %ld) are not within max_images = %d", fn, image_base, (long)image_base + N, max_images);
    const VocLayout L = voc_layout(num_classes, capacity, max_images, 0);
    if (ws_bytes < L.bytes) {
        set_error("%s: workspace of %zu bytes, %zu needed", fn, ws_bytes, L.bytes);
        return FRCNN_ERR_WORKSPACE;
    }
    const EvalStrides is = {prob_stride, boxes_stride, keep_idx_stride, conf_count_stride};
    FRCNN_CUDA_OK(launch_plain(voc_append_kernel, dim3(N, cdiv(num_classes - 1, kAppendWarps)), dim3(kAppendWarps * 32), 0,
                               (cudaStream_t)stream, prob, boxes, keep_idx, conf_count, im_scale, R_cap, num_classes, is, image_base,
                               capacity, max_images, at<unsigned long long>(ws, L.total), at<int2>(ws, L.seg),
                               at<float4>(ws, L.pool_box), at<float>(ws, L.pool_score)));
    return FRCNN_OK;
}

extern "C" int frcnn_voc_eval(int num_classes, int capacity, int max_images, int max_gt, int n_images, const int* gt_offsets,
                              const float* gt_boxes, const int* gt_labels, const unsigned char* gt_difficult, int n_gt,
                              double iou_thresh, double* out, void* ws, size_t ws_bytes, void* stream) {
    FRCNN_ENTRY();
    const char* fn = "frcnn_voc_eval";
    FRCNN_REQUIRE(gt_offsets, "%s: gt_offsets is NULL", fn);
    FRCNN_REQUIRE(gt_boxes, "%s: gt_boxes is NULL", fn);
    FRCNN_REQUIRE(gt_labels, "%s: gt_labels is NULL", fn);
    FRCNN_REQUIRE(gt_difficult, "%s: gt_difficult is NULL", fn);
    FRCNN_REQUIRE(out, "%s: out is NULL", fn);
    FRCNN_REQUIRE(ws, "%s: ws is NULL", fn);
    VOC_REQUIRE_SHAPE(fn, num_classes, capacity, max_images);
    FRCNN_REQUIRE(max_gt >= 0, "%s: max_gt must be >= 0 (got %d)", fn, max_gt);
    FRCNN_REQUIRE(n_images >= 0 && n_images <= max_images, "%s: n_images must be in [0, max_images = %d] (got %d)", fn, max_images,
                  n_images);
    FRCNN_REQUIRE(n_gt >= 0 && n_gt <= max_gt, "%s: n_gt must be in [0, max_gt = %d] (got %d)", fn, max_gt, n_gt);
    FRCNN_REQUIRE(isfinite(iou_thresh), "%s: iou_thresh must be finite", fn);
    const VocLayout L = voc_layout(num_classes, capacity, max_images, max_gt);
    if (ws_bytes < L.bytes) {
        set_error("%s: workspace of %zu bytes, %zu needed", fn, ws_bytes, L.bytes);
        return FRCNN_ERR_WORKSPACE;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const int K = num_classes - 1, tiles = cdiv(capacity, kSortTile);
    const unsigned long long* total = at<unsigned long long>(ws, L.total);
    if (n_gt > 0) FRCNN_CUDA_OK(cudaMemsetAsync(at<unsigned char>(ws, L.claimed), 0, (size_t)n_gt, st));
    FRCNN_CUDA_OK(launch_plain(voc_class_offsets_kernel, dim3(K), dim3(kScanThreads), 0, st, at<const int2>(ws, L.seg), max_images,
                               at<int>(ws, L.seg_off), at<int>(ws, L.class_count)));
    const long segs = (long)K * max_images;
    FRCNN_CUDA_OK(launch_plain(voc_match_kernel, dim3((unsigned)((segs + kMatchWarps - 1) / kMatchWarps)), dim3(kMatchWarps * 32), 0,
                               st, num_classes, max_images, n_images, n_gt, gt_offsets, gt_boxes, gt_labels, gt_difficult, iou_thresh,
                               total, capacity, at<const int2>(ws, L.seg), at<const float4>(ws, L.pool_box),
                               at<const float>(ws, L.pool_score), at<const int>(ws, L.seg_off), at<const int>(ws, L.class_count),
                               at<unsigned char>(ws, L.flags), at<unsigned long long>(ws, L.keys[0]), at<int>(ws, L.vals[0]),
                               at<int>(ws, L.vals[1]), at<unsigned char>(ws, L.claimed)));
    const int passes = cdiv(32 + class_bits(num_classes), 8);
    int b = 0;
    for (int p = 0; p < passes; ++p, b ^= 1) {
        FRCNN_CUDA_OK(launch_plain(voc_radix_hist_kernel, dim3(tiles), dim3(kSortThreads), 0, st,
                                   at<const unsigned long long>(ws, L.keys[b]), total, capacity, 8 * p, tiles, at<int>(ws, L.hist)));
        FRCNN_CUDA_OK(launch_plain(voc_radix_rows_kernel, dim3(kRadix), dim3(kScanThreads), 0, st, at<int>(ws, L.hist), tiles,
                                   at<int>(ws, L.row_total)));
        FRCNN_CUDA_OK(launch_plain(voc_radix_scatter_kernel, dim3(tiles), dim3(kSortThreads), 0, st,
                                   at<const unsigned long long>(ws, L.keys[b]), at<const int>(ws, L.vals[b]), total, capacity, 8 * p,
                                   tiles, at<const int>(ws, L.hist), at<const int>(ws, L.row_total),
                                   at<unsigned long long>(ws, L.keys[b ^ 1]), at<int>(ws, L.vals[b ^ 1])));
    }
    FRCNN_CUDA_OK(launch_plain(voc_curve_kernel, dim3(K), dim3(kScanThreads), 0, st, at<const int>(ws, L.class_count), total,
                               capacity, at<const int>(ws, L.vals[b]), at<const unsigned char>(ws, L.flags), n_gt, gt_labels, gt_difficult,
                               at<int>(ws, L.tp_cum), at<int>(ws, L.fp_cum), at<double>(ws, L.env), out));
    FRCNN_CUDA_OK(launch_plain(voc_finish_kernel, dim3(1), dim3(1), 0, st, num_classes, total, capacity, out));
    return FRCNN_OK;
}
