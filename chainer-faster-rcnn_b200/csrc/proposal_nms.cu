// proposal_nms.cu -- the ProposalLayer and greedy-NMS path on device.
//
// Replaces (all under /root/reference): models/proposal_layer.py:102-221 (anchor grid, decode, clip,
// min-size filter, sort, top-N, NMS, top-N), models/bbox_transform.py:41-109, models/cpu_nms.pyx:18-69
// (the live NMS), and retires models/gpu_nms.pyx + models/nms_kernel.cu (dead on the live path, Q2).
//
// All box arithmetic is float32 with ONE rounding per operation (explicit __f*_rn intrinsics: no FMA
// contraction), in the reference's operation order, so results are bit-identical to the CPU oracle.
// These are HBM/latency-bound integer/float kernels -- no tensor cores by design.
//
// Pipeline (5 launches, no host sync, data-dependent counts stay on device):
//   1. rpn_decode_kernel   one thread per anchor: [2A-way softmax ->] fg score, anchor from index,
//                          decode + clip + min-size test -> box[i], score[i], sort key[i] (0 = filtered)
//   2. topk_sort_kernel    ONE CTA: 4-pass radix select of the pre_nms_top_n-th key, order-preserving
//                          compaction of the survivors' (key | ~index) composites
//   3. rank_scatter_kernel chip-wide rank-by-counting of the unique composites = argsort(key desc, index
//                          asc); scatters box / score / index to the sorted position
//   4. nms_mask_kernel     upper-triangular 64x64 IoU tiles -> uint64 suppression bitmask
//   5. nms_scan_kernel     ONE CTA walks the mask (device-side; the reference copies it to the host,
//                          nms_kernel.cu:124-139), stops at post_nms_top_n, gathers the output rows
#include "common.cuh"
#include "nms_math.cuh"

namespace frcnn {

// ------------------------------------------------------------------------------------------ 1. decode
struct DecodeArgs {
    const float* cls; long cls_cs, cls_ps; int cls_is_logits;
    const float* bbox; long bbox_cs, bbox_ps;
    const double* anchors;
    int A, H, W, feat_stride, im_h, im_w, min_size;
    float4* boxes; float* scores; uint32_t* keys;
};

__global__ void rpn_decode_kernel(const DecodeArgs a) {
    grid_dep_wait();
    const int n = a.A * a.H * a.W;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int pix = i / a.A, an = i - pix * a.A;
    const int h = pix / a.W, w = pix - h * a.W;

    // fg score: channel A+an of rpn_cls_prob (models/proposal_layer.py:152-154)
    float score;
    if (a.cls_is_logits) {
        // F.softmax over ALL 2A channels (models/region_proposal_network.py:119, SURVEY Q1):
        // y = x - max; e = exp(y); e / sum(e), sum in ascending channel order.
        const float* c = a.cls + (long)pix * a.cls_ps;
        float m = c[0];
        for (int k = 1; k < 2 * a.A; ++k) m = fmaxf(m, c[(long)k * a.cls_cs]);
        float s = 0.0f, mine = 0.0f;
        for (int k = 0; k < 2 * a.A; ++k) {
            float e = det_expf(__fsub_rn(c[(long)k * a.cls_cs], m));
            s = __fadd_rn(s, e);
            if (k == a.A + an) mine = e;
        }
        score = __fdiv_rn(mine, s);
    } else {
        score = a.cls[(long)(a.A + an) * a.cls_cs + (long)pix * a.cls_ps];
    }

    // anchor (models/proposal_layer.py:207-221): float64 base + integer shift, cast to float32
    const double sx = (double)(w * a.feat_stride), sy = (double)(h * a.feat_stride);
    const float ax1 = (float)(a.anchors[4 * an + 0] + sx);
    const float ay1 = (float)(a.anchors[4 * an + 1] + sy);
    const float ax2 = (float)(a.anchors[4 * an + 2] + sx);
    const float ay2 = (float)(a.anchors[4 * an + 3] + sy);
    // deltas: bbox_trans[(h*W+w)*A + an, j] = rpn_bbox_pred[4*an + j, h, w]  (:138)
    const float* d = a.bbox + (long)pix * a.bbox_ps + (long)(4 * an) * a.bbox_cs;
    const float dx = d[0], dy = d[a.bbox_cs], dw = d[2 * a.bbox_cs], dh = d[3 * a.bbox_cs];

    // bbox_transform_inv (models/bbox_transform.py:51-74)
    const float bw = __fadd_rn(__fsub_rn(ax2, ax1), 1.0f);
    const float bh = __fadd_rn(__fsub_rn(ay2, ay1), 1.0f);
    const float cx = __fadd_rn(ax1, __fmul_rn(0.5f, bw));
    const float cy = __fadd_rn(ay1, __fmul_rn(0.5f, bh));
    const float pcx = __fadd_rn(__fmul_rn(dx, bw), cx);
    const float pcy = __fadd_rn(__fmul_rn(dy, bh), cy);
    const float pw = __fmul_rn(det_expf(dw), bw);
    const float ph = __fmul_rn(det_expf(dh), bh);
    float x1 = __fsub_rn(pcx, __fmul_rn(0.5f, pw));
    float y1 = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
    float x2 = __fadd_rn(pcx, __fmul_rn(0.5f, pw));
    float y2 = __fadd_rn(pcy, __fmul_rn(0.5f, ph));
    // clip_boxes (models/bbox_transform.py:87-98): max(min(v, bound), 0)
    const float wmax = (float)(a.im_w - 1), hmax = (float)(a.im_h - 1);
    x1 = fmaxf(fminf(x1, wmax), 0.0f);
    y1 = fmaxf(fminf(y1, hmax), 0.0f);
    x2 = fmaxf(fminf(x2, wmax), 0.0f);
    y2 = fmaxf(fminf(y2, hmax), 0.0f);
    // filter_boxes (models/bbox_transform.py:105-108)
    const float ws = __fadd_rn(__fsub_rn(x2, x1), 1.0f);
    const float hs = __fadd_rn(__fsub_rn(y2, y1), 1.0f);
    const bool ok = (ws >= (float)a.min_size) && (hs >= (float)a.min_size) && (score == score);

    a.boxes[i] = make_float4(x1, y1, x2, y2);
    a.scores[i] = score;
    a.keys[i] = ok ? float_to_ordered(score) : 0u;
}

__global__ void dets_keys_kernel(const float* dets, int n, float4* boxes, float* scores, uint32_t* keys) {
    grid_dep_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* d = dets + 5l * i;
    boxes[i] = make_float4(d[0], d[1], d[2], d[3]);
    scores[i] = d[4];
    keys[i] = float_to_ordered(d[4]);     // never 0: every det is a candidate (cpu_nms has no filter)
}

// ------------------------------------------------------------------------------------------ 2. select + sort
constexpr int kSortThreads = 1024;

// Exclusive prefix sum over blockDim.x values (one per thread); returns the exclusive prefix,
// *total = sum of all.  `red` is a 33-entry smem scratch.
__device__ __forceinline__ unsigned long long block_exclusive_scan(unsigned long long v, unsigned long long* red,
                                                                   unsigned long long* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) red[wid] = x;
    __syncthreads();
    if (wid == 0) {
        unsigned long long w = lane < nw ? red[lane] : 0ull;
        unsigned long long xs = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned long long y = __shfl_up_sync(0xffffffffu, xs, o);
            if (lane >= o) xs += y;
        }
        red[lane] = xs - w;             // exclusive warp offsets
        if (lane == 31) red[32] = xs;   // grand total
    }
    __syncthreads();
    unsigned long long res = red[wid] + x - v;
    *total = red[32];
    __syncthreads();
    return res;
}

struct SortArgs {
    const uint32_t* keys; int n; int top_k;
    const float4* boxes; const float* scores;
    float4* sorted_boxes; float* sorted_scores; int* sorted_idx; int* num_sorted;
    float* dbg_dets; int* dbg_idx; int* dbg_num;
    long long* dbg_clocks;     // optional: 8 phase timestamps (clock64 of thread 0)
    unsigned long long* comp_out;   // [k_cap] selected composites (key desc | index), unordered
};

// Selection step (ONE CTA): count, 4-pass radix select of the top_k-th key, order-preserving compaction.
// dynamic smem: uint64 comp[P] (P >= min(top_k, n)) followed, when it fits, by a copy of the n keys
// (the select passes then never touch global memory again).
__global__ void __launch_bounds__(kSortThreads, 1) topk_sort_kernel(const SortArgs a, const int P, const int cache_keys) {
    grid_dep_wait();
    extern __shared__ unsigned long long comp[];
    __shared__ unsigned int hist[256];
    __shared__ unsigned int whist[32 * 256];
    __shared__ unsigned long long red[33];
    __shared__ unsigned int s_prefix, s_need;
    const int tid = threadIdx.x, lane = tid & 31;
    const int n = a.n;
    const int n_pad = (n + 31) & ~31;                 // whole warps iterate together (warp-aggregated atomics)
    uint32_t* skeys = reinterpret_cast<uint32_t*>(comp + P);
    const uint32_t* keys = a.keys;
#define SORT_MARK(i) do { if (a.dbg_clocks && tid == 0) a.dbg_clocks[i] = clock64(); } while (0)
    SORT_MARK(0);

    // ---- count candidates (key != 0), filling the smem copy on the way
    unsigned int cnt = 0;
    for (int i = tid; i < n; i += kSortThreads) {
        const uint32_t k = a.keys[i];
        if (cache_keys) skeys[i] = k;
        cnt += k != 0u;
    }
    unsigned long long tot;
    block_exclusive_scan(cnt, red, &tot);             // (has the barriers that publish skeys)
    if (cache_keys) keys = skeys;
    const int n_valid = (int)tot;
    const int K = n_valid < a.top_k ? n_valid : a.top_k;      // how many we keep
    SORT_MARK(1);

    // ---- radix select: the K-th largest key T (MSB-first, 8 bits per pass)
    unsigned int prefix = 0, need = (unsigned int)K;     // need = rank (1-based) inside the current bucket
    if (K > 0 && K < n_valid) {
        for (int pass = 0; pass < 4; ++pass) {
            const int shift = 24 - 8 * pass;
            const unsigned int mask_hi = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
            // per-warp private histograms (whist[warp][digit]; bank = digit % 32): a warp whose active lanes all hold the same
            // digit -- the rule in the first passes, where the keys share their leading bits -- adds its count with ONE
            // atomic, any other warp lets every lane add 1 to its own bin.  (The first version elected group leaders with
            // __match_any_sync for every key: 43 k of the kernel's 60 k cycles, profiles/r02_sort_profile.txt.)
            for (int i = tid; i < 32 * 256; i += kSortThreads) whist[i] = 0;
            __syncthreads();
            unsigned int* mine_h = whist + (tid >> 5) * 256;
            for (int i = tid; i < n_pad; i += kSortThreads) {
                const unsigned int k = i < n ? keys[i] : 0u;
                const bool act = k != 0u && (k & mask_hi) == prefix;
                const unsigned int digit = (k >> shift) & 255u;
                const unsigned int amask = __ballot_sync(0xffffffffu, act);
                if (amask == 0u) continue;
                const unsigned int lead = __shfl_sync(0xffffffffu, digit, __ffs(amask) - 1);
                const unsigned int same = __ballot_sync(0xffffffffu, act && digit == lead);
                if (same == amask) {
                    if (lane == __ffs(amask) - 1) atomicAdd(&mine_h[lead], (unsigned int)__popc(amask));
                } else if (act) {
                    atomicAdd(&mine_h[digit], 1u);
                }
            }
            __syncthreads();
            if (tid < 256) {
                unsigned int acc_h = 0;
#pragma unroll 8
                for (int w = 0; w < 32; ++w) acc_h += whist[w * 256 + tid];
                hist[tid] = acc_h;
            }
            __syncthreads();
            // suffix counts: bin b is chosen if  sum(hist[b+1..255]) < need <= sum(hist[b..255])
            unsigned long long v = tid < 256 ? (unsigned long long)hist[255 - tid] : 0ull;   // reversed
            unsigned long long t2;
            unsigned long long above = block_exclusive_scan(v, red, &t2);   // count in bins > b
            if (tid < 256) {
                const unsigned int b = 255 - tid;
                if (above < need && need <= above + v) {
                    s_prefix = prefix | (b << shift);
                    s_need = need - (unsigned int)above;
                }
            }
            __syncthreads();
            prefix = s_prefix;
            need = s_need;
            __syncthreads();
        }
    }
    SORT_MARK(2);
    // Now: keys > T are all taken; among keys == T the `need` lowest indices are taken.
    const unsigned int T = (K > 0 && K < n_valid) ? prefix : 1u;       // K == n_valid: take every candidate
    const bool take_all = !(K > 0 && K < n_valid);

    // ---- order-preserving compaction into comp[] (each thread owns a contiguous index range)
    const int chunk = (n + kSortThreads - 1) / kSortThreads;
    const int i0 = tid * chunk, i1 = min(n, i0 + chunk);
    unsigned int c_gt = 0, c_eq = 0;
    for (int i = i0; i < i1; ++i) {
        const unsigned int k = keys[i];
        if (k == 0u) continue;
        if (take_all || k > T) ++c_gt; else if (k == T) ++c_eq;
    }
    unsigned long long packed = ((unsigned long long)c_eq << 32) | c_gt, tot2;
    unsigned long long pre = block_exclusive_scan(packed, red, &tot2);
    unsigned int gt_before = (unsigned int)(pre & 0xFFFFFFFFu), eq_before = (unsigned int)(pre >> 32);
    const unsigned int gt_total = (unsigned int)(tot2 & 0xFFFFFFFFu);
    const unsigned int eq_take = take_all ? 0u : need;
    for (int i = i0; i < i1; ++i) {
        const unsigned int k = keys[i];
        if (k == 0u) continue;
        // composite: ascending order == (key descending, index ascending)
        const unsigned long long c = ((unsigned long long)(~k) << 32) | (unsigned int)i;
        if (take_all || k > T) {
            comp[gt_before++] = c;
        } else if (k == T) {
            if (eq_before < eq_take) comp[gt_total + eq_before] = c;
            ++eq_before;
        }
    }
    __syncthreads();
    SORT_MARK(3);
    // ---- hand the K selected composites (unordered) to the chip-wide rank kernel
    for (int r = tid; r < K; r += kSortThreads) a.comp_out[r] = comp[r];
    SORT_MARK(4);
    SORT_MARK(5);
#undef SORT_MARK
    if (tid == 0) {
        *a.num_sorted = K;
        if (a.dbg_num) *a.dbg_num = K;
    }
}

// Ordering step: rank-by-counting across the whole chip.  The composites are unique (they contain the
// index), so rank(i) = #{j : comp[j] < comp[i]} is a permutation; 6000^2 64-bit compares spread over the
// whole chip, where a single-CTA bitonic network of the same 6000 elements is instruction-issue bound on one SM.  Each block ranks 32 elements (8 threads per element, each scanning 1/8 of the list from
// a shared-memory copy) and scatters box / score / index straight to the sorted position.
constexpr int kRankThreads = 256, kRankPerBlock = 32;
__global__ void __launch_bounds__(kRankThreads) rank_scatter_kernel(const SortArgs a) {
    grid_dep_wait();
    extern __shared__ unsigned long long scomp[];
    const int K = *a.num_sorted;
    const int e0 = blockIdx.x * kRankPerBlock;
    if (e0 >= K) return;
    for (int i = threadIdx.x; i < K; i += kRankThreads) scomp[i] = a.comp_out[i];
    __syncthreads();
    const int e = e0 + (threadIdx.x >> 3), part = threadIdx.x & 7;
    const bool live = e < K;
    const unsigned long long mine = live ? scomp[e] : 0ull;
    int cnt = 0;
    for (int j = part; j < K; j += 8) cnt += scomp[j] < mine;
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 1);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 2);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 4);
    if (live && part == 0) {
        const int r = cnt;
        const int idx = (int)(mine & 0xFFFFFFFFull);
        const float4 b = a.boxes[idx];
        const float s = a.scores[idx];
        a.sorted_boxes[r] = b;
        a.sorted_scores[r] = s;
        a.sorted_idx[r] = idx;
        if (a.dbg_dets) {
            float* o = a.dbg_dets + 5l * r;
            o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w; o[4] = s;
        }
        if (a.dbg_idx) a.dbg_idx[r] = idx;
    }
}


// ------------------------------------------------------------------------------------------ 3. IoU bitmask
// grid (col_blocks, col_blocks); only blocks with col >= row do work.  mask[row_box][col_block].
// Thread = one row box against the block's 64 column boxes (shared memory, broadcast reads, areas precomputed): one
// branch-free suppress_word64() per thread, ~25 instructions a pair.  (Pairs that branched on their decision path
// diverged the warp on almost every column: 38 us for 6000 boxes, ~4x the instruction-issue bound.)
__global__ void __launch_bounds__(64) nms_mask_kernel(const float4* boxes, const int* n_ptr, int n_cap,
                                                      double thr_d, float thr_f, int mode,
                                                      unsigned long long* mask, int col_blocks) {
    grid_dep_wait();
    const int n = n_ptr ? min(*n_ptr, n_cap) : n_cap;
    const int rb = blockIdx.y, cb = blockIdx.x;
    if (cb < rb || rb * 64 >= n || cb * 64 >= n) return;
    __shared__ float4 cbox[64];
    __shared__ float carea[64];
    const int t = threadIdx.x;
    const int ccount = min(64, n - cb * 64);
    {
        const float4 b = t < ccount ? boxes[cb * 64 + t] : make_float4(0.f, 0.f, 0.f, 0.f);
        cbox[t] = b;
        carea[t] = box_area(b);
    }
    __syncthreads();
    const int ri = rb * 64 + t;
    if (ri >= n) return;
    const float4 a = boxes[ri];
    const int start = (rb == cb) ? t + 1 : 0;               // the diagonal block: pairs (i, j > i) only
    unsigned long long live = ccount < 64 ? (1ull << ccount) - 1ull : ~0ull;       // columns [start, ccount)
    live = start < 64 ? (live >> start) << start : 0ull;
    mask[(long)ri * col_blocks + cb] = suppress_word64(a, box_area(a), cbox, carea, live, pretest_bounds(thr_f), thr_d, thr_f, mode);
}

// ------------------------------------------------------------------------------------------ 4. mask scan
struct ScanArgs {
    const unsigned long long* mask; int col_blocks;
    const int* n_ptr; int n_cap; int max_keep;
    const int* index_map;          // optional: sorted position -> original index
    int* keep_out; int* num_out;   // optional
    const float4* sorted_boxes; const float* sorted_scores;   // optional gather
    float* out_rois; float* out_scores; int out_cap;
    int diag_in_smem;
};

__global__ void __launch_bounds__(256, 1) nms_scan_kernel(const ScanArgs a) {
    grid_dep_wait();
    extern __shared__ unsigned long long removed[];   // [col_blocks]
    __shared__ unsigned long long tile[256][4];       // the current super-block's rows x its own four 64-column words
    __shared__ int s_keep[256];
    __shared__ int s_nk, s_total;
    __shared__ int s_keep_all[2048];                  // positions of the first 2048 survivors (for the gather)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = a.n_ptr ? min(*a.n_ptr, a.n_cap) : a.n_cap;
    const int nb = (n + 63) / 64;
    const int nsb = (nb + 3) / 4;
    const int limit = a.max_keep > 0 ? a.max_keep : 0x7fffffff;
    for (int w = tid; w < a.col_blocks; w += blockDim.x) removed[w] = 0ull;
    if (tid == 0) s_total = 0;
    // The greedy chain is serial in the 64-row blocks, and every step that has to wait for L2 (the kept rows' mask words for
    // the blocks ahead) costs ~0.7 us: with one such step per block the scan took 75 us on 94 blocks.  Here FOUR blocks form
    // a super-block: its 256 x 256-bit corner of the mask (8 KB) is staged in shared memory -- requested one super-block
    // ahead, so that latency is off the chain -- and warp 0 resolves all four blocks from shared memory alone; only the fold
    // of the super-block's kept rows into the words beyond it goes to L2, once per 256 rows.
    unsigned long long pf[4];
    auto request = [&](int sb) {                      // thread t: row sb*256 + t, words 4sb .. 4sb+3
        const long row = (long)sb * 256 + tid;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int w = 4 * sb + j;
            pf[j] = (row < n && w < nb) ? a.mask[row * a.col_blocks + w] : 0ull;
        }
    };
    if (nsb > 0) request(0);
    __syncthreads();

    for (int sb = 0; sb < nsb; ++sb) {
#pragma unroll
        for (int j = 0; j < 4; ++j) tile[tid][j] = pf[j];
        __syncthreads();
        if (sb + 1 < nsb) request(sb + 1);            // in flight while this super-block is resolved and folded
        if (warp == 0) {
            int total = s_total, nk = 0;
            for (int j = 0; j < 4 && 4 * sb + j < nb && total < limit; ++j) {
                const int blk = 4 * sb + j;
                const int rows = min(64, n - blk * 64);
                unsigned long long cand = ~removed[blk];
                if (rows < 64) cand &= (1ull << rows) - 1ull;
                while (cand != 0ull && total < limit) {
                    const int i = __ffsll((long long)cand) - 1;
                    const int lr = 64 * j + i;                      // row inside the super-block
                    if (lane == 0) {
                        s_keep[nk] = lr;
                        const int pos = blk * 64 + i;
                        if (a.keep_out) a.keep_out[total] = a.index_map ? a.index_map[pos] : pos;
                        if (total < 2048) s_keep_all[total] = pos;
                    }
                    ++nk;
                    ++total;
                    cand &= ~tile[lr][j];
                    cand &= ~(1ull << i);
                    if (lane > j && lane < 4 && 4 * sb + lane < nb) removed[4 * sb + lane] |= tile[lr][lane];    // later blocks of this super-block
                }
                __syncwarp();                    // lanes 1..3's words are read by every lane in the next round
            }
            if (lane == 0) { s_nk = nk; s_total = total; }
        }
        __syncthreads();
        const int nk = s_nk;
        if (s_total >= limit) break;
        // Fold the kept rows of this super-block into `removed` for the blocks beyond it: nk x W mask words, spread over ALL
        // threads (item = (kept row, word)), 8 independent loads in flight per thread, OR-ed into shared memory with atomics.
        const int w0 = 4 * (sb + 1);
        const int W = nb - w0;
        const int items = W > 0 ? nk * W : 0;
        const unsigned long long* base = a.mask + (long)(sb * 256) * a.col_blocks + w0;
        for (int it0 = tid; it0 < items; it0 += 8 * 256) {
            unsigned long long m[8];
            int wv[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int it = it0 + u * 256;
                m[u] = 0ull;
                wv[u] = 0;
                if (it < items) {
                    const int k = it / W, w = it - k * W;
                    wv[u] = w;
                    m[u] = base[(long)s_keep[k] * a.col_blocks + w];
                }
            }
#pragma unroll
            for (int u = 0; u < 8; ++u)
                if (m[u] != 0ull) atomicOr(&removed[w0 + wv[u]], m[u]);
        }
        __syncthreads();
    }
    __syncthreads();
    const int total = s_total;
    if (tid == 0 && a.num_out) *a.num_out = total;
    if (a.out_rois) {
        for (int r = tid; r < a.out_cap; r += blockDim.x) {
            float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
            float s = 0.f;
            if (r < total && r < 2048) {
                const int pos = s_keep_all[r];
                b = a.sorted_boxes[pos];
                s = a.sorted_scores[pos];
            }
            reinterpret_cast<float4*>(a.out_rois)[r] = b;
            if (a.out_scores) a.out_scores[r] = s;
        }
    }
}

// ------------------------------------------------------------------------------------------ workspace carving
struct NmsWs {
    float4* boxes; float* scores; uint32_t* keys;             // [n_all]
    float4* sorted_boxes; float* sorted_scores; int* sorted_idx;  // [k_cap]
    int* num_sorted;
    unsigned long long* mask;                                  // [k_cap * col_blocks]
    unsigned long long* comp;                                  // [k_cap]
    int col_blocks;
    size_t total;
};

static NmsWs carve(void* ws, int n_all, int k_cap) {
    NmsWs w;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    char* base = static_cast<char*>(ws);
    w.col_blocks = cdiv(k_cap, 64);
    size_t o_boxes = take(sizeof(float4) * (size_t)n_all);
    size_t o_scores = take(sizeof(float) * (size_t)n_all);
    size_t o_keys = take(sizeof(uint32_t) * (size_t)n_all);
    size_t o_sb = take(sizeof(float4) * (size_t)k_cap);
    size_t o_ss = take(sizeof(float) * (size_t)k_cap);
    size_t o_si = take(sizeof(int) * (size_t)k_cap);
    size_t o_ns = take(sizeof(int) * 4);
    size_t o_mask = take(sizeof(unsigned long long) * (size_t)k_cap * w.col_blocks);
    size_t o_comp = take(sizeof(unsigned long long) * (size_t)k_cap);
    w.total = off;
    w.boxes = reinterpret_cast<float4*>(base + o_boxes);
    w.scores = reinterpret_cast<float*>(base + o_scores);
    w.keys = reinterpret_cast<uint32_t*>(base + o_keys);
    w.sorted_boxes = reinterpret_cast<float4*>(base + o_sb);
    w.sorted_scores = reinterpret_cast<float*>(base + o_ss);
    w.sorted_idx = reinterpret_cast<int*>(base + o_si);
    w.num_sorted = reinterpret_cast<int*>(base + o_ns);
    w.mask = reinterpret_cast<unsigned long long*>(base + o_mask);
    w.comp = reinterpret_cast<unsigned long long*>(base + o_comp);
    return w;
}

static long long* g_sort_clocks = nullptr;     // debug hook, see frcnn_debug_sort_clocks

static int next_pow2(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

// sort (top-k) + mask + scan, shared by frcnn_proposals and frcnn_nms
static int run_sort_nms(const NmsWs& w, int n_all, int top_k, double thresh, int mode, int max_keep,
                        int* keep_out, int* num_out, float* out_rois, float* out_scores, int out_cap,
                        float* dbg_dets, int* dbg_idx, int* dbg_num, bool map_to_original, cudaStream_t stream) {
    const int k_cap = top_k < n_all ? top_k : n_all;
    const int P = next_pow2(k_cap < 2 ? 2 : k_cap);
    SortArgs sa;
    sa.keys = w.keys; sa.n = n_all; sa.top_k = top_k;
    sa.boxes = w.boxes; sa.scores = w.scores;
    sa.sorted_boxes = w.sorted_boxes; sa.sorted_scores = w.sorted_scores; sa.sorted_idx = w.sorted_idx;
    sa.num_sorted = w.num_sorted;
    sa.dbg_dets = dbg_dets; sa.dbg_idx = dbg_idx; sa.dbg_num = dbg_num;
    sa.dbg_clocks = g_sort_clocks;
    sa.comp_out = w.comp;
    size_t sort_smem = sizeof(unsigned long long) * (size_t)P;
    const size_t keys_bytes = sizeof(uint32_t) * (size_t)n_all;
    const int cache_keys = sort_smem + keys_bytes <= 188 * 1024;     // smem copy of the keys when it fits (34 KB of static smem on top)
    if (cache_keys) sort_smem += keys_bytes;
    FRCNN_CUDA_OK(cudaFuncSetAttribute(topk_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sort_smem));
    FRCNN_CUDA_OK(launch_pdl(topk_sort_kernel, dim3(1), dim3(kSortThreads), sort_smem, stream, sa, P, cache_keys));
    const size_t rank_smem = sizeof(unsigned long long) * (size_t)k_cap;
    FRCNN_CUDA_OK(cudaFuncSetAttribute(rank_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rank_smem));
    FRCNN_CUDA_OK(launch_pdl(rank_scatter_kernel, dim3(cdiv(k_cap, kRankPerBlock)), dim3(kRankThreads), rank_smem, stream, sa));

    const int cbs = cdiv(k_cap, 64);
    dim3 grid(cbs, cbs);
    FRCNN_CUDA_OK(launch_pdl(nms_mask_kernel, grid, dim3(64), 0, stream, (const float4*)w.sorted_boxes, (const int*)w.num_sorted,
                             k_cap, thresh, (float)thresh, mode, w.mask, w.col_blocks));

    ScanArgs sc;
    sc.mask = w.mask; sc.col_blocks = w.col_blocks;
    sc.n_ptr = w.num_sorted; sc.n_cap = k_cap; sc.max_keep = max_keep;
    sc.index_map = map_to_original ? w.sorted_idx : nullptr;
    sc.keep_out = keep_out; sc.num_out = num_out;
    sc.sorted_boxes = w.sorted_boxes; sc.sorted_scores = w.sorted_scores;
    sc.out_rois = out_rois; sc.out_scores = out_scores; sc.out_cap = out_cap;
    const size_t scan_smem = sizeof(unsigned long long) * (size_t)w.col_blocks;
    sc.diag_in_smem = 0;
    FRCNN_CUDA_OK(launch_pdl(nms_scan_kernel, dim3(1), dim3(256), scan_smem, stream, sc));
    return FRCNN_OK;
}

}  // namespace frcnn

using namespace frcnn;

extern "C" size_t frcnn_proposals_workspace_bytes(int A, int H, int W, int pre_nms_top_n) {
    FRCNN_ENTRY();
    if (A <= 0 || H <= 0 || W <= 0 || pre_nms_top_n <= 0) return 0;
    const long n_all = (long)A * H * W;
    const int k_cap = (int)(pre_nms_top_n < n_all ? pre_nms_top_n : n_all);
    return carve(nullptr, (int)n_all, k_cap).total;
}

extern "C" int frcnn_proposals(const float* cls, long cls_chan_stride, long cls_pix_stride, int cls_is_logits,
                               const float* bbox, long bbox_chan_stride, long bbox_pix_stride, const double* anchors,
                               int A, int H, int W, int feat_stride, int im_h, int im_w, int min_size,
                               int pre_nms_top_n, int post_nms_top_n, double nms_thresh, float* out_rois,
                               float* out_scores, int* out_count, float* dbg_sorted_dets, int* dbg_sorted_anchor_idx,
                               int* dbg_num_sorted, void* ws, size_t ws_bytes, void* stream_) {
    FRCNN_ENTRY();
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    FRCNN_REQUIRE(cls && bbox && anchors && out_rois && out_count && ws, "frcnn_proposals: NULL argument");
    FRCNN_REQUIRE(A > 0 && A <= 32 && H > 0 && W > 0, "frcnn_proposals: bad shape A=%d H=%d W=%d", A, H, W);
    FRCNN_REQUIRE(pre_nms_top_n > 0 && pre_nms_top_n <= 16384, "frcnn_proposals: pre_nms_top_n must be in [1,16384] (got %d)", pre_nms_top_n);
    FRCNN_REQUIRE(post_nms_top_n > 0 && post_nms_top_n <= 2048, "frcnn_proposals: post_nms_top_n must be in [1,2048] (got %d)", post_nms_top_n);
    const long n_all_l = (long)A * H * W;
    FRCNN_REQUIRE(n_all_l < (1l << 24), "frcnn_proposals: too many anchors (%ld)", n_all_l);
    const int n_all = (int)n_all_l;
    const int k_cap = pre_nms_top_n < n_all ? pre_nms_top_n : n_all;
    NmsWs w = carve(ws, n_all, k_cap);
    if (ws_bytes < w.total) {
        set_error("frcnn_proposals: workspace %zu < required %zu", ws_bytes, w.total);
        return FRCNN_ERR_WORKSPACE;
    }
    DecodeArgs da;
    da.cls = cls; da.cls_cs = cls_chan_stride; da.cls_ps = cls_pix_stride; da.cls_is_logits = cls_is_logits;
    da.bbox = bbox; da.bbox_cs = bbox_chan_stride; da.bbox_ps = bbox_pix_stride;
    da.anchors = anchors;
    da.A = A; da.H = H; da.W = W; da.feat_stride = feat_stride; da.im_h = im_h; da.im_w = im_w; da.min_size = min_size;
    da.boxes = w.boxes; da.scores = w.scores; da.keys = w.keys;
    FRCNN_CUDA_OK(launch_pdl(rpn_decode_kernel, dim3(cdiv(n_all, 128)), dim3(128), 0, stream, da));
    return run_sort_nms(w, n_all, pre_nms_top_n, nms_thresh, FRCNN_NMS_GE_DOUBLE, post_nms_top_n, nullptr, out_count,
                        out_rois, out_scores, post_nms_top_n, dbg_sorted_dets, dbg_sorted_anchor_idx, dbg_num_sorted,
                        false, stream);
}

extern "C" size_t frcnn_nms_workspace_bytes(int n) {
    FRCNN_ENTRY();
    if (n <= 0) return 256;
    return carve(nullptr, n, n).total;
}

extern "C" int frcnn_nms(const float* dets, int n, double thresh, int mode, int max_keep, int* keep_out,
                         int* num_out, void* ws, size_t ws_bytes, void* stream_) {
    FRCNN_ENTRY();
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    FRCNN_REQUIRE(num_out != nullptr, "frcnn_nms: num_out is NULL");
    FRCNN_REQUIRE(n >= 0 && n <= 16384, "frcnn_nms: n must be in [0,16384] (got %d)", n);
    FRCNN_REQUIRE(mode == FRCNN_NMS_GE_DOUBLE || mode == FRCNN_NMS_GT_FLOAT, "frcnn_nms: bad mode %d", mode);
    if (n == 0) {
        FRCNN_CUDA_OK(cudaMemsetAsync(num_out, 0, sizeof(int), stream));
        return FRCNN_OK;
    }
    FRCNN_REQUIRE(dets && keep_out && ws, "frcnn_nms: NULL argument");
    NmsWs w = carve(ws, n, n);
    if (ws_bytes < w.total) {
        set_error("frcnn_nms: workspace %zu < required %zu", ws_bytes, w.total);
        return FRCNN_ERR_WORKSPACE;
    }
    FRCNN_CUDA_OK(launch_pdl(dets_keys_kernel, dim3(cdiv(n, 256)), dim3(256), 0, stream, dets, n, w.boxes, w.scores, w.keys));
    return run_sort_nms(w, n, n, thresh, mode, max_keep, keep_out, num_out, nullptr, nullptr, 0, nullptr, nullptr,
                        nullptr, true, stream);
}

// Debug / profiling hook (not part of the drop-in surface): device buffer of 8 int64 that receives the
// per-phase clock64() stamps of the next topk_sort_kernel launches; NULL disables.
extern "C" void frcnn_debug_sort_clocks(long long* dev_buf) { g_sort_clocks = dev_buf; }
