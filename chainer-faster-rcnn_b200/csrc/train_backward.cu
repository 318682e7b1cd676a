// train_backward.cu -- the memory-bound kernels of the conv backward pass (SURVEY.md 8f rank 1, train_rpn.py step).
//
// The dense parts of backward run on the SAME wgmma kernel as forward (conv_gemm_sm90.cu):
//   data gradient    dX = conv(dY, W rotated 180 deg, in/out swapped)      -> frcnn_conv2d with frcnn_pack_conv_weights_dgrad
//   weight gradient  dW[r][s] = sum_pixels dY[p] (x) X[p + (r-1, s-1)]      -> frcnn_gemm_nt_splitk over a zero-padded,
//                                                                            pixel-contiguous ("transposed") copy of dY and X
// This file holds what surrounds them (all HBM-bound, 16-byte accesses along channels on the NHWC side):
//   frcnn_grad_prepare      ReLU mask (and 2x2 ceil-mode max-pool routing) of an incoming gradient, hi/lo re-split, NHWC
//                           output for the next dgrad and the transposed padded copy for the wgrad GEMM
//                           (Chainer F.relu / F.max_pooling_2d backward, /root/reference models/vgg16.py:38-82 graph)
//   frcnn_act_transpose3    forward activation -> three column-shifted transposed planes (the GEMM's B operand)
//   frcnn_wgrad_reduce      split-K partials -> dW in the reference's OIHW float32 layout (fixed order: deterministic)
//   frcnn_bias_grad         db[c] = sum over pixels of dY
//   frcnn_optimizer_update  WeightDecay(rate) hook + MomentumSGD / Adam / AdaGrad / RMSprop on the float32 masters, the
//                           hyper-parameters read from device memory; frcnn_sgd_momentum(_bf16g) are its MomentumSGD rule
//                           with them passed by value (train_rpn.py:165-167)
#include "common.cuh"

namespace frcnn {

__device__ __forceinline__ float bf(const __nv_bfloat16 v) { return __bfloat162float(v); }

struct PrepArgs {
    // source gradient: bf16 hi/lo NHWC [Hs][Ws][C]  (Hs,Ws = H,W or the pooled size), or fp32 [H*W][ld] (src_f32)
    const __nv_bfloat16 *g_hi, *g_lo;
    const float* g_f32; int ld_f32;
    // forward activation the gradient flows into (post-ReLU output Y [H][W][C]); NULL = no mask
    const __nv_bfloat16 *y_hi, *y_lo;
    // pooled forward activation P [ceil(H/2)][ceil(W/2)][C] when the gradient arrives at pooled resolution; NULL otherwise
    const __nv_bfloat16 *p_hi, *p_lo;
    int H, W, C, Wp;
    long Kp;
    __nv_bfloat16 *o_hi, *o_lo;      // NHWC [H][W][C] out (optional)
    __nv_bfloat16 *t_hi, *t_lo;      // transposed [planes][C][t_ld] out (optional); image n's block at columns [n*Kp, (n+1)*Kp)
    long t_ld;                       // N*Kp
    int c_blocks;                    // blockIdx.z = image * c_blocks + 64-channel block
    int planes;                      // 1: plane at q; 3: planes shifted by -1/0/+1 pixel
    int times2;                      // multiply the result by 2 (the 1/(1-ratio) of a ratio-0.5 dropout), correctly rounded
    int route;                       // ROUTE_*: how the source reaches pixel (h, w)
};

// ROUTE_PLAIN: the source at (h, w), or routed through the 2x2 ceil-mode pool when p is given (frcnn_grad_prepare);
// ROUTE_POOL3: the 3x3/2 cover_all max-pool backward, p [pool3s2_out(H)][pool3s2_out(W)][C] (frcnn_maxpool3x3s2_backward);
// ROUTE_STRIDE2: the source [ceil(H/2)][ceil(W/2)][C] at the even pixels (2i, 2j), 0 elsewhere (frcnn_grad_prepare_stride2).
enum { ROUTE_PLAIN = 0, ROUTE_POOL3 = 1, ROUTE_STRIDE2 = 2 };

constexpr int PAD_LEFT = 8;          // zero columns left of pixel 0 in the transposed layout: every 8-pixel group starts 16-B aligned

// per-halfword mask (0xFFFF where equal) of VALUE equality hi+lo == hi'+lo' for two packed bf16 pairs.  The pooled map is a
// re-split of the maximum's float value, and a re-split may move half an ulp between hi and lo (ties), so the bit patterns
// of equal values can differ: the float sums (exact in fp32) are compared.
__device__ __forceinline__ uint32_t eq_values(uint32_t ah, uint32_t al, uint32_t bh, uint32_t bl) {
    const float a0 = __uint_as_float(ah << 16) + __uint_as_float(al << 16);
    const float b0 = __uint_as_float(bh << 16) + __uint_as_float(bl << 16);
    const float a1 = __uint_as_float(ah & 0xFFFF0000u) + __uint_as_float(al & 0xFFFF0000u);
    const float b1 = __uint_as_float(bh & 0xFFFF0000u) + __uint_as_float(bl & 0xFFFF0000u);
    return (a0 == b0 ? 0x0000FFFFu : 0u) | (a1 == b1 ? 0xFFFF0000u : 0u);
}

__device__ __forceinline__ void ld4(const __nv_bfloat16* p, long off, uint32_t w[4]) {
    const uint4 v = *reinterpret_cast<const uint4*>(p + off);
    w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
}

// 8 floats -> 4 words of bf16 hi and 4 words of bf16 lo (element j in the low/high half of word j/2)
__device__ __forceinline__ void pack8(const float v[8], uint32_t hw[4], uint32_t lw[4]) {
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        __nv_bfloat16 h0, l0, h1, l1;
        split_bf16(v[2 * m], h0, l0);
        split_bf16(v[2 * m + 1], h1, l1);
        hw[m] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        lw[m] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
}

// per-halfword mask of y > 0 for packed bf16 words read as int16: (0, +inf] -- +0, negatives and every NaN are excluded, as
// Chainer's `y > 0` excludes them
__device__ __forceinline__ uint32_t positive_mask(uint32_t y) { return __vcmpgts2(y, 0u) & __vcmplts2(y, 0x7F817F81u); }

// x2 on each bf16 of a packed pair, correctly rounded: exact for finite values (subnormals included), +-inf for an overflow,
// inf stays inf and NaN stays NaN
__device__ __forceinline__ uint32_t times2_bf16x2(uint32_t x) {
    __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&x);
    v = __hmul2(v, __floats2bfloat162_rn(2.f, 2.f));
    return *reinterpret_cast<const uint32_t*>(&v);
}

// The values of 8 split pairs, read as pool_pair_value reads them (an infinite hi stands alone).
__device__ __forceinline__ void pair_values(const __nv_bfloat16* hi, const __nv_bfloat16* lo, long off, float v[8]) {
    uint32_t hw[4], lw[4] = {0u, 0u, 0u, 0u};
    ld4(hi, off, hw);
    if (lo) ld4(lo, off, lw);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int m = j >> 1, sh = (j & 1) * 16;
        v[j] = pool_pair_value(__uint_as_float(((hw[m] >> sh) & 0xFFFFu) << 16), __uint_as_float(((lw[m] >> sh) & 0xFFFFu) << 16));
    }
}

// F.max_pooling_2d(3, stride=2, pad=0, cover_all=True) backward at pixel (r, c) of the H x W pool input, as a gather: window
// (i, j) covers rows [2i, min(2i+3, H)) and columns [2j, min(2j+3, W)) and sends g[i][j] to the FIRST element in scan order
// whose value equals p[i][j] (values compared as floats: +0 == -0, NaN equals nothing).  Up to four windows cover a pixel;
// their contributions are summed in fp32 in ascending (i, j) order starting from +0, then masked by y > 0 and re-split.
__device__ __forceinline__ void pool3_words(const PrepArgs& a, int r, int c, int c8, uint32_t hw[4], uint32_t lw[4]) {
    const int ph = (a.H - 2) / 2 + 1, pw = (a.W - 2) / 2 + 1;
    const long self = ((long)r * a.W + c) * a.C + c8 * 8;
    float yv[8], acc[8];
    pair_values(a.y_hi, a.y_lo, self, yv);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    const int i0 = r < 2 ? 0 : (r - 1) / 2, i1 = min(r / 2, ph - 1);
    const int j0 = c < 2 ? 0 : (c - 1) / 2, j1 = min(c / 2, pw - 1);
    for (int i = i0; i <= i1; ++i) {
        for (int j = j0; j <= j1; ++j) {
            const long q = ((long)i * pw + j) * a.C + c8 * 8;
            float pv[8], gv[8];
            pair_values(a.p_hi, a.p_lo, q, pv);
            pair_values(a.g_hi, a.g_lo, q, gv);
            bool hit[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) hit[k] = yv[k] == pv[k];
            const int w_end = min(2 * j + 3, a.W);
            for (int e = 0; e < 9; ++e) {                   // the window elements before (r, c) in scan order
                const int rr = 2 * i + e / 3, cc = 2 * j + e % 3;
                if (rr == r && cc == c) break;
                if (cc >= w_end) continue;
                float ev[8];
                pair_values(a.y_hi, a.y_lo, ((long)rr * a.W + cc) * a.C + c8 * 8, ev);
#pragma unroll
                for (int k = 0; k < 8; ++k) hit[k] = hit[k] && !(ev[k] == pv[k]);
            }
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (hit[k]) acc[k] = __fadd_rn(acc[k], gv[k]);
        }
    }
    pack8(acc, hw, lw);
    uint32_t yh[4];
    ld4(a.y_hi, self, yh);
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        const uint32_t keep = positive_mask(yh[m]);          // y > 0
        hw[m] &= keep;
        lw[m] &= keep;
    }
}

// The (masked / routed) gradient of 8 channels (chunk c8) at pixel (h, w) as packed bf16 words -- integer SIMD only:
//   * a value is the pair (hi, lo) with hi = bf16(v), lo = bf16(v - hi): v > 0 iff hi > 0 (read as int16, NaN excluded);
//     equality of two values is tested on the exact float sums (eq_values);
//   * F.max_pooling_2d backward: the incoming gradient goes to the FIRST element of the 2x2 ceil-mode window (scan order)
//     whose value equals the pooled maximum;  F.relu backward: gy where y > 0.
// Masked elements become +0 in both planes; kept elements keep the source's (hi, lo) words untouched (an fp32 source is
// split into (hi, lo) first).
__device__ __forceinline__ void prep_words(const PrepArgs& a, int h, int w, int c8, uint32_t hw[4], uint32_t lw[4]) {
    if (a.route == ROUTE_POOL3) {
        pool3_words(a, h, w, c8, hw, lw);
        return;
    }
    const long off = ((long)h * a.W + w) * a.C + c8 * 8;
    uint32_t keep[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
    uint32_t yh[4], yl[4] = {0u, 0u, 0u, 0u};
    if (a.y_hi != nullptr) {
        ld4(a.y_hi, off, yh);
#pragma unroll
        for (int m = 0; m < 4; ++m) keep[m] = positive_mask(yh[m]);          // y > 0
    }
    if (a.g_f32 != nullptr) {
        const float* g = a.g_f32 + ((long)h * a.W + w) * a.ld_f32 + c8 * 8;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (c8 * 8 + j < a.ld_f32) ? g[j] : 0.f;
        pack8(v, hw, lw);
#pragma unroll
        for (int m = 0; m < 4; ++m) { hw[m] &= keep[m]; lw[m] &= keep[m]; }
        return;
    }
    if (a.y_hi != nullptr && a.y_lo) ld4(a.y_lo, off, yl);
    long goff = off;
    if (a.route == ROUTE_STRIDE2) {                         // odd rows and columns receive nothing
        if ((h | w) & 1) {
#pragma unroll
            for (int m = 0; m < 4; ++m) hw[m] = lw[m] = 0u;
            return;
        }
        goff = ((long)(h >> 1) * ((a.W + 1) / 2) + (w >> 1)) * a.C + c8 * 8;
    }
    if (a.p_hi != nullptr) {
        const int Wq = (a.W + 1) / 2;
        const int ph = h >> 1, pw = w >> 1;
        goff = ((long)ph * Wq + pw) * a.C + c8 * 8;
        uint32_t pmh[4], pml[4] = {0u, 0u, 0u, 0u};
        ld4(a.p_hi, goff, pmh);
        if (a.p_lo) ld4(a.p_lo, goff, pml);
#pragma unroll
        for (int m = 0; m < 4; ++m) keep[m] &= eq_values(yh[m], yl[m], pmh[m], pml[m]);               // I am a maximum
        const int h0 = ph * 2, w0 = pw * 2;
        for (int e = 0; e < 4; ++e) {                       // ... and no earlier window element is
            const int eh = h0 + (e >> 1), ew = w0 + (e & 1);
            if (eh == h && ew == w) break;
            if (eh >= a.H || ew >= a.W) continue;
            const long eo = ((long)eh * a.W + ew) * a.C + c8 * 8;
            uint32_t eh4[4], el4[4] = {0u, 0u, 0u, 0u};
            ld4(a.y_hi, eo, eh4);
            if (a.y_lo) ld4(a.y_lo, eo, el4);
#pragma unroll
            for (int m = 0; m < 4; ++m) keep[m] &= ~eq_values(eh4[m], el4[m], pmh[m], pml[m]);
        }
    }
    ld4(a.g_hi, goff, hw);
    if (a.g_lo) ld4(a.g_lo, goff, lw);
    else { lw[0] = lw[1] = lw[2] = lw[3] = 0u; }
#pragma unroll
    for (int m = 0; m < 4; ++m) { hw[m] &= keep[m]; lw[m] &= keep[m]; }
    if (a.times2) {
#pragma unroll
        for (int m = 0; m < 4; ++m) { hw[m] = times2_bf16x2(hw[m]); lw[m] = times2_bf16x2(lw[m]); }
    }
}

// One block = 256 pixels x 64 channels of one image row, two phases with a 16-byte-granular exchange through shared memory:
//   phase 1  thread = (pixel, 16-byte channel chunk): the 8 lanes of a pixel read its 8 chunks = one 128-B line (coalesced),
//            evaluate prep_words, write the NHWC output (coalesced) and park the (hi, lo) vectors in smem, XOR-swizzled;
//   phase 2  thread = (chunk = warp, 8-pixel group = lane): reads its 8 (+2) pixels' vectors back (conflict-free), transposes
//            IN REGISTERS (byte_perm) -- per channel 8 consecutive pixels = one aligned 16-byte vector -- and stores: one
//            instruction writes 32 x 16 B = 512 contiguous bytes of ONE channel row.
// (Lane = chunk in both phases scatters every store over 8 rows 1.2 MB apart; lane = group in both phases makes every load
// touch 32 lines: each ran at a third of the HBM rate.)
constexpr int PREP_PX = 256;
constexpr int PREP_SMEM = (PREP_PX + 2) * 128 * 2;        // rows -1 .. 256, 128 B per plane

// Image n of a batch: every NHWC pointer moves by one image, the transposed planes by one Kp block.  The source g and the
// pooled map p are smaller than the H x W map, by a size that depends on the route: the 2x2 ceil pool's
// [ceil(H/2)][ceil(W/2)], the 3x3/2 cover_all pool's [(H-2)/2+1][(W-2)/2+1] (pool3_words), the stride-2 subsample's
// [ceil(H/2)][ceil(W/2)] with no p.
__device__ __forceinline__ void prep_image(PrepArgs& a, int n) {
    if (n == 0) return;
    const long img = (long)a.H * a.W * a.C;
    const long pooled = a.route == ROUTE_POOL3 ? (long)((a.H - 2) / 2 + 1) * ((a.W - 2) / 2 + 1) * a.C
                                               : (long)((a.H + 1) / 2) * ((a.W + 1) / 2) * a.C;
    const long g_img = (a.p_hi != nullptr || a.route == ROUTE_STRIDE2) ? pooled : img;
    if (a.g_hi) a.g_hi += n * g_img;
    if (a.g_lo) a.g_lo += n * g_img;
    if (a.g_f32) a.g_f32 += n * (long)a.H * a.W * a.ld_f32;
    if (a.y_hi) a.y_hi += n * img;
    if (a.y_lo) a.y_lo += n * img;
    if (a.p_hi) a.p_hi += n * pooled;
    if (a.p_lo) a.p_lo += n * pooled;
    if (a.o_hi) a.o_hi += n * img;
    if (a.o_lo) a.o_lo += n * img;
    if (a.t_hi) a.t_hi += n * a.Kp;
    if (a.t_lo) a.t_lo += n * a.Kp;
}

template <int PLANES>
__global__ void __launch_bounds__(256) grad_prepare_kernel(PrepArgs a) {
    extern __shared__ uint4 prep_smem[];
    uint4* s_hi = prep_smem;                                // [258][8] 16-byte units, unit column = c8 ^ ((row >> 3) & 7)
    uint4* s_lo = prep_smem + (PREP_PX + 2) * 8;
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int img = blockIdx.z / a.c_blocks;
    prep_image(a, img);
    const int h = blockIdx.y, w0 = blockIdx.x * PREP_PX, c0 = (blockIdx.z - img * a.c_blocks) * 8;      // c0 in chunks
    // ---- phase 1
    {
        const int c8l = t & 7, c8 = c0 + c8l;
        const bool c_ok = c8 * 8 < a.C;
        for (int it = 0; it < (PLANES == 3 ? 9 : 8); ++it) {
            int row;                                        // smem row = pixel - w0 + 1
            if (it < 8) row = 1 + it * 32 + (t >> 3);
            else { if (t >= 16) break; row = (t >> 3) ? PREP_PX + 1 : 0; }         // the two halo pixels
            const int w = w0 + row - 1;
            uint32_t hw[4], lw[4];
            const bool live = c_ok && w >= 0 && w < a.W;
            if (live) {
                prep_words(a, h, w, c8, hw, lw);
            } else {
#pragma unroll
                for (int m = 0; m < 4; ++m) hw[m] = lw[m] = 0u;
            }
            if (live && it < 8 && a.o_hi != nullptr) {
                const long off = ((long)h * a.W + w) * a.C + c8 * 8;
                *reinterpret_cast<uint4*>(a.o_hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                if (a.o_lo) *reinterpret_cast<uint4*>(a.o_lo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            }
            const int u = row * 8 + (c8l ^ ((row >> 3) & 7));
            s_hi[u] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            s_lo[u] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        }
    }
    if (a.t_hi == nullptr) return;
    __syncthreads();
    // ---- phase 2
    constexpr int NPX = PLANES == 3 ? 10 : 8;
    constexpr int FIRST = PLANES == 3 ? 0 : 1;              // first smem row relative to the group's row 8*lane
    const int c8l = warp, c8 = c0 + c8l;
    const int wg = w0 + lane * 8;
    if (wg >= a.W || c8 * 8 >= a.C) return;
    uint32_t hw[NPX][4], lw[NPX][4];
#pragma unroll
    for (int i = 0; i < NPX; ++i) {
        const int row = lane * 8 + FIRST + i;
        const int u = row * 8 + (c8l ^ ((row >> 3) & 7));
        const uint4 vh = s_hi[u], vl = s_lo[u];
        hw[i][0] = vh.x; hw[i][1] = vh.y; hw[i][2] = vh.z; hw[i][3] = vh.w;
        lw[i][0] = vl.x; lw[i][1] = vl.y; lw[i][2] = vl.z; lw[i][3] = vl.w;
    }
    const long k0 = (long)(h + 1) * a.Wp + PAD_LEFT + wg;          // multiple of 8
#pragma unroll
    for (int pl = 0; pl < PLANES; ++pl) {
        // plane pl at k holds pixel k + pl - 1 (PLANES == 3) / pixel k (PLANES == 1): window starts at array index pl / 0
        const int b0 = PLANES == 3 ? pl : 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t sel = (j & 1) ? 0x7632u : 0x5410u;
            const int m = j >> 1;
            uint4 vh, vl;
            vh.x = __byte_perm(hw[b0 + 0][m], hw[b0 + 1][m], sel);
            vh.y = __byte_perm(hw[b0 + 2][m], hw[b0 + 3][m], sel);
            vh.z = __byte_perm(hw[b0 + 4][m], hw[b0 + 5][m], sel);
            vh.w = __byte_perm(hw[b0 + 6][m], hw[b0 + 7][m], sel);
            const long row = ((long)pl * a.C + c8 * 8 + j) * a.t_ld + k0;
            *reinterpret_cast<uint4*>(a.t_hi + row) = vh;
            if (a.t_lo) {
                vl.x = __byte_perm(lw[b0 + 0][m], lw[b0 + 1][m], sel);
                vl.y = __byte_perm(lw[b0 + 2][m], lw[b0 + 3][m], sel);
                vl.z = __byte_perm(lw[b0 + 4][m], lw[b0 + 5][m], sel);
                vl.w = __byte_perm(lw[b0 + 6][m], lw[b0 + 7][m], sel);
                *reinterpret_cast<uint4*>(a.t_lo + row) = vl;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ split-K partials -> dW (OIHW fp32)
__global__ void wgrad_reduce_kernel(const float* __restrict__ parts, int groups, int splits, int Mp, int M, int ld, int N,
                                    float* __restrict__ dw, float scale) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long total = (long)M * N * groups;
    if (t >= total) return;
    const int g = (int)(t % groups);
    const long mn = t / groups;
    const int n = (int)(mn % N), m = (int)(mn / N);
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += parts[(((long)g * splits + s) * Mp + m) * ld + n];
    dw[t] = acc * scale;                         // OIHW: ((m*N + n)*groups + g), g = r*3 + s
}

// ------------------------------------------------------------------------------------------ bias gradient from the transposed dY
__global__ void __launch_bounds__(256) bias_grad_kernel(const __nv_bfloat16* __restrict__ t_hi, const __nv_bfloat16* __restrict__ t_lo,
                                                        long Kp, float* __restrict__ db, float scale) {
    __shared__ float s_w[8];
    const int c = blockIdx.x;
    const __nv_bfloat16* rh = t_hi + (long)c * Kp;
    const __nv_bfloat16* rl = t_lo ? t_lo + (long)c * Kp : nullptr;
    float acc = 0.f;
    for (long k = (long)threadIdx.x * 8; k < Kp; k += 256 * 8) {        // Kp % 64 == 0
        const uint4 h4 = *reinterpret_cast<const uint4*>(rh + k);
        const __nv_bfloat16* hb = reinterpret_cast<const __nv_bfloat16*>(&h4);
        uint4 l4 = make_uint4(0, 0, 0, 0);
        if (rl) l4 = *reinterpret_cast<const uint4*>(rl + k);
        const __nv_bfloat16* lb = reinterpret_cast<const __nv_bfloat16*>(&l4);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc += bf(hb[j]) + bf(lb[j]);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float a = 0.f;
        for (int w = 0; w < 8; ++w) a += s_w[w];
        db[c] = a * scale;
    }
}

// ------------------------------------------------------------------------------------------ optimizers
// Chainer v1's update_one_cpu of each rule after the WeightDecay hook, in float32 with every operation rounded on its own
// in the order NumPy evaluates it (explicit _rn intrinsics: nothing may be contracted).  h: the rule's hyper layout
// (include/frcnn_b200.h), h[0] the decay rate.  s0 / s1: the rule's state (s1 only for Adam).
struct OptHyper { float h[FRCNN_OPT_HYPER_LEN]; };

template <int RULE>
__device__ __forceinline__ void optimizer_one(float& w, float& s0, float& s1, const float g, const OptHyper& p) {
    const float* h = p.h;
    const float gi = __fmaf_rn(h[0], w, g);                  // WeightDecay: g += rate * w
    if (RULE == FRCNN_OPT_MOMENTUM_SGD) {                    // v = momentum*v - lr*g; w += v
        s0 = __fsub_rn(__fmul_rn(h[2], s0), __fmul_rn(h[1], gi));
        w = __fadd_rn(w, s0);
    } else if (RULE == FRCNN_OPT_ADAM) {                     // m += (1-beta1)*(g-m); v += (1-beta2)*(g*g-v); w -= lr_t*m / (sqrt(v)+eps)
        s0 = __fadd_rn(s0, __fmul_rn(h[2], __fsub_rn(gi, s0)));
        s1 = __fadd_rn(s1, __fmul_rn(h[3], __fsub_rn(__fmul_rn(gi, gi), s1)));
        w = __fsub_rn(w, __fdiv_rn(__fmul_rn(h[1], s0), __fadd_rn(__fsqrt_rn(s1), h[4])));
    } else if (RULE == FRCNN_OPT_ADAGRAD) {                  // h += g*g; w -= lr*g / (sqrt(h)+eps)
        s0 = __fadd_rn(s0, __fmul_rn(gi, gi));
        w = __fsub_rn(w, __fdiv_rn(__fmul_rn(h[1], gi), __fadd_rn(__fsqrt_rn(s0), h[2])));
    } else {                                                 // ms *= alpha; ms += (1-alpha)*g*g; w -= lr*g / (sqrt(ms)+eps)
        s0 = __fadd_rn(__fmul_rn(s0, h[2]), __fmul_rn(__fmul_rn(h[3], gi), gi));
        w = __fsub_rn(w, __fdiv_rn(__fmul_rn(h[1], gi), __fadd_rn(__fsqrt_rn(s0), h[4])));
    }
}

__device__ __forceinline__ float grad_value(const float g) { return g; }
__device__ __forceinline__ float grad_value(const __nv_bfloat16 g) { return __bfloat162float(g); }

// One element per thread.  hyper: the device array frcnn_optimizer_update reads at run time (a captured launch follows
// whatever was written there before the replay); NULL: the by-value `by_value` of frcnn_sgd_momentum(_bf16g).
template <int RULE, typename G>
__global__ void optimizer_kernel(float* __restrict__ w, float* __restrict__ s0, float* __restrict__ s1, const G* __restrict__ g,
                                 long n, const float* __restrict__ hyper, OptHyper by_value) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    OptHyper p = by_value;
    if (hyper) {
#pragma unroll
        for (int k = 0; k < FRCNN_OPT_HYPER_LEN; ++k) p.h[k] = hyper[k];
    }
    float wi = w[i], a = s0[i], b = RULE == FRCNN_OPT_ADAM ? s1[i] : 0.f;
    optimizer_one<RULE>(wi, a, b, grad_value(g[i]), p);
    s0[i] = a;
    if (RULE == FRCNN_OPT_ADAM) s1[i] = b;
    w[i] = wi;
}

// bf16 gradient bucket (BASELINE config #5: "bf16, NCCL grad allreduce"): the fp32 gradients of a bucket are rounded to bf16
// for the all-reduce (half the bytes on the wire), the fp32 masters / momentum are updated from the reduced bf16 values.
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long n) {
    const long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        const float4 v = *reinterpret_cast<const float4*>(src + i);            // src + i is 16-B aligned (bucket starts are)
        __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
        uint2 o;
        o.x = *reinterpret_cast<const uint32_t*>(&a);
        o.y = *reinterpret_cast<const uint32_t*>(&b);
        *reinterpret_cast<uint2*>(dst + i) = o;
    } else {
        for (long k = i; k < n; ++k) dst[k] = __float2bfloat16_rn(src[k]);
    }
}

// ------------------------------------------------------------------------------------------ dgrad weight packing
// out[t][ci][co] (bf16 hi/lo, co padded to Cout_pad) = W[co][ci][kh-1-r][kw-1-s], t = r*kw + s: the data gradient of a
// stride-1 "same" convolution is the convolution of dY with the 180-degree rotated, in/out-swapped filter.
__global__ void pack_weights_dgrad_kernel(const float* __restrict__ w, int Cout, int Cin, int taps, int Cout_pad,
                                          __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long total = (long)taps * Cin * Cout_pad;
    if (t >= total) return;
    const int co = (int)(t % Cout_pad);
    const int ci = (int)((t / Cout_pad) % Cin);
    const int tap = (int)(t / ((long)Cout_pad * Cin));
    float v = 0.f;
    if (co < Cout) v = w[((long)co * Cin + ci) * taps + (taps - 1 - tap)];
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[t] = h;
    if (lo) lo[t] = l;
}

}  // namespace frcnn

using namespace frcnn;

static long padded_pixels(int H, int W, int* wp_out) {
    const int Wp = (W + PAD_LEFT + 1 + 7) / 8 * 8;        // 8 zero columns left (aligned groups), >= 1 right
    if (wp_out) *wp_out = Wp;
    const long raw = (long)(H + 2) * Wp;
    return (raw + 63) / 64 * 64;
}

template <typename G>
static int optimizer_launch(int rule, float* w, float* s0, float* s1, const G* g, long n, const float* hyper, OptHyper by_value,
                            cudaStream_t stream) {
    if (n == 0) return FRCNN_OK;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    switch (rule) {
    case FRCNN_OPT_MOMENTUM_SGD:
        optimizer_kernel<FRCNN_OPT_MOMENTUM_SGD, G><<<blocks, 256, 0, stream>>>(w, s0, s1, g, n, hyper, by_value); break;
    case FRCNN_OPT_ADAM: optimizer_kernel<FRCNN_OPT_ADAM, G><<<blocks, 256, 0, stream>>>(w, s0, s1, g, n, hyper, by_value); break;
    case FRCNN_OPT_ADAGRAD: optimizer_kernel<FRCNN_OPT_ADAGRAD, G><<<blocks, 256, 0, stream>>>(w, s0, s1, g, n, hyper, by_value); break;
    default: optimizer_kernel<FRCNN_OPT_RMSPROP, G><<<blocks, 256, 0, stream>>>(w, s0, s1, g, n, hyper, by_value); break;
    }
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

static OptHyper sgd_hyper(float lr, float momentum, float weight_decay) {
    OptHyper p = {};
    p.h[0] = weight_decay; p.h[1] = lr; p.h[2] = momentum;
    return p;
}

static int grad_prepare(const char* fn, const void* g_hi, const void* g_lo, const float* g_f32, int ld_f32, const void* y_hi,
                        const void* y_lo, const void* p_hi, const void* p_lo, int N, int H, int W, int C, void* o_hi, void* o_lo,
                        void* t_hi, void* t_lo, int planes, int times2, cudaStream_t stream, int route = ROUTE_PLAIN) {
    FRCNN_REQUIRE(N >= 1, "%s: N = %d < 1", fn, N);
    FRCNN_REQUIRE(H > 0 && W > 0 && C > 0 && C % 8 == 0, "%s: bad shape H=%d W=%d C=%d (C %% 8 == 0)", fn, H, W, C);
    FRCNN_REQUIRE((g_hi != nullptr) != (g_f32 != nullptr), "%s: give the source as bf16 planes OR fp32", fn);
    FRCNN_REQUIRE(!g_f32 || (ld_f32 >= 1 && !p_hi), "%s: fp32 source needs ld_f32 and no pooling", fn);
    FRCNN_REQUIRE(!p_hi || y_hi, "%s: pooled routing needs the un-pooled forward activation", fn);
    FRCNN_REQUIRE(planes == 1 || planes == 3, "%s: planes must be 1 or 3", fn);
    FRCNN_REQUIRE(o_hi || t_hi, "%s: no output requested", fn);
    FRCNN_REQUIRE(route != ROUTE_POOL3 || (g_hi && y_hi && p_hi && H >= 2 && W >= 2 && !times2),
                  "%s: needs the pooled gradient, y and p, and a pool input of at least 2 x 2 (got H=%d W=%d)", fn, H, W);
    FRCNN_REQUIRE(route != ROUTE_STRIDE2 || (g_hi && !p_hi && !times2), "%s: needs a bf16 source and no pooled map", fn);
    PrepArgs a;
    a.g_hi = (const __nv_bfloat16*)g_hi; a.g_lo = (const __nv_bfloat16*)g_lo; a.g_f32 = g_f32; a.ld_f32 = ld_f32;
    a.y_hi = (const __nv_bfloat16*)y_hi; a.y_lo = (const __nv_bfloat16*)y_lo;
    a.p_hi = (const __nv_bfloat16*)p_hi; a.p_lo = (const __nv_bfloat16*)p_lo;
    a.H = H; a.W = W; a.C = C;
    a.Kp = padded_pixels(H, W, &a.Wp);
    a.o_hi = (__nv_bfloat16*)o_hi; a.o_lo = (__nv_bfloat16*)o_lo; a.t_hi = (__nv_bfloat16*)t_hi; a.t_lo = (__nv_bfloat16*)t_lo;
    a.t_ld = (long)N * a.Kp;
    a.planes = planes;
    a.times2 = times2 ? 1 : 0;
    a.route = route;
    a.c_blocks = cdiv(C, 64);
    FRCNN_REQUIRE(!times2 || !g_f32, "%s: times2 is not available for an fp32 source", fn);
    const long gz = (long)N * a.c_blocks;
    FRCNN_REQUIRE(H <= 65535 && gz <= 65535, "%s: image too tall / too many channels or images for one launch", fn);
    dim3 grid(cdiv(W, 256), H, (unsigned)gz);
    static bool attr_set = false;
    if (!attr_set) {
        FRCNN_CUDA_OK(cudaFuncSetAttribute(grad_prepare_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, PREP_SMEM));
        FRCNN_CUDA_OK(cudaFuncSetAttribute(grad_prepare_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, PREP_SMEM));
        attr_set = true;
    }
    if (planes == 3) grad_prepare_kernel<3><<<grid, 256, PREP_SMEM, stream>>>(a);
    else grad_prepare_kernel<1><<<grid, 256, PREP_SMEM, stream>>>(a);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" {

long frcnn_padded_pixels(int H, int W, int* row_pitch) { return padded_pixels(H, W, row_pitch); }

int frcnn_grad_prepare(const void* g_hi, const void* g_lo, const float* g_f32, int ld_f32, const void* y_hi, const void* y_lo,
                       const void* p_hi, const void* p_lo, int H, int W, int C, void* o_hi, void* o_lo, void* t_hi, void* t_lo,
                       int planes, int times2, void* stream) {
    FRCNN_ENTRY();
    return grad_prepare("grad_prepare", g_hi, g_lo, g_f32, ld_f32, y_hi, y_lo, p_hi, p_lo, 1, H, W, C, o_hi, o_lo, t_hi, t_lo,
                        planes, times2, (cudaStream_t)stream);
}

int frcnn_grad_prepare_batch(const void* g_hi, const void* g_lo, const float* g_f32, int ld_f32, const void* y_hi,
                             const void* y_lo, const void* p_hi, const void* p_lo, int N, int H, int W, int C, void* o_hi,
                             void* o_lo, void* t_hi, void* t_lo, int planes, int times2, void* stream) {
    FRCNN_ENTRY();
    return grad_prepare("grad_prepare_batch", g_hi, g_lo, g_f32, ld_f32, y_hi, y_lo, p_hi, p_lo, N, H, W, C, o_hi, o_lo, t_hi,
                        t_lo, planes, times2, (cudaStream_t)stream);
}

int frcnn_maxpool3x3s2_backward(const void* g_hi, const void* g_lo, const void* y_hi, const void* y_lo, const void* p_hi,
                                const void* p_lo, int H, int W, int C, void* o_hi, void* o_lo, void* t_hi, void* t_lo, void* stream) {
    FRCNN_ENTRY();
    return grad_prepare("maxpool3x3s2_backward", g_hi, g_lo, nullptr, 0, y_hi, y_lo, p_hi, p_lo, 1, H, W, C, o_hi, o_lo, t_hi,
                        t_lo, 1, 0, (cudaStream_t)stream, ROUTE_POOL3);
}

int frcnn_grad_prepare_stride2(const void* g_hi, const void* g_lo, const void* y_hi, const void* y_lo, int H, int W, int C,
                               void* o_hi, void* o_lo, void* t_hi, void* t_lo, int planes, void* stream) {
    FRCNN_ENTRY();
    return grad_prepare("grad_prepare_stride2", g_hi, g_lo, nullptr, 0, y_hi, y_lo, nullptr, nullptr, 1, H, W, C, o_hi, o_lo,
                        t_hi, t_lo, planes, 0, (cudaStream_t)stream, ROUTE_STRIDE2);
}

int frcnn_maxpool3x3s2_backward_batch(const void* g_hi, const void* g_lo, const void* y_hi, const void* y_lo, const void* p_hi,
                                      const void* p_lo, int N, int H, int W, int C, void* o_hi, void* o_lo, void* t_hi, void* t_lo,
                                      void* stream) {
    FRCNN_ENTRY();
    return grad_prepare("maxpool3x3s2_backward_batch", g_hi, g_lo, nullptr, 0, y_hi, y_lo, p_hi, p_lo, N, H, W, C, o_hi, o_lo,
                        t_hi, t_lo, 1, 0, (cudaStream_t)stream, ROUTE_POOL3);
}

int frcnn_grad_prepare_stride2_batch(const void* g_hi, const void* g_lo, const void* y_hi, const void* y_lo, int N, int H, int W,
                                     int C, void* o_hi, void* o_lo, void* t_hi, void* t_lo, int planes, void* stream) {
    FRCNN_ENTRY();
    return grad_prepare("grad_prepare_stride2_batch", g_hi, g_lo, nullptr, 0, y_hi, y_lo, nullptr, nullptr, N, H, W, C, o_hi,
                        o_lo, t_hi, t_lo, planes, 0, (cudaStream_t)stream, ROUTE_STRIDE2);
}

int frcnn_wgrad_reduce(const float* parts, int groups, int splits, int M_parts, int M, int ld, int N, float scale, float* dw,
                       void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(parts && dw && groups >= 1 && splits >= 1 && M > 0 && M_parts >= M && N > 0 && ld >= N, "wgrad_reduce: bad arguments");
    const long total = (long)M * N * groups;
    wgrad_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(parts, groups, splits, M_parts, M, ld, N, dw, scale);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_bias_grad(const void* t_hi, const void* t_lo, int C, long Kp, float scale, float* db, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(t_hi && db && C > 0 && Kp > 0 && Kp % 64 == 0, "bias_grad: bad arguments");
    bias_grad_kernel<<<C, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)t_hi, (const __nv_bfloat16*)t_lo, Kp, db, scale);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_sgd_momentum(float* w, float* v, const float* g, long n, float lr, float momentum, float weight_decay, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(w && v && g && n >= 0, "sgd_momentum: bad arguments");
    return optimizer_launch(FRCNN_OPT_MOMENTUM_SGD, w, v, nullptr, g, n, nullptr, sgd_hyper(lr, momentum, weight_decay),
                            (cudaStream_t)stream);
}

int frcnn_cast_f32_bf16(const float* src, void* dst_bf16, long n, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(src && dst_bf16 && n >= 0, "cast_f32_bf16: bad arguments");
    FRCNN_REQUIRE((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst_bf16) & 7) == 0,
                  "cast_f32_bf16: src must be 16-byte and dst 8-byte aligned");
    if (n == 0) return FRCNN_OK;
    const long threads = (n + 3) / 4;
    cast_f32_bf16_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(src, (__nv_bfloat16*)dst_bf16, n);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_sgd_momentum_bf16g(float* w, float* v, const void* g_bf16, long n, float lr, float momentum, float weight_decay,
                             void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(w && v && g_bf16 && n >= 0, "sgd_momentum_bf16g: bad arguments");
    return optimizer_launch(FRCNN_OPT_MOMENTUM_SGD, w, v, nullptr, (const __nv_bfloat16*)g_bf16, n, nullptr,
                            sgd_hyper(lr, momentum, weight_decay), (cudaStream_t)stream);
}

int frcnn_optimizer_update(int rule, float* w, float* s0, float* s1, const void* g, int g_bf16, long n, const float* hyper,
                           void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(rule >= FRCNN_OPT_MOMENTUM_SGD && rule <= FRCNN_OPT_RMSPROP, "optimizer_update: unknown rule %d", rule);
    FRCNN_REQUIRE(w && s0 && g && hyper, "optimizer_update: null pointer");
    FRCNN_REQUIRE((s1 != nullptr) == (rule == FRCNN_OPT_ADAM), "optimizer_update: s1 must be %s for rule %d",
                  rule == FRCNN_OPT_ADAM ? "given" : "NULL", rule);
    FRCNN_REQUIRE(g_bf16 == 0 || g_bf16 == 1, "optimizer_update: g_bf16 must be 0 or 1 (got %d)", g_bf16);
    FRCNN_REQUIRE(n >= 0, "optimizer_update: n = %ld < 0", n);
    const OptHyper unused = {};
    if (g_bf16)
        return optimizer_launch(rule, w, s0, s1, (const __nv_bfloat16*)g, n, hyper, unused, (cudaStream_t)stream);
    return optimizer_launch(rule, w, s0, s1, (const float*)g, n, hyper, unused, (cudaStream_t)stream);
}

int frcnn_pack_conv_weights_dgrad(const float* w_oihw, int Cout, int Cin, int kh, int kw, int Cout_pad, void* w_hi, void* w_lo,
                                  void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(w_oihw && w_hi && Cout > 0 && Cin > 0 && kh > 0 && kw > 0 && Cout_pad >= Cout && Cout_pad % 8 == 0,
                  "pack_conv_weights_dgrad: bad arguments");
    const long total = (long)kh * kw * Cin * Cout_pad;
    pack_weights_dgrad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        w_oihw, Cout, Cin, kh * kw, Cout_pad, (__nv_bfloat16*)w_hi, (__nv_bfloat16*)w_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

}  // extern "C"
