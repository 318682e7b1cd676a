// head_ops.cu -- the memory-bound kernels around the dense contractions:
//   frcnn_pack_image / frcnn_pack_conv_weights / frcnn_unpack_nhwc : layout + bf16 hi/lo conversion
//   frcnn_maxpool2x2_ceil : F.MaxPooling2D(2,2) ceil mode        (/root/reference models/vgg16.py:43,48,55,62)
//   frcnn_roi_pool        : F.roi_pooling_2d(.., 7, 7, 1/16)     (models/faster_rcnn.py:123-126)
//   frcnn_head_decode     : softmax + per-class decode + clip    (models/faster_rcnn.py:175-178)
//   frcnn_detect          : per-class NMS + confidence filter    (forward.py:48-57)
//   frcnn_detection_lists_batch : the detection lists drawn     (forward.py:50-59)
// All are HBM/L2-bound: 16-byte vector accesses along the channel axis (NHWC), grids sized to
// cover the tensor with >= 2 waves of 132 SMs where the tensor is large enough.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"
#include "nms_math.cuh"
#include "raw_photo.cuh"

namespace frcnn {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// 8 consecutive channels as bf16 hi (+lo) <-> 8 floats
struct F8 { float v[8]; };

__device__ __forceinline__ F8 load8(const __nv_bfloat16* hi, const __nv_bfloat16* lo, long off) {
    F8 r;
    const uint4 h = *reinterpret_cast<const uint4*>(hi + off);
    const uint32_t hw[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        r.v[2 * j] = __uint_as_float(hw[j] << 16);
        r.v[2 * j + 1] = __uint_as_float(hw[j] & 0xFFFF0000u);
    }
    if (lo) {
        const uint4 l = *reinterpret_cast<const uint4*>(lo + off);
        const uint32_t lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            r.v[2 * j] += __uint_as_float(lw[j] << 16);          // exact: hi+lo has <= 24 significant bits
            r.v[2 * j + 1] += __uint_as_float(lw[j] & 0xFFFF0000u);
        }
    }
    return r;
}

__device__ __forceinline__ void store8(__nv_bfloat16* hi, __nv_bfloat16* lo, long off, const F8& r) {
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        __nv_bfloat16 h0, l0, h1, l1;
        split_bf16(r.v[2 * j], h0, l0);
        split_bf16(r.v[2 * j + 1], h1, l1);
        hw[j] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        lw[j] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
    *reinterpret_cast<uint4*>(hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    if (lo) *reinterpret_cast<uint4*>(lo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

// ------------------------------------------------------------------------------------------ pack / unpack
__global__ void pack_image_kernel(const float* x, int C, int H, int W, int Cp, __nv_bfloat16* hi, __nv_bfloat16* lo) {
    const long total = (long)H * W * Cp;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cp);
        const long p = i / Cp;
        const float v = c < C ? x[(long)c * H * W + p] : 0.0f;
        __nv_bfloat16 h, l;
        split_bf16(v, h, l);
        hi[i] = h;
        if (lo) lo[i] = l;
    }
}

__global__ void pack_weights_kernel(const float* w, int Cout, int Cin, int taps, int Cp, __nv_bfloat16* hi,
                                    __nv_bfloat16* lo, int perm, int pc, int ph, int pw) {
    // dst [tap][o][c'] ; src OIHW: w[(o*Cin + c)*taps + tap]
    const long total = (long)taps * Cout * Cp;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int cdst = (int)(i % Cp);
        const long t = i / Cp;
        const int o = (int)(t % Cout);
        const int tap = (int)(t / Cout);
        float v = 0.0f;
        if (cdst < Cin) {
            int csrc = cdst;
            if (perm) {     // dst K order (h,w,c)  <-  src K order (c,h,w)
                const int c = cdst % pc, hw = cdst / pc;
                csrc = c * (ph * pw) + hw;
            }
            v = w[((long)o * Cin + csrc) * taps + tap];
        }
        __nv_bfloat16 h, l;
        split_bf16(v, h, l);
        hi[i] = h;
        if (lo) lo[i] = l;
    }
}

// First-layer im2col: (C<=3,H,W) fp32 -> [H][W][32] bf16 hi/lo with K index (r*3+s)*C + c (zero padded
// borders, zeros for k >= 9*C).  conv1_1 (C_in = 3, K = 27) then runs as ONE 64-byte-row k-block per tile
// instead of nine 32-byte-row blocks.  One thread per pixel; neighbouring threads share their loads in L1.
// The source element (c, h, w) is x[c*sc + h*sh + w*sw]: (H*W, W, 1) for a dense (C,H,W) image, (1, W*C, C) for the
// (H,W,C) memory that forward.py:45's `img.transpose([2, 0, 1]).astype(np.float32)` actually leaves behind (astype keeps
// the transposed strides), so that such a caller's buffer is uploaded as it is and permuted here for free.
__global__ void pack_image_im2col_kernel(const float* x, int C, int H, int W, long sc, long sh, long sw, __nv_bfloat16* hi,
                                         __nv_bfloat16* lo) {
    // One thread per pixel: its 9 taps x C channels are 9*C scalar loads that coalesce across the warp (consecutive
    // threads = consecutive w), then 4 + 4 16-byte stores of the pixel's 64-byte hi / lo rows.
    const long total = (long)H * W;
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < total; p += (long)gridDim.x * blockDim.x) {
        const int h = (int)(p / W), w = (int)(p % W);
        if (C != 3) {                                   // generic (C = 1, 2): one 8-value chunk at a time
            for (int q = 0; q < 4; ++q) {
                F8 f;
                for (int j = 0; j < 8; ++j) {
                    const int k = 8 * q + j;
                    float val = 0.0f;
                    if (k < 9 * C) {
                        const int tap = k / C, c = k - tap * C;
                        const int hh = h + tap / 3 - 1, ww = w + tap % 3 - 1;
                        if (hh >= 0 && hh < H && ww >= 0 && ww < W) val = x[c * sc + hh * sh + ww * sw];
                    }
                    f.v[j] = val;
                }
                store8(hi, lo, p * 32 + 8 * q, f);
            }
            continue;
        }
        float v[32];                                    // C == 3: every index below is a compile-time constant (registers)
#pragma unroll
        for (int k = 0; k < 32; ++k) v[k] = 0.0f;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int hh = h + tap / 3 - 1, ww = w + tap % 3 - 1;
            if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
                const long o = hh * sh + ww * sw;
#pragma unroll
                for (int c = 0; c < 3; ++c) v[tap * 3 + c] = x[c * sc + o];
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            F8 f;
#pragma unroll
            for (int j = 0; j < 8; ++j) f.v[j] = v[8 * q + j];
            store8(hi, lo, p * 32 + 8 * q, f);
        }
    }
}

// Compact first-layer input: (C<=3,H,W) fp32 (any strides) -> [H][W+2][8] bf16 hi/lo: 8 channels per pixel (3 used), one
// zero pixel left and right of every row.  conv1_1 (models/vgg16.py:39) then reads, for output pixel (h, w) and kernel row
// r, the 32 contiguous values of stored pixels w .. w+3 of row h+r-1 through a SLIDING-WINDOW tensor map (frcnn_conv3x3_c8):
// 19 MB written here instead of the 77 MB of the [H][W][32] im2col copy, and nothing re-read from HBM four times.
// A batch: image blockIdx.y reads x + blockIdx.y * sn and writes its own plane, out_elems elements further on.  A canvas
// batch (extents != NULL): only the image's own eh x ew pixels are read, every other stored pixel of its plane is 0.
__global__ void pack_image_c8_kernel(const float* x, int C, int H, int W, long sc, long sh, long sw, __nv_bfloat16* hi,
                                     __nv_bfloat16* lo, long slack_pixels, long sn, long out_elems, const int* extents) {
    x += blockIdx.y * sn;
    hi += blockIdx.y * out_elems;
    if (lo) lo += blockIdx.y * out_elems;
    const int eh = extents ? canvas_extent(extents, blockIdx.y, 0, 0, H) : H;
    const int ew = extents ? canvas_extent(extents, blockIdx.y, 1, 0, W) : W;
    const int WP = W + 2;
    const long total = (long)H * WP + slack_pixels;
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < total; p += (long)gridDim.x * blockDim.x) {
        F8 f;
#pragma unroll
        for (int j = 0; j < 8; ++j) f.v[j] = 0.0f;
        if (p < (long)H * WP) {
            const int h = (int)(p / WP), wp = (int)(p % WP);
            if (h < eh && wp >= 1 && wp <= ew) {
                const long o = h * sh + (long)(wp - 1) * sw;
                for (int c = 0; c < C; ++c) f.v[c] = x[c * sc + o];
            }
        }
        store8(hi, lo, p * 8, f);
    }
}

// conv1_1 weights for frcnn_conv3x3_c8: OIHW (Cout, Cin<=3, 3, 3) -> [3 (kernel row r)][Cout][32], k = dx*8 + c holds
// W[co][c][r][dx] for dx < 3, c < Cin, zero elsewhere (the 4th pixel of the window and channels 3..7 multiply zeros).
__global__ void pack_weights_c8_kernel(const float* w, int Cout, int Cin, __nv_bfloat16* hi, __nv_bfloat16* lo) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 3 * Cout * 32) return;
    const int k = t % 32, co = (t / 32) % Cout, r = t / (32 * Cout);
    const int dx = k / 8, c = k % 8;
    float v = 0.0f;
    if (dx < 3 && c < Cin) v = w[((co * Cin + c) * 3 + r) * 3 + dx];
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[t] = h;
    if (lo) lo[t] = l;
}

// Caller-side preprocessing (forward.py:34-45, img_preprocessing): uint8 BGR HWC image -> float32(pixel - mean)
// -> cv.resize(INTER_LINEAR) -> (3,H,W) float32.  One thread per output pixel, all three channels; the arithmetic is
// bilinear_bgr8 (raw_photo.cuh).
struct PreArgs {
    const unsigned char* src; int h0, w0;
    double m0, m1, m2, sx, sy;
    int H, W;
    float* out;
};

__global__ void preprocess_bgr8_kernel(const PreArgs a) {
    const long total = (long)a.H * a.W;
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < total; p += (long)gridDim.x * blockDim.x) {
        const int y = (int)(p / a.W), x = (int)(p % a.W);
        float v[3];
        bilinear_bgr8(a.src, a.w0, bilinear_tap(y, a.sy, a.h0), bilinear_tap(x, a.sx, a.w0), a.m0, a.m1, a.m2, v);
#pragma unroll
        for (int c = 0; c < 3; ++c) a.out[((long)c * a.H + y) * a.W + x] = v[c];
    }
}

// Raw photos straight into a canvas batch's first-layer planes: preprocess_bgr8_kernel + pack_image_c8_kernel(extents) for
// all N slots in one launch, without the float32 image in between.  Image blockIdx.y is the dense uint8 (h0, w0, 3) block at
// arena + src_off[n]; its resized extent, source size, offset and 1 / im_scale are device arrays read here, so a captured
// launch serves any mix of sizes.  One block per stored row [Wc+2][8] of the slot (the last one also zeroes the 8 slack
// pixels): the row's y taps are computed once per thread, and every stored pixel outside the extent is written as 0.  A
// slot whose source does not lie inside [0, arena_bytes) or whose source size is not positive is an empty slot (raw_slot).
struct PreCanvasArgs {
    const unsigned char* arena; long long arena_bytes;
    const long long* src_off; const int* src_hw; const double* inv_scale; const int* extents;
    int Hc, Wc;
    double m0, m1, m2;
    __nv_bfloat16 *hi, *lo;
    long out_elems;
};
__global__ void preprocess_bgr8_canvas_kernel(const PreCanvasArgs a) {
    const int n = blockIdx.y, h = blockIdx.x, WP = a.Wc + 2;
    __nv_bfloat16* hi = a.hi + n * a.out_elems;
    __nv_bfloat16* lo = a.lo ? a.lo + n * a.out_elems : nullptr;
    const RawSlot s = raw_slot(a.arena, a.arena_bytes, a.src_off, a.src_hw, a.inv_scale, a.extents, n, a.Hc, a.Wc);
    F8 f;
#pragma unroll
    for (int j = 0; j < 8; ++j) f.v[j] = 0.0f;
    const long row = (long)h * WP;
    if (h < s.eh) {
        const BilinearTap ty = bilinear_tap(h, s.inv_scale, s.h0);
        for (int wp = threadIdx.x; wp < WP; wp += blockDim.x) {
            F8 g = f;
            if (wp >= 1 && wp <= s.ew) bilinear_bgr8(s.src, s.w0, ty, bilinear_tap(wp - 1, s.inv_scale, s.w0), a.m0, a.m1, a.m2, g.v);
            store8(hi, lo, (row + wp) * 8, g);
        }
    } else {
        for (int wp = threadIdx.x; wp < WP; wp += blockDim.x) store8(hi, lo, (row + wp) * 8, f);
    }
    if (h == a.Hc - 1 && threadIdx.x < 8) store8(hi, lo, (row + WP + threadIdx.x) * 8, f);
}

// OIHW 3x3 weights (Cin <= 3) -> [1][Cout][32] bf16 hi/lo with the same K order as pack_image_im2col_kernel.
__global__ void pack_weights_im2col_kernel(const float* w, int Cout, int Cin, __nv_bfloat16* hi, __nv_bfloat16* lo) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Cout * 32) return;
    const int o = i / 32, k = i % 32;
    float v = 0.0f;
    if (k < 9 * Cin) {
        const int tap = k / Cin, c = k % Cin;
        v = w[((long)o * Cin + c) * 9 + tap];
    }
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
}

__global__ void unpack_nhwc_kernel(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int H, int W, int C, float* y) {
    const long total = (long)H * W * C;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long p = i / C;
        float v = __bfloat162float(hi[i]);
        if (lo) v += __bfloat162float(lo[i]);
        y[(long)c * H * W + p] = v;
    }
}

// ------------------------------------------------------------------------------------------ max-pool 2x2/2 ceil
// A batch [N][H][W][C]: image blockIdx.y reads x + blockIdx.y * H*W*C and writes y + blockIdx.y * Ho*Wo*C.
// Every kernel of this file with a kBatch parameter takes the image from blockIdx.y when it is true; the one-image entry
// points launch the kBatch = false instantiation, where the image is the constant 0 and the offsets fold away.
template <bool kBatch>
__global__ void maxpool_kernel(const __nv_bfloat16* xh, const __nv_bfloat16* xl, int H, int W, int C,
                               __nv_bfloat16* yh, __nv_bfloat16* yl) {
    grid_dep_wait();
    if (kBatch) {
        const long xo = blockIdx.y * ((long)H * W * C), yo = blockIdx.y * ((long)((H + 1) / 2) * ((W + 1) / 2) * C);
        xh += xo;
        yh += yo;
        if (xl) xl += xo;
        if (yl) yl += yo;
    }
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2, C8 = C / 8;
    const long total = (long)Ho * Wo * C8;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        const long p = i / C8;
        const int wo = (int)(p % Wo), ho = (int)(p / Wo);
        F8 m;
        bool first = true;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const int h = 2 * ho + dy, w = 2 * wo + dx;
                if (h < H && w < W) {       // ceil mode: partial windows use the valid elements only
                    const F8 v = load8(xh, xl, ((long)h * W + w) * C + 8 * c8);
                    if (first) { m = v; first = false; }
                    else {
#pragma unroll
                        for (int j = 0; j < 8; ++j) m.v[j] = fmaxf(m.v[j], v.v[j]);
                    }
                }
            }
        store8(yh, yl, ((long)ho * Wo + wo) * C + 8 * c8, m);
    }
}

// ------------------------------------------------------------------------------------------ RoI max pooling
// Caffe / Chainer-v1 GPU semantics (see the oracle's orc_roi_pool): round() half away from zero, float32 bin sizes, empty
// bin -> 0; the bins of any RoI, NaN and infinite coordinates included, follow roi_coord / roi_bin (common.cuh).  The bounds
// of the PH row bands and the PW column bins are computed ONCE per RoI.  NaN features are ignored (max.bf16x2 returns the
// other operand, set.gt / set.eq are false), so a non-empty window with no number above -inf keeps its start, -inf.
//
// The maximum is taken on the PACKED bf16 pairs, not on converted floats.  A feature value is v = hi + lo with hi = RN_bf16(v)
// and |lo| <= ulp(hi)/2 (split_bf16), and rounding is monotone, so v_a > v_b  <=>  hi_a > hi_b, or hi_a == hi_b and lo_a > lo_b:
// the maximum of v over a window is the lexicographic maximum of (hi, lo) (max.bf16x2 / set.{gt,eq}.u32.bf16x2 on two
// channels per instruction).  The result IS one input pixel's (hi, lo) pair and is stored as it is: its VALUE hi + lo is
// exactly what the float formulation produced (max of the floats), without the unpack / add per loaded pixel and the 8
// float -> bf16 pair conversions per output item.  (The float formulation re-split the maximum; the re-split of hi + lo gives
// the same pair back except when lo is exactly +-ulp(hi)/2 -- a rounding midpoint, 0.08 % of random values -- where it may
// name the same value by its other neighbour: tests/test_host_cpu.py::test_packed_pair_maximum_is_the_maximum_of_the_values.)
//
// History of this kernel, all variants bit-exact and measured on the same workload (profiles/r02_roi_pool_window_experiment_negative.txt):
// per-bin gather, float compares 25 us; the same on packed pairs 26 us (a third fewer instructions, same time: ncu shows no
// saturated unit, a latency chain); bands staged in shared memory with a barrier pair per output row 44 us; this one 21 us.
constexpr int kRoiMaxBins = 32;

__device__ __forceinline__ uint32_t bf2_max(uint32_t a, uint32_t b) {
    uint32_t d;
    asm("max.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t bf2_eq_mask(uint32_t a, uint32_t b) {       // 0xFFFF per half where a == b (as values)
    uint32_t d;
    asm("set.eq.u32.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
constexpr uint32_t kBf2NegInf = 0xFF80FF80u;

// Bin-column walker: one CTA per (RoI, channel slice), one thread per (output column pw, 8 channels) -- NO shared-memory
// staging and no barrier inside the RoI.  The thread walks the window's rows top to bottom ONCE: per row it folds the pixels
// of its bin's columns [ws, we) into a row value, per output row ph it folds the band's row values, and because band ph+1
// starts at he[ph] or he[ph]-1 (floor / ceil of the SAME product, see the bounds) the only row two bands can share is the
// last one folded -- it is kept in registers, so every window row is loaded exactly once per bin column (82 MB of distinct
// window pixels at the headline workload where a thread per BIN requests 185 MB and re-derives every bin from scratch).  All folds are the lexicographic maximum of the packed (hi, lo) pairs (see above), streaming: h' = max(h, b.h),
// l' = b.h > h ? b.l : (b.h == h ? max(l, b.l) : l).  Rows are taken two at a time so that a tall RoI's chain of L2 round
// trips is halved.  All RoIs are resident at once (300 CTAs of 448 threads): the kernel time is the tallest RoI's chain.
struct Pair8 { uint4 h, l; };

__device__ __forceinline__ void lex_fold(uint32_t& h, uint32_t& l, uint32_t bh, uint32_t bl) {
    uint32_t gt, eq;
    asm("set.gt.u32.bf16x2 %0, %1, %2;" : "=r"(gt) : "r"(bh), "r"(h));
    eq = bf2_eq_mask(bh, h);
    const uint32_t lm = bf2_max(l, bl);
    const uint32_t t = (lm & eq) | (l & ~eq);
    l = (bl & gt) | (t & ~gt);
    h = bf2_max(h, bh);
}
template <bool LO>
__device__ __forceinline__ void lex_fold8(Pair8& a, const uint4 bh, const uint4 bl) {
    if (LO) {
        lex_fold(a.h.x, a.l.x, bh.x, bl.x);
        lex_fold(a.h.y, a.l.y, bh.y, bl.y);
        lex_fold(a.h.z, a.l.z, bh.z, bl.z);
        lex_fold(a.h.w, a.l.w, bh.w, bl.w);
    } else {
        a.h.x = bf2_max(a.h.x, bh.x);
        a.h.y = bf2_max(a.h.y, bh.y);
        a.h.z = bf2_max(a.h.z, bh.z);
        a.h.w = bf2_max(a.h.w, bh.w);
    }
}
__device__ __forceinline__ Pair8 pair8_neg_inf() {
    Pair8 p;
    p.h = make_uint4(kBf2NegInf, kBf2NegInf, kBf2NegInf, kBf2NegInf);
    p.l = p.h;
    return p;
}

constexpr int kRoiColMaxThreads = 448;        // 7 output columns x 64 channel groups; two CTAs of 72 registers per SM
template <bool LO, bool kBatch>
__global__ void __launch_bounds__(kRoiColMaxThreads, 2) roi_pool_col_kernel(const __nv_bfloat16* __restrict__ fh, const __nv_bfloat16* __restrict__ fl,
                                                                         int H, int W, int C, const float* __restrict__ rois,
                                                                         const int* __restrict__ count, int R_cap, int PH, int PW, float scale,
                                                                         __nv_bfloat16* __restrict__ oh, __nv_bfloat16* __restrict__ ol,
                                                                         float* __restrict__ of32, int c8_per_cta, int slices,
                                                                         long rois_is, long count_is, long out_is,
                                                                         const int* __restrict__ extents, int halvings) {
    grid_dep_wait();
    // a canvas batch: the bins are clamped to the image's own map (bh x bw), the addressing keeps the canvas width W
    const int bh = extents ? canvas_extent(extents, blockIdx.y, 0, halvings, H) : H;
    const int bw = extents ? canvas_extent(extents, blockIdx.y, 1, halvings, W) : W;
    if (kBatch) {                      // image blockIdx.y: its feature map [H][W][C], RoIs, count and output rows
        const long img = blockIdx.y;
        const long fo = img * ((long)H * W * C), oo = img * out_is;
        fh += fo;
        if (LO) fl += fo;
        rois += img * rois_is;
        if (count) count += img * count_is;
        if (oh) oh += oo;
        if (ol) ol += oo;
        if (of32) of32 += oo;
    }
    __shared__ int s_ws[kRoiMaxBins], s_we[kRoiMaxBins], s_hs[kRoiMaxBins], s_he[kRoiMaxBins];
    const int C8 = C / 8;
    const int R = count ? min(*count, R_cap) : R_cap;
    const int tid = threadIdx.x;
    const int pw = tid / c8_per_cta, c8l = tid - pw * c8_per_cta;
    for (int blk = blockIdx.x; blk < R_cap * slices; blk += gridDim.x) {
        const int r = blk / slices, c8 = (blk - r * slices) * c8_per_cta + c8l;
        const bool valid = r < R;                            // CTA-uniform
        if (valid && tid < max(PH, PW)) {                    // the bin rule of common.cuh (roi_coord / roi_bin)
            const float4 roi = reinterpret_cast<const float4*>(rois)[r];
            if (tid < PH) {
                const int2 b = roi_bin(roi_coord(roi.y, scale), roi_coord(roi.w, scale), PH, tid, bh);
                s_hs[tid] = b.x;
                s_he[tid] = b.y;
            }
            if (tid < PW) {
                const int2 b = roi_bin(roi_coord(roi.x, scale), roi_coord(roi.z, scale), PW, tid, bw);
                s_ws[tid] = b.x;
                s_we[tid] = b.y;
            }
        }
        __syncthreads();
        if (pw < PW && c8 < C8) {
            const int ws = valid ? s_ws[pw] : 0, bwid = valid ? s_we[pw] - ws : 0;
            int prev_y = -1;                                 // the last row folded, and its row value
            Pair8 prev = pair8_neg_inf();
            for (int ph = 0; ph < PH; ++ph) {
                uint4 mh = make_uint4(0u, 0u, 0u, 0u), ml = mh;          // empty bin / row past the count -> 0
                const int hs = valid ? s_hs[ph] : 0, he = valid ? s_he[ph] : 0;
                if (he > hs && bwid > 0) {
                    Pair8 acc = pair8_neg_inf();
                    int y = hs;
                    if (y == prev_y) {                       // the row this band shares with the previous one
                        acc = prev;
                        ++y;
                    }
                    for (; y < he; y += 2) {
                        const bool two = y + 1 < he;         // warp-uniform
                        Pair8 ra = pair8_neg_inf(), rb = ra;
                        const long o = ((long)y * W + ws) * C + 8 * c8;
                        const uint4* ph0 = reinterpret_cast<const uint4*>(fh + o);
                        const uint4* pl0 = reinterpret_cast<const uint4*>(LO ? fl + o : fh + o);
                        const long row = (long)W * C8;       // one image row in uint4 units
                        if (two) {
                            for (int x = 0; x < bwid; ++x) {
                                const uint4 ha = __ldg(ph0 + (long)x * C8), hb = __ldg(ph0 + row + (long)x * C8);
                                uint4 la = ha, lb = hb;
                                if (LO) { la = __ldg(pl0 + (long)x * C8); lb = __ldg(pl0 + row + (long)x * C8); }
                                lex_fold8<LO>(ra, ha, la);
                                lex_fold8<LO>(rb, hb, lb);
                            }
                            lex_fold8<LO>(acc, ra.h, ra.l);
                            lex_fold8<LO>(acc, rb.h, rb.l);
                            prev = rb;
                            prev_y = y + 1;
                        } else {
                            for (int x = 0; x < bwid; ++x) {
                                const uint4 ha = __ldg(ph0 + (long)x * C8);
                                uint4 la = ha;
                                if (LO) la = __ldg(pl0 + (long)x * C8);
                                lex_fold8<LO>(ra, ha, la);
                            }
                            lex_fold8<LO>(acc, ra.h, ra.l);
                            prev = ra;
                            prev_y = y;
                        }
                    }
                    mh = acc.h;
                    if (LO) ml = acc.l;
                }
                const long off = (((long)r * PH + ph) * PW + pw) * C + 8 * c8;
                if (oh) {
                    *reinterpret_cast<uint4*>(oh + off) = mh;
                    if (ol) *reinterpret_cast<uint4*>(ol + off) = ml;
                }
                if (of32) {
                    const uint32_t hw[4] = {mh.x, mh.y, mh.z, mh.w}, lw[4] = {ml.x, ml.y, ml.z, ml.w};
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        v[2 * j] = pool_pair_value(__uint_as_float(hw[j] << 16), __uint_as_float(lw[j] << 16));
                        v[2 * j + 1] = pool_pair_value(__uint_as_float(hw[j] & 0xFFFF0000u), __uint_as_float(lw[j] & 0xFFFF0000u));
                    }
                    float4* d = reinterpret_cast<float4*>(of32 + off);
                    d[0] = make_float4(v[0], v[1], v[2], v[3]);
                    d[1] = make_float4(v[4], v[5], v[6], v[7]);
                }
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------ head decode
// One thread per (roi, class): softmax over classes (every thread recomputes max/sum of its row --
// 21 values, L1-resident) and bbox_transform_inv + clip_boxes for its class's 4 deltas.  Image blockIdx.y of a batch
// reads and writes its own rows, (image) * (the array's image stride) elements on.  im_info (optional, device [N][2]):
// image n's clip bounds (im_h, im_w), in place of the launch's one pair.
struct DecodeStrides { long in, rois, count, prob, boxes; };
template <bool kBatch>
__global__ void head_decode_kernel(const float* scores, const float* deltas, int ld, const float* rois,
                                   const int* count, int R_cap, int NC, int im_h, int im_w, float* prob,
                                   float* boxes, const DecodeStrides is, const int* im_info) {
    grid_dep_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R_cap * NC) return;
    if (im_info) {
        im_h = __ldg(im_info + 2 * blockIdx.y);
        im_w = __ldg(im_info + 2 * blockIdx.y + 1);
    }
    if (kBatch) {
        const long img = blockIdx.y;
        scores += img * is.in;
        deltas += img * is.in;
        rois += img * is.rois;
        if (count) count += img * is.count;
        prob += img * is.prob;
        boxes += img * is.boxes;
    }
    const int r = i / NC, c = i - r * NC;
    const int R = count ? min(*count, R_cap) : R_cap;
    float p = 0.0f;
    float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < R) {
        const float* s = scores + (long)r * ld;
        float m = s[0];
        for (int k = 1; k < NC; ++k) m = fmaxf(m, s[k]);
        float sum = 0.0f, mine = 0.0f;
        for (int k = 0; k < NC; ++k) {
            const float e = det_expf(__fsub_rn(s[k], m));
            sum = __fadd_rn(sum, e);
            if (k == c) mine = e;
        }
        p = __fdiv_rn(mine, sum);
        const float4 a = reinterpret_cast<const float4*>(rois)[r];
        const float* d = deltas + (long)r * ld + 4 * c;
        const float bw = __fadd_rn(__fsub_rn(a.z, a.x), 1.0f), bh = __fadd_rn(__fsub_rn(a.w, a.y), 1.0f);
        const float cx = __fadd_rn(a.x, __fmul_rn(0.5f, bw)), cy = __fadd_rn(a.y, __fmul_rn(0.5f, bh));
        const float pcx = __fadd_rn(__fmul_rn(d[0], bw), cx), pcy = __fadd_rn(__fmul_rn(d[1], bh), cy);
        const float pw = __fmul_rn(det_expf(d[2]), bw), ph = __fmul_rn(det_expf(d[3]), bh);
        const float wmax = (float)(im_w - 1), hmax = (float)(im_h - 1);
        box.x = clip_coord(__fsub_rn(pcx, __fmul_rn(0.5f, pw)), wmax);
        box.y = clip_coord(__fsub_rn(pcy, __fmul_rn(0.5f, ph)), hmax);
        box.z = clip_coord(__fadd_rn(pcx, __fmul_rn(0.5f, pw)), wmax);
        box.w = clip_coord(__fadd_rn(pcy, __fmul_rn(0.5f, ph)), hmax);
    }
    prob[i] = p;
    reinterpret_cast<float4*>(boxes)[i] = box;
}

// ------------------------------------------------------------------------------------------ per-class detection
// One CTA per foreground class, R <= 2048 rows: rank by counting in the score order of nms_math.cuh, then the greedy
// suppression with cpu_nms's exact decision.  detect_kernel builds the R x R/64 "i suppresses j" bitmask in shared memory
// (upper triangle), and ONE warp walks its rows in rank order keeping `removed` in registers (lane w owns word w; R <= 2048
// = 32 words) -- the greedy chain costs a shuffle + a few ALU ops per row instead of a block-wide barrier per kept box (the
// barrier version: 85 us for 300 rows x 20 classes; the bitmask: 40 us).
constexpr int kDetThreads = 256;                      // detect_barrier_kernel
constexpr int kDetMaskThreads = 1024;                 // detect_kernel: 20 CTAs on 132 SMs -- the rank and mask phases scale with the CTA
constexpr int kDetMaxR = 2048;

// Image blockIdx.y of a batch: its prob / boxes rows, count and keep_idx / keep_count / conf_count outputs lie
// (image) * (the array's image stride) elements on.  Applied to the base pointers once, here at entry.
struct DetectStrides { long prob, boxes, count, keep_idx, keep_count, conf_count; };
__device__ __forceinline__ void detect_image_bases(const DetectStrides& is, const float*& prob, const float*& boxes,
                                                   const int*& count, int*& keep_idx, int*& keep_count, int*& conf_count) {
    const long img = blockIdx.y;
    prob += img * is.prob;
    boxes += img * is.boxes;
    if (count) count += img * is.count;
    keep_idx += img * is.keep_idx;
    keep_count += img * is.keep_count;
    conf_count += img * is.conf_count;
}

template <bool kBatch>
__global__ void __launch_bounds__(kDetMaskThreads) detect_kernel(const float* prob, const float* boxes, const int* count,
                                                             int R_cap, int NC, double thr, float conf,
                                                             int* keep_idx, int* keep_count, int* conf_count,
                                                             const DetectStrides is) {
    grid_dep_wait();
    if (kBatch) detect_image_bases(is, prob, boxes, count, keep_idx, keep_count, conf_count);
    extern __shared__ __align__(16) unsigned char dsm[];
    const int R = count ? min(*count, R_cap) : R_cap;
    const int words = (R_cap + 63) >> 6;                             // uint64 words per mask row
    float4* sbox = reinterpret_cast<float4*>(dsm);                   // [64*words] boxes by rank (entries >= R are never used: masked)
    unsigned long long* mask = reinterpret_cast<unsigned long long*>(sbox + 64 * words);   // [R_cap][words]: row i = who i suppresses
    uint32_t* skey = reinterpret_cast<uint32_t*>(mask + (size_t)R_cap * words);       // [R_cap] score keys by roi
    int* order = reinterpret_cast<int*>(skey + R_cap);               // [R_cap] roi index by rank
    float* sarea = reinterpret_cast<float*>(order + R_cap);          // [64*words] box areas by rank
    __shared__ int s_nge;                                            // rows with score >= conf: ranks [0, s_nge) after the sort
    const int cls = blockIdx.x + 1, tid = threadIdx.x;
    if (tid == 0) s_nge = 0;
    __syncthreads();
    {
        int nge = 0;
        for (int r = tid; r < R; r += kDetMaskThreads) {
            const float s = prob[(long)r * NC + cls];
            skey[r] = float_to_ordered(s);
            nge += s >= conf;
        }
        if (nge) atomicAdd(&s_nge, nge);
    }
    __syncthreads();
    // rank: a permutation of [0, R), and the rows with score >= conf come first whatever else the rows hold.  (The same
    // prologue as detect_barrier_kernel's; as a shared function it cost this kernel 2%: R left the uniform registers.)
    for (int r = tid; r < R; r += kDetMaskThreads) {
        const uint32_t s = skey[r];
        int rank = 0;
        for (int q = 0; q < R; ++q) rank += ahead(skey[q], q, s, r);
        order[rank] = r;
        const float4 b = reinterpret_cast<const float4*>(boxes)[(long)r * NC + cls];
        sbox[rank] = b;
        sarea[rank] = box_area(b);
    }
    __syncthreads();
    // mask rows: item = (word w, row i) with w >= i/64 (upper triangle), i fastest: the lanes of a warp work on consecutive
    // rows i against the SAME 64 columns, so sbox[j] is a broadcast read and sbox[i] a conflict-free one (with w fastest the
    // lanes read 5 different boxes 1 KB apart = the same banks: measured 4x slower).
    // The pair loop of suppress_word64(), written out: at this kernel's 64-register cap the shared routine needs 8 more bytes
    // of stack; with the `pt.on` select the compiler specialises the loop for the common case instead.
    const int nw = (R + 63) >> 6;
    const float thr_f = (float)thr;
    const PreTest pt = pretest_bounds(thr_f);
    for (int it = tid; it < R * nw; it += kDetMaskThreads) {
        const int w = it / R, i = it - w * R;
        unsigned long long bits = 0ull;
        if (w >= (i >> 6)) {
            const float4 a = sbox[i];
            const float area_a = sarea[i];
            const int j0 = w << 6;
            uint32_t sup_w[2] = {0u, 0u}, und_w[2] = {0u, 0u};
#pragma unroll
            for (int j = 0; j < 64; ++j) {
                float inter, uni;
                inter_union(a, area_a, sbox[j0 + j], sarea[j0 + j], inter, uni);
                uint32_t sure, und;
                pretest(inter, uni, pt, sure, und);
                sup_w[j >> 5] |= sure << (j & 31);
                und_w[j >> 5] |= und << (j & 31);
            }
            const int lo = max(i + 1 - j0, 0), hi = min(R - j0, 64);              // live columns [lo, hi) of this word
            unsigned long long live = hi < 64 ? (1ull << hi) - 1ull : ~0ull;
            live = lo < 64 ? (live >> lo) << lo : 0ull;
            bits = ((unsigned long long)sup_w[0] | ((unsigned long long)sup_w[1] << 32)) & live;
            const unsigned long long und = pt.on ? ((unsigned long long)und_w[0] | ((unsigned long long)und_w[1] << 32)) & live : live;
            bits = resolve_undecided(bits, und, [&](int j) { const float4 b = sbox[j0 + j]; return iou(a, box_area(a), b, box_area(b)); },
                                     thr, thr_f, FRCNN_NMS_GE_DOUBLE);
        }
        mask[(size_t)i * words + w] = bits;
    }
    __syncthreads();
    if (tid < 32) {
        const int lane = tid;
        const int n_ge = s_nge;
        unsigned long long removed = 0ull;                // lane w: suppression state of ranks [64w, 64w+64)
        int nk = 0, nconf = 0;
        // The loop-carried chain is removed -> shuffle -> bit test -> OR.  The row's mask word and its RoI index do not depend on
        // it: they are loaded four rows ahead, so that no shared-memory latency sits on the chain (it did: a load issued after
        // the test stalls the in-order warp at its first use, ~2x the chain itself).  "score >= conf" of the kept row is a rank
        // comparison: the rows are sorted by descending score, so the rows with score >= conf are exactly ranks [0, n_ge).
        for (int i0 = 0; i0 < R; i0 += 4) {
            unsigned long long m[4];
            int o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int i = i0 + k;
                m[k] = (i < R && lane < nw) ? mask[(size_t)i * words + lane] : 0ull;
                o[k] = i < R ? order[i] : 0;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int i = i0 + k;
                if (i >= R) break;                        // warp-uniform
                const unsigned long long word = __shfl_sync(0xffffffffu, removed, i >> 6);
                if ((word >> (i & 63)) & 1ull) continue;  // warp-uniform
                if (lane == 0) keep_idx[(long)(cls - 1) * R_cap + nk] = o[k];
                ++nk;
                if (i < n_ge) nconf = nk;
                removed |= m[k];
            }
        }
        for (int k = nk + lane; k < R_cap; k += 32) keep_idx[(long)(cls - 1) * R_cap + k] = -1;
        if (lane == 0) {
            keep_count[cls - 1] = nk;
            conf_count[cls - 1] = nconf;
        }
    }
}

// Fallback for R_cap too large for the bitmask to fit in shared memory (R_cap > ~1100): survivors are resolved with one
// block-wide barrier per kept box.
template <bool kBatch>
__global__ void __launch_bounds__(kDetThreads) detect_barrier_kernel(const float* prob, const float* boxes, const int* count,
                                                             int R_cap, int NC, double thr, float conf,
                                                             int* keep_idx, int* keep_count, int* conf_count,
                                                             const DetectStrides is) {
    grid_dep_wait();
    if (kBatch) detect_image_bases(is, prob, boxes, count, keep_idx, keep_count, conf_count);
    extern __shared__ __align__(16) unsigned char dsm[];
    const int R = count ? min(*count, R_cap) : R_cap;
    float4* sbox = reinterpret_cast<float4*>(dsm);                   // [R_cap] boxes by rank
    uint32_t* skey = reinterpret_cast<uint32_t*>(sbox + R_cap);      // [R_cap] score keys by roi
    int* order = reinterpret_cast<int*>(skey + R_cap);               // [R_cap] roi index by rank
    unsigned char* dead = reinterpret_cast<unsigned char*>(order + R_cap);  // [R_cap] by rank
    __shared__ int s_nconf, s_nge;                                   // s_nge: rows with score >= conf = ranks [0, s_nge)
    const int cls = blockIdx.x + 1, tid = threadIdx.x;
    if (tid == 0) { s_nconf = 0; s_nge = 0; }
    __syncthreads();
    {
        int nge = 0;
        for (int r = tid; r < R; r += kDetThreads) {
            const float s = prob[(long)r * NC + cls];
            skey[r] = float_to_ordered(s);
            nge += s >= conf;
        }
        if (nge) atomicAdd(&s_nge, nge);
    }
    __syncthreads();
    for (int r = tid; r < R; r += kDetThreads) {             // the order of detect_kernel
        const uint32_t s = skey[r];
        int rank = 0;
        for (int q = 0; q < R; ++q) rank += ahead(skey[q], q, s, r);
        order[rank] = r;
        sbox[rank] = reinterpret_cast<const float4*>(boxes)[(long)r * NC + cls];
        dead[rank] = 0;
    }
    __syncthreads();
    const int n_ge = s_nge;
    // greedy pass: for pivot i (ascending rank), all threads mark later candidates it suppresses
    int nk = 0;
    for (int i = 0; i < R; ++i) {
        if (dead[i]) { continue; }          // uniform: dead[] is only written before a barrier
        const float4 a = sbox[i];
        if (tid == 0) {
            keep_idx[(long)(cls - 1) * R_cap + nk] = order[i];
            if (i < n_ge) s_nconf = nk + 1;
        }
        ++nk;
        for (int j = i + 1 + tid; j < R; j += kDetThreads) {
            const float4 b = sbox[j];
            // box_area(a) stays in the loop: hoisted, it would sit on the serial path of every pivot
            if (!dead[j] && suppresses(iou(a, box_area(a), b, box_area(b)), thr, (float)thr, FRCNN_NMS_GE_DOUBLE)) dead[j] = 1;
        }
        __syncthreads();
    }
    for (int k = nk + tid; k < R_cap; k += kDetThreads) keep_idx[(long)(cls - 1) * R_cap + k] = -1;
    __syncthreads();
    if (tid == 0) {
        keep_count[cls - 1] = nk;
        conf_count[cls - 1] = s_nconf;
    }
}

// ------------------------------------------------------------------------------------------ detection lists
// The list forward.py:50-59 draws (preprocess.result_detections) from the per-class NMS lists of frcnn_detect: for class
// c = 1 .. NC-1 in order, the first conf_count[c-1] entries r of its keep list give the row
//     (c, int(x1 / im_scale), int(y1 / im_scale), int(x2 / im_scale), int(y2 / im_scale)),  score prob[r, c].
// `boxes[r, 4c:4c+4] / im_scale` divides a float32 row by a Python float; under NumPy >= 2 (NEP 50, the repository's NumPy)
// the Python float is a weak scalar, so the quotient is the float32 division by float32(im_scale) -- __fdiv_rn by the
// round-to-nearest float of the double -- and int() truncates it toward zero.  (Multiplying by a float reciprocal, or dividing
// in double, gives different bits.)  The one deviation: NaN and +-inf make int() raise and a quotient outside the int32
// range has no int32 value; here they convert as cvt.rzi.s32.f32 does (NaN -> 0, saturation to the int32 range), the rule
// of roi_coord (DESIGN.md 2).  The graph's boxes are clipped to the image, so it never gets there.
// One CTA per image: the classes go in chunks of kListThreads, a block scan over the chunk's counts gives every class its
// output offset, and then the chunk's rows are written in parallel (row t finds its class by a binary search of the offsets).
constexpr int kListThreads = 256;
struct ListStrides { long prob, boxes, keep_idx, conf_count; };

__global__ void __launch_bounds__(kListThreads) detection_lists_kernel(const float* prob, const float* boxes, const int* keep_idx,
                                                                     const int* conf_count, const double* im_scale, int R_cap,
                                                                     int NC, const ListStrides is, int* dets, float* scores,
                                                                     int* det_count) {
    grid_dep_wait();
    const long img = blockIdx.x;
    prob += img * is.prob;
    boxes += img * is.boxes;
    keep_idx += img * is.keep_idx;
    conf_count += img * is.conf_count;
    const long cap = (long)(NC - 1) * R_cap;
    dets += img * cap * 5;
    scores += img * cap;
    const float s = __double2float_rn(im_scale[img]);
    __shared__ int s_rel[kListThreads];                  // output offset of the chunk's classes, relative to the chunk
    __shared__ int s_warp[kListThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int carry = 0;                                       // rows of the classes before the chunk
    for (int c0 = 0; c0 < NC - 1; c0 += kListThreads) {
        const int k = c0 + tid;
        const int n = k < NC - 1 ? min(max(conf_count[k], 0), R_cap) : 0;
        int incl = n;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += v;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kListThreads / 32; ++w) {
            before += w < warp ? s_warp[w] : 0;
            total += s_warp[w];
        }
        s_rel[tid] = before + incl - n;
        __syncthreads();
        const int nc = min(kListThreads, NC - 1 - c0);
        for (int t = tid; t < total; t += kListThreads) {
            int lo = 0, hi = nc;                         // the last class j with s_rel[j] <= t (it holds row t: t < s_rel[j+1])
            while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (s_rel[mid] <= t) lo = mid; else hi = mid;
            }
            const int c = c0 + lo + 1;
            const int r = keep_idx[(long)(c - 1) * R_cap + (t - s_rel[lo])];
            int* d = dets + (long)(carry + t) * 5;
            d[0] = c;
            if (r >= 0 && r < R_cap) {
                const float* b = boxes + (long)r * 4 * NC + 4 * c;
#pragma unroll
                for (int q = 0; q < 4; ++q) d[1 + q] = __float2int_rz(__fdiv_rn(b[q], s));
                scores[carry + t] = prob[(long)r * NC + c];
            } else {                                     // not an index frcnn_detect writes: nothing is read
#pragma unroll
                for (int q = 0; q < 4; ++q) d[1 + q] = 0;
                scores[carry + t] = 0.0f;
            }
        }
        carry += total;
        __syncthreads();                                 // s_rel / s_warp are rewritten by the next chunk
    }
    if (tid == 0) det_count[img] = carry;
}

static int grid_for(long total, int block) {
    long g = (total + block - 1) / block;
    const long cap = 132l * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace frcnn

using namespace frcnn;

extern "C" int frcnn_version(void) { return 100; }
extern "C" const char* frcnn_last_error(void) { return g_err; }

namespace frcnn {
static int pdl_default() {
    // off unless FRCNN_PDL=1: the persistent conv CTAs own every SM's shared memory until they exit, so a dependent kernel
    // cannot become resident early anyway
    const char* e = getenv("FRCNN_PDL");
    return (e != nullptr && e[0] == '1') ? 1 : 0;
}
static thread_local int g_pdl = -1;          // -1: not set by this thread -> environment default
bool pdl_enabled() { return (g_pdl < 0 ? pdl_default() : g_pdl) != 0; }
}  // namespace frcnn
extern "C" void frcnn_set_programmatic_launch(int on) { frcnn::g_pdl = on < 0 ? -1 : (on ? 1 : 0); }

extern "C" int frcnn_pack_image(const float* x_chw, int C, int H, int W, int C_pad, void* y_hi, void* y_lo,
                                void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(x_chw && y_hi && C > 0 && H > 0 && W > 0 && C_pad >= C && C_pad % 8 == 0,
                  "frcnn_pack_image: bad arguments (C=%d H=%d W=%d C_pad=%d)", C, H, W, C_pad);
    const long total = (long)H * W * C_pad;
    pack_image_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        x_chw, C, H, W, C_pad, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" int frcnn_pack_conv_weights(const float* w_oihw, int Cout, int Cin, int kh, int kw, int Cin_pad, void* w_hi,
                                       void* w_lo, int perm_chw_to_hwc, int pc, int ph, int pw, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(w_oihw && w_hi && Cout > 0 && Cin > 0 && kh > 0 && kw > 0 && Cin_pad >= Cin && Cin_pad % 8 == 0,
                  "frcnn_pack_conv_weights: bad arguments");
    FRCNN_REQUIRE(!perm_chw_to_hwc || (pc * ph * pw == Cin && Cin_pad == Cin),
                  "frcnn_pack_conv_weights: permutation needs pc*ph*pw == Cin == Cin_pad");
    const long total = (long)kh * kw * Cout * Cin_pad;
    pack_weights_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        w_oihw, Cout, Cin, kh * kw, Cin_pad, (__nv_bfloat16*)w_hi, (__nv_bfloat16*)w_lo, perm_chw_to_hwc, pc, ph, pw);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" int frcnn_preprocess_bgr8(const unsigned char* img_hwc, int h0, int w0, double mean_b, double mean_g,
                                     double mean_r, double im_scale, int H, int W, float* out_chw, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(img_hwc && out_chw && h0 > 0 && w0 > 0 && H > 0 && W > 0 && im_scale > 0.0,
                  "frcnn_preprocess_bgr8: bad arguments");
    PreArgs a;
    a.src = img_hwc; a.h0 = h0; a.w0 = w0;
    a.m0 = mean_b; a.m1 = mean_g; a.m2 = mean_r;
    a.sx = 1.0 / im_scale; a.sy = 1.0 / im_scale;
    a.H = H; a.W = W; a.out = out_chw;
    preprocess_bgr8_kernel<<<grid_for((long)H * W, 256), 256, 0, (cudaStream_t)stream>>>(a);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" int frcnn_pack_image_im2col3x3_strided(const float* x, int C, int H, int W, long stride_c, long stride_h,
                                                  long stride_w, void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(x && y_hi && C > 0 && C <= 3 && H > 0 && W > 0, "frcnn_pack_image_im2col3x3: needs 1 <= C <= 3 (got %d)", C);
    FRCNN_REQUIRE(stride_c > 0 && stride_h > 0 && stride_w > 0, "frcnn_pack_image_im2col3x3_strided: strides must be positive");
    pack_image_im2col_kernel<<<grid_for((long)H * W, 128), 128, 0, (cudaStream_t)stream>>>(
        x, C, H, W, stride_c, stride_h, stride_w, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" size_t frcnn_image_c8_elems(int H, int W) {
    return (H > 0 && W > 0) ? ((size_t)H * (W + 2) + 8) * 8 : 0;          // 8 slack pixels behind the last row, zeroed by the pack
}

extern "C" int frcnn_pack_image_c8(const float* x, int C, int H, int W, long stride_c, long stride_h, long stride_w, void* y_hi,
                                   void* y_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(x && y_hi && C > 0 && C <= 3 && H > 0 && W > 0, "frcnn_pack_image_c8: needs 1 <= C <= 3 (got %d)", C);
    FRCNN_REQUIRE(stride_c > 0 && stride_h > 0 && stride_w > 0, "frcnn_pack_image_c8: strides must be positive");
    const long total = (long)H * (W + 2) + 8;
    pack_image_c8_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(x, C, H, W, stride_c, stride_h, stride_w,
                                                                                (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo, 8, 0, 0,
                                                                                nullptr);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

namespace frcnn {
static int pack_image_c8_n(const char* fn, const float* x, int N, int C, int H, int W, long stride_n, long stride_c, long stride_h,
                           long stride_w, const int* extents, void* y_hi, void* y_lo, cudaStream_t stream) {
    FRCNN_REQUIRE(x && y_hi && N >= 1 && N <= 65535 && C > 0 && C <= 3 && H > 0 && W > 0,
                  "%s: needs 1 <= N <= 65535 and 1 <= C <= 3 (got N=%d C=%d)", fn, N, C);
    FRCNN_REQUIRE(stride_n > 0 && stride_c > 0 && stride_h > 0 && stride_w > 0, "%s: strides must be positive", fn);
    const long total = (long)H * (W + 2) + 8;
    const dim3 grid(grid_for(total, 256), N);
    pack_image_c8_kernel<<<grid, 256, 0, stream>>>(x, C, H, W, stride_c, stride_h, stride_w, (__nv_bfloat16*)y_hi,
                                                   (__nv_bfloat16*)y_lo, 8, stride_n, (long)frcnn_image_c8_elems(H, W), extents);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}
}  // namespace frcnn

extern "C" int frcnn_pack_image_c8_batch(const float* x, int N, int C, int H, int W, long stride_n, long stride_c, long stride_h,
                                         long stride_w, void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    return pack_image_c8_n("frcnn_pack_image_c8_batch", x, N, C, H, W, stride_n, stride_c, stride_h, stride_w, nullptr, y_hi, y_lo,
                           (cudaStream_t)stream);
}

extern "C" int frcnn_pack_image_c8_batch_ext(const float* x, int N, int C, int H, int W, long stride_n, long stride_c,
                                             long stride_h, long stride_w, const int* extents, void* y_hi, void* y_lo,
                                             void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(extents, "frcnn_pack_image_c8_batch_ext: extents is NULL");
    return pack_image_c8_n("frcnn_pack_image_c8_batch_ext", x, N, C, H, W, stride_n, stride_c, stride_h, stride_w, extents, y_hi,
                           y_lo, (cudaStream_t)stream);
}

extern "C" int frcnn_preprocess_bgr8_canvas(const unsigned char* arena, long long arena_bytes, const long long* src_off,
                                             const int* src_hw, const double* inv_scale, const int* extents, int N, int Hc,
                                             int Wc, double mean_b, double mean_g, double mean_r, void* y_hi, void* y_lo,
                                             void* stream) {
    FRCNN_ENTRY();
    const char* fn = "frcnn_preprocess_bgr8_canvas";
    FRCNN_REQUIRE(arena, "%s: arena is NULL", fn);
    FRCNN_REQUIRE(arena_bytes > 0, "%s: arena_bytes must be positive (got %lld)", fn, arena_bytes);
    FRCNN_REQUIRE(src_off, "%s: src_off is NULL", fn);
    FRCNN_REQUIRE(src_hw, "%s: src_hw is NULL", fn);
    FRCNN_REQUIRE(inv_scale, "%s: inv_scale is NULL", fn);
    FRCNN_REQUIRE(extents, "%s: extents is NULL", fn);
    FRCNN_REQUIRE(y_hi, "%s: y_hi is NULL", fn);
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "%s: needs 1 <= N <= 65535 (got N=%d)", fn, N);
    FRCNN_REQUIRE(Hc > 0 && Wc > 0, "%s: the canvas must be positive (got Hc=%d Wc=%d)", fn, Hc, Wc);
    PreCanvasArgs a;
    a.arena = arena; a.arena_bytes = arena_bytes;
    a.src_off = src_off; a.src_hw = src_hw; a.inv_scale = inv_scale; a.extents = extents;
    a.Hc = Hc; a.Wc = Wc;
    a.m0 = mean_b; a.m1 = mean_g; a.m2 = mean_r;
    a.hi = (__nv_bfloat16*)y_hi; a.lo = (__nv_bfloat16*)y_lo;
    a.out_elems = (long)frcnn_image_c8_elems(Hc, Wc);
    preprocess_bgr8_canvas_kernel<<<dim3(Hc, N), 128, 0, (cudaStream_t)stream>>>(a);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" int frcnn_pack_conv_weights_c8(const float* w_oihw, int Cout, int Cin, void* w_hi, void* w_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(w_oihw && w_hi && Cout > 0 && Cin > 0 && Cin <= 3, "frcnn_pack_conv_weights_c8: needs 1 <= Cin <= 3");
    pack_weights_c8_kernel<<<cdiv(3 * Cout * 32, 128), 128, 0, (cudaStream_t)stream>>>(w_oihw, Cout, Cin, (__nv_bfloat16*)w_hi,
                                                                                     (__nv_bfloat16*)w_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" int frcnn_pack_image_im2col3x3(const float* x_chw, int C, int H, int W, void* y_hi, void* y_lo, void* stream) {
    return frcnn_pack_image_im2col3x3_strided(x_chw, C, H, W, (long)H * W, W, 1, y_hi, y_lo, stream);
}

extern "C" int frcnn_pack_conv_weights_im2col3x3(const float* w_oihw, int Cout, int Cin, void* w_hi, void* w_lo,
                                                 void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(w_oihw && w_hi && Cout > 0 && Cin > 0 && Cin <= 3, "frcnn_pack_conv_weights_im2col3x3: needs 1 <= Cin <= 3");
    pack_weights_im2col_kernel<<<cdiv(Cout * 32, 128), 128, 0, (cudaStream_t)stream>>>(
        w_oihw, Cout, Cin, (__nv_bfloat16*)w_hi, (__nv_bfloat16*)w_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" int frcnn_unpack_nhwc(const void* x_hi, const void* x_lo, int H, int W, int C, float* y_chw, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(x_hi && y_chw && H > 0 && W > 0 && C > 0, "frcnn_unpack_nhwc: bad arguments");
    const long total = (long)H * W * C;
    unpack_nhwc_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x_hi, (const __nv_bfloat16*)x_lo, H, W, C, y_chw);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

namespace frcnn {
static int maxpool2x2_n(const char* fn, const void* x_hi, const void* x_lo, int N, int H, int W, int C, void* y_hi, void* y_lo,
                        cudaStream_t stream) {
    FRCNN_REQUIRE(x_hi && y_hi && H > 0 && W > 0 && C > 0 && C % 8 == 0, "%s: bad arguments (C=%d)", fn, C);
    FRCNN_REQUIRE((x_lo == nullptr) == (y_lo == nullptr), "%s: lo planes must both be given or both NULL", fn);
    const long total = (long)((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
    FRCNN_CUDA_OK(launch_pdl(N > 1 ? maxpool_kernel<true> : maxpool_kernel<false>, dim3(grid_for(total, 256), N), dim3(256), 0, stream, (const __nv_bfloat16*)x_hi,
                             (const __nv_bfloat16*)x_lo, H, W, C, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo));
    return FRCNN_OK;
}

static int roi_pool_n(const char* fn, const void* feat_hi, const void* feat_lo, int N, int H, int W, int C, const float* rois,
                      long rois_stride, const int* counts, long count_stride, int R_cap, int outh, int outw, float scale, void* out_hi,
                      void* out_lo, float* out_f32, long out_stride, cudaStream_t stream, const int* extents = nullptr,
                      int halvings = 0) {
    FRCNN_REQUIRE(halvings >= 0 && halvings <= 30, "%s: halvings must be in [0,30] (got %d)", fn, halvings);
    FRCNN_REQUIRE(feat_hi && rois && (out_hi || out_f32) && H > 0 && W > 0 && C > 0 && C % 8 == 0 && R_cap > 0 &&
                      outh > 0 && outw > 0,
                  "%s: bad arguments", fn);
    FRCNN_REQUIRE(!out_lo || out_hi, "%s: out_lo without out_hi", fn);
    FRCNN_REQUIRE(outw < kRoiMaxBins && outh < kRoiMaxBins, "%s: outh and outw must be < %d", fn, kRoiMaxBins);
    if (N > 1) {
        const long rows = (long)R_cap * outh * outw * C;
        FRCNN_REQUIRE(rois_stride >= 0 && rois_stride % 4 == 0, "%s: rois image stride must be a multiple of 4 and >= 0", fn);
        FRCNN_REQUIRE(!counts || count_stride >= 0, "%s: count image stride must be >= 0", fn);
        FRCNN_REQUIRE(out_stride >= rows && out_stride % 8 == 0, "%s: output image stride %ld overlaps (needs a multiple of 8, >= %ld)",
                      fn, out_stride, rows);
    }
    int c8_per_cta = 1;                                      // a power of two: the slice's channel groups are contiguous
    while (2 * c8_per_cta <= C / 8 && 2 * c8_per_cta * outw <= kRoiColMaxThreads) c8_per_cta *= 2;
    const int slices = (C / 8 + c8_per_cta - 1) / c8_per_cta;
    const int threads = ((outw * c8_per_cta + 31) / 32) * 32;
    const long ctas = (long)R_cap * slices;
    const dim3 grid((unsigned)(ctas < 132l * 64 ? ctas : 132l * 64), N);
    if (feat_lo) {
        FRCNN_CUDA_OK(launch_pdl(N > 1 ? roi_pool_col_kernel<true, true> : roi_pool_col_kernel<true, false>, grid, dim3(threads), 0, stream, (const __nv_bfloat16*)feat_hi,
                                 (const __nv_bfloat16*)feat_lo, H, W, C, rois, counts, R_cap, outh, outw, scale, (__nv_bfloat16*)out_hi,
                                 (__nv_bfloat16*)out_lo, out_f32, c8_per_cta, slices, rois_stride, count_stride, out_stride,
                                 extents, halvings));
    } else {
        FRCNN_CUDA_OK(launch_pdl(N > 1 ? roi_pool_col_kernel<false, true> : roi_pool_col_kernel<false, false>, grid, dim3(threads), 0, stream, (const __nv_bfloat16*)feat_hi,
                                 (const __nv_bfloat16*)feat_lo, H, W, C, rois, counts, R_cap, outh, outw, scale, (__nv_bfloat16*)out_hi,
                                 (__nv_bfloat16*)out_lo, out_f32, c8_per_cta, slices, rois_stride, count_stride, out_stride,
                                 extents, halvings));
    }
    return FRCNN_OK;
}

static int head_decode_n(const char* fn, int N, const float* scores, const float* deltas, int ld, const float* rois,
                         const int* counts, int R_cap, int num_classes, int im_h, int im_w, float* out_prob, float* out_boxes,
                         const DecodeStrides& is, cudaStream_t stream, const int* im_info = nullptr) {
    FRCNN_REQUIRE(scores && deltas && rois && out_prob && out_boxes && R_cap > 0 && num_classes > 0 && ld >= num_classes,
                  "%s: bad arguments", fn);
    if (N > 1) {
        FRCNN_REQUIRE(is.in >= 0 && is.rois >= 0 && is.rois % 4 == 0 && (!counts || is.count >= 0),
                      "%s: input image strides must be >= 0 (rois: a multiple of 4)", fn);
        FRCNN_REQUIRE(is.prob >= (long)R_cap * num_classes, "%s: prob image stride %ld overlaps (needs >= %ld)", fn, is.prob,
                      (long)R_cap * num_classes);
        FRCNN_REQUIRE(is.boxes >= 4l * R_cap * num_classes && is.boxes % 4 == 0,
                      "%s: boxes image stride %ld overlaps (needs a multiple of 4, >= %ld)", fn, is.boxes, 4l * R_cap * num_classes);
    }
    const int total = R_cap * num_classes;
    FRCNN_CUDA_OK(launch_pdl(N > 1 ? head_decode_kernel<true> : head_decode_kernel<false>, dim3(cdiv(total, 128), N), dim3(128), 0, stream, scores, deltas, ld, rois, counts, R_cap,
                             num_classes, im_h, im_w, out_prob, out_boxes, is, im_info));
    return FRCNN_OK;
}

static int detect_n(const char* fn, int N, const float* prob, const float* boxes, const int* counts, int R_cap, int num_classes,
                    double nms_thresh, float conf, int* keep_idx, int* keep_count, int* conf_count, const DetectStrides& is,
                    cudaStream_t stream) {
    FRCNN_REQUIRE(prob && boxes && keep_idx && keep_count && conf_count && num_classes > 1, "%s: bad arguments", fn);
    FRCNN_REQUIRE(R_cap > 0 && R_cap <= kDetMaxR, "%s: R_cap must be in [1,%d] (got %d)", fn, kDetMaxR, R_cap);
    if (N > 1) {
        FRCNN_REQUIRE(is.prob >= 0 && is.boxes >= 0 && is.boxes % 4 == 0 && (!counts || is.count >= 0),
                      "%s: input image strides must be >= 0 (boxes: a multiple of 4)", fn);
        FRCNN_REQUIRE(is.keep_idx >= (long)(num_classes - 1) * R_cap, "%s: keep_idx image stride %ld overlaps (needs >= %ld)", fn,
                      is.keep_idx, (long)(num_classes - 1) * R_cap);
        FRCNN_REQUIRE(is.keep_count >= num_classes - 1 && is.conf_count >= num_classes - 1,
                      "%s: keep_count / conf_count image strides %ld / %ld overlap (need >= %d)", fn, is.keep_count, is.conf_count,
                      num_classes - 1);
    }
    const size_t words = (size_t)(R_cap + 63) / 64;
    size_t smem = (size_t)R_cap * (sizeof(float) + sizeof(int) + 8 * words) + 64 * words * (sizeof(float4) + sizeof(float)) + 16;
    const dim3 grid(num_classes - 1, N);
    if (smem > 200 * 1024) {
        smem = (size_t)R_cap * (sizeof(float) + sizeof(int) + sizeof(float4) + 1) + 16;
        auto kern = N > 1 ? detect_barrier_kernel<true> : detect_barrier_kernel<false>;
        FRCNN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        FRCNN_CUDA_OK(launch_pdl(kern, grid, dim3(kDetThreads), smem, stream, prob, boxes, counts, R_cap, num_classes,
                                 nms_thresh, conf, keep_idx, keep_count, conf_count, is));
        return FRCNN_OK;
    }
    auto kern = N > 1 ? detect_kernel<true> : detect_kernel<false>;
    FRCNN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FRCNN_CUDA_OK(launch_pdl(kern, grid, dim3(kDetMaskThreads), smem, stream, prob, boxes, counts, R_cap, num_classes,
                             nms_thresh, conf, keep_idx, keep_count, conf_count, is));
    return FRCNN_OK;
}
}  // namespace frcnn

#define FRCNN_REQUIRE_BATCH(fn, N) FRCNN_REQUIRE((N) >= 1 && (N) <= 65535, "%s: N must be in [1,65535] (got %d)", fn, (int)(N))

extern "C" int frcnn_maxpool2x2_ceil(const void* x_hi, const void* x_lo, int H, int W, int C, void* y_hi, void* y_lo,
                                     void* stream) {
    FRCNN_ENTRY();
    return maxpool2x2_n("frcnn_maxpool2x2_ceil", x_hi, x_lo, 1, H, W, C, y_hi, y_lo, (cudaStream_t)stream);
}

extern "C" int frcnn_maxpool2x2_ceil_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int C, void* y_hi, void* y_lo,
                                           void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE_BATCH("frcnn_maxpool2x2_ceil_batch", N);
    return maxpool2x2_n("frcnn_maxpool2x2_ceil_batch", x_hi, x_lo, N, H, W, C, y_hi, y_lo, (cudaStream_t)stream);
}

extern "C" int frcnn_roi_pool(const void* feat_hi, const void* feat_lo, int H, int W, int C, const float* rois,
                              const int* count, int R_cap, int outh, int outw, float scale, void* out_hi, void* out_lo,
                              float* out_f32, void* stream) {
    FRCNN_ENTRY();
    return roi_pool_n("frcnn_roi_pool", feat_hi, feat_lo, 1, H, W, C, rois, 0, count, 0, R_cap, outh, outw, scale, out_hi, out_lo,
                      out_f32, 0, (cudaStream_t)stream);
}

extern "C" int frcnn_roi_pool_batch(const void* feat_hi, const void* feat_lo, int N, int H, int W, int C, const float* rois,
                                    long rois_stride, const int* counts, long count_stride, int R_cap, int outh, int outw, float scale,
                                    void* out_hi, void* out_lo, float* out_f32, long out_stride, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE_BATCH("frcnn_roi_pool_batch", N);
    return roi_pool_n("frcnn_roi_pool_batch", feat_hi, feat_lo, N, H, W, C, rois, rois_stride, counts, count_stride, R_cap, outh, outw,
                      scale, out_hi, out_lo, out_f32, out_stride, (cudaStream_t)stream);
}

extern "C" int frcnn_head_decode(const float* scores, const float* deltas, int ld, const float* rois, const int* count,
                                 int R_cap, int num_classes, int im_h, int im_w, float* out_prob, float* out_boxes,
                                 void* stream) {
    FRCNN_ENTRY();
    const DecodeStrides is = {0, 0, 0, 0, 0};
    return head_decode_n("frcnn_head_decode", 1, scores, deltas, ld, rois, count, R_cap, num_classes, im_h, im_w, out_prob, out_boxes,
                         is, (cudaStream_t)stream);
}

extern "C" int frcnn_head_decode_batch(int N, const float* scores, const float* deltas, int ld, long in_stride, const float* rois,
                                       long rois_stride, const int* counts, long count_stride, int R_cap, int num_classes, int im_h,
                                       int im_w, float* out_prob, long prob_stride, float* out_boxes, long boxes_stride,
                                       void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE_BATCH("frcnn_head_decode_batch", N);
    const DecodeStrides is = {in_stride, rois_stride, count_stride, prob_stride, boxes_stride};
    return head_decode_n("frcnn_head_decode_batch", N, scores, deltas, ld, rois, counts, R_cap, num_classes, im_h, im_w, out_prob,
                         out_boxes, is, (cudaStream_t)stream);
}

extern "C" int frcnn_roi_pool_batch_ext(const void* feat_hi, const void* feat_lo, int N, int H, int W, int C, const float* rois,
                                        long rois_stride, const int* counts, long count_stride, int R_cap, int outh, int outw,
                                        float scale, const int* extents, int halvings, void* out_hi, void* out_lo, float* out_f32,
                                        long out_stride, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE_BATCH("frcnn_roi_pool_batch_ext", N);
    FRCNN_REQUIRE(extents, "frcnn_roi_pool_batch_ext: extents is NULL");
    return roi_pool_n("frcnn_roi_pool_batch_ext", feat_hi, feat_lo, N, H, W, C, rois, rois_stride, counts, count_stride, R_cap, outh,
                      outw, scale, out_hi, out_lo, out_f32, out_stride, (cudaStream_t)stream, extents, halvings);
}

extern "C" int frcnn_head_decode_batch_ext(int N, const float* scores, const float* deltas, int ld, long in_stride, const float* rois,
                                           long rois_stride, const int* counts, long count_stride, int R_cap, int num_classes,
                                           const int* im_info, float* out_prob, long prob_stride, float* out_boxes,
                                           long boxes_stride, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE_BATCH("frcnn_head_decode_batch_ext", N);
    FRCNN_REQUIRE(im_info, "frcnn_head_decode_batch_ext: im_info is NULL");
    const DecodeStrides is = {in_stride, rois_stride, count_stride, prob_stride, boxes_stride};
    return head_decode_n("frcnn_head_decode_batch_ext", N, scores, deltas, ld, rois, counts, R_cap, num_classes, 0, 0, out_prob,
                         out_boxes, is, (cudaStream_t)stream, im_info);
}

namespace frcnn {
__global__ void bbox_decode_kernel(const float* boxes, const float* trans, int N, int K, int clip, int im_h, int im_w,
                                   int min_size, float* out, unsigned char* ok_flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * K) return;
    const int n = i / K;
    float4 o;
    if (trans == nullptr) {        // clip / filter only: `boxes` is [N, 4K]
        o = reinterpret_cast<const float4*>(boxes)[i];
    } else {
        const float4 a = reinterpret_cast<const float4*>(boxes)[n];
        const float4 d = reinterpret_cast<const float4*>(trans)[i];
        const float bw = __fadd_rn(__fsub_rn(a.z, a.x), 1.0f), bh = __fadd_rn(__fsub_rn(a.w, a.y), 1.0f);
        const float cx = __fadd_rn(a.x, __fmul_rn(0.5f, bw)), cy = __fadd_rn(a.y, __fmul_rn(0.5f, bh));
        const float pcx = __fadd_rn(__fmul_rn(d.x, bw), cx), pcy = __fadd_rn(__fmul_rn(d.y, bh), cy);
        const float pw = __fmul_rn(det_expf(d.z), bw), ph = __fmul_rn(det_expf(d.w), bh);
        o.x = __fsub_rn(pcx, __fmul_rn(0.5f, pw));
        o.y = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
        o.z = __fadd_rn(pcx, __fmul_rn(0.5f, pw));
        o.w = __fadd_rn(pcy, __fmul_rn(0.5f, ph));
    }
    if (clip) {
        const float wmax = (float)(im_w - 1), hmax = (float)(im_h - 1);
        o.x = clip_coord(o.x, wmax);
        o.y = clip_coord(o.y, hmax);
        o.z = clip_coord(o.z, wmax);
        o.w = clip_coord(o.w, hmax);
    }
    reinterpret_cast<float4*>(out)[i] = o;
    if (ok_flags) {
        const float ws = __fadd_rn(__fsub_rn(o.z, o.x), 1.0f), hs = __fadd_rn(__fsub_rn(o.w, o.y), 1.0f);
        ok_flags[i] = (ws >= (float)min_size && hs >= (float)min_size) ? 1 : 0;
    }
}
}  // namespace frcnn

extern "C" int frcnn_bbox_decode(const float* boxes, const float* trans, int N, int K, int clip, int im_h, int im_w,
                                 int min_size, float* out, unsigned char* ok_flags, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 0 && K > 0, "frcnn_bbox_decode: bad N=%d K=%d", N, K);
    if (N == 0) return FRCNN_OK;
    FRCNN_REQUIRE(boxes && out, "frcnn_bbox_decode: NULL argument");   // trans == NULL: clip / filter only
    FRCNN_REQUIRE(!ok_flags || K == 1, "frcnn_bbox_decode: ok_flags needs K == 1");
    bbox_decode_kernel<<<cdiv(N * K, 128), 128, 0, (cudaStream_t)stream>>>(boxes, trans, N, K, clip, im_h, im_w, min_size,
                                                                          out, ok_flags);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" int frcnn_detect(const float* prob, const float* boxes, const int* count, int R_cap, int num_classes,
                            double nms_thresh, float conf, int* keep_idx, int* keep_count, int* conf_count,
                            void* stream) {
    FRCNN_ENTRY();
    const DetectStrides is = {0, 0, 0, 0, 0, 0};
    return detect_n("frcnn_detect", 1, prob, boxes, count, R_cap, num_classes, nms_thresh, conf, keep_idx, keep_count, conf_count, is,
                    (cudaStream_t)stream);
}

extern "C" int frcnn_detect_batch(int N, const float* prob, long prob_stride, const float* boxes, long boxes_stride,
                                  const int* counts, long count_stride, int R_cap, int num_classes, double nms_thresh, float conf,
                                  int* keep_idx, long keep_idx_stride, int* keep_count, long keep_count_stride, int* conf_count,
                                  long conf_count_stride, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE_BATCH("frcnn_detect_batch", N);
    const DetectStrides is = {prob_stride, boxes_stride, count_stride, keep_idx_stride, keep_count_stride, conf_count_stride};
    return detect_n("frcnn_detect_batch", N, prob, boxes, counts, R_cap, num_classes, nms_thresh, conf, keep_idx, keep_count, conf_count,
                    is, (cudaStream_t)stream);
}

extern "C" int frcnn_detection_lists_batch(int N, const float* prob, long prob_stride, const float* boxes, long boxes_stride,
                                           const int* keep_idx, long keep_idx_stride, const int* conf_count, long conf_count_stride,
                                           const double* im_scale, int R_cap, int num_classes, int* out_dets, float* out_scores,
                                           int* out_det_count, void* stream) {
    FRCNN_ENTRY();
    const char* fn = "frcnn_detection_lists_batch";
    FRCNN_REQUIRE(prob, "%s: prob is NULL", fn);
    FRCNN_REQUIRE(boxes, "%s: boxes is NULL", fn);
    FRCNN_REQUIRE(keep_idx, "%s: keep_idx is NULL", fn);
    FRCNN_REQUIRE(conf_count, "%s: conf_count is NULL", fn);
    FRCNN_REQUIRE(im_scale, "%s: im_scale is NULL", fn);
    FRCNN_REQUIRE(out_dets, "%s: out_dets is NULL", fn);
    FRCNN_REQUIRE(out_scores, "%s: out_scores is NULL", fn);
    FRCNN_REQUIRE(out_det_count, "%s: out_det_count is NULL", fn);
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "%s: N must be in [1,65535] (got N=%d)", fn, N);
    FRCNN_REQUIRE(R_cap >= 1, "%s: R_cap must be >= 1 (got R_cap=%d)", fn, R_cap);
    FRCNN_REQUIRE(num_classes >= 2, "%s: num_classes must be >= 2 (got num_classes=%d)", fn, num_classes);
    FRCNN_REQUIRE((long)(num_classes - 1) * R_cap * 5 <= 0x7fffffffl, "%s: (num_classes-1) * R_cap = %ld rows is too large", fn,
                  (long)(num_classes - 1) * R_cap);
    FRCNN_REQUIRE(prob_stride >= 0 && boxes_stride >= 0 && keep_idx_stride >= 0 && conf_count_stride >= 0,
                  "%s: image strides must be >= 0", fn);
    const ListStrides is = {prob_stride, boxes_stride, keep_idx_stride, conf_count_stride};
    FRCNN_CUDA_OK(launch_pdl(detection_lists_kernel, dim3(N), dim3(kListThreads), 0, (cudaStream_t)stream, prob, boxes, keep_idx,
                             conf_count, im_scale, R_cap, num_classes, is, out_dets, out_scores, out_det_count));
    return FRCNN_OK;
}
