// raw_photo.cuh -- the resize of forward.py's img_preprocessing (bilinear) and of the VOC training dataset (bicubic) on raw
// uint8 BGR photos, and the descriptor rule of a canvas batch's raw-photo slots: the one statement of each for every kernel
// that reads raw photos (head_ops.cu: preprocess_bgr8_kernel, preprocess_bgr8_canvas_kernel; resnet_ops.cu:
// preprocess_canvas_im2col_kernel).
#pragma once
#include "common.cuh"

namespace frcnn {

// OpenCV's float bilinear (cv.resize INTER_LINEAR), restated: coordinate / floor / fraction in double, weight cast to
// float, h = fma(S[x1] - S[x0], tx, S[x0]) on both source rows, out = fma(h1 - h0, ty, h0).
//
// One axis of the resize: output index o of a source axis of n pixels -> the two source indices and the weight of the
// second.  Whatever inv_scale holds (0, negative, huge, +-inf, NaN), i0 and i1 end up inside [0, n - 1]: the conversion to
// int saturates, and an index clamped to either end gets weight 0.
struct BilinearTap { int i0, i1; float t; };
__device__ __forceinline__ BilinearTap bilinear_tap(int o, double inv_scale, int n) {
    const double f = ((double)o + 0.5) * inv_scale - 0.5;
    BilinearTap r;
    r.i0 = (int)floor(f);
    r.t = (float)(f - (double)r.i0);
    if (r.i0 < 0) { r.i0 = 0; r.t = 0.0f; }
    if (r.i0 >= n - 1) { r.i0 = n - 1; r.t = 0.0f; }
    r.i1 = min(r.i0 + 1, n - 1);
    return r;
}

// The resized, mean-subtracted pixel at taps (y, x) of a dense uint8 (h0, w0, 3) image: out[c], c = B, G, R.
__device__ __forceinline__ void bilinear_bgr8(const unsigned char* src, int w0, const BilinearTap& y, const BilinearTap& x,
                                              double m0, double m1, double m2, float out[3]) {
    const unsigned char* r0 = src + (long)y.i0 * w0 * 3;
    const unsigned char* r1 = src + (long)y.i1 * w0 * 3;
    const double mean[3] = {m0, m1, m2};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float p00 = (float)((double)r0[x.i0 * 3 + c] - mean[c]);
        const float p01 = (float)((double)r0[x.i1 * 3 + c] - mean[c]);
        const float p10 = (float)((double)r1[x.i0 * 3 + c] - mean[c]);
        const float p11 = (float)((double)r1[x.i1 * 3 + c] - mean[c]);
        const float ha = __fmaf_rn(__fsub_rn(p01, p00), x.t, p00);
        const float hb = __fmaf_rn(__fsub_rn(p11, p10), x.t, p10);
        out[c] = __fmaf_rn(__fsub_rn(hb, ha), y.t, ha);
    }
}

// OpenCV's float bicubic (cv.resize INTER_CUBIC, the VOC dataset's resize), restated from OpenCV's generic path -- what
// cv2 computes for float32 images when IPP is off; with IPP on, cv2 hands float cubic to Intel IPP, whose rounding differs
// in the last bits (DESIGN.md section 5).  Per axis: the coordinate f = float((o + 0.5) * inv_scale - 0.5) (double
// product and difference, then rounded to float), s = floor(f), t = f - s, coefficients from A = -0.75 in float
// (interpolateCubic), taps s-1 .. s+2 clamped to [0, n - 1] (replicate).  No operation is contracted into an FMA.
// Whatever inv_scale holds, every index stays inside [0, n - 1] and the weights stay finite: a non-finite t becomes 0.
struct CubicTap { int i[4]; float w[4]; bool border; };
__device__ __forceinline__ CubicTap cubic_tap(int o, double inv_scale, int n) {
    const float f = (float)__dsub_rn(__dmul_rn((double)o + 0.5, inv_scale), 0.5);
    float fl = floorf(f);
    float t = __fsub_rn(f, fl);
    if (!(t >= 0.0f && t < 1.0f)) t = 0.0f;                      // f = +-inf or NaN
    fl = fminf(fmaxf(fl, -2.0f), (float)n + 1.0f);               // NaN -> -2; no int overflow below
    const int s = (int)fl;
    CubicTap r;
    r.border = s < 1 || s + 2 >= n;     // OpenCV's border columns (xmin / xmax): their horizontal sum starts from 0.0f
#pragma unroll
    for (int k = 0; k < 4; ++k) r.i[k] = min(max(s - 1 + k, 0), n - 1);
    const float x1 = __fadd_rn(t, 1.0f), y = __fsub_rn(1.0f, t);
    r.w[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(-0.75f, x1), -3.75f), x1), -6.0f), x1), -3.0f);
    r.w[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, t), 2.25f), t), t), 1.0f);
    r.w[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, y), 2.25f), y), y), 1.0f);
    r.w[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.0f, r.w[0]), r.w[1]), r.w[2]);
    return r;
}

// The taps of the horizontally mirrored source (p[:, ::-1]): the flipped image's column i is the source's column n - 1 - i.
// The weights and the border flag stay those computed on the flipped image's own columns, so cubic_bgr8 with the mirrored
// taps equals the resize of the flipped image bit for bit.
__device__ __forceinline__ void mirror_taps(CubicTap& t, int n) {
#pragma unroll
    for (int k = 0; k < 4; ++k) t.i[k] = n - 1 - t.i[k];
}

// The resized, mean-subtracted pixel (y, x) of a dense uint8 (h0, w0, 3) image resized to W columns: out[c], c = B, G, R.
// Each tap's pixel is float(double(u8) - mean_c), the reference's in-place float32 mean subtraction before its resize.
// Horizontal pass: ((p0 + p1) + p2) + p3 per source row (0.0f + p0 first on a border column).  Vertical pass: OpenCV sums
// a row's first 4 * floor(3W / 4) floats in its 4-lane vector loop as ((q3 + q2) + q1) + q0 and the rest in scalar code as
// ((q0 + q1) + q2) + q3; element 3x + c follows the rule of its position.  The result is not clamped.
__device__ __forceinline__ void cubic_bgr8(const unsigned char* src, int w0, const CubicTap& ty, const CubicTap& tx, int x, int W,
                                           double m0, double m1, double m2, float out[3]) {
    const double mean[3] = {m0, m1, m2};
    const int vec_end = (3 * W) & ~3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float q[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const unsigned char* row = src + (long)ty.i[k] * w0 * 3 + c;
            float h = __fmul_rn((float)((double)row[tx.i[0] * 3] - mean[c]), tx.w[0]);
            if (tx.border) h = __fadd_rn(0.0f, h);
#pragma unroll
            for (int j = 1; j < 4; ++j) h = __fadd_rn(h, __fmul_rn((float)((double)row[tx.i[j] * 3] - mean[c]), tx.w[j]));
            q[k] = __fmul_rn(h, ty.w[k]);
        }
        out[c] = 3 * x + c < vec_end ? __fadd_rn(__fadd_rn(__fadd_rn(q[3], q[2]), q[1]), q[0])
                                     : __fadd_rn(__fadd_rn(__fadd_rn(q[0], q[1]), q[2]), q[3]);
    }
}

// Slot n of a raw-photo canvas batch, as the kernels may use it.  Its source is the dense uint8 (h0, w0, 3) block at
// arena + src_off[n]; the slot is live only when that block has a positive size and lies inside [0, arena_bytes)
// (64-bit arithmetic).  A slot that is not live is empty: extent 0 x 0, and src is the arena itself, never read.  The
// extent (the resized H, W) is clamped to the Hc x Wc slot, and bilinear_tap / cubic_tap keep every source index inside h0 x w0
// whatever inv_scale holds, so no descriptor value moves an access outside the arena or the slot.
struct RawSlot { const unsigned char* src; int h0, w0, eh, ew; double inv_scale; };
__device__ __forceinline__ RawSlot raw_slot(const unsigned char* arena, long long arena_bytes, const long long* src_off,
                                            const int* src_hw, const double* inv_scale, const int* extents, int n, int Hc,
                                            int Wc) {
    RawSlot s;
    s.h0 = __ldg(src_hw + 2 * n);
    s.w0 = __ldg(src_hw + 2 * n + 1);
    const long long off = __ldg(src_off + n);
    const bool live = s.h0 > 0 && s.w0 > 0 && off >= 0 && off <= arena_bytes && (long long)s.h0 * s.w0 <= (arena_bytes - off) / 3;
    s.src = live ? arena + off : arena;
    s.eh = live ? canvas_extent(extents, n, 0, 0, Hc) : 0;
    s.ew = live ? canvas_extent(extents, n, 1, 0, Wc) : 0;
    s.inv_scale = __ldg(inv_scale + n);
    return s;
}

// The augmentation draw of a training slot whose step seed is `seed` (frcnn_voc_augment_batch): the flip is the top bit of
// sample_key(seed ^ mix64(3), 0), the index among S scale candidates ((sample_key(seed ^ mix64(3), 1) >> 32) * S) >> 32.
// Salt 3 sets it apart from the other draws of the same seed: the subsampling's keys (seed, seed ^ BG_SEED_XOR) and the
// dropout masks (seed ^ mix64(1), seed ^ mix64(2)).
constexpr unsigned long long AUG_SALT = 3;
__device__ __forceinline__ void aug_draw(unsigned long long seed, int S, int& flip, int& scale_index) {
    const unsigned long long s = seed ^ mix64(AUG_SALT);
    flip = (int)(sample_key(s, 0) >> 63);
    scale_index = (int)(((sample_key(s, 1) >> 32) * (unsigned long long)S) >> 32);
}

}  // namespace frcnn
