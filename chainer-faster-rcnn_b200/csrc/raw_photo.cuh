// raw_photo.cuh -- the resize of forward.py's img_preprocessing on raw uint8 BGR photos, and the descriptor rule of a
// canvas batch's raw-photo slots: the one statement of both for every kernel that reads raw photos (head_ops.cu:
// preprocess_bgr8_kernel, preprocess_bgr8_canvas_kernel; resnet_ops.cu: preprocess_bgr8_canvas_im2col_kernel).
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

// Slot n of a raw-photo canvas batch, as the kernels may use it.  Its source is the dense uint8 (h0, w0, 3) block at
// arena + src_off[n]; the slot is live only when that block has a positive size and lies inside [0, arena_bytes)
// (64-bit arithmetic).  A slot that is not live is empty: extent 0 x 0, and src is the arena itself, never read.  The
// extent (the resized H, W) is clamped to the Hc x Wc slot, and bilinear_tap keeps every source index inside h0 x w0
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

}  // namespace frcnn
