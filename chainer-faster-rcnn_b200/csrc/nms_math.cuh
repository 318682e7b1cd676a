// nms_math.cuh -- the arithmetic every NMS path shares: the score order, the "+1" box area, the exact IoU of
// models/cpu_nms.pyx, the product pre-test that decides most pairs without a division, and the float64 IoU of
// models/bbox.pyx used for the training targets.  The kernels differ in thread mapping, shared-memory layout, word
// width and greedy chain; the decision "box i suppresses box j" and the rank of a row are made here and nowhere else.
//
// All float arithmetic is one rounding per operation (explicit __f*_rn / __d*_rn intrinsics: no FMA contraction), in
// the reference's operation order, so every decision is bit-identical to the CPU oracle.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/frcnn_b200.h"

namespace frcnn {

// ------------------------------------------------------------------------------------------ score order
// The project's one score order (DESIGN §2): score descending; -0.0 equals +0.0; every NaN, whatever its sign and payload,
// ranks below every number, -inf included; equal scores go to the lower index.
//
// float_to_ordered maps a float to a uint32 key with larger float => larger key, -0.0 and +0.0 on the same key and every
// NaN on key 1, below -inf's 0x007FFFFF.  Key 0 is never produced: it marks filtered-out rows and padding, which therefore
// rank behind every real row.
__device__ __forceinline__ uint32_t float_to_ordered(float f) {
    if (f != f) return 1u;
    uint32_t b = __float_as_uint(f);
    if (b == 0x80000000u) b = 0u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// 1 if the row (key t, index q) comes before the row (key s, index r) in that order, else 0, without a branch: the oracle's
// orc_cmp_desc on keys.  Summed over all q, it is the rank of row r: a permutation of [0, n) since (key, index) pairs are
// unique.
__device__ __forceinline__ int ahead(uint32_t t, int q, uint32_t s, int r) {
    return (int)(t > s) | ((int)(t == s) & (int)(q < r));
}

// ------------------------------------------------------------------------------------------ float32 IoU (cpu_nms.pyx)
// models/cpu_nms.pyx:25: (x2 - x1 + 1) * (y2 - y1 + 1)
__device__ __forceinline__ float box_area(const float4 b) {
    return __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.0f), __fadd_rn(__fsub_rn(b.w, b.y), 1.0f));
}

// models/cpu_nms.pyx:58-65: intersection and union of the pair
__device__ __forceinline__ void inter_union(const float4 a, float area_a, const float4 b, float area_b, float& inter, float& uni) {
    const float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y), xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
    const float w = fmaxf(0.0f, __fadd_rn(__fsub_rn(xx2, xx1), 1.0f));
    const float h = fmaxf(0.0f, __fadd_rn(__fsub_rn(yy2, yy1), 1.0f));
    inter = __fmul_rn(w, h);
    uni = __fsub_rn(__fadd_rn(area_a, area_b), inter);
}

// models/cpu_nms.pyx:65, true float32 division
__device__ __forceinline__ float iou(const float4 a, float area_a, const float4 b, float area_b) {
    float inter, uni;
    inter_union(a, area_a, b, area_b, inter, uni);
    return __fdiv_rn(inter, uni);
}

// The compare: cpu_nms.pyx:66's `ovr >= thresh` with thresh a Python float (FRCNN_NMS_GE_DOUBLE), or nms_kernel.cu's
// float `>` (FRCNN_NMS_GT_FLOAT, the `_nms` entry point).
__device__ __forceinline__ bool suppresses(float ovr, double thr_d, float thr_f, int mode) {
    return mode == FRCNN_NMS_GE_DOUBLE ? ((double)ovr >= thr_d) : (ovr > thr_f);
}

// ------------------------------------------------------------------------------------------ product pre-test
// A division per pair is what the mask kernels cannot afford, and a branch per pair diverges the lanes of a warp (they work
// on different rows), so every pair first takes the same straight-line products test: with u = area_a + area_b - inter,
// "inter / u against thr" is certain whenever u > 0 and inter lies outside [thr*u*(1-1e-5), thr*u*(1+1e-5)], because the
// float roundings involved are < 1e-6 relative.  A disjoint pair has inter == 0 < lo*u.  Everything else -- within 1e-5 of
// the threshold, u <= 0 or NaN (degenerate boxes), and every pair when thr <= 1e-3 -- is only RECORDED as undecided, and
// resolve_undecided() takes it through iou() and suppresses() after the loop.  The band holds for both compare modes.
struct PreTest {
    float lo, hi;
    bool on;   // false: lo / hi are -inf / +inf
};

// thr <= 1e-3 (or NaN) turns the pre-test off: bounds of -inf / +inf leave every pair undecided.
__device__ __forceinline__ PreTest pretest_bounds(float thr_f) {
    const bool on = thr_f > 1e-3f;
    return {on ? thr_f * (1.0f - 1e-5f) : -INFINITY, on ? thr_f * (1.0f + 1e-5f) : INFINITY, on};
}

// sure = 1: the pair surely suppresses; und = 1: the products cannot say.  (sure = und = 0: surely not.)
__device__ __forceinline__ void pretest(float inter, float uni, const PreTest p, uint32_t& sure, uint32_t& und) {
    const bool pos = uni > 0.0f;
    const bool yes = pos && inter > p.hi * uni, no = pos && inter < p.lo * uni;     // a product into a compare cannot contract
    sure = yes;
    und = !(yes || no);
}

__device__ __forceinline__ int lowest_bit(uint32_t w) { return __ffs((int)w) - 1; }
__device__ __forceinline__ int lowest_bit(unsigned long long w) { return __ffsll((long long)w) - 1; }

// The exact decision for every undecided bit of a word (rare): bit k of the result is suppresses(iou_of(k)) where `und`
// has it, `sure`'s bit elsewhere.  Word = uint32_t for 16- or 32-column words, unsigned long long for 64.
template <typename Word, typename IouOf>
__device__ __forceinline__ Word resolve_undecided(Word sure, Word und, IouOf iou_of, double thr_d, float thr_f, int mode) {
    while (und != 0) {
        const int k = lowest_bit(und);
        und &= und - 1;
        sure = (sure & ~((Word)1 << k)) | ((Word)suppresses(iou_of(k), thr_d, thr_f, mode) << k);
    }
    return sure;
}

// Bit j of the result: row box `a` (area `area_a`) suppresses column box cbox[j], for the `live` columns j < 64 (the others
// are 0; cbox / carea entries of dead columns may hold anything).  The 64-pair loop is fully unrolled and branch-free, with
// compile-time bit positions in 32-bit halves (no 64-bit variable shift); only the undecided pairs are divided afterwards.
__device__ __forceinline__ unsigned long long suppress_word64(const float4 a, float area_a, const float4* cbox, const float* carea,
                                                              unsigned long long live, const PreTest p, double thr_d, float thr_f,
                                                              int mode) {
    uint32_t sure_w[2] = {0u, 0u}, und_w[2] = {0u, 0u};
#pragma unroll
    for (int j = 0; j < 64; ++j) {
        float inter, uni;
        inter_union(a, area_a, cbox[j], carea[j], inter, uni);
        uint32_t sure, und;
        pretest(inter, uni, p, sure, und);
        sure_w[j >> 5] |= sure << (j & 31);
        und_w[j >> 5] |= und << (j & 31);
    }
    const unsigned long long sure = ((unsigned long long)sure_w[0] | ((unsigned long long)sure_w[1] << 32)) & live;
    const unsigned long long und = ((unsigned long long)und_w[0] | ((unsigned long long)und_w[1] << 32)) & live;
    return resolve_undecided(sure, und, [&](int j) { return iou(a, area_a, cbox[j], carea[j]); }, thr_d, thr_f, mode);
}

// ------------------------------------------------------------------------------------------ float64 IoU (bbox.pyx)
// models/bbox.pyx:35-38: the query box's area, hoisted out of the box loop as the reference does
__device__ __forceinline__ double box_area_f64(double x1, double y1, double x2, double y2) {
    return __dmul_rn(__dadd_rn(__dsub_rn(x2, x1), 1.0), __dadd_rn(__dsub_rn(y2, y1), 1.0));
}

// models/bbox.pyx:39-55, same operation order: IoU of box b with query box q of area q_area; 0 when they do not overlap.
__device__ __forceinline__ double iou_f64(const double b[4], const double q[4], double q_area) {
    const double iw = __dadd_rn(__dsub_rn(fmin(b[2], q[2]), fmax(b[0], q[0])), 1.0);
    if (!(iw > 0.0)) return 0.0;
    const double ih = __dadd_rn(__dsub_rn(fmin(b[3], q[3]), fmax(b[1], q[1])), 1.0);
    if (!(ih > 0.0)) return 0.0;
    const double inter = __dmul_rn(iw, ih);
    return __ddiv_rn(inter, __dsub_rn(__dadd_rn(box_area_f64(b[0], b[1], b[2], b[3]), q_area), inter));
}

}  // namespace frcnn
