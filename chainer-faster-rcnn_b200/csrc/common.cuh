// common.cuh -- error plumbing and small device helpers shared by all kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/frcnn_b200.h"

namespace frcnn {

void set_error(const char* fmt, ...);

#define FRCNN_CUDA_OK(expr)                                                                          \
    do {                                                                                             \
        cudaError_t _e = (expr);                                                                     \
        if (_e != cudaSuccess) {                                                                     \
            ::frcnn::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return FRCNN_ERR_CUDA;                                                                   \
        }                                                                                            \
    } while (0)

#define FRCNN_REQUIRE(cond, ...)              \
    do {                                      \
        if (!(cond)) {                        \
            ::frcnn::set_error(__VA_ARGS__);  \
            return FRCNN_ERR_ARG;             \
        }                                     \
    } while (0)

#define FRCNN_LAUNCH_OK() FRCNN_CUDA_OK(cudaGetLastError())

// First statement of every entry point: drop a stale, non-sticky error that an EARLIER runtime call of this host thread
// (the framework's, another library's) may have left behind -- cudaGetLastError() after a <<<>>> launch reports the last
// error of the calling thread, whoever caused it.
#define FRCNN_ENTRY() ((void)cudaGetLastError())

// ------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  The forward path is a chain of ~35 dependent kernels; launched with the
// programmatic-stream-serialization attribute a kernel's CTAs may become resident while the previous kernel drains
// (its CTAs exit one by one), run their prologue (barrier init, tensor-map prefetch, argument setup)
// and then block in grid_dep_wait() until the previous grid has completed and its writes are visible.  EVERY kernel
// launched through launch_pdl() must call grid_dep_wait() before its first global-memory access.  Inside a stream
// capture the attribute becomes a programmatic edge of the CUDA graph.  frcnn_set_programmatic_launch(0) turns the
// attribute off for the calling thread (plain stream order; grid_dep_wait() is then a no-op).
bool pdl_enabled();

__device__ __forceinline__ void grid_dep_wait() {
#if defined(__CUDA_ARCH__)
    asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// launch without the attribute; the launch status comes back directly (no cudaGetLastError involved)
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_plain(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                       Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------
// Deterministic float32 exp: the same fixed sequence of correctly rounded IEEE-754 binary32
// operations as the oracle's specification (fma / mul / add / rint), so device results are
// bit-identical to the CPU oracle on every host.  Replaces xp.exp at models/bbox_transform.py:62-63
// and the exp inside F.softmax (models/region_proposal_network.py:119, models/faster_rcnn.py:178).
__device__ __forceinline__ float pow2i(int k) { return __uint_as_float((uint32_t)(k + 127) << 23); }

__device__ __forceinline__ float det_expf(float x) {
    if (x != x) return x;
    x = x > 88.8f ? 88.8f : x;
    x = x < -104.0f ? -104.0f : x;
    const float LOG2E = 1.44269504088896341f;
    const float LN2_HI = 0.693359375f;
    const float LN2_LO = -2.12194440e-4f;
    float n = rintf(__fmul_rn(x, LOG2E));
    float r = __fmaf_rn(n, -LN2_HI, x);
    r = __fmaf_rn(n, -LN2_LO, r);
    float p = 1.9875691500e-4f;
    p = __fmaf_rn(p, r, 1.3981999507e-3f);
    p = __fmaf_rn(p, r, 8.3334519073e-3f);
    p = __fmaf_rn(p, r, 4.1665795894e-2f);
    p = __fmaf_rn(p, r, 1.6666665459e-1f);
    p = __fmaf_rn(p, r, 5.0000001201e-1f);
    float r2 = __fmul_rn(r, r);
    p = __fmaf_rn(p, r2, r);
    p = __fadd_rn(p, 1.0f);
    int ni = (int)n;
    int h = ni / 2;
    return __fmul_rn(__fmul_rn(p, pow2i(h)), pow2i(ni - h));
}

// clip_boxes (models/bbox_transform.py:87-98): max(min(v, bound), 0) for one coordinate, the clip of every decode kernel.
// NumPy's minimum / maximum propagate NaN, CUDA's fminf / fmaxf return the other operand, so NaN is passed through
// explicitly: a NaN coordinate stays NaN, and its box then fails every min-size test and suppresses nothing, as in the
// oracle.
__device__ __forceinline__ float clip_coord(float v, float bound) {
    return v != v ? v : fmaxf(fminf(v, bound), 0.0f);
}

// bf16 hi/lo split of an fp32 value: v ~= hi + lo with 16 significant bits ("bf16x3" operands).
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(v);
    lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// The value a split pair stands for in RoI pooling: hi + lo, or hi itself when hi is +-inf or NaN (split_bf16 of +-inf
// leaves lo = NaN, and inf + NaN would turn an infinite feature into a NaN one).
__device__ __forceinline__ float pool_pair_value(float hi, float lo) { return isfinite(hi) ? __fadd_rn(hi, lo) : hi; }

// RoI-pooling bins, the one rule of the forward (roi_pool_col_kernel) and the backward (roi_pool_backward_kernel), restated
// by the oracle's orc_roi_pool and tests/backward_ref.py (DESIGN §2).  A RoI coordinate becomes roundf(coord * scale) in
// float32, converted to int32 with NaN -> 0 and saturation (cvt.rzi.s32.f32, as Chainer's GPU kernel converts it).  The
// extent, the bin bounds and the shift by the start are 64-bit integers, then clamped to [0, L]: no step overflows, and a
// RoI far larger than the map pools the whole map into its first bins.
__device__ __forceinline__ int roi_coord(float c, float scale) { return __float2int_rz(roundf(__fmul_rn(c, scale))); }

// [x, y) of bin i of P over the scaled RoI extent [s, e] along an axis of L pixels; empty when y <= x.
__device__ __forceinline__ int2 roi_bin(int s, int e, int P, int i, int L) {
    const long long ext = max((long long)e - s + 1, 1ll);
    const float b = __fdiv_rn(__ll2float_rn(ext), (float)P);
    const long long lo = (long long)floorf(__fmul_rn((float)i, b)) + s, hi = (long long)ceilf(__fmul_rn((float)(i + 1), b)) + s;
    return make_int2((int)min(max(lo, 0ll), (long long)L), (int)min(max(hi, 0ll), (long long)L));
}

// Canvas batches (the *_ext entries): image n of N sits at the top-left of its [Hc][Wc] slot and its true size is
// extents[2n] x extents[2n+1] (device memory, read at run time, so one captured graph serves any mix of sizes).  After
// `halvings` ceil-mode 2x2 pools the extent is ceil(e / 2^halvings) (repeated ceil-halving).  Every extent is clamped to
// [0, limit] (the canvas at that resolution): a bad extent can never move a read or write outside the buffers.
__device__ __forceinline__ int canvas_extent(const int* extents, int img, int axis, int halvings, int limit) {
    long long e = max(__ldg(extents + 2 * img + axis), 0);
    e = (e + (1ll << halvings) - 1) >> halvings;
    return (int)min(e, (long long)limit);
}

// The counter hash of device-side sampling (include/frcnn_b200.h, frcnn_anchor_targets mode 1): the anchor-target and
// proposal-target subsampling and the dropout masks all draw through this one key, so their rules cannot drift apart.
__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {       // splitmix64 finaliser
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// key(seed, i): the top 32 bits hash (seed, i), the low 32 bits are i, so keys are distinct and a hash tie goes to the
// lower index
__device__ __forceinline__ unsigned long long sample_key(unsigned long long seed, int i) {
    return (mix64(seed ^ ((unsigned long long)(unsigned)i * 0xD6E8FEB86659FD93ull)) & 0xFFFFFFFF00000000ull) | (unsigned)i;
}
constexpr unsigned long long BG_SEED_XOR = 0xA5A5A5A5DEADBEEFull;     // the negatives / background draw with seed ^ this

}  // namespace frcnn
