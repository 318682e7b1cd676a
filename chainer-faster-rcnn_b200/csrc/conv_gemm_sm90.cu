// conv_gemm_sm90.cu -- implicit-GEMM 3x3 / 1x1 convolution (and plain GEMM) on Hopper tensor cores:
// TMA -> swizzled shared memory -> wgmma (bf16 operands, fp32 accumulators in registers) -> epilogue with fused
// bias + ReLU (+ residual, + bf16 hi/lo split, + optional fused 2x2 ceil-mode max-pool) -> TMA tensor stores (bf16) or
// global stores (fp32, pooled bf16).
//
// Replaces, for the forward path: L.Convolution2D at the reference's models/vgg16.py:39-67 and
// models/region_proposal_network.py:53-57, L.Linear at models/faster_rcnn.py:33-36, and (fused)
// F.MaxPooling2D(2,2) at models/vgg16.py:43,48,55,62.
//
// Mapping (NHWC activations, tap-major K-major weights):
//   M = output pixels, tiled as TH x TW patches of 128 pixels;  N = output channels (BN per tile);
//   K = taps x Cin, walked as (tap, BK-channel block) "k-blocks".
//   The A operand of k-block (tap=(r,s), cb) is ONE 3-D TMA box {BK ch, TW, TH} of the input at
//   spatial offset (r-1, s-1): out-of-bounds rows/columns are zero-filled by the TMA unit, which
//   is exactly the conv's zero padding -- no im2col buffer, no halo handling in the kernel.
//   The box lands in smem as 128 rows x (2*BK) B, the canonical K-major swizzled wgmma tile.
//
// Kernel structure: persistent, one CTA per SM, three warpgroups:
//   warpgroup 0    : TMA producer (one elected lane of warp 0), smem ring with full/empty mbarriers
//   warpgroups 1-2 : MMA + epilogue; warpgroup c owns pixel rows 64c .. 64c+63 of the tile (m64nBNk16 wgmma) and
//                    keeps its accumulators in registers.  The producer runs ahead into the next tile while they
//                    finish the epilogue of the current one.
//
// "bf16x3" mode (lo planes present): per k-block the stage holds A_hi, A_lo, B_hi, B_lo; A_hi*B_hi goes into the
// main accumulator and A_lo*B_hi + A_hi*B_lo into a separate correction accumulator (the tensor-core accumulator
// truncates on every add; see DESIGN.md 2), added once in the epilogue with a round-to-nearest fp32 add.
//
// Long K (PROMOTE): every acc_chunk k-blocks the main accumulator is added into a register total with round-to-nearest
// adds and restarted, so the truncation bias of the tensor-core sum grows with acc_chunk, not with K.
//
// Epilogue: per 32-channel chunk a warpgroup transposes its 64 x 32 fp32 fragment through shared memory so that a
// thread owns 16 consecutive channels of one pixel.  fp32 and fused-pool results are stored from registers; unpooled
// bf16 hi / lo results are staged in the same shared tile and leave as one TMA tensor store per plane (the map clips what
// lies outside the output).  The issuing thread only waits for a store to have read the tile before the next chunk
// reuses it, so the global writes drain behind the next tile's main loop; they are waited for once, before the CTA exits.
#include <cuda.h>
#include <stdlib.h>

#include <mutex>

#include "common.cuh"
#include "sm90_ptx.cuh"

namespace frcnn {

// Division by a launch-constant divisor without the ~25-instruction software division the compiler emits for `x / p.field`
// (every role recomputes the tile coordinates once per tile).  Granlund-Montgomery round-up multiplier: exact for every
// 32-bit unsigned x and d >= 1.
struct FastDiv {
    uint32_t m, s1, s2, d;
};
__device__ __forceinline__ int fd_div(int x, const FastDiv& f) {
    const uint32_t q = __umulhi(f.m, (uint32_t)x);
    return (int)(((((uint32_t)x - q) >> f.s1) + q) >> f.s2);
}
static inline FastDiv make_fastdiv(int d_) {
    FastDiv f;
    const uint32_t d = d_ > 0 ? (uint32_t)d_ : 1u;
    uint32_t l = 0;
    while ((1ull << l) < d) ++l;                       // l = ceil(log2 d)
    f.m = (uint32_t)(((1ull << 32) * ((1ull << l) - d)) / d + 1);
    f.s1 = l < 1 ? l : 1;
    f.s2 = l - f.s1;
    f.d = d;
    return f;
}

struct ConvParams {
    int H, W, Cout;
    int taps, ksize, cin_blocks;
    int kw, pad_h, pad_w;                // tap -> (r, s) = (tap / kw, tap % kw); A box origin (w0 + s - pad_w, h0 + r - pad_h)
    int TH, TW, tiles_h, tiles_w, n_tiles, num_tiles;
    FastDiv fd_tiles_w, fd_n_tiles, fd_tiles_per_part;   // set by launch_conv() once the three divisors are final
    int num_stages, relu, pool;
    int acc_chunk;                       // PROMOTE: k-blocks per tensor-core partial sum
    int ld_f32, n_cover;
    int b_res;                           // 1 (per-tap path, one N tile, few k-blocks): ALL weight tiles are loaded once per CTA and stay
                                         // resident in shared memory; the ring then carries A tiles only (conv1_1: one 24 KB load per CTA)
    float* y_f32;
    __nv_bfloat16 *y_hi, *y_lo;          // bf16 outputs [H][W][Cout] (pooled: [ceil(H/2)][ceil(W/2)][Cout])
    const float* bias;
    const int* m_valid;
    const __nv_bfloat16 *res_hi, *res_lo;   // optional residual [H][W][Cout] (hi + lo) added before the ReLU (ResNet shortcut)
    // split-K GEMM mode (frcnn_gemm_nt_splitk): the tile space is n_parts x tiles_per_part, part = group * splits + split;
    // a split covers k-blocks [split*kb_per_split, ...) of kb_total; group g shifts the B operand's K coordinate by
    // (g/3-1)*g_row_stride and reads plane g%3 of B (the 3x3 taps of a padded pixel axis: a TMA box must start 16-B
    // aligned, so the +-1 column shifts are three pre-shifted planes); every part writes its own fp32 slab
    // y_f32 + part*part_stride.  n_parts == 1: an ordinary convolution.
    int n_parts, tiles_per_part, splits, kb_per_split, kb_total, g_row_stride;
    long part_stride;
    // batch: n_img images of one H x W shape, [n_img][H][W][C] (A through a 4-D tensor map {C, W, H, image} when n_img > 1).
    // Pixel tile mt is tile mt % img_tiles of image mt / img_tiles; each image keeps the one-image plan, and the fp32 output,
    // the residual and the pooled bf16 output are addressed in the tile's own image at img_pix (img_opix pooled) pixels per
    // image; the unpooled bf16 outputs are stored through a 4-D map.
    int n_img, img_tiles;
    FastDiv fd_img_tiles;
    long img_pix, img_opix;
    // canvas batch (frcnn_*_batch_ext): image n's true size at this layer's input resolution is canvas_extent(extents, n,
    // ., ext_halvings, H / W); every output pixel outside it is written as 0, the zero padding the next convolution reads.
    // NULL: every pixel of the H x W image is live.
    const int* extents;
    int ext_halvings;
};

// Pixel tile mt -> (image, first row, first column).  Past the last tile (odd count, CTA pairs) the row lies below the
// last image: loads read zeros and nothing is stored.
__device__ __forceinline__ void tile_origin(const ConvParams& p, int mt, int& img, int& h0, int& w0) {
    img = 0;
    if (p.n_img > 1) {
        img = min(fd_div(mt, p.fd_img_tiles), p.n_img - 1);
        mt -= img * p.img_tiles;
    }
    const int th_i = fd_div(mt, p.fd_tiles_w);
    h0 = th_i * p.TH;
    w0 = (mt - th_i * p.tiles_w) * p.TW;
}

constexpr int kNumThreads = 384;          // warpgroup 0 producer, warpgroups 1-2 MMA + epilogue
constexpr int kTileM = 128;
constexpr int kWgRows = 64;               // pixel rows per MMA warpgroup
constexpr int kScratchLd = 36;            // fp32 row pitch of the epilogue transpose tile (16-B aligned rows)
constexpr int kScratchBytes = 2 * kWgRows * kScratchLd * 4;
constexpr int kBarrierBytes = 512;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;    // 128 * 40 + 256 * 232 <= 64K registers

template <int BN, int BK>
struct Cfg {
    static constexpr int ROW_BYTES = BK * 2;
    static constexpr int A_BYTES = kTileM * ROW_BYTES;
    static constexpr int B_BYTES = BN * ROW_BYTES;
};

// split-K GEMM mode helpers (ConvParams::n_parts > 1); an ordinary convolution has one part covering everything
__device__ __forceinline__ int part_k0(const ConvParams& p, int part) {
    return p.n_parts > 1 ? (part % p.splits) * p.kb_per_split : 0;
}
__device__ __forceinline__ int part_kblocks(const ConvParams& p, int part, int num_kb) {
    if (p.n_parts <= 1) return num_kb;
    const int k0 = (part % p.splits) * p.kb_per_split;
    return min(p.kb_per_split, p.kb_total - k0);
}
__device__ __forceinline__ int part_b_shift(const ConvParams& p, int part) {
    if (p.n_parts <= 1 || p.g_row_stride == 0) return 0;
    return ((part / p.splits) / 3 - 1) * p.g_row_stride;       // multiple of 8 elements: TMA box starts stay 16-B aligned
}
__device__ __forceinline__ int part_b_plane(const ConvParams& p, int part) {
    return (p.n_parts > 1 && p.g_row_stride != 0) ? (part / p.splits) % 3 : -1;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b, float& ra, float& rb) {
    // returns packed (bf16(a), bf16(b)); ra/rb = residuals a - hi, b - hi (exact in fp32)
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    const uint32_t u = *reinterpret_cast<const uint32_t*>(&h);
    ra = a - __uint_as_float(u << 16);
    rb = b - __uint_as_float(u & 0xFFFF0000u);
    return u;
}

// Position of 16-byte unit j (0..3: channels 8j .. 8j+7 of a 32-channel chunk) of staged pixel `spix` in a warpgroup's
// bf16 staging plane: 64 B per pixel, in the 64-byte swizzle the output tensor maps use (16-byte unit index XOR bits 7-8
// of the offset); every plane starts on a 512-byte boundary.  A quarter-warp's eight consecutive pixels hit eight
// distinct bank groups.
__device__ __forceinline__ uint32_t stage_off(int spix, int j) {
    return (uint32_t)(spix * 64 + ((j ^ ((spix >> 1) & 3)) << 4));
}

// One 16-channel run of one pixel: bias, residual, ReLU, validity, the fp32 store and the bf16 hi / lo split.  Unpooled,
// the packed hi / lo values are returned in hv / lv for the TMA store (whose tensor map clips pixels outside the image)
// and the function returns true; with the fused 2x2 pool, one lane per window stores them here.
// (ext_h, ext_w): the image's extent (H, W without a canvas); pixels outside it are stored as 0.
__device__ __forceinline__ bool epilogue_run(const ConvParams& p, float (&v)[16], int part, int img, int h, int w, int n,
                                             int lane, int m_valid, int ext_h, int ext_w, uint4 (&hv)[2], uint4 (&lv)[2]) {
    const bool in_img = (h < p.H) && (w < p.W);
    const long ipix = (long)h * p.W + w;
    const long pix = img * p.img_pix + ipix;
    const bool live = in_img && h < ext_h && w < ext_w && ipix < m_valid;
    if (p.bias != nullptr) {                    // split-K partial sums carry no bias (the reduction adds it once)
        const float4* b4 = reinterpret_cast<const float4*>(p.bias + n);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 b = __ldg(b4 + j);
            v[4 * j + 0] += b.x;
            v[4 * j + 1] += b.y;
            v[4 * j + 2] += b.z;
            v[4 * j + 3] += b.w;
        }
    }
    if (p.res_hi != nullptr && in_img && n < p.Cout) {
        // residual add (h + shortcut) of a bottleneck block, fused ahead of the ReLU
        const long ro = pix * p.Cout + n;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const uint4 rh = __ldg(reinterpret_cast<const uint4*>(p.res_hi + ro) + q);
            const __nv_bfloat16* hb = reinterpret_cast<const __nv_bfloat16*>(&rh);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[8 * q + j] += __bfloat162float(hb[j]);
            if (p.res_lo != nullptr) {
                const uint4 rl = __ldg(reinterpret_cast<const uint4*>(p.res_lo + ro) + q);
                const __nv_bfloat16* lb = reinterpret_cast<const __nv_bfloat16*>(&rl);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[8 * q + j] += __bfloat162float(lb[j]);
            }
        }
    }
    if (p.relu) {
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.0f);
    }
    if (!live) {
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = 0.0f;
    }
    if (in_img && p.y_f32 != nullptr && n < p.ld_f32) {
        float4* dst = reinterpret_cast<float4*>(p.y_f32 + (long)part * p.part_stride + pix * p.ld_f32 + n);
#pragma unroll
        for (int j = 0; j < 4; ++j) dst[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    }
    if (p.y_hi == nullptr || n >= p.Cout) return false;      // CTA-uniform condition
    bool writer = true;
    long opix = 0;
    if (p.pool) {
        // F.MaxPooling2D(2,2) ceil mode fused: the tile is 8 x 16 pixels and a warp holds two consecutive tile rows, so the
        // 2x2 window is lanes {l, l^1, l^16, l^17}.  Out-of-image pixels were zeroed above and every valid value is >= 0
        // (ReLU), so the max over the valid part of a partial window is unchanged (Chainer cover_all=True).
        const int tw_mask = p.TW;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            float m = fmaxf(v[j], __shfl_xor_sync(0xffffffffu, v[j], 1));
            v[j] = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, tw_mask));
        }
        writer = in_img && (lane & (1 | tw_mask)) == 0;
        opix = img * p.img_opix + (long)(h >> 1) * ((p.W + 1) >> 1) + (w >> 1);
    }
    if (writer) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            float ra[8], d0, d1;
            hv[q].x = pack_bf16x2(v[8 * q + 0], v[8 * q + 1], ra[0], ra[1]);
            hv[q].y = pack_bf16x2(v[8 * q + 2], v[8 * q + 3], ra[2], ra[3]);
            hv[q].z = pack_bf16x2(v[8 * q + 4], v[8 * q + 5], ra[4], ra[5]);
            hv[q].w = pack_bf16x2(v[8 * q + 6], v[8 * q + 7], ra[6], ra[7]);
            lv[q].x = pack_bf16x2(ra[0], ra[1], d0, d1);
            lv[q].y = pack_bf16x2(ra[2], ra[3], d0, d1);
            lv[q].z = pack_bf16x2(ra[4], ra[5], d0, d1);
            lv[q].w = pack_bf16x2(ra[6], ra[7], d0, d1);
        }
    }
    if (!p.pool) return true;
    // a pooled chunk is 16 pixels per warpgroup, written by a quarter of the threads: direct stores cost less here than
    // staging them for a TMA store (two more warpgroup barriers per chunk)
    if (writer) {
        uint4* dh = reinterpret_cast<uint4*>(p.y_hi + opix * p.Cout + n);
        dh[0] = hv[0];
        dh[1] = hv[1];
        if (p.y_lo != nullptr) {
            uint4* dl = reinterpret_cast<uint4*>(p.y_lo + opix * p.Cout + n);
            dl[0] = lv[0];
            dl[1] = lv[1];
        }
    }
    return false;
}

template <int BN, int BK, bool X3, bool PROMOTE, int CG>
__global__ void __launch_bounds__(kNumThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                 const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                 const __grid_constant__ CUtensorMap tm_y_hi, const __grid_constant__ CUtensorMap tm_y_lo,
                 const ConvParams p) {
    using C = Cfg<BN, BK>;
    constexpr int NACC = BN / 2;           // fp32 accumulator registers per thread of an m64nBN fragment
    extern __shared__ uint8_t smem_raw[];
    // 1024-B alignment required by SWIZZLE_128B tiles.
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

    // [resident weight tiles][ring of S stages][epilogue transpose tiles][barriers]
    constexpr int planes = X3 ? 2 : 1;
    const bool bres = p.b_res != 0;
    const int bres_bytes = bres ? p.taps * p.cin_blocks * planes * C::B_BYTES : 0;       // resident weight tiles, k-block major
    const int stage_bytes = bres ? planes * C::A_BYTES : planes * (C::A_BYTES + C::B_BYTES);
    const int a_lo_off = bres ? C::A_BYTES : C::A_BYTES + C::B_BYTES;                     // A_lo inside a stage
    const int S = p.num_stages;
    uint8_t* bres_base = smem;
    uint8_t* ring = bres_base + bres_bytes;
    float* scratch = reinterpret_cast<float*>(ring + (size_t)S * stage_bytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(scratch) + kScratchBytes);
    uint64_t* full_bar = bars;            // [S]
    uint64_t* empty_bar = bars + S;       // [S]
    uint64_t* bres_bar = bars + 2 * S;    // [1]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    // CG = 2: a cluster of two CTAs works on two neighbouring pixel tiles of the same N tile; each CTA loads half of the
    // weight tile and multicasts it into both, so a stage is refilled only when the MMA warps of BOTH CTAs released it
    const uint32_t rank = CG == 2 ? ptx::cluster_ctarank() : 0u;
    const int tile0 = CG == 2 ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
    const int tile_step = CG == 2 ? (int)(gridDim.x >> 1) : (int)gridDim.x;

    if (warp == 0 && lane == 0) {
        ptx::prefetch_tensormap(&tm_a_hi);
        ptx::prefetch_tensormap(&tm_b_hi);
        if (X3) {
            ptx::prefetch_tensormap(&tm_a_lo);
            ptx::prefetch_tensormap(&tm_b_lo);
        }
        if (p.y_hi != nullptr && !p.pool) ptx::prefetch_tensormap(&tm_y_hi);
        if (p.y_lo != nullptr && !p.pool) ptx::prefetch_tensormap(&tm_y_lo);
        for (int i = 0; i < S; ++i) {
            ptx::mbar_init(&full_bar[i], 1);
            ptx::mbar_init(&empty_bar[i], 8 * CG);     // one arrive per MMA warp of every CTA that reads the stage
        }
        ptx::mbar_init(bres_bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();
    if constexpr (CG == 2) ptx::cluster_sync();      // the peer's barriers are initialised before any multicast / remote arrive
    // programmatic dependent launch: everything above overlapped the previous kernel's drain; from here on this kernel
    // reads the previous kernel's output (TMA loads, residual, m_valid) and overwrites buffers it may still be reading
    grid_dep_wait();

    const int num_kb = p.taps * p.cin_blocks;

    if (wg == 0) {
        // ================================ TMA producer ================================
        ptx::setmaxnreg_dec<kProducerRegs>();
        if (warp == 0 && ptx::elect_one()) {
            // the weight tile: one TMA box, or (CG = 2) this CTA's half of it, multicast to the same offset in both CTAs
            auto load_b = [&](uint8_t* dst, const CUtensorMap* tm, uint64_t* bar, int k, int n, int plane) {
                if constexpr (CG == 2) {
                    constexpr int half = BN / 2;
                    ptx::tma_load_3d_multicast(dst + rank * half * C::ROW_BYTES, tm, bar, k, n + (int)rank * half, plane, 0x3);
                } else {
                    ptx::tma_load_3d(dst, tm, bar, k, n, plane);
                }
            };
            int stage = 0;
            uint32_t phase = 0;
            if (bres) {                  // one N tile: every weight tile of the layer, once, for all of this CTA's pixel tiles
                ptx::mbar_arrive_expect_tx(bres_bar, (uint32_t)bres_bytes);
                for (int kb = 0; kb < num_kb; ++kb) {
                    const int tap = kb / p.cin_blocks, cb = kb - tap * p.cin_blocks;
                    uint8_t* sb = bres_base + (size_t)kb * planes * C::B_BYTES;
                    ptx::tma_load_3d(sb, &tm_b_hi, bres_bar, cb * BK, 0, tap);
                    if (X3) ptx::tma_load_3d(sb + C::B_BYTES, &tm_b_lo, bres_bar, cb * BK, 0, tap);
                }
            }
            for (int tile = tile0; tile < p.num_tiles; tile += tile_step) {
                const int part = fd_div(tile, p.fd_tiles_per_part), t2 = tile - part * p.tiles_per_part;
                const int mq = fd_div(t2, p.fd_n_tiles), nt = t2 - mq * p.n_tiles;
                const int mt = mq * CG + (int)rank;      // past the last pixel tile (odd count): loads zeros, stores nothing
                int img, h0, w0;
                tile_origin(p, mt, img, h0, w0);
                const int n0 = nt * BN;
                // one image: the 3-D map; a batch: the 4-D map, whose out-of-bounds fill pads every image on its own
                auto load_a = [&](uint8_t* dst, const CUtensorMap* tm, uint64_t* bar, int k, int w, int h) {
                    if (p.n_img > 1) ptx::tma_load_4d(dst, tm, bar, k, w, h, img);
                    else ptx::tma_load_3d(dst, tm, bar, k, w, h);
                };
                const int nkb = part_kblocks(p, part, num_kb);
                const int ka = part_k0(p, part) * BK, kboff = ka + part_b_shift(p, part);
                const int bplane = part_b_plane(p, part);
                for (int kb = 0; kb < nkb; ++kb) {
                    const int tap = kb / p.cin_blocks;
                    const int btap = bplane >= 0 ? bplane : tap;
                    const int cb = kb - tap * p.cin_blocks;
                    const int r = tap / p.kw, s = tap - r * p.kw;
                    if constexpr (CG == 2) ptx::mbar_wait_cluster(&empty_bar[stage], phase ^ 1);
                    else ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* st = ring + (size_t)stage * stage_bytes;
                    ptx::mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)stage_bytes);
                    load_a(st, &tm_a_hi, &full_bar[stage], ka + cb * BK, w0 + s - p.pad_w, h0 + r - p.pad_h);
                    if (!bres) load_b(st + C::A_BYTES, &tm_b_hi, &full_bar[stage], kboff + cb * BK, n0, btap);
                    if (X3) {
                        uint8_t* st2 = st + a_lo_off;
                        load_a(st2, &tm_a_lo, &full_bar[stage], ka + cb * BK, w0 + s - p.pad_w, h0 + r - p.pad_h);
                        if (!bres) load_b(st2 + C::A_BYTES, &tm_b_lo, &full_bar[stage], kboff + cb * BK, n0, btap);
                    }
                    if (++stage == S) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ================================ MMA + epilogue ================================
        ptx::setmaxnreg_inc<kConsumerRegs>();
        const int c = wg - 1;                    // rows 64c .. 64c+63 of every tile
        const int t = threadIdx.x - 128 * wg;    // thread within the warpgroup
        const int wq = t >> 5;                   // warp within the warpgroup
        float* scr = scratch + c * kWgRows * kScratchLd;
        // transposed ownership in the epilogue: pixel row er of this warpgroup, channels 16*eh .. 16*eh+15 of each 32-chunk
        const int er = t & 63, eh = t >> 6;
        const int row = c * kWgRows + er;
        const int row_h = row / p.TW, row_w = row - row_h * p.TW;
        // unpooled bf16 outputs leave through TMA tensor stores of the warpgroup's 64 pixels, a box of its 64 / TW whole tile
        // rows (TW = 128: half a row); the 32-channel hi and lo planes of a chunk are staged in the transpose tile (2 x 4 KB)
        uint8_t* stg = reinterpret_cast<uint8_t*>(scr);
        const int box_dw = (kWgRows * c) % p.TW, box_dh = (kWgRows * c) / p.TW;
        const int m_valid = p.m_valid ? *p.m_valid : 0x7fffffff;
        const uint32_t a_off = (uint32_t)(c * kWgRows * C::ROW_BYTES);     // this warpgroup's 64 rows of the A tile
        float acc[NACC];
        float corr[X3 ? NACC : 1];
        float tot[PROMOTE ? NACC : 1];
        int stage = 0;
        uint32_t phase = 0;
        // a stage is free for the producer(s) once this warp's MMAs on it have retired: tell every CTA that loaded into it
        auto release = [&](int st) {
            if constexpr (CG == 2) {
                ptx::mbar_arrive_cluster(&empty_bar[st], 0);
                ptx::mbar_arrive_cluster(&empty_bar[st], 1);
            } else {
                ptx::mbar_arrive(&empty_bar[st]);
            }
        };
        if (bres) ptx::mbar_wait(bres_bar, 0);   // the resident weight tiles have landed
        for (int tile = tile0; tile < p.num_tiles; tile += tile_step) {
            const int part = fd_div(tile, p.fd_tiles_per_part), t2 = tile - part * p.tiles_per_part;
            const int mq = fd_div(t2, p.fd_n_tiles), nt = t2 - mq * p.n_tiles;
            const int mt = mq * CG + (int)rank;
            int img, h0, w0;
            tile_origin(p, mt, img, h0, w0);
            const int n0 = nt * BN;
            const int nkb = part_kblocks(p, part, num_kb);
            const int ext_h = p.extents ? canvas_extent(p.extents, img, 0, p.ext_halvings, p.H) : p.H;
            const int ext_w = p.extents ? canvas_extent(p.extents, img, 1, p.ext_halvings, p.W) : p.W;
    #pragma unroll
            for (int i = 0; i < NACC; ++i) {
                acc[i] = 0.0f;
                if constexpr (X3) corr[i] = 0.0f;
                if constexpr (PROMOTE) tot[i] = 0.0f;
            }
            int prev = -1;                       // stage whose wgmma group may still be reading it
            for (int kb = 0; kb < nkb; ++kb) {
                ptx::mbar_wait(&full_bar[stage], phase);
                const uint32_t st = ptx::smem_u32(ring + (size_t)stage * stage_bytes);
                const uint32_t sbw = bres ? ptx::smem_u32(bres_base + (size_t)kb * planes * C::B_BYTES) : st + C::A_BYTES;
                const uint64_t a_hi = ptx::make_smem_desc(st + a_off, C::ROW_BYTES);
                const uint64_t b_hi = ptx::make_smem_desc(sbw, C::ROW_BYTES);
                const bool fresh = PROMOTE ? (kb % p.acc_chunk == 0) : (kb == 0);
                ptx::fence_operand(acc);
                ptx::wgmma_fence();
    #pragma unroll
                for (int k = 0; k < BK / 16; ++k)      // advance 16 elements (32 B) along K inside the swizzle span: +2 in (addr>>4)
                    ptx::wgmma_bf16(acc, a_hi + 2 * k, b_hi + 2 * k, (fresh && k == 0) ? 0u : 1u);
                if constexpr (X3) {
                    const uint64_t a_lo = ptx::make_smem_desc(st + a_lo_off + a_off, C::ROW_BYTES);
                    const uint64_t b_lo = ptx::make_smem_desc(bres ? sbw + C::B_BYTES : st + a_lo_off + C::A_BYTES, C::ROW_BYTES);
    #pragma unroll
                    for (int k = 0; k < BK / 16; ++k) ptx::wgmma_bf16(corr, a_lo + 2 * k, b_hi + 2 * k, 1u);
    #pragma unroll
                    for (int k = 0; k < BK / 16; ++k) ptx::wgmma_bf16(corr, a_hi + 2 * k, b_lo + 2 * k, 1u);
                }
                ptx::wgmma_commit();
                const bool promote_now = PROMOTE && (kb % p.acc_chunk == p.acc_chunk - 1 || kb == nkb - 1);
                if (promote_now) {
                    ptx::wgmma_wait<0>();
                    ptx::fence_operand(acc);
                    if constexpr (PROMOTE) {
    #pragma unroll
                        for (int i = 0; i < NACC; ++i) tot[i] = __fadd_rn(tot[i], acc[i]);
                    }
                    if (lane == 0) {
                        if (prev >= 0) release(prev);
                        release(stage);
                    }
                    prev = -1;
                } else {
                    ptx::wgmma_wait<1>();            // the previous k-block's MMAs are done: its stage may be refilled
                    if (prev >= 0 && lane == 0) release(prev);
                    prev = stage;
                }
                if (++stage == S) { stage = 0; phase ^= 1; }
            }
            ptx::wgmma_wait<0>();
            ptx::fence_operand(acc);
            if constexpr (X3) ptx::fence_operand(corr);
            if (prev >= 0 && lane == 0) release(prev);

    #pragma unroll
            for (int ch = 0; ch < BN / 32; ++ch) {
                if (n0 + ch * 32 >= p.n_cover) break;   // CTA-uniform: nothing is stored past the covered columns
                // the previous chunk's TMA stores have read the staging tile (their global writes may still be in flight)
                if (t == 0) ptx::bulk_wait_group_read0();
                ptx::named_bar_sync(1 + c, 128);       // ... and every thread has read the previous chunk's transpose tile
    #pragma unroll
                for (int i = 4 * ch; i < 4 * ch + 4; ++i) {
    #pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        float v0, v1;
                        if constexpr (PROMOTE) {
                            v0 = tot[4 * i + 2 * hh];
                            v1 = tot[4 * i + 2 * hh + 1];
                        } else {
                            v0 = acc[4 * i + 2 * hh];
                            v1 = acc[4 * i + 2 * hh + 1];
                        }
                        if constexpr (X3) {
                            // the ~2^-8-sized correction products, added with one round-to-nearest fp32 add
                            v0 += corr[4 * i + 2 * hh];
                            v1 += corr[4 * i + 2 * hh + 1];
                        }
                        const int r = 16 * wq + (lane >> 2) + 8 * hh, col = 8 * (i - 4 * ch) + 2 * (lane & 3);
                        *reinterpret_cast<float2*>(scr + r * kScratchLd + col) = make_float2(v0, v1);
                    }
                }
                ptx::named_bar_sync(1 + c, 128);
                float v[16];
    #pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 f = *reinterpret_cast<const float4*>(scr + er * kScratchLd + 16 * eh + 4 * q);
                    v[4 * q + 0] = f.x;
                    v[4 * q + 1] = f.y;
                    v[4 * q + 2] = f.z;
                    v[4 * q + 3] = f.w;
                }
                const int nc = n0 + ch * 32;
                uint4 hv[2], lv[2];
                if (epilogue_run(p, v, part, img, h0 + row_h, w0 + row_w, nc + 16 * eh, lane, m_valid, ext_h, ext_w, hv, lv)) {
                    // CTA-uniform: an unpooled bf16 chunk
                    ptx::named_bar_sync(1 + c, 128);       // every thread has read its transposed values: the tile is free
                    const uint32_t sh = ptx::smem_u32(stg);
                    ptx::st_shared_v4(sh + stage_off(er, 2 * eh), hv[0]);
                    ptx::st_shared_v4(sh + stage_off(er, 2 * eh + 1), hv[1]);
                    if (p.y_lo != nullptr) {
                        ptx::st_shared_v4(sh + 4096 + stage_off(er, 2 * eh), lv[0]);
                        ptx::st_shared_v4(sh + 4096 + stage_off(er, 2 * eh + 1), lv[1]);
                    }
                    ptx::fence_proxy_async_smem();
                    ptx::named_bar_sync(1 + c, 128);
                    if (t == 0) {
                        const int bw = w0 + box_dw, bh = h0 + box_dh;
                        if (p.n_img > 1) {
                            ptx::tma_store_4d(&tm_y_hi, stg, nc, bw, bh, img);
                            if (p.y_lo != nullptr) ptx::tma_store_4d(&tm_y_lo, stg + 4096, nc, bw, bh, img);
                        } else {
                            ptx::tma_store_3d(&tm_y_hi, stg, nc, bw, bh);
                            if (p.y_lo != nullptr) ptx::tma_store_3d(&tm_y_lo, stg + 4096, nc, bw, bh);
                        }
                        ptx::bulk_commit_group();
                    }
                }
            }
        }
        // no tile reads another tile's output, so the stores drain behind the following tiles' main loops; they must be
        // complete before the CTA exits (the staging tile stays valid until they have read it)
        if (t == 0) ptx::bulk_wait_group0();
    }
    if constexpr (CG == 2) ptx::cluster_sync();      // the peer may still multicast into our stages / arrive on our barriers
}

// ------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    // Resolved through the runtime so the library has no link-time dependency on libcuda.so
    // (it must dlopen on a CPU-only box for the symbol/ABI tests).
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

// 3-D bf16 tensor map: dims (innermost first) {d0,d1,d2}, row pitch d0 elements, box {b0,b1,b2};
// swizzle span = the box's inner extent in bytes (32 / 64 / 128).
// Encoded maps are cached per thread, keyed by (base, dims, box): an eager caller of frcnn_forward_vgg16 re-encodes
// nothing after its first image (six driver calls per conv launch otherwise); graph replay never comes here.
struct TmapKey {
    const void* base;
    uint64_t d0, d1, d2, d3, s3;
    uint32_t b0, b1, b2;
    bool operator==(const TmapKey& o) const {
        return base == o.base && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && d3 == o.d3 && s3 == o.s3 && b0 == o.b0 &&
               b1 == o.b1 && b2 == o.b2;
    }
};
constexpr int kTmapCacheSlots = 512;
struct TmapCache {
    TmapKey key[kTmapCacheSlots];
    CUtensorMap map[kTmapCacheSlots];
    bool used[kTmapCacheSlots];
};
static TmapCache* tmap_cache() {
    static thread_local TmapCache* c = nullptr;
    if (c == nullptr) c = new TmapCache();          // value-initialised: used[] all false
    return c;
}

static int make_tmap_3d(CUtensorMap* tm, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0,
                        uint32_t b1, uint32_t b2, uint64_t stride1_bytes = 0, uint64_t stride2_bytes = 0, uint64_t d3 = 0,
                        uint64_t stride3_bytes = 0) {
    // stride1_bytes / stride2_bytes != 0: explicit byte strides of dimensions 1 and 2 (a SLIDING-WINDOW map when stride1 is
    // smaller than the dimension-0 extent: neighbouring "rows" overlap in memory, tests/experiments/tma_overlap_probe.cu); the cache key folds them into d1 / d2's upper bits
    // d3 > 0: a 4-D map (a batch of d3 images, stride3_bytes apart, box extent 1 along it)
    const TmapKey key{base, d0, d1 | (stride1_bytes << 32), d2 | (stride2_bytes << 32), d3, stride3_bytes, b0, b1, b2};
    uint64_t hsh = reinterpret_cast<uintptr_t>(base) * 0x9E3779B97F4A7C15ull;
    hsh ^= (d0 * 31 + d1) * 0xC2B2AE3D27D4EB4Full + d2 * 0x165667B19E3779F9ull + b0 * 131 + b1 * 17 + b2 + d3 * 0x27D4EB2Full;
    const int slot = (int)((hsh >> 20) % kTmapCacheSlots);
    TmapCache* cache = tmap_cache();
    if (cache->used[slot] && cache->key[slot] == key) {
        *tm = cache->map[slot];
        return FRCNN_OK;
    }
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) {
        set_error("cuTensorMapEncodeTiled not available from the driver");
        return FRCNN_ERR_CUDA;
    }
    cuuint64_t dims[4] = {d0, d1, d2, d3};
    cuuint64_t strides[3] = {stride1_bytes ? stride1_bytes : d0 * 2, stride2_bytes ? stride2_bytes : d0 * d1 * 2,
                             stride3_bytes ? stride3_bytes : d0 * d1 * d2 * 2};
    cuuint32_t box[4] = {b0, b1, b2, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUtensorMapSwizzle sw = (b0 * 2 == 128) ? CU_TENSOR_MAP_SWIZZLE_128B
                                            : (b0 * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, d3 > 0 ? 4 : 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): dims {%llu,%llu,%llu} box {%u,%u,%u} base %p", (int)r,
                  (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, b0, b1, b2, base);
        return FRCNN_ERR_CUDA;
    }
    cache->key[slot] = key;
    cache->map[slot] = *tm;
    cache->used[slot] = true;
    return FRCNN_OK;
}

// Tuning overrides (frcnn_conv2d_set_*): per calling thread, read when a launch is enqueued (and therefore fixed inside
// a captured graph) -- two engines driven from different threads cannot disturb each other.
static int env_int(const char* name) {
    const char* v = getenv(name);
    return v ? atoi(v) : 0;
}
// FRCNN_CONV_MAX_CTAS: a process-wide default for frcnn_conv2d_set_max_ctas (each thread starts from it)
static thread_local int g_force_bn = 0, g_force_th = 0, g_force_tw = 0, g_force_cg = 0, g_max_ctas = env_int("FRCNN_CONV_MAX_CTAS"),
                        g_smem_reserve = 0;

static int device_sm_count() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    return sms;
}

// The plan of the calling thread's last conv / GEMM launch (frcnn_conv2d_last_plan), in the order
// BN, BK, x3, promote, CG, TH, TW, stages, grid, num_tiles, n_parts, splits.
constexpr int kPlanFields = 12;
static thread_local int g_last_plan[kPlanFields] = {};

// Bytes of one ring stage and of the stage-independent part of the dynamic shared memory (alignment slack, barriers, the
// epilogue's transpose tiles and, with resident weights, every weight tile of the layer).
static void conv_smem_layout(int BN, int BK, bool x3, int bres_kblocks, int* stage_bytes, int* fixed) {
    const int planes = x3 ? 2 : 1;
    const int a_bytes = kTileM * BK * 2, b_bytes = BN * BK * 2;
    *stage_bytes = bres_kblocks > 0 ? planes * a_bytes : planes * (a_bytes + b_bytes);
    *fixed = 1024 /*align slack*/ + kBarrierBytes + kScratchBytes + bres_kblocks * planes * b_bytes;
}

// Pipeline stages that fit the shared-memory budget (at most 20).  The budget is the whole SM by default;
// frcnn_conv2d_set_smem_reserve leaves a slice of every SM to other kernels, so that the small kernels of ANOTHER image in
// flight (decode, NMS, RoI pooling, a host caller's per-class NMS) can become resident next to a convolution instead of
// waiting for one of its CTAs to retire.
static int conv_stages(int BN, int BK, bool x3, int bres_kblocks) {
    int stage_bytes, fixed;
    conv_smem_layout(BN, BK, x3, bres_kblocks, &stage_bytes, &fixed);
    const int stages = (227 * 1024 - g_smem_reserve - fixed) / stage_bytes;
    return stages > 20 ? 20 : stages;
}

template <int BN, int BK, bool X3, bool PROMOTE, int CG>
static int launch_conv(const CUtensorMap* tm, ConvParams p, cudaStream_t stream) {
    p.fd_tiles_w = make_fastdiv(p.tiles_w);
    p.fd_n_tiles = make_fastdiv(p.n_tiles);
    p.fd_tiles_per_part = make_fastdiv(p.tiles_per_part);
    p.fd_img_tiles = make_fastdiv(p.img_tiles);
    const int bres_kblocks = p.b_res ? p.taps * p.cin_blocks : 0;
    int stage_bytes, fixed;
    conv_smem_layout(BN, BK, X3, bres_kblocks, &stage_bytes, &fixed);
    const int stages = conv_stages(BN, BK, X3, bres_kblocks);
    if (stages < 2) {
        set_error("conv tile BN=%d BK=%d x3=%d does not fit 2 pipeline stages", BN, BK, (int)X3);
        return FRCNN_ERR_ARG;
    }
    p.num_stages = stages;
    const size_t smem = (size_t)stages * stage_bytes + fixed;
    auto kern = conv_gemm_kernel<BN, BK, X3, PROMOTE, CG>;
    FRCNN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int ctas = device_sm_count();
    if (g_max_ctas > 0 && g_max_ctas < ctas) ctas = g_max_ctas;      // several images in flight: each launch takes a share of the SMs
    const int units = ctas / CG > 0 ? ctas / CG : 1;     // CTAs (CG = 1) or CTA pairs (CG = 2) resident at once
    const int grid = CG * (p.num_tiles < units ? p.num_tiles : units);
    const int plan[kPlanFields] = {BN, BK, X3 ? 1 : 0, PROMOTE ? 1 : 0, CG, p.TH, p.TW, stages, grid, p.num_tiles, p.n_parts,
                                   p.splits};
    for (int i = 0; i < kPlanFields; ++i) g_last_plan[i] = plan[i];
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kNumThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (CG == 2) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = 2;
        attr[na].val.clusterDim.y = 1;
        attr[na].val.clusterDim.z = 1;
        ++na;
    }
    if (pdl_enabled()) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    FRCNN_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], p));
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

}  // namespace frcnn

using namespace frcnn;

extern "C" void frcnn_conv2d_set_cta_group(int cta_group) { g_force_cg = cta_group; }

extern "C" void frcnn_conv2d_set_max_ctas(int max_ctas) { g_max_ctas = max_ctas; }

extern "C" void frcnn_conv2d_set_smem_reserve(int bytes) { g_smem_reserve = bytes < 0 ? 0 : (bytes > 96 * 1024 ? 96 * 1024 : bytes); }

extern "C" void frcnn_conv2d_set_tile(int block_n, int tile_h, int tile_w) {
    g_force_bn = block_n;
    g_force_th = tile_h;
    g_force_tw = tile_w;
}

extern "C" int frcnn_conv2d_last_plan(int* out, int n) {
    for (int i = 0; out != nullptr && i < n && i < kPlanFields; ++i) out[i] = g_last_plan[i];
    return kPlanFields;
}

namespace {
struct GemmExtra {          // split-K GEMM mode of the same kernel (frcnn_gemm_nt_splitk)
    int groups, row_stride, splits;
    long part_stride;
    int bn = 0;             // 0: the weight-gradient rule (128 / 64); else the N tile to use (64, 128, 256)
    int nacc = 1;           // > 1: long K, every split promotes its tensor-core partial sums into a register total
};
struct ResExtra {           // residual input of frcnn_conv2d_res
    const void *hi, *lo;
};
struct WinExtra {           // frcnn_conv3x3_c8: 3x3 convolution over a compact [H][W+2][8] image through a sliding-window map
    int row_pixels;         // pixels per stored row (W + 2: one zero column on each side)
    long image_elems;       // elements per image of a batch (frcnn_image_c8_elems)
};
}  // namespace

// n_img > 1: a batch of n_img images of the same shape, [n_img][H][W][C] (compact first layer: n_img planes of
// frcnn_image_c8_elems), every image planned, tiled and computed exactly as a one-image launch would.
static int conv2d_impl(const void* x_hi, const void* x_lo, int H, int W, int Cin, const void* w_hi,
                       const void* w_lo, const float* bias, int Cout, int ksize, int relu, int fuse_pool2x2,
                       void* y_hi, void* y_lo, float* y_f32, int ld_f32, const int* m_valid, void* stream_,
                       const GemmExtra* ge, const ResExtra* re = nullptr, const WinExtra* we = nullptr, int n_img = 1,
                       const int* extents = nullptr, int ext_halvings = 0) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    for (int& v : g_last_plan) v = 0;          // a call that launches nothing leaves an empty record
    FRCNN_REQUIRE(n_img >= 1 && (n_img == 1 || (!ge && !m_valid)), "frcnn_conv2d: bad batch of %d images", n_img);
    FRCNN_REQUIRE(!extents || (!ge && !m_valid && ext_halvings >= 0 && ext_halvings <= 30),
                  "frcnn_conv2d: extents need a plain convolution and 0 <= halvings <= 30 (got %d)", ext_halvings);
    FRCNN_REQUIRE(x_hi && w_hi && (bias || ge), "frcnn_conv2d: x_hi, w_hi and bias are required");
    FRCNN_REQUIRE((x_lo == nullptr) == (w_lo == nullptr), "frcnn_conv2d: x_lo and w_lo must both be given (bf16x3) or both NULL");
    FRCNN_REQUIRE(ksize == 1 || ksize == 3, "frcnn_conv2d: ksize must be 1 or 3 (got %d)", ksize);
    FRCNN_REQUIRE(H > 0 && W > 0 && Cin > 0 && Cout > 0, "frcnn_conv2d: bad shape H=%d W=%d Cin=%d Cout=%d", H, W, Cin, Cout);
    FRCNN_REQUIRE(Cin % 8 == 0, "frcnn_conv2d: Cin must be a multiple of 8 (16-byte TMA rows), got %d", Cin);
    FRCNN_REQUIRE(y_hi || y_f32, "frcnn_conv2d: no output requested");
    FRCNN_REQUIRE(!y_hi || Cout % 32 == 0, "frcnn_conv2d: bf16 output needs Cout %% 32 == 0 (got %d)", Cout);
    FRCNN_REQUIRE(!y_f32 || (ld_f32 % 32 == 0 && ld_f32 >= Cout), "frcnn_conv2d: ld_f32 must be a multiple of 32 and >= Cout");
    FRCNN_REQUIRE(!y_lo || y_hi, "frcnn_conv2d: y_lo without y_hi");
    FRCNN_REQUIRE(!fuse_pool2x2 || (y_hi && relu && !y_f32 && !m_valid),
                  "frcnn_conv2d: fuse_pool2x2 needs a bf16 output, relu=1, no fp32 output and no m_valid");

    const int BK = (Cin >= 64) ? 64 : (Cin >= 32 ? 32 : 16);
    FRCNN_REQUIRE(BK != 32 || Cin == 32, "frcnn_conv2d: Cin in (32,64) is not supported (use 16, 32 or >= 64)");
    const bool x3 = x_lo != nullptr;

    // ---- pixel tile: minimise padded pixels (the fused pool needs the 8x16 tile: 2x2 windows inside a warp)
    static const int shapes[6][2] = {{8, 16}, {16, 8}, {4, 32}, {2, 64}, {1, 128}, {32, 4}};
    int TH = 8, TW = 16;
    const bool forced_tile = g_force_th > 0 && g_force_tw > 0 && g_force_th * g_force_tw == kTileM;
    if (fuse_pool2x2) {
        TH = 8;
        TW = 16;
    } else if (forced_tile) {
        TH = g_force_th;
        TW = g_force_tw;
    } else {
        long best = -1;
        for (auto& s : shapes) {
            long t = (long)cdiv(H, s[0]) * cdiv(W, s[1]);
            if (best < 0 || t < best) { best = t; TH = s[0]; TW = s[1]; }
        }
    }
    const int tiles_h = cdiv(H, TH), tiles_w = cdiv(W, TW);
    const long m_tiles = (long)tiles_h * tiles_w;

    // ---- long K: the tensor-core partial sum is restarted every 8 k-blocks and promoted into a register total
    const bool promote = (ge == nullptr && ksize * ksize * cdiv(Cin, BK) >= 256) || (ge != nullptr && ge->nacc > 1);
    // ---- N tile.  The accumulators live in the registers of the two MMA warpgroups: BN / 2 fp32 per thread for each of
    // the main, correction (bf16x3) and promoted (long K) sums, within the 232 registers a consumer thread gets
    const int bn_cap = promote ? (x3 ? 64 : 128) : (x3 ? 128 : 256);
    const int cout_cover = y_f32 ? (ld_f32 > Cout ? ld_f32 : Cout) : Cout;
    int BN = 0;
    if (g_force_bn == 64 || g_force_bn == 128 || g_force_bn == 256) {
        BN = g_force_bn;
    } else if (ge != nullptr && ge->bn != 0) {
        BN = ge->bn;
    } else if (ge != nullptr) {
        // split-K GEMM mode has tiles to spare (groups x splits): N = 128 halves the re-reads of A
        BN = cout_cover >= 128 ? 128 : 64;
    } else {
        // minimise waves x shared-memory fill per k-block (A tile + B tile bytes): the main loop streams both operands
        // from L2 for every k-block, so a wider N tile costs less per output channel but quantises into fewer tiles
        const int sms = device_sm_count();
        double best = 0;
        const int cand[3] = {256, 128, 64};
        for (int i = 0; i < 3; ++i) {
            if (cand[i] > bn_cap) continue;
            if (cand[i] > 64 && cand[i] > cout_cover && cand[i] / 2 >= cout_cover) continue;  // too wide
            const long tiles = m_tiles * cdiv(cout_cover, cand[i]);
            const double t = (double)cdiv((int)tiles, sms) * (kTileM + cand[i]);
            if (BN == 0 || t < best) { best = t; BN = cand[i]; }
        }
    }
    while (BN > bn_cap) BN /= 2;
    if (BN != 64 && BN != 128 && BN != 256) BN = 128;      // an N tile without a kernel (160): the nearest smaller one
    // a shared-memory reserve (frcnn_conv2d_set_smem_reserve) can leave less than two pipeline stages of a wide N tile
    // (bf16x3 BN = 128 above 81,408 B): narrow the tile until two fit; launch_conv reports the case where BN = 64 does not
    {
        const int kblocks = (we != nullptr ? 3 : ksize * ksize) * cdiv(Cin, BK);
        auto bres_kblocks = [&](int bn) {
            return (we != nullptr && cdiv(cout_cover, bn) == 1 && ge == nullptr && kblocks <= 16) ? kblocks : 0;
        };
        while (BN > 64 && conv_stages(BN, BK, x3, bres_kblocks(BN)) < 2) BN /= 2;
    }

    ConvParams p;
    p.H = H; p.W = W; p.Cout = Cout;
    p.ksize = ksize; p.taps = ksize * ksize; p.cin_blocks = cdiv(Cin, BK);
    p.kw = ksize; p.pad_h = p.pad_w = (ksize - 1) / 2;
    if (we != nullptr) {
        // K = 3 image rows x (4 pixels x 8 channels): one k-block of 32 per row r, its A box starting at stored pixel w0 of row
        // h0 + r - 1 (the left zero column is stored, rows -1 and H are the TMA unit's out-of-bounds zero fill)
        FRCNN_REQUIRE(Cin == 32 && ksize == 3 && !fuse_pool2x2 && !m_valid && !ge && !re, "conv3x3_c8: bad configuration");
        p.taps = 3; p.kw = 1; p.pad_h = 1; p.pad_w = 0;
    }
    p.TH = TH; p.TW = TW; p.tiles_h = tiles_h; p.tiles_w = tiles_w;
    p.n_tiles = cdiv(cout_cover, BN);
    // CTA pairs (a cluster of 2 sharing each weight tile through TMA multicast) only on request: on an H100 the pair's
    // lockstep over one stage ring made the whole 600x1000 forward 1.9x slower than single CTAs (5.55 vs 2.96 ms / image)
    const int CG = (g_force_cg == 2 && BK == 64 && we == nullptr) ? 2 : 1;
    FRCNN_REQUIRE(n_img * m_tiles * p.n_tiles < (1l << 30), "frcnn_conv2d: too many tiles");
    // a batch only multiplies the pixel tiles: the tile shape and N tile above are the one-image plan
    p.n_img = n_img;
    p.img_tiles = (int)m_tiles;
    p.img_pix = (long)H * W;
    p.img_opix = (long)((H + 1) / 2) * ((W + 1) / 2);
    p.num_tiles = (int)(cdiv((int)(n_img * m_tiles), CG) * p.n_tiles);     // tiles (CG = 1) or pair-tiles (CG = 2)
    p.tiles_per_part = p.num_tiles;
    p.n_parts = 1; p.splits = 1; p.kb_per_split = p.kb_total = p.taps * p.cin_blocks; p.g_row_stride = 0; p.part_stride = 0;
    if (ge != nullptr) {
        FRCNN_REQUIRE(ksize == 1 && BK == 64 && Cin % 64 == 0 && y_f32 && !y_hi && !m_valid, "gemm_nt_splitk: bad configuration");
        p.kb_total = p.cin_blocks;
        p.kb_per_split = cdiv(p.kb_total, ge->splits);
        p.splits = cdiv(p.kb_total, p.kb_per_split);             // every split non-empty
        p.n_parts = ge->groups * p.splits;
        p.g_row_stride = ge->groups == 9 ? ge->row_stride : 0;
        FRCNN_REQUIRE(ge->groups == 1 || (ge->row_stride > 0 && ge->row_stride % 8 == 0),
                      "gemm_nt_splitk: row_stride must be a positive multiple of 8 (16-byte aligned TMA box starts)");
        p.part_stride = ge->part_stride;
        FRCNN_REQUIRE((long)p.num_tiles * p.n_parts < (1l << 30), "gemm_nt_splitk: too many tiles");
        p.num_tiles *= p.n_parts;
    }
    p.num_stages = 0;
    p.acc_chunk = 8;
    p.relu = relu;
    p.pool = fuse_pool2x2 ? 1 : 0;
    p.ld_f32 = ld_f32;
    p.n_cover = cdiv(cout_cover, 32) * 32;
    p.y_hi = static_cast<__nv_bfloat16*>(y_hi);
    p.y_lo = static_cast<__nv_bfloat16*>(y_lo);
    // resident weights: the compact first layer (3 k-blocks, one N tile): fetched once per CTA instead of once per tile
    p.b_res = (we != nullptr && p.n_tiles == 1 && ge == nullptr && p.taps * p.cin_blocks <= 16) ? 1 : 0;
    p.y_f32 = y_f32;
    p.bias = bias;
    p.m_valid = m_valid;
    p.res_hi = re ? (const __nv_bfloat16*)re->hi : nullptr;
    p.res_lo = re ? (const __nv_bfloat16*)re->lo : nullptr;
    p.extents = extents;
    p.ext_halvings = ext_halvings;
    FRCNN_REQUIRE(!re || (re->hi && !fuse_pool2x2 && Cout % 32 == 0), "frcnn_conv2d_res: residual needs res_hi, Cout %% 32 == 0 and no fused pool");

    CUtensorMap tm[6];      // A hi / lo, B hi / lo, bf16 output hi / lo
    int rc;
    const uint64_t as1 = we ? 16 : 0, as2 = we ? (uint64_t)we->row_pixels * 16 : 0;     // sliding window: one pixel (8 ch) per step
    const uint64_t an = n_img > 1 ? n_img : 0, as3 = (n_img > 1 && we) ? (uint64_t)we->image_elems * 2 : 0;
    if ((rc = make_tmap_3d(&tm[0], x_hi, Cin, W, H, BK, TW, TH, as1, as2, an, as3)) != FRCNN_OK) return rc;
    const int b_planes = (ge != nullptr && ge->groups == 9) ? 3 : p.taps;
    if ((rc = make_tmap_3d(&tm[2], w_hi, Cin, Cout, b_planes, BK, BN / CG, 1)) != FRCNN_OK) return rc;
    if (x3) {
        if ((rc = make_tmap_3d(&tm[1], x_lo, Cin, W, H, BK, TW, TH, as1, as2, an, as3)) != FRCNN_OK) return rc;
        if ((rc = make_tmap_3d(&tm[3], w_lo, Cin, Cout, b_planes, BK, BN / CG, 1)) != FRCNN_OK) return rc;
    } else {
        tm[1] = tm[0];
        tm[3] = tm[2];
    }
    // unpooled bf16 outputs: one TMA store box per MMA warpgroup and 32-channel chunk (its 64 pixels); the map clips the
    // rows, columns and channels outside the output.  A batch stores through a 4-D map {C, W, H, image}.
    tm[4] = tm[0];
    tm[5] = tm[0];
    if (y_hi != nullptr && !fuse_pool2x2) {
        const uint32_t bw = TW < kWgRows ? TW : kWgRows, bh = TW < kWgRows ? kWgRows / TW : 1;
        if ((rc = make_tmap_3d(&tm[4], y_hi, Cout, W, H, 32, bw, bh, 0, 0, an)) != FRCNN_OK) return rc;
        if (y_lo != nullptr && (rc = make_tmap_3d(&tm[5], y_lo, Cout, W, H, 32, bw, bh, 0, 0, an)) != FRCNN_OK) return rc;
    }

#define FRCNN_DISPATCH(BN_, BK_, X3_, PROMOTE_, CG_) \
    if (BN == BN_ && BK == BK_ && x3 == X3_ && promote == PROMOTE_ && CG == CG_) \
        return launch_conv<BN_, BK_, X3_, PROMOTE_, CG_>(tm, p, stream);
    FRCNN_DISPATCH(256, 64, false, false, 1)
    FRCNN_DISPATCH(256, 64, false, false, 2)
    FRCNN_DISPATCH(128, 64, false, false, 1)
    FRCNN_DISPATCH(128, 64, false, false, 2)
    FRCNN_DISPATCH(64, 64, false, false, 1)
    FRCNN_DISPATCH(64, 64, false, false, 2)
    FRCNN_DISPATCH(128, 64, true, false, 1)
    FRCNN_DISPATCH(128, 64, true, false, 2)
    FRCNN_DISPATCH(64, 64, true, false, 1)
    FRCNN_DISPATCH(64, 64, true, false, 2)
    FRCNN_DISPATCH(128, 64, false, true, 1)
    FRCNN_DISPATCH(128, 64, false, true, 2)
    FRCNN_DISPATCH(64, 64, false, true, 1)
    FRCNN_DISPATCH(64, 64, false, true, 2)
    FRCNN_DISPATCH(64, 64, true, true, 1)
    FRCNN_DISPATCH(64, 64, true, true, 2)
    FRCNN_DISPATCH(128, 32, false, false, 1)
    FRCNN_DISPATCH(64, 32, false, false, 1)
    FRCNN_DISPATCH(128, 32, true, false, 1)
    FRCNN_DISPATCH(64, 32, true, false, 1)
    FRCNN_DISPATCH(256, 16, false, false, 1)
    FRCNN_DISPATCH(128, 16, false, false, 1)
    FRCNN_DISPATCH(64, 16, false, false, 1)
    FRCNN_DISPATCH(128, 16, true, false, 1)
    FRCNN_DISPATCH(64, 16, true, false, 1)
#undef FRCNN_DISPATCH
    set_error("frcnn_conv2d: no kernel for BN=%d BK=%d x3=%d long-K=%d CG=%d", BN, BK, (int)x3, (int)promote, CG);
    return FRCNN_ERR_ARG;
}

extern "C" int frcnn_conv2d(const void* x_hi, const void* x_lo, int H, int W, int Cin, const void* w_hi,
                            const void* w_lo, const float* bias, int Cout, int ksize, int relu, int fuse_pool2x2,
                            void* y_hi, void* y_lo, float* y_f32, int ld_f32, const int* m_valid, void* stream_) {
    FRCNN_ENTRY();
    return conv2d_impl(x_hi, x_lo, H, W, Cin, w_hi, w_lo, bias, Cout, ksize, relu, fuse_pool2x2, y_hi, y_lo, y_f32, ld_f32,
                       m_valid, stream_, nullptr);
}

extern "C" int frcnn_conv2d_res(const void* x_hi, const void* x_lo, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                                const float* bias, int Cout, int ksize, int relu, const void* res_hi, const void* res_lo,
                                void* y_hi, void* y_lo, void* stream_) {
    FRCNN_ENTRY();
    ResExtra re{res_hi, res_lo};
    return conv2d_impl(x_hi, x_lo, H, W, Cin, w_hi, w_lo, bias, Cout, ksize, relu, 0, y_hi, y_lo, nullptr, 0, nullptr, stream_,
                       nullptr, &re);
}

extern "C" int frcnn_conv3x3_c8(const void* x_hi, const void* x_lo, int H, int W, const void* w_hi, const void* w_lo,
                                const float* bias, int Cout, int relu, void* y_hi, void* y_lo, void* stream_) {
    FRCNN_ENTRY();
    WinExtra we{W + 2, 0};
    return conv2d_impl(x_hi, x_lo, H, W, 32, w_hi, w_lo, bias, Cout, 3, relu, 0, y_hi, y_lo, nullptr, 0, nullptr, stream_, nullptr,
                       nullptr, &we);
}

extern "C" int frcnn_conv2d_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int Cin, const void* w_hi,
                                  const void* w_lo, const float* bias, int Cout, int ksize, int relu, int fuse_pool2x2,
                                  void* y_hi, void* y_lo, float* y_f32, int ld_f32, void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1, "frcnn_conv2d_batch: N must be >= 1 (got %d)", N);
    return conv2d_impl(x_hi, x_lo, H, W, Cin, w_hi, w_lo, bias, Cout, ksize, relu, fuse_pool2x2, y_hi, y_lo, y_f32, ld_f32,
                       nullptr, stream_, nullptr, nullptr, nullptr, N);
}

extern "C" int frcnn_conv3x3_c8_batch(const void* x_hi, const void* x_lo, int N, int H, int W, const void* w_hi,
                                      const void* w_lo, const float* bias, int Cout, int relu, void* y_hi, void* y_lo,
                                      void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && H > 0 && W > 0, "frcnn_conv3x3_c8_batch: bad shape N=%d H=%d W=%d", N, H, W);
    WinExtra we{W + 2, (long)frcnn_image_c8_elems(H, W)};
    return conv2d_impl(x_hi, x_lo, H, W, 32, w_hi, w_lo, bias, Cout, 3, relu, 0, y_hi, y_lo, nullptr, 0, nullptr, stream_, nullptr,
                       nullptr, &we, N);
}

extern "C" int frcnn_conv2d_batch_ext(const void* x_hi, const void* x_lo, int N, int H, int W, int Cin, const void* w_hi,
                                      const void* w_lo, const float* bias, int Cout, int ksize, int relu, int fuse_pool2x2,
                                      void* y_hi, void* y_lo, float* y_f32, int ld_f32, const int* extents, int halvings,
                                      void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && extents, "frcnn_conv2d_batch_ext: needs N >= 1 (got %d) and the device extents", N);
    return conv2d_impl(x_hi, x_lo, H, W, Cin, w_hi, w_lo, bias, Cout, ksize, relu, fuse_pool2x2, y_hi, y_lo, y_f32, ld_f32,
                       nullptr, stream_, nullptr, nullptr, nullptr, N, extents, halvings);
}

// the residual is [N][H][W][Cout] like the output: the epilogue reads it at the output pixel's own image offset, and a pixel
// outside a canvas extent is zeroed after the add, whatever the residual holds there
extern "C" int frcnn_conv2d_res_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int Cin, const void* w_hi,
                                      const void* w_lo, const float* bias, int Cout, int ksize, int relu, const void* res_hi,
                                      const void* res_lo, void* y_hi, void* y_lo, void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1, "frcnn_conv2d_res_batch: N must be >= 1 (got %d)", N);
    ResExtra re{res_hi, res_lo};
    return conv2d_impl(x_hi, x_lo, H, W, Cin, w_hi, w_lo, bias, Cout, ksize, relu, 0, y_hi, y_lo, nullptr, 0, nullptr, stream_,
                       nullptr, &re, nullptr, N);
}

extern "C" int frcnn_conv2d_res_batch_ext(const void* x_hi, const void* x_lo, int N, int H, int W, int Cin, const void* w_hi,
                                          const void* w_lo, const float* bias, int Cout, int ksize, int relu, const void* res_hi,
                                          const void* res_lo, void* y_hi, void* y_lo, const int* extents, int halvings,
                                          void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && extents, "frcnn_conv2d_res_batch_ext: needs N >= 1 (got %d) and the device extents", N);
    ResExtra re{res_hi, res_lo};
    return conv2d_impl(x_hi, x_lo, H, W, Cin, w_hi, w_lo, bias, Cout, ksize, relu, 0, y_hi, y_lo, nullptr, 0, nullptr, stream_,
                       nullptr, &re, nullptr, N, extents, halvings);
}

extern "C" int frcnn_conv3x3_c8_batch_ext(const void* x_hi, const void* x_lo, int N, int H, int W, const void* w_hi,
                                          const void* w_lo, const float* bias, int Cout, int relu, const int* extents,
                                          void* y_hi, void* y_lo, void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && H > 0 && W > 0 && extents, "frcnn_conv3x3_c8_batch_ext: bad shape N=%d H=%d W=%d or NULL extents",
                  N, H, W);
    WinExtra we{W + 2, (long)frcnn_image_c8_elems(H, W)};
    return conv2d_impl(x_hi, x_lo, H, W, 32, w_hi, w_lo, bias, Cout, 3, relu, 0, y_hi, y_lo, nullptr, 0, nullptr, stream_, nullptr,
                       nullptr, &we, N, extents, 0);
}

extern "C" int frcnn_gemm_nt_splitk_splits(int K, int splits) {
    FRCNN_ENTRY();
    const int kb = cdiv(K, 64), per = cdiv(kb, splits < 1 ? 1 : splits);
    return cdiv(kb, per);
}

extern "C" int frcnn_gemm_nt_splitk(const void* a_hi, const void* a_lo, int M, int K, const void* b_hi, const void* b_lo,
                                    int N, int groups, int row_stride, int splits, const float* zero_bias, float* parts,
                                    int ld, void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(groups == 1 || groups == 9, "gemm_nt_splitk: groups must be 1 or 9 (got %d)", groups);
    FRCNN_REQUIRE(M > 0 && N > 0 && K > 0 && K % 64 == 0, "gemm_nt_splitk: bad shape M=%d N=%d K=%d (K %% 64 == 0)", M, N, K);
    FRCNN_REQUIRE(splits >= 1 && parts && zero_bias, "gemm_nt_splitk: splits >= 1, parts and a zero bias vector of ld floats are required");
    GemmExtra ge{groups, row_stride, splits, (long)M * ld};
    return conv2d_impl(a_hi, a_lo, 1, M, K, b_hi, b_lo, zero_bias, N, 1, 0, 0, nullptr, nullptr, parts, ld, nullptr, stream_, &ge);
}

// Internal entry of linear_swapab.cu: parts[split][M][ld] = A[M,K] . B[N,K]^T over that split's K range, no bias, N tile
// `bn`, each split promoting its partial sums when nacc > 1 (long K).  Returns the effective number of splits through *splits_out.
namespace frcnn {
int gemm_nt_splitk_parts(const void* a_hi, const void* a_lo, int M, int K, const void* b_hi, const void* b_lo, int N, int splits,
                         int bn, int nacc, float* parts, int ld, int* splits_out, void* stream_) {
    FRCNN_REQUIRE(M > 0 && N > 0 && K > 0 && K % 64 == 0 && splits >= 1 && parts, "gemm_nt_splitk_parts: bad arguments");
    GemmExtra ge{1, 0, splits, (long)M * ld};
    ge.bn = bn;
    ge.nacc = nacc;
    if (splits_out) *splits_out = frcnn_gemm_nt_splitk_splits(K, splits);
    return conv2d_impl(a_hi, a_lo, 1, M, K, b_hi, b_lo, nullptr, N, 1, 0, 0, nullptr, nullptr, parts, ld, nullptr, stream_, &ge);
}
}  // namespace frcnn
