// linear_swapab.cu -- frcnn_linear: y = act(x . W^T + b) for a SMALL number of rows (the R <= 300 RoIs of the head).
//
// Replaces L.Linear + F.relu at /root/reference models/faster_rcnn.py:33-36,127-134 (fc6, fc7, cls_score | bbox_pred).
//
// Why not the convolution's orientation (RoIs = pixel rows of the 128-row tile): 300 rows occupy 384 tile rows (22 % of
// the tensor work multiplies zeros) and the 3 tiles of fc6 walk K = 25,088 serially.  Here the operands are swapped: the
// WEIGHT rows are the M side (4096 = 32 full tiles), the RoIs are the N side (300 -> 320 = 5 tiles of N = 64: 6.7 %
// padding), and K is split so that every SM has about one unit of work; a long split additionally promotes its
// tensor-core partial sums into a register total every 8 k-blocks (the tensor core's fp32 accumulator truncates on
// every add, DESIGN.md 2).  Per split the GEMM (conv_gemm_kernel in split-K "NT" mode) writes an fp32 slab
// parts[split][channel][roi]; `linear_reduce_kernel` sums the slabs in fixed order (deterministic), adds the bias, applies
// ReLU, zeroes the rows past the device-side RoI count, transposes through shared memory and writes [roi][channel] as
// bf16 hi/lo planes (the next layer's operand) and/or fp32.
#include "common.cuh"

namespace frcnn {

int gemm_nt_splitk_parts(const void* a_hi, const void* a_lo, int M, int K, const void* b_hi, const void* b_lo, int N, int splits,
                         int bn, int nacc, float* parts, int ld, int* splits_out, void* stream_);

constexpr int kRedC = 64, kRedR = 32, kRedThreads = 256;

// parts [S][Mrows][ld] fp32 (row = output channel, column = RoI)  ->  y[r][c], r < seg_rows, c < Cout (rows >= R_cap are 0).
// A batch of images: blockIdx.y = image * rblocks + row block; image i owns parts columns [i*seg_rows, (i+1)*seg_rows), output
// rows [i*seg_rows, (i+1)*seg_rows) and RoI count m_valid[i * count_stride].  One image: rblocks = gridDim.y, seg_rows = R_cap.
__global__ void __launch_bounds__(kRedThreads) linear_reduce_kernel(const float* __restrict__ parts, int S, long part_stride, int ld,
                                                                    const float* __restrict__ bias, int Cout, int R_cap,
                                                                    const int* __restrict__ m_valid, int relu,
                                                                    __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo,
                                                                    float* __restrict__ y_f32, int ld_f32, int seg_rows, int rblocks,
                                                                    int count_stride) {
    __shared__ float tile[kRedC][kRedR + 1];
    grid_dep_wait();
    const int img = blockIdx.y / rblocks;
    const int c0 = blockIdx.x * kRedC, r0 = (blockIdx.y - img * rblocks) * kRedR;
    parts += (long)img * seg_rows;
    if (y_hi != nullptr) y_hi += (long)img * seg_rows * Cout;
    if (y_lo != nullptr) y_lo += (long)img * seg_rows * Cout;
    if (y_f32 != nullptr) y_f32 += (long)img * seg_rows * ld_f32;
    const int R = m_valid ? min(m_valid[(long)img * count_stride], R_cap) : R_cap;
    // load phase: thread = (channel row, 4 consecutive RoI columns): one 16-byte load per split (ld % 32 == 0 keeps every row
    // 128-byte aligned), all splits' loads of a thread independent; summed in split order (deterministic)
    {
        const int cl = threadIdx.x >> 3, rq = (threadIdx.x & 7) * 4;
#pragma unroll
        for (int j = 0; j < kRedC / 32; ++j) {
            const int c = c0 + cl + 32 * j;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (c < Cout) {
                const float* src = parts + (long)c * ld + r0 + rq;
                int s = 0;
                for (; s + 4 <= S; s += 4) {
                    float4 t[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) t[u] = *reinterpret_cast<const float4*>(src + (long)(s + u) * part_stride);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        v.x = __fadd_rn(v.x, t[u].x); v.y = __fadd_rn(v.y, t[u].y);
                        v.z = __fadd_rn(v.z, t[u].z); v.w = __fadd_rn(v.w, t[u].w);
                    }
                }
                for (; s < S; ++s) {
                    const float4 t = *reinterpret_cast<const float4*>(src + (long)s * part_stride);
                    v.x = __fadd_rn(v.x, t.x); v.y = __fadd_rn(v.y, t.y); v.z = __fadd_rn(v.z, t.z); v.w = __fadd_rn(v.w, t.w);
                }
                const float b = bias[c];
                v.x = __fadd_rn(v.x, b); v.y = __fadd_rn(v.y, b); v.z = __fadd_rn(v.z, b); v.w = __fadd_rn(v.w, b);
                if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            }
            const int r = r0 + rq;                       // rows past the RoI count are zero
            float* t = &tile[cl + 32 * j][rq];
            t[0] = r + 0 < R ? v.x : 0.f;
            t[1] = r + 1 < R ? v.y : 0.f;
            t[2] = r + 2 < R ? v.z : 0.f;
            t[3] = r + 3 < R ? v.w : 0.f;
        }
    }
    __syncthreads();
    // store phase: thread = (RoI row, 2 adjacent channels): a warp writes 64 consecutive channels (128 B of bf16) of one row
    {
        const int cp = (threadIdx.x & 31) * 2, rl = threadIdx.x >> 5;
        const int c = c0 + cp;
#pragma unroll
        for (int k = 0; k < kRedR / 8; ++k) {
            const int r = r0 + rl + 8 * k;
            if (r >= seg_rows) continue;
            const float v0 = tile[cp][rl + 8 * k], v1 = tile[cp + 1][rl + 8 * k];
            if (y_hi != nullptr && c < Cout) {
                __nv_bfloat16 h0, l0, h1, l1;
                split_bf16(v0, h0, l0);
                split_bf16(v1, h1, l1);
                if ((Cout & 1) == 0) {                      // even row pitch: 4-byte aligned pairs
                    __nv_bfloat162 hh, ll;
                    hh.x = h0; hh.y = h1; ll.x = l0; ll.y = l1;
                    *reinterpret_cast<__nv_bfloat162*>(y_hi + (long)r * Cout + c) = hh;
                    if (y_lo != nullptr) *reinterpret_cast<__nv_bfloat162*>(y_lo + (long)r * Cout + c) = ll;
                } else {
                    y_hi[(long)r * Cout + c] = h0;
                    if (y_lo != nullptr) y_lo[(long)r * Cout + c] = l0;
                    if (c + 1 < Cout) {
                        y_hi[(long)r * Cout + c + 1] = h1;
                        if (y_lo != nullptr) y_lo[(long)r * Cout + c + 1] = l1;
                    }
                }
            }
            if (y_f32 != nullptr) {
                if (c < ld_f32) y_f32[(long)r * ld_f32 + c] = v0;               // columns [Cout, ld_f32) are zero
                if (c + 1 < ld_f32) y_f32[(long)r * ld_f32 + c + 1] = v1;
            }
        }
    }
}

struct LinearPlan {
    int ld, bn, splits, nacc, m_rows;
    size_t parts_bytes;
};

static LinearPlan plan_linear(int R_cap, int K, int Cout) {
    LinearPlan lp;
    lp.ld = (R_cap + 31) / 32 * 32;
    // N tile: least padding, then the wider tile
    const int cand[3] = {256, 128, 64};
    long best = -1;
    lp.bn = 128;
    for (int bn : cand) {
        const long padded = (long)cdiv(lp.ld, bn) * bn;
        if (best < 0 || padded < best) { best = padded; lp.bn = bn; }
    }
    const int kb = K / 64;
    const int m_tiles = cdiv(Cout, 128);
    const int base = m_tiles * cdiv(lp.ld, lp.bn);
    int sms = 132;
    {
        int dev = 0;
        if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    const int slots = sms;
    // splits: minimise (waves x k-blocks per unit) + the reduction's traffic; a unit keeps >= 2 k-blocks
    const double red_cost = (double)cdiv(Cout, 128) * 128 * lp.ld * 8.0 / 5e6 / 0.75;       // one slab written + read, in k-block times
    double best_cost = 0;
    lp.splits = 1;
    for (int s = 1; s <= 16 && s * 2 <= (kb > 1 ? kb : 2); ++s) {       // <= 16 slabs: the reduction reads them one after another
        const int per = cdiv(kb, s);
        if (cdiv(kb, per) != s) continue;                   // not an effective split count
        const double cost = (double)cdiv(base * s, slots) * per + red_cost * s;
        if (s == 1 || cost < best_cost) { best_cost = cost; lp.splits = s; }
    }
    const int per = cdiv(kb, lp.splits);
    // long K per split: promote the tensor-core partial sums (conv2d_impl then narrows the N tile to fit the registers)
    lp.nacc = (per >= 64) ? 2 : 1;
    lp.m_rows = Cout;
    lp.parts_bytes = (size_t)lp.splits * Cout * lp.ld * sizeof(float);
    return lp;
}

}  // namespace frcnn

using namespace frcnn;

extern "C" size_t frcnn_linear_workspace_bytes(int R_cap, int K, int Cout) {
    FRCNN_ENTRY();
    if (R_cap <= 0 || K <= 0 || Cout <= 0 || K % 64 != 0) return 0;
    return align_up(plan_linear(R_cap, K, Cout).parts_bytes, 256);
}

extern "C" int frcnn_linear(const void* x_hi, const void* x_lo, int R_cap, int K, const void* w_hi, const void* w_lo,
                            const float* bias, int Cout, int relu, const int* m_valid, void* y_hi, void* y_lo, float* y_f32,
                            int ld_f32, void* workspace, size_t workspace_bytes, void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(x_hi && w_hi && bias && workspace, "frcnn_linear: x_hi, w_hi, bias and workspace are required");
    FRCNN_REQUIRE((x_lo == nullptr) == (w_lo == nullptr), "frcnn_linear: x_lo and w_lo must both be given (bf16x3) or both NULL");
    FRCNN_REQUIRE(R_cap > 0 && Cout > 0 && K > 0 && K % 64 == 0, "frcnn_linear: bad shape R_cap=%d K=%d Cout=%d (K %% 64 == 0)", R_cap, K, Cout);
    FRCNN_REQUIRE(y_hi || y_f32, "frcnn_linear: no output requested");
    FRCNN_REQUIRE(!y_lo || y_hi, "frcnn_linear: y_lo without y_hi");
    FRCNN_REQUIRE(!y_f32 || ld_f32 >= Cout, "frcnn_linear: ld_f32 must be >= Cout");
    const LinearPlan lp = plan_linear(R_cap, K, Cout);
    if (workspace_bytes < lp.parts_bytes) {
        set_error("frcnn_linear: workspace %zu < required %zu", workspace_bytes, lp.parts_bytes);
        return FRCNN_ERR_WORKSPACE;
    }
    float* parts = static_cast<float*>(workspace);
    int S = 0;
    // swapped operands: A = weights [Cout, K] (the M side), B = activations [R_cap, K] (the N side; rows past R_cap are
    // zero-filled by the TMA unit)
    int rc = gemm_nt_splitk_parts(w_hi, w_lo, Cout, K, x_hi, x_lo, R_cap, lp.splits, lp.bn, lp.nacc, parts, lp.ld, &S, stream_);
    if (rc != FRCNN_OK) return rc;
    const int cols = y_f32 ? (ld_f32 > Cout ? ld_f32 : Cout) : Cout;
    dim3 grid(cdiv(cols, kRedC), cdiv(R_cap, kRedR));
    FRCNN_CUDA_OK(launch_pdl(linear_reduce_kernel, grid, dim3(kRedThreads), 0, static_cast<cudaStream_t>(stream_),
                             (const float*)parts, S, (long)Cout * lp.ld, lp.ld, bias, Cout, R_cap, m_valid, relu,
                             (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo, y_f32, ld_f32, R_cap, (int)grid.y, 0));
    return FRCNN_OK;
}

extern "C" size_t frcnn_linear_batch_workspace_bytes(int N, int R_cap, int K, int Cout) {
    FRCNN_ENTRY();
    if (N <= 0 || R_cap <= 0 || K <= 0 || Cout <= 0 || K % 64 != 0) return 0;
    return align_up((size_t)N * plan_linear(R_cap, K, Cout).parts_bytes, 256);
}

extern "C" int frcnn_linear_batch(const void* x_hi, const void* x_lo, int N, int R_cap, int K, const void* w_hi, const void* w_lo,
                                  const float* bias, int Cout, int relu, const int* counts, int count_stride, void* y_hi, void* y_lo,
                                  float* y_f32, int ld_f32, void* workspace, size_t workspace_bytes, void* stream_) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(x_hi && w_hi && bias && workspace, "frcnn_linear_batch: x_hi, w_hi, bias and workspace are required");
    FRCNN_REQUIRE((x_lo == nullptr) == (w_lo == nullptr), "frcnn_linear_batch: x_lo and w_lo must both be given (bf16x3) or both NULL");
    FRCNN_REQUIRE(N >= 1 && R_cap > 0 && Cout > 0 && K > 0 && K % 64 == 0,
                  "frcnn_linear_batch: bad shape N=%d R_cap=%d K=%d Cout=%d (K %% 64 == 0)", N, R_cap, K, Cout);
    FRCNN_REQUIRE(y_hi || y_f32, "frcnn_linear_batch: no output requested");
    FRCNN_REQUIRE(!y_lo || y_hi, "frcnn_linear_batch: y_lo without y_hi");
    FRCNN_REQUIRE(!y_f32 || ld_f32 >= Cout, "frcnn_linear_batch: ld_f32 must be >= Cout");
    FRCNN_REQUIRE(count_stride >= 0, "frcnn_linear_batch: count_stride must be >= 0");
    // the one-image plan (N tile, splits, partial-sum promotion): every image's sums are those of frcnn_linear
    const LinearPlan lp = plan_linear(R_cap, K, Cout);
    const int rows = N * lp.ld;
    FRCNN_REQUIRE((long)N * lp.ld < (1l << 30), "frcnn_linear_batch: too many rows");
    const size_t need = (size_t)N * lp.parts_bytes;
    if (workspace_bytes < need) {
        set_error("frcnn_linear_batch: workspace %zu < required %zu", workspace_bytes, need);
        return FRCNN_ERR_WORKSPACE;
    }
    float* parts = static_cast<float*>(workspace);
    int S = 0;
    // the N side is all images' segments of lp.ld rows back to back: parts[split][Cout][N * lp.ld]
    int rc = gemm_nt_splitk_parts(w_hi, w_lo, Cout, K, x_hi, x_lo, rows, lp.splits, lp.bn, lp.nacc, parts, rows, &S, stream_);
    if (rc != FRCNN_OK) return rc;
    const int cols = y_f32 ? (ld_f32 > Cout ? ld_f32 : Cout) : Cout;
    const int rblocks = lp.ld / kRedR;
    dim3 grid(cdiv(cols, kRedC), N * rblocks);
    FRCNN_CUDA_OK(launch_pdl(linear_reduce_kernel, grid, dim3(kRedThreads), 0, static_cast<cudaStream_t>(stream_),
                             (const float*)parts, S, (long)Cout * rows, rows, bias, Cout, R_cap, counts, relu,
                             (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo, y_f32, ld_f32, lp.ld, rblocks, count_stride));
    return FRCNN_OK;
}
