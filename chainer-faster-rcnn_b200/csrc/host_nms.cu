// host_nms.cu -- the HOST-array NMS entry points: `_nms` (the reference's only FFI, models/gpu_nms.hpp:9-10, called from
// models/gpu_nms.pyx:16-29) and frcnn_cpu_nms_host (behind models.cpu_nms.cpu_nms: /root/reference models/cpu_nms.pyx:18-69,
// called per class by forward.py:48-57 and by models/proposal_layer.py:176-178).
//
// The caller hands over HOST arrays and wants a HOST keep list back, 20 times per image with n <= 300 rows
// (forward.py's per-class loop), so what matters here is the round trip, not the arithmetic.  Per calling thread the library
// keeps one context: a stream, a MAPPED pinned staging block (dets in, keep list + completion flag out) and a device
// workspace -- nothing is allocated or freed per call (the reference mallocs and frees its device scratch on every call,
// nms_kernel.cu:100-108,142-143).  n <= 2048: ONE single-CTA kernel reads the boxes straight from the mapped host block
// (zero-copy over PCIe), ranks them by counting (the score order of nms_math.cuh), resolves the greedy suppression with a
// lazily built IoU bitmask (cpu_nms.pyx's decision, or `_nms`'s float `>`), writes the keep list into the mapped block and
// raises a flag the host thread polls: no cudaMemcpy, no cudaStreamSynchronize on this path.
// n > 2048: the chip-wide pipeline of frcnn_nms (sort, 64x64 IoU bitmask, device-side scan) on the context's buffers.
#include <stdint.h>
#include <string.h>

#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#include "common.cuh"
#include "nms_math.cuh"

namespace frcnn {

constexpr int kSmallMax = 2048;

// The small-n kernel (n <= 2048, which covers every call of forward.py's per-class loop; 123 KB of shared memory at n = 2048):
// one CTA of up to 1024 threads, launched once per call -- so its code runs COLD (instruction fetches from L2) and what it costs is
// roughly proportional to the code it touches: the first version (every loop unrolled, 46 KB of SASS, the whole upper
// triangle of IoU tests) spent 33 us on 300 rows, 18 of them in a bitmask phase that runs at half its issue rate.  Hence
// compact rolled loops, ONE shared IoU routine, and lazy evaluation: a suppressed box's row of the bitmask is never
// needed, so only the 64x64 diagonal blocks are computed up front; after a block's greedy chain is resolved (one warp, 64
// dependent steps on 32-bit halves), all threads test just the KEPT rows of that block against the later columns and OR
// the results straight into the `removed` words.
// Phases: (1) the dense rows, coalesced 16-byte reads of the mapped host block; (2) rank by counting, all threads;
// (3) diagonal blocks; (4) per 64-rank block: resolve, then kept rows x later columns; (5) keep list + count to the mapped
// block in wide writes, fence, flag.
constexpr int kFastThreadsMax = 1024;

// bits[k] = box `i` (rank) suppresses box j0 + k, k < 16 (columns >= n read box n - 1; the caller masks them): the pairs of
// suppress_word64() in a rolled loop, for code size.  (With `if (decided) ... else divide` in the loop the compiler made
// three divergent branches per pair, which ran at a third of the issue rate.)
__device__ __forceinline__ unsigned sup_bits16(const float4* __restrict__ sbox, const float* __restrict__ area, int i, int j0, int n,
                                               const PreTest pt, double thr_d, float thr_f, int mode) {
    const float4 a = sbox[i];
    const float area_a = area[i];
    unsigned sb = 0u, ub = 0u;
#pragma unroll 4
    for (int k = 0; k < 16; ++k) {
        const int j = min(j0 + k, n - 1);
        float inter, uni;
        inter_union(a, area_a, sbox[j], area[j], inter, uni);
        uint32_t sure, und;
        pretest(inter, uni, pt, sure, und);
        sb |= sure << k;
        ub |= und << k;
    }
    auto iou_of = [&](int k) {
        const int j = min(j0 + k, n - 1);
        return iou(a, area_a, sbox[j], area[j]);
    };
    return resolve_undecided(sb, ub, iou_of, thr_d, thr_f, mode);
}

__global__ void __launch_bounds__(kFastThreadsMax) nms_small_fast_kernel(const float* __restrict__ dets, int n, int sd, int presorted,
                                                                         double thr_d, float thr_f, int mode, volatile int* out,
                                                                         int ticket, int clk_off) {
    extern __shared__ __align__(16) unsigned char sm[];
    const int T = blockDim.x, tid = threadIdx.x;
    // diagnostics: SM clock at the phase boundaries, for frcnn_host_nms_phase_cycles (thread 0, 6 x 64 bit past the keep list)
    volatile long long* clk = reinterpret_cast<volatile long long*>(out + clk_off);
#define FRCNN_NMS_STAMP(k) do { if (tid == 0) clk[k] = clock64(); } while (0)
    FRCNN_NMS_STAMP(0);
    const int nw = (n + 63) >> 6, n4 = (n + 3) & ~3;
    // shared-memory carve-up (every region a multiple of 16 bytes): see fast_smem_bytes()
    float4* sbox = reinterpret_cast<float4*>(sm);                                    // [n] boxes by rank
    unsigned long long* diag = reinterpret_cast<unsigned long long*>(sbox + n);      // [nw * 64] diagonal-block rows
    float* flat = reinterpret_cast<float*>(diag + (size_t)nw * 64);                  // [n * sd -> x4] rows as the host wrote them
    float* area = flat + ((n * sd + 3) & ~3);                                        // [n4] box areas by rank
    uint32_t* skey = reinterpret_cast<uint32_t*>(area + n4);                         // [n4] score keys by row
    int* order = reinterpret_cast<int*>(skey + n4);                                  // [n4] row by rank
    int* s_keep = order + n4;                                                        // [n4] keep list
    unsigned* removed32 = reinterpret_cast<unsigned*>(s_keep + n4);                  // [2 nw -> x4] suppressed ranks
    int* s_kl = reinterpret_cast<int*>(removed32 + ((2 * nw + 3) & ~3));             // [64] kept rows of the current block + [1] count
    {   // (1)
        const int total = n * sd, nv = total >> 2;
        const float4* src4 = reinterpret_cast<const float4*>(dets);
        float4* dst4 = reinterpret_cast<float4*>(flat);
        for (int k = tid; k < nv; k += T) dst4[k] = src4[k];
        for (int k = (nv << 2) + tid; k < total; k += T) flat[k] = dets[k];
        for (int k = tid; k < 2 * nw; k += T) removed32[k] = 0u;
        for (int k = tid; k < nw * 64; k += T) diag[k] = 0ull;
    }
    __syncthreads();
    FRCNN_NMS_STAMP(1);
    // (2) rank by counting with ALL threads: `parts` threads per row, each counts the rows ahead() of its own in a slice of
    // the densely re-packed keys, four per 16-byte broadcast load; the partial counts meet in shared-memory atomics.
    if (!presorted) {
        for (int r = tid; r < n4; r += T) {
            skey[r] = r < n ? float_to_ordered(flat[r * sd + 4]) : 0u;   // padding never counts: key 0 is below every row's
            order[r] = 0;                                // order[] doubles as the rank counters until the scatter below
        }
        __syncthreads();
        const int parts = max(1, min(T / n, 8));
        const int per4 = (n4 / 4 + parts - 1) / parts;   // float4 groups per part
        for (int it = tid; it < n * parts; it += T) {
            const int part = it / n, r = it - part * n;
            const uint32_t s = skey[r];
            const int g0 = part * per4, g1 = min(n4 / 4, g0 + per4);
            int cnt = 0;
#pragma unroll 2
            for (int g = g0; g < g1; ++g) {
                const uint4 t = reinterpret_cast<const uint4*>(skey)[g];
                const int q = g << 2;
                cnt += ahead(t.x, q + 0, s, r) + ahead(t.y, q + 1, s, r) + ahead(t.z, q + 2, s, r) + ahead(t.w, q + 3, s, r);
            }
            if (cnt) atomicAdd(&order[r], cnt);
        }
        __syncthreads();
    }
    {
        int my_rank[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {                    // n <= 2 T (checked by the host)
            const int r = tid + u * T;
            my_rank[u] = r < n ? (presorted ? r : order[r]) : 0;
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int r = tid + u * T;
            if (r < n) {
                const float* d = flat + r * sd;
                const float4 bx = make_float4(d[0], d[1], d[2], d[3]);
                order[my_rank[u]] = r;
                sbox[my_rank[u]] = bx;
                area[my_rank[u]] = box_area(bx);
            }
        }
    }
    __syncthreads();
    FRCNN_NMS_STAMP(2);
    const PreTest pt = pretest_bounds(thr_f);
    // (3) diagonal blocks: item = (block b, 16-column quarter qd, local row il), il fastest
    for (int it = tid; it < nw * 256; it += T) {
        const int b = it >> 8, qd = (it >> 6) & 3, il = it & 63;
        const int i = (b << 6) + il, j0 = (b << 6) + (qd << 4);
        if (i >= n || j0 >= n || (qd << 4) + 15 <= il) continue;
        unsigned bits = sup_bits16(sbox, area, i, j0, n, pt, thr_d, thr_f, mode);
        // keep j > i and j < n
        const int lo = il + 1 - (qd << 4);                                   // first valid k
        if (lo > 0) bits &= ~((1u << lo) - 1u);
        const int hi = n - j0;                                               // valid k < hi
        if (hi < 16) bits &= (1u << hi) - 1u;
        reinterpret_cast<unsigned short*>(diag)[((size_t)i << 2) + qd] = (unsigned short)bits;
    }
    __syncthreads();
    FRCNN_NMS_STAMP(3);
    // (4)
    int nk = 0;                                         // warp 0's running keep count (uniform over its lanes)
    for (int b = 0; b < nw; ++b) {
        const int r0 = b << 6;
        if (tid < 32) {
            // little-endian halves of the 64-bit rows: .x = columns r0..r0+31, .y = r0+32..r0+63
            const uint2* drow = reinterpret_cast<const uint2*>(diag + r0);
            const uint2 d0 = drow[tid], d1 = drow[32 + tid];          // rows r0 + tid, r0 + 32 + tid (rows >= n are zero)
            unsigned cur_lo = removed32[2 * b], cur_hi = removed32[2 * b + 1];
            unsigned bit = 1u;                          // walks off the dependent chain: test-to-predicate + select + OR per rank
#pragma unroll 8
            for (int i = 0; i < 32; ++i) {              // rows r0 .. r0+31: the serial chain runs on cur_lo only
                const unsigned rl = __shfl_sync(0xffffffffu, d0.x, i), rh = __shfl_sync(0xffffffffu, d0.y, i);
                if (!(cur_lo & bit)) {
                    cur_lo |= rl;
                    cur_hi |= rh;
                }
                bit += bit;
            }
            bit = 1u;
#pragma unroll 8
            for (int i = 0; i < 32; ++i) {              // rows r0+32 .. r0+63: their low halves are empty (upper triangle)
                const unsigned rh = __shfl_sync(0xffffffffu, d1.y, i);
                if (!(cur_hi & bit)) cur_hi |= rh;
                bit += bit;
            }
            const int rows = min(64, n - r0);
            const unsigned v_lo = rows >= 32 ? 0xffffffffu : ((1u << rows) - 1u);
            const unsigned v_hi = rows >= 64 ? 0xffffffffu : (rows > 32 ? ((1u << (rows - 32)) - 1u) : 0u);
            const unsigned k_lo = ~cur_lo & v_lo, k_hi = ~cur_hi & v_hi;
            const int c_lo = __popc(k_lo);
            const unsigned below = (1u << tid) - 1u;
            if ((k_lo >> tid) & 1u) {
                const int pos = __popc(k_lo & below);
                s_keep[nk + pos] = order[r0 + tid];
                s_kl[pos] = tid;
            }
            if ((k_hi >> tid) & 1u) {
                const int pos = c_lo + __popc(k_hi & below);
                s_keep[nk + pos] = order[r0 + 32 + tid];
                s_kl[pos] = 32 + tid;
            }
            const int kb = c_lo + __popc(k_hi);
            nk += kb;
            if (tid == 0) s_kl[64] = kb;
        }
        if (b + 1 == nw) break;                         // uniform
        __syncthreads();
        {
            const int kb = s_kl[64], c0 = r0 + 64;
            const int ncq = (n - c0 + 15) >> 4;         // 16-column groups to the right of this block
            for (int it = tid; it < kb * ncq; it += T) {
                const int cq = it / kb, k = it - cq * kb;       // k fastest: a warp = different kept rows, same columns
                const int i = r0 + s_kl[k], j0 = c0 + (cq << 4);
                unsigned bits = sup_bits16(sbox, area, i, j0, n, pt, thr_d, thr_f, mode);
                const int hi = n - j0;
                if (hi < 16) bits &= (1u << hi) - 1u;
                if (bits) atomicOr(&removed32[j0 >> 5], bits << (j0 & 16));
            }
        }
        __syncthreads();
    }
    if (tid >= 32) return;
    __syncwarp();
    FRCNN_NMS_STAMP(4);
    // (5)
    for (int k = tid; k < nk; k += 32) out[2 + k] = s_keep[k];
    if (tid == 0) out[1] = nk;
    FRCNN_NMS_STAMP(5);
    __threadfence_system();                            // keep list + count visible to the host before the flag
    __syncwarp();
    if (tid == 0) out[0] = ticket;
#undef FRCNN_NMS_STAMP
}

static size_t fast_smem_bytes(int n, int sd) {
    const size_t nw = (size_t)(n + 63) / 64, n4 = (size_t)(n + 3) & ~(size_t)3;
    return (size_t)n * 16 + nw * 64 * 8 + 4 * (((size_t)n * sd + 3) & ~(size_t)3) + 4 * n4 * 4 + 4 * ((2 * nw + 3) & ~(size_t)3) +
           4 * 68;
}

struct HostNmsCtx {
    int device = -1;
    cudaStream_t stream = nullptr;
    float* h_in = nullptr;          // mapped pinned: dets
    int* h_out = nullptr;           // mapped pinned: flag, count, keep[]
    float* d_in = nullptr;          // device aliases of the two blocks
    int* d_out = nullptr;
    int cap = 0;                    // rows the blocks hold
    char* d_ws = nullptr;           // device scratch of the large-n path
    size_t ws_bytes = 0;
    int ticket = 0;
    size_t smem_attr_fast = 48 * 1024;   // largest dynamic shared-memory size set on nms_small_fast_kernel by this thread so far
    long fast_calls = 0;
    long long last_launch_ns = 0, last_wait_ns = 0;   // host side of the last small-n call: the launch call, the flag poll
    // No destructor on purpose: cudaFreeHost / cudaFree at THREAD EXIT synchronise the whole device and hold the context lock
    // for milliseconds, stalling every other caller thread that is still running (measured: two of six threads took 3x as
    // long, profiles/r02_api_threads_diag_before_plan_pool.txt).  A thread's ~50 KB of pinned staging and its stream stay
    // allocated until the process exits.
};

static thread_local HostNmsCtx t_ctx;

static int ctx_prepare(HostNmsCtx& c, int device_id, int n, bool large) {
    if (c.device != device_id) {
        if (c.device >= 0) {
            cudaSetDevice(c.device);
            if (c.h_in) cudaFreeHost(c.h_in);
            if (c.h_out) cudaFreeHost(c.h_out);
            if (c.d_ws) cudaFree(c.d_ws);
            if (c.stream) cudaStreamDestroy(c.stream);
            c.h_in = nullptr; c.h_out = nullptr; c.d_ws = nullptr; c.stream = nullptr; c.cap = 0; c.ws_bytes = 0;
        }
        FRCNN_CUDA_OK(cudaSetDevice(device_id));
        FRCNN_CUDA_OK(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
        c.device = device_id;
    } else {
        FRCNN_CUDA_OK(cudaSetDevice(device_id));
    }
    if (n > c.cap) {
        const int cap = n < 1024 ? 1024 : (n + 1023) / 1024 * 1024;
        if (c.h_in) cudaFreeHost(c.h_in);
        if (c.h_out) cudaFreeHost(c.h_out);
        c.h_in = nullptr; c.h_out = nullptr; c.cap = 0;
        FRCNN_CUDA_OK(cudaHostAlloc((void**)&c.h_in, sizeof(float) * 5 * (size_t)cap, cudaHostAllocMapped));
        FRCNN_CUDA_OK(cudaHostAlloc((void**)&c.h_out, sizeof(int) * ((size_t)cap + 2 + 16), cudaHostAllocMapped));   // + 6 phase clocks
        FRCNN_CUDA_OK(cudaHostGetDevicePointer((void**)&c.d_in, c.h_in, 0));
        FRCNN_CUDA_OK(cudaHostGetDevicePointer((void**)&c.d_out, c.h_out, 0));
        c.h_out[0] = 0;
        c.cap = cap;
    }
    if (large) {
        const size_t need = align_up(sizeof(float) * 5 * (size_t)n, 256) + align_up(sizeof(int) * (size_t)n, 256) + 256 +
                            frcnn_nms_workspace_bytes(n);
        if (need > c.ws_bytes) {
            if (c.d_ws) cudaFree(c.d_ws);
            c.d_ws = nullptr; c.ws_bytes = 0;
            FRCNN_CUDA_OK(cudaMalloc((void**)&c.d_ws, need));
            c.ws_bytes = need;
        }
    }
    return FRCNN_OK;
}

static int nms_host_impl(const float* dets_host, int n, int dim, double thresh, int mode, int presorted, int* keep_out_host,
                         int device_id) {
    if (n < 0 || dim < 4 || (!presorted && dim < 5)) { set_error("nms host: bad n=%d dim=%d", n, dim); return FRCNN_ERR_ARG; }
    if (n == 0) return 0;
    if (n > 16384) { set_error("nms host: n=%d > 16384 (the device pipeline's limit; see INTEGRATION.md)", n); return FRCNN_ERR_ARG; }
    if (!dets_host || !keep_out_host) { set_error("nms host: NULL argument"); return FRCNN_ERR_ARG; }
    HostNmsCtx& ctx = t_ctx;
    const bool large = n > kSmallMax;
    // device_id < 0: the calling thread's CURRENT device (cpu_nms has no device argument: a process that owns GPU 3 must
    // not be moved to GPU 0 by its per-class NMS).  An explicit id (`_nms`, gpu_nms.pyx:16) is honoured and the caller's
    // current device restored afterwards.
    int prev_dev = 0;
    FRCNN_CUDA_OK(cudaGetDevice(&prev_dev));
    if (device_id < 0) device_id = prev_dev;
    struct Restore {
        int dev, prev;
        ~Restore() { if (dev != prev) cudaSetDevice(prev); }
    } restore{device_id, prev_dev};
    int rc = ctx_prepare(ctx, device_id, n, large);
    if (rc != FRCNN_OK) return rc;
    if (!large) {
        // stage rows densely as [n, dim'] (dim' = 4 or 5) in the mapped block
        const int sd = presorted ? 4 : 5;
        if (dim == sd) {
            memcpy(ctx.h_in, dets_host, sizeof(float) * (size_t)sd * n);
        } else {
            for (int i = 0; i < n; ++i)
                for (int j = 0; j < sd; ++j) ctx.h_in[(size_t)sd * i + j] = dets_host[(size_t)dim * i + j];
        }
        const int ticket = ++ctx.ticket == 0 ? ++ctx.ticket : ctx.ticket;
        const size_t fast_smem = fast_smem_bytes(n, sd);
        const auto t_launch0 = std::chrono::steady_clock::now();
        if (fast_smem > ctx.smem_attr_fast) {            // raise the kernel's dynamic shared-memory limit only when needed
            FRCNN_CUDA_OK(cudaFuncSetAttribute(nms_small_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fast_smem));
            ctx.smem_attr_fast = fast_smem;
        }
        const int threads = n > 128 ? kFastThreadsMax : 256;
        FRCNN_CUDA_OK(launch_plain(nms_small_fast_kernel, dim3(1), dim3(threads), fast_smem, ctx.stream, (const float*)ctx.d_in, n,
                                   sd, presorted, thresh, (float)thresh, mode, (volatile int*)ctx.d_out, ticket, (ctx.cap + 2 + 1) & ~1));
        ctx.fast_calls++;
        // poll the completion flag in mapped memory; if it does not show up soon, fall back to a stream sync (which also
        // surfaces an execution error)
        volatile int* flag = ctx.h_out;
        const auto t0 = std::chrono::steady_clock::now();
        ctx.last_launch_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(t0 - t_launch0).count();
        long spins = 0;
        while (flag[0] != ticket) {
            if ((++spins & 0x3ff) == 0 &&
                std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > 0.25) {
                FRCNN_CUDA_OK(cudaStreamSynchronize(ctx.stream));
                if (flag[0] != ticket) { set_error("nms host: kernel finished without raising its flag"); return FRCNN_ERR_CUDA; }
                break;
            }
        }
        ctx.last_wait_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
        const int num = flag[1];
        memcpy(keep_out_host, (const void*)(ctx.h_out + 2), sizeof(int) * (size_t)num);
        return num;
    }
    // ---- large n: the chip-wide pipeline on the context's buffers.  [n,5] staging: a pre-sorted input without scores
    // gets strictly descending synthetic scores so the internal (stable) sort is the identity.
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j < 4; ++j) ctx.h_in[5 * (size_t)i + j] = dets_host[(size_t)dim * i + j];
        ctx.h_in[5 * (size_t)i + 4] = presorted ? (float)(n - i) : dets_host[(size_t)dim * i + 4];
    }
    const size_t dets_b = align_up(sizeof(float) * 5 * (size_t)n, 256), keep_b = align_up(sizeof(int) * (size_t)n, 256);
    float* d_dets = reinterpret_cast<float*>(ctx.d_ws);
    int* d_keep = reinterpret_cast<int*>(ctx.d_ws + dets_b);
    int* d_num = reinterpret_cast<int*>(ctx.d_ws + dets_b + keep_b);
    void* d_ws = ctx.d_ws + dets_b + keep_b + 256;
    FRCNN_CUDA_OK(cudaMemcpyAsync(d_dets, ctx.h_in, sizeof(float) * 5 * (size_t)n, cudaMemcpyHostToDevice, ctx.stream));
    rc = frcnn_nms(d_dets, n, thresh, mode, 0, d_keep, d_num, d_ws, ctx.ws_bytes - (dets_b + keep_b + 256), ctx.stream);
    if (rc != FRCNN_OK) return rc;
    FRCNN_CUDA_OK(cudaMemcpyAsync(ctx.h_out + 1, d_num, sizeof(int), cudaMemcpyDeviceToHost, ctx.stream));
    FRCNN_CUDA_OK(cudaMemcpyAsync(ctx.h_out + 2, d_keep, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, ctx.stream));
    FRCNN_CUDA_OK(cudaStreamSynchronize(ctx.stream));
    const int num = ctx.h_out[1];
    memcpy(keep_out_host, ctx.h_out + 2, sizeof(int) * (size_t)num);
    return num;
}

}  // namespace frcnn

using namespace frcnn;

extern "C" void _nms(int* keep_out, int* num_out, const float* boxes_host, int boxes_num, int boxes_dim,
                     float nms_overlap_thresh, int device_id) {
    FRCNN_ENTRY();
    int r = nms_host_impl(boxes_host, boxes_num, boxes_dim, (double)nms_overlap_thresh, FRCNN_NMS_GT_FLOAT, 1, keep_out,
                          device_id);
    *num_out = r < 0 ? -1 : r;
}

// Diagnostics of the calling thread's LAST small-n call: out8[0..5] = SM clock stamps (kernel entry, rows read, ranked,
// diagonal blocks built, chain resolved, keep list written), out8[6] = host nanoseconds inside the launch call, out8[7] =
// host nanoseconds polling the completion flag.  Returns 0 if this thread has not made such a call.
extern "C" int frcnn_host_nms_phase_cycles(long long* out8) {
    FRCNN_ENTRY();
    if (!out8 || t_ctx.fast_calls == 0 || !t_ctx.h_out) return 0;
    const long long* c = reinterpret_cast<const long long*>(t_ctx.h_out + ((t_ctx.cap + 2 + 1) & ~1));
    for (int i = 0; i < 6; ++i) out8[i] = c[i];
    out8[6] = t_ctx.last_launch_ns;
    out8[7] = t_ctx.last_wait_ns;
    return 1;
}

// Host-side helper of the in-graph per-class NMS hand-off (models.cpu_nms): is `dets` [R,5] bit for bit the (boxes of class c
// | score of class c) rows of the result block the model call just returned?  Tries class `hint` first, then every other
// foreground class; returns the class (1 .. num_classes-1) or 0 if none matches.  Pure host code, no CUDA call.
extern "C" int frcnn_match_class_dets(const float* dets, int R, const float* boxes, int ld_boxes, const float* prob, int ld_prob,
                                      int num_classes, int hint) {
    if (!dets || !boxes || !prob || R <= 0 || num_classes < 2) return 0;
    const uint32_t* d = reinterpret_cast<const uint32_t*>(dets);
    auto same = [&](int c) {
        const uint32_t* b = reinterpret_cast<const uint32_t*>(boxes) + 4 * c;
        const uint32_t* q = reinterpret_cast<const uint32_t*>(prob) + c;
        for (int r = 0; r < R; ++r) {
            const uint32_t* dr = d + 5 * (size_t)r;
            const uint32_t* br = b + (size_t)r * ld_boxes;
            if (dr[4] != q[(size_t)r * ld_prob] || dr[0] != br[0] || dr[1] != br[1] || dr[2] != br[2] || dr[3] != br[3]) return false;
        }
        return true;
    };
    if (hint >= 1 && hint < num_classes && same(hint)) return hint;
    for (int c = 1; c < num_classes; ++c)
        if (c != hint && same(c)) return c;
    return 0;
}

extern "C" int frcnn_cpu_nms_host(const float* dets_host, int n, double thresh, int* keep_out_host, int device_id) {
    FRCNN_ENTRY();
    return nms_host_impl(dets_host, n, 5, thresh, FRCNN_NMS_GE_DOUBLE, 0, keep_out_host, device_id);
}

// ------------------------------------------------------------------------------------------ host staging helpers
// Pinned host blocks and explicit async copies for the host-array front ends (engine.ForwardPlan.forward_host,
// engine.StreamRunner): the image upload and the result download go through cudaMemcpyAsync on the plan's stream from /
// to memory this library pinned itself, so that their cost is the link's (measured: 7.2 MB in 0.136 ms = 53 GB/s,
// profiles/r02_h2d_probe.txt) and does not depend on a framework's pinned-memory heuristics.
extern "C" void* frcnn_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (bytes == 0) return nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
        set_error("frcnn_host_alloc: cudaHostAlloc(%zu) failed: %s", bytes, cudaGetErrorString(cudaGetLastError()));
        return nullptr;
    }
    return p;
}

extern "C" int frcnn_host_free(void* p) {
    FRCNN_ENTRY();
    if (p != nullptr) FRCNN_CUDA_OK(cudaFreeHost(p));
    return FRCNN_OK;
}

extern "C" int frcnn_memcpy_h2d_async(void* dst_device, const void* src_host, size_t bytes, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(dst_device && src_host, "frcnn_memcpy_h2d_async: NULL pointer");
    FRCNN_CUDA_OK(cudaMemcpyAsync(dst_device, src_host, bytes, cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)));
    return FRCNN_OK;
}

extern "C" int frcnn_memcpy_d2h_async(void* dst_host, const void* src_device, size_t bytes, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(dst_host && src_device, "frcnn_memcpy_d2h_async: NULL pointer");
    FRCNN_CUDA_OK(cudaMemcpyAsync(dst_host, src_device, bytes, cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)));
    return FRCNN_OK;
}

extern "C" int frcnn_stream_synchronize(void* stream) {
    FRCNN_ENTRY();
    FRCNN_CUDA_OK(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
    return FRCNN_OK;
}

// Pageable -> pinned staging copy on a few host threads that SLEEP between jobs (condition variable, no spinning).  The
// first version used the framework's parallel copy: 64 OpenMP workers that spin for milliseconds after every parallel
// region; with one such region per image the process ran into ~70 ms stalls (CPU-quota throttling on the GPU boxes,
// profiles/r02_host_api_profile.txt).  4 workers move the 7.2 MB image in ~0.15-0.2 ms and cost nothing when idle.
namespace frcnn {
class CopyPool {
  public:
    static CopyPool& get() {
        static CopyPool* p = new CopyPool();          // leaked on purpose: worker threads must not be joined at exit
        return *p;
    }
    void copy(char* dst, const char* src, size_t bytes) {
        const int parts = kWorkers + 1;
        const size_t chunk = ((bytes / parts) + 4095) & ~size_t(4095);
        if (bytes < (1u << 20) || chunk == 0) { memcpy(dst, src, bytes); return; }
        std::unique_lock<std::mutex> run(run_mu_);      // one job at a time (callers from several threads queue here)
        {
            std::lock_guard<std::mutex> g(mu_);
            dst_ = dst; src_ = src; bytes_ = bytes; chunk_ = chunk;
            pending_ = kWorkers;
            ++job_;
        }
        cv_.notify_all();
        const size_t o = (size_t)kWorkers * chunk;       // the caller copies the last part itself
        if (o < bytes) memcpy(dst + o, src + o, bytes - o);
        std::unique_lock<std::mutex> g(mu_);
        done_.wait(g, [&] { return pending_ == 0; });
    }

  private:
    static constexpr int kWorkers = 3;
    CopyPool() {
        for (int i = 0; i < kWorkers; ++i) std::thread([this, i] { work(i); }).detach();
    }
    void work(int i) {
        unsigned long seen = 0;
        for (;;) {
            std::unique_lock<std::mutex> g(mu_);
            cv_.wait(g, [&] { return job_ != seen; });
            seen = job_;
            char* d = dst_; const char* s = src_;
            const size_t bytes = bytes_, chunk = chunk_;
            g.unlock();
            const size_t o = (size_t)i * chunk;
            if (o < bytes) memcpy(d + o, s + o, o + chunk <= bytes ? chunk : bytes - o);
            g.lock();
            if (--pending_ == 0) done_.notify_one();
        }
    }
    std::mutex mu_, run_mu_;
    std::condition_variable cv_, done_;
    char* dst_ = nullptr; const char* src_ = nullptr;
    size_t bytes_ = 0, chunk_ = 0;
    int pending_ = 0;
    unsigned long job_ = 0;
};
}  // namespace frcnn

extern "C" int frcnn_host_copy(void* dst, const void* src, size_t bytes) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(dst && src, "frcnn_host_copy: NULL pointer");
    frcnn::CopyPool::get().copy(static_cast<char*>(dst), static_cast<const char*>(src), bytes);
    return FRCNN_OK;
}

// Upload of a PAGEABLE host buffer through a pinned staging block, pipelined: chunk k is copied into the staging block by
// the calling thread while chunk k-1 is already on the wire (cudaMemcpyAsync on `stream`), so the image costs
// max(host memcpy, DMA) + one chunk instead of their sum -- and no helper thread is involved (the GPU boxes give the process
// a 16-CPU quota; a thread pool that wakes for every image costs more than it saves there, profiles/r02_host_api_profile.txt).
// `staging` must hold `bytes` (the whole image: the chunks of an image never share staging memory, so the host never waits).
extern "C" int frcnn_upload_pageable(void* dst_device, const void* src_host, void* staging_pinned, size_t bytes, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(dst_device && src_host && staging_pinned, "frcnn_upload_pageable: NULL pointer");
    const size_t chunk = 1u << 20;
    for (size_t o = 0; o < bytes; o += chunk) {
        const size_t n = bytes - o < chunk ? bytes - o : chunk;
        memcpy(static_cast<char*>(staging_pinned) + o, static_cast<const char*>(src_host) + o, n);
        FRCNN_CUDA_OK(cudaMemcpyAsync(static_cast<char*>(dst_device) + o, static_cast<char*>(staging_pinned) + o, n,
                                      cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)));
    }
    return FRCNN_OK;
}
