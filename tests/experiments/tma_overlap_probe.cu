// Hardware probe (not product code): does a TILED tensor map whose dimension-1 stride (16 B = one 8-channel pixel) is smaller
// than the dimension-0 extent (32 elements = 64 B = 4 pixels) encode and load correctly?  That "sliding window" map lets
// conv1_1 read, for every output pixel, the 4-pixel x 8-channel neighbourhood of one image row straight from a compact
// NHWC8 image (zero border columns in memory, zero rows by TMA out-of-bounds fill) instead of from a 4x larger im2col copy.
// Image: [H][W+2][8] bf16, value(h, wp, c) = h*1000 + wp*8 + c (exact in fp32; bf16 rounding irrelevant: we compare bits).
// Map: dims {32, W, H}, strides {16 B, (W+2)*16 B}, box {32, TW, TH}, SWIZZLE_64B.  Tile at (0, w0, h0) must hold, at smem row
// (y*TW + x), chunk j (16 B, XOR-swizzled with ((row>>1)&3)), the 8 channels of padded pixel (h0+y, w0+x+j); rows with
// h0+y outside [0,H) must be zero.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -I ../../chainer-faster-rcnn_b200/csrc -o tma_overlap_probe tma_overlap_probe.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda.h>
#include <cuda_bf16.h>
#include "sm90_ptx.cuh"

constexpr int TW = 16, TH = 8;

__global__ void probe(const __grid_constant__ CUtensorMap tm, int w0, int h0, uint16_t* out) {
    __shared__ __align__(1024) uint8_t tile[TW * TH * 64];
    __shared__ uint64_t bar;
    if (threadIdx.x == 0) { ptx::mbar_init(&bar, 1); ptx::fence_barrier_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        ptx::mbar_arrive_expect_tx(&bar, TW * TH * 64);
        ptx::tma_load_3d(tile, &tm, &bar, 0, w0, h0);
    }
    ptx::mbar_wait(&bar, 0);
    for (int i = threadIdx.x; i < TW * TH * 32; i += blockDim.x) out[i] = reinterpret_cast<uint16_t*>(tile)[i];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
int main() {
    void* fp = nullptr; cudaDriverEntryPointQueryResult q;
    cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q);
    EncodeTiledFn enc = (EncodeTiledFn)fp;
    const int H = 21, W = 37, WP = W + 2;
    std::vector<__nv_bfloat16> img((size_t)H * WP * 8 + 64);
    for (int h = 0; h < H; ++h) for (int wp = 0; wp < WP; ++wp) for (int c = 0; c < 8; ++c)
        img[((size_t)h * WP + wp) * 8 + c] = __float2bfloat16((wp == 0 || wp == WP - 1) ? 0.0f : (float)((h * 64 + wp) % 251 + c * 0.0f + 1));
    for (size_t i = (size_t)H * WP * 8; i < img.size(); ++i) img[i] = __float2bfloat16(0.0f);
    __nv_bfloat16* d; uint16_t* dout;
    cudaMalloc(&d, img.size() * 2); cudaMalloc(&dout, TW * TH * 64);
    cudaMemcpy(d, img.data(), img.size() * 2, cudaMemcpyHostToDevice);
    CUtensorMap tm;
    cuuint64_t dims[3] = {32, (cuuint64_t)W, (cuuint64_t)H};
    cuuint64_t str[2] = {16, (cuuint64_t)WP * 16};
    cuuint32_t box[3] = {32, TW, TH}, es[3] = {1, 1, 1};
    CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, d, dims, str, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    printf("cuTensorMapEncodeTiled(dims {32,%d,%d}, strides {16, %d}) -> %d\n", W, H, WP * 16, (int)r);
    if (r != CUDA_SUCCESS) return 2;
    std::vector<uint16_t> ho(TW * TH * 32);
    int bad_total = 0;
    const int cases[][2] = {{0, 0}, {16, 8}, {32, 16}, {0, -1}, {16, 15}, {-1, 0}};
    for (auto& cs : cases) {
        const int w0 = cs[0], h0 = cs[1];
        cudaMemset(dout, 0xFF, TW * TH * 64);
        probe<<<1, 128>>>(tm, w0, h0, dout);
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { printf("w0 %d h0 %d: CUDA error %s\n", w0, h0, cudaGetErrorString(e)); return 1; }
        cudaMemcpy(ho.data(), dout, ho.size() * 2, cudaMemcpyDeviceToHost);
        int bad = 0;
        for (int y = 0; y < TH; ++y) for (int x = 0; x < TW; ++x) {
            const int row = y * TW + x, sw = (row >> 1) & 3;
            for (int j = 0; j < 4; ++j) for (int c = 0; c < 8; ++c) {
                const int h = h0 + y, w = w0 + x;               // dim-1 coordinate w, dim-2 coordinate h
                uint16_t want = 0;
                if (h >= 0 && h < H && w >= 0 && w < W) {
                    const __nv_bfloat16 v = img[((size_t)h * WP + (w + j)) * 8 + c];
                    want = *reinterpret_cast<const uint16_t*>(&v);
                }
                const uint16_t got = ho[row * 32 + ((j ^ sw) * 8) + c];
                if (got != want) ++bad;
            }
        }
        printf("tile (w0 %3d, h0 %3d): %d mismatching elements of %d\n", w0, h0, bad, TW * TH * 32);
        bad_total += bad;
    }
    printf(bad_total == 0 ? "TMA_OVERLAP_OK\n" : "TMA_OVERLAP_MISMATCH\n");
    return bad_total == 0 ? 0 : 1;
}
