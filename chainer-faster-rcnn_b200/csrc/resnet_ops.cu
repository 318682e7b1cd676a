// resnet_ops.cu -- the memory-bound kernels a ResNet trunk adds around the tensor-core convolutions (SURVEY.md 8f rank 2,
// BASELINE config #4).  The reference's trunk is chainer.links.model.vision.resnet.ResNetLayers (un-vendored;
// /root/reference models/resnet.py:11-45 only subclasses it and returns 'res5'); its published structure is restated:
//   conv1 7x7/2 pad 3 + BN + ReLU          -> frcnn_pack_image_im2col (K = 147 -> 160) + a 1x1 tensor-core GEMM (BN folded)
//   pool1 max 3x3/2, pad 0, cover_all      -> frcnn_maxpool3x3s2_ceil
//   bottleneck 1x1(/s) - 3x3 - 1x1 + shortcut, BN folded into every conv, ReLU after the add
//                                          -> frcnn_conv2d / frcnn_conv2d_res (residual add fused into the epilogue);
//                                             a stride-2 1x1 convolution = frcnn_subsample2x + a stride-1 1x1 convolution
// All three kernels are HBM-bound: 16-byte accesses along the channel axis of the NHWC bf16 hi/lo planes.
// frcnn_preprocess_bgr8_canvas_im2col feeds conv1 of a canvas batch straight from raw uint8 photos.
#include "common.cuh"
#include "raw_photo.cuh"

namespace frcnn {

// The values of 8 split pairs (pool_pair_value: an infinite hi stands alone, its lo is the NaN of inf - inf).
__device__ __forceinline__ void load8f(const __nv_bfloat16* hi, const __nv_bfloat16* lo, long off, float v[8]) {
    const uint4 h = *reinterpret_cast<const uint4*>(hi + off);
    const __nv_bfloat16* hb = reinterpret_cast<const __nv_bfloat16*>(&h);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = __bfloat162float(hb[j]);
    if (lo) {
        const uint4 l = *reinterpret_cast<const uint4*>(lo + off);
        const __nv_bfloat16* lb = reinterpret_cast<const __nv_bfloat16*>(&l);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = pool_pair_value(v[j], __bfloat162float(lb[j]));
    }
}

__device__ __forceinline__ void store8f(__nv_bfloat16* hi, __nv_bfloat16* lo, long off, const float v[8]) {
    __align__(16) __nv_bfloat16 h[8];
    __align__(16) __nv_bfloat16 l[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) split_bf16(v[j], h[j], l[j]);
    *reinterpret_cast<uint4*>(hi + off) = *reinterpret_cast<const uint4*>(h);
    if (lo) *reinterpret_cast<uint4*>(lo + off) = *reinterpret_cast<const uint4*>(l);
}

// Output size of a ksize / stride / pad convolution over e input pixels (0 when not even one window fits).  C division
// truncates towards zero, so a negative numerator is answered before it is divided.
__host__ __device__ __forceinline__ int conv_out(int e, int ks, int stride, int pad) {
    const int t = e + 2 * pad - ks;
    return t < 0 ? 0 : t / stride + 1;
}

// Output size of the 3x3 / 2, pad 0, cover_all max-pool over c pixels: ceil((c - 3) / 2) + 1 = (c - 2) / 2 + 1, 0 for c <= 1.
__host__ __device__ __forceinline__ int pool3s2_out(int c) { return c < 2 ? 0 : (c - 2) / 2 + 1; }

// General first-layer im2col: (C,H,W) fp32 -> [Ho][Wo][Kp] bf16 hi/lo, K index (r*ks + s)*C + c, zero padded borders,
// zeros for k >= ks*ks*C.  One thread per 8 consecutive k of one output pixel; blockIdx.y is the image of a batch
// ((N,C,H,W) in, [N][Ho][Wo][Kp] out).  extents (a canvas batch; NULL: every image fills H x W): image n is extents[2n] x
// extents[2n+1] input pixels, a tap outside it reads as the zero padding and every output pixel outside
// conv_out(extent) is written as 0.
__global__ void im2col_kernel(const float* __restrict__ x, int C, int H, int W, int ks, int stride, int pad, int Ho, int Wo,
                              int Kp, const int* __restrict__ extents, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const int k8n = Kp / 8;
    const long total = (long)Ho * Wo * k8n;
    const int kmax = ks * ks * C;
    const int img = blockIdx.y;
    x += (long)img * C * H * W;
    hi += (long)img * Ho * Wo * Kp;
    if (lo) lo += (long)img * Ho * Wo * Kp;
    int eh = H, ew = W, oh = Ho, ow = Wo;
    if (extents) {
        eh = canvas_extent(extents, img, 0, 0, H);
        ew = canvas_extent(extents, img, 1, 0, W);
        oh = conv_out(eh, ks, stride, pad);
        ow = conv_out(ew, ks, stride, pad);
    }
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int k8 = (int)(t % k8n);
        const long p = t / k8n;
        const int wo = (int)(p % Wo), ho = (int)(p / Wo);
        const bool live = ho < oh && wo < ow;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = k8 * 8 + j;
            float val = 0.f;
            if (live && k < kmax) {
                const int tap = k / C, c = k - tap * C;
                const int hh = ho * stride - pad + tap / ks, ww = wo * stride - pad + tap % ks;
                if (hh >= 0 && hh < eh && ww >= 0 && ww < ew) val = x[((long)c * H + hh) * W + ww];
            }
            v[j] = val;
        }
        store8f(hi, lo, p * Kp + k8 * 8, v);
    }
}

// Raw photos straight into the first-layer im2col planes of a canvas batch: preprocess_bgr8_kernel (kCubic: the VOC
// dataset's bicubic, cubic_bgr8), a copy into a zeroed canvas and im2col_kernel(extents) for all N slots in one launch, bit
// for bit.  Slot blockIdx.y is raw_slot's; one CTA
// per (band of `band` output rows, tile of `tile` output columns).  The CTA first stages the resized, mean-subtracted input
// window its outputs read -- rows [ho0*stride - pad, +rows), columns [wo0*stride - pad, +cols), float32 [rows][cols][3] in
// shared memory, 0 outside the image's extent -- so each input pixel's bilinear is computed once per CTA instead of once
// per covering output pixel, then writes the tile's [Wo][Kp] rows as 16-byte hi/lo stores, reading every K index through
// a table of its window offset.  Every output pixel outside conv_out(extent) and every k >= ks*ks*3 is written as 0.
// kFlip (cubic only): a slot whose flip[n] is nonzero is resized from its mirrored source (mirror_taps).
struct PreIm2colArgs {
    const unsigned char* arena; long long arena_bytes;
    const long long* src_off; const int* src_hw; const double* inv_scale; const int* extents;
    int Hc, Wc, ks, stride, pad, Kp, Ho, Wo;
    int band, tile, tiles, cols;        // output rows per band, output columns per tile, tiles per band, staged row pitch
    double m0, m1, m2;
    __nv_bfloat16 *hi, *lo;
    const int* flip;                    // kFlip: device int32 [N]
};
template <bool kCubic, bool kFlip = false>
__global__ void __launch_bounds__(256) preprocess_canvas_im2col_kernel(const PreIm2colArgs a) {
    extern __shared__ float smem[];
    const int kmax = a.ks * a.ks * 3;
    int* tab = reinterpret_cast<int*>(smem);           // [kmax]: window offset of K index k
    float* win = smem + kmax;                          // [rows][a.cols][3]
    const int n = blockIdx.y;
    const int ho0 = (int)(blockIdx.x / a.tiles) * a.band, wo0 = (int)(blockIdx.x % a.tiles) * a.tile;
    const int nb = min(a.band, a.Ho - ho0), nt = min(a.tile, a.Wo - wo0);
    const RawSlot s = raw_slot(a.arena, a.arena_bytes, a.src_off, a.src_hw, a.inv_scale, a.extents, n, a.Hc, a.Wc);
    const int oh = conv_out(s.eh, a.ks, a.stride, a.pad), ow = conv_out(s.ew, a.ks, a.stride, a.pad);
    const bool any = ho0 < oh && wo0 < ow;             // CTA-uniform: a tile wholly outside the image only writes zeros
    const bool mirror = kFlip && __ldg(a.flip + n) != 0;
    if (any) {
        for (int k = threadIdx.x; k < kmax; k += blockDim.x) {
            const int tap = k / 3, c = k - tap * 3;
            tab[k] = ((tap / a.ks) * a.cols + tap % a.ks) * 3 + c;
        }
        const int y0 = ho0 * a.stride - a.pad, x0 = wo0 * a.stride - a.pad;
        const int rows = a.stride * (nb - 1) + a.ks, cols = a.stride * (nt - 1) + a.ks;
        for (int p = threadIdx.x; p < rows * cols; p += blockDim.x) {
            const int i = p / cols, j = p - i * cols, y = y0 + i, x = x0 + j;
            float v[3] = {0.0f, 0.0f, 0.0f};
            if (y >= 0 && y < s.eh && x >= 0 && x < s.ew) {
                if (kCubic && kFlip) {
                    CubicTap tx = cubic_tap(x, s.inv_scale, s.w0);
                    if (mirror) mirror_taps(tx, s.w0);
                    cubic_bgr8(s.src, s.w0, cubic_tap(y, s.inv_scale, s.h0), tx, x, s.ew, a.m0, a.m1, a.m2, v);
                } else if (kCubic)
                    cubic_bgr8(s.src, s.w0, cubic_tap(y, s.inv_scale, s.h0), cubic_tap(x, s.inv_scale, s.w0), x, s.ew, a.m0, a.m1,
                               a.m2, v);
                else
                    bilinear_bgr8(s.src, s.w0, bilinear_tap(y, s.inv_scale, s.h0), bilinear_tap(x, s.inv_scale, s.w0), a.m0, a.m1,
                                  a.m2, v);
            }
            float* w = win + (i * a.cols + j) * 3;
            w[0] = v[0];
            w[1] = v[1];
            w[2] = v[2];
        }
    }
    __syncthreads();
    const int k8n = a.Kp / 8;
    const long img = (long)n * a.Ho * a.Wo;
    for (int t = threadIdx.x; t < nb * nt * k8n; t += blockDim.x) {
        const int k8 = t % k8n, q = t / k8n, wl = q % nt, hl = q / nt;
        const bool live = any && ho0 + hl < oh && wo0 + wl < ow;
        const float* w = win + (hl * a.stride * a.cols + wl * a.stride) * 3;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = k8 * 8 + j;
            v[j] = live && k < kmax ? w[tab[k]] : 0.0f;
        }
        store8f(a.hi, a.lo, ((img + (long)(ho0 + hl) * a.Wo + wo0 + wl) * a.Kp) + k8 * 8, v);
    }
}

// The VOC dataset's box scaling on the device: gt[n][g] = (f32(box) * f32(im_scale) for the four coordinates, the label
// unchanged) for g < count[n] (clamped to [0, max_gt]), 0 for the rows after it; gt_counts[n] = that count.  One thread per
// (slot, row, column).  kFlip: a slot whose flip[n] is nonzero first mirrors its boxes in the photo's w0 = src_hw[2n+1]
// columns, py-faster-rcnn's inclusive flip in float32: x1' = (f32(w0) - x2) - 1, x2' = (f32(w0) - x1) - 1.
template <bool kFlip>
__global__ void voc_scale_gt_kernel(const float* __restrict__ scale, const int* __restrict__ count, const float* __restrict__ raw,
                                    const int* __restrict__ src_hw, const int* __restrict__ flip, int N, int max_gt,
                                    float* __restrict__ gt, int* __restrict__ gt_counts) {
    const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (i >= (long)N * max_gt * 5) return;
    const int n = (int)(i / ((long)max_gt * 5)), g = (int)(i / 5 % max_gt), j = (int)(i % 5);
    const int cnt = min(max(__ldg(count + n), 0), max_gt);
    float v = raw[i];
    if (kFlip && (j == 0 || j == 2) && __ldg(flip + n) != 0)
        v = __fsub_rn(__fsub_rn((float)__ldg(src_hw + 2 * n + 1), raw[j == 0 ? i + 2 : i - 2]), 1.0f);
    gt[i] = g < cnt ? (j < 4 ? __fmul_rn(v, __ldg(scale + n)) : v) : 0.0f;
    if (g == 0 && j == 0) gt_counts[n] = cnt;
}

// frcnn_voc_augment_batch: one thread per slot.  draw 1 / 2 first writes the slot's aug_draw into choice (2: the flip as 0);
// then the chosen candidate (index clamped to [0, S-1]) becomes the slot's descriptors.  A slot without a source stays
// empty: extent and clip bounds 0 x 0, inv_scale, scale and flip 0.
__global__ void voc_augment_kernel(const unsigned long long* __restrict__ seeds, int N, int S, const int* __restrict__ cand_hw,
                                   const double* __restrict__ cand_inv, const float* __restrict__ cand_scale,
                                   const int* __restrict__ src_hw, int draw, int* __restrict__ choice, int* __restrict__ flip,
                                   int* __restrict__ extents, int* __restrict__ im_info, double* __restrict__ inv_scale,
                                   float* __restrict__ scale) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    if (draw) {
        int f, k;
        aug_draw(__ldg(seeds + n), S, f, k);
        choice[2 * n] = draw == 1 ? f : 0;
        choice[2 * n + 1] = k;
    }
    const int k = min(max(choice[2 * n + 1], 0), S - 1), c = n * S + k;
    const bool live = __ldg(src_hw + 2 * n) > 0 && __ldg(src_hw + 2 * n + 1) > 0;
    const int h = live ? __ldg(cand_hw + 2 * c) : 0, w = live ? __ldg(cand_hw + 2 * c + 1) : 0;
    extents[2 * n] = im_info[2 * n] = h;
    extents[2 * n + 1] = im_info[2 * n + 1] = w;
    inv_scale[n] = live ? __ldg(cand_inv + c) : 0.0;
    scale[n] = live ? __ldg(cand_scale + c) : 0.0f;
    flip[n] = live && choice[2 * n] != 0 ? 1 : 0;
}

// OIHW (Cout, C, ks, ks) fp32 -> [1][Cout][Kp] bf16 hi/lo in the K order of im2col_kernel; scale[o] (optional) multiplies
// output channel o (a folded test-mode BatchNorm).
__global__ void pack_weights_im2col_general_kernel(const float* __restrict__ w, const float* __restrict__ scale, int Cout, int C,
                                                   int ks, int Kp, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Cout * Kp) return;
    const int o = i / Kp, k = i % Kp;
    float v = 0.f;
    if (k < ks * ks * C) {
        const int tap = k / C, c = k % C;
        v = w[((long)o * C + c) * ks * ks + tap];
        if (scale) v = __fmul_rn(v, scale[o]);
    }
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
}

// F.max_pooling_2d(x, 3, stride=2) with Chainer's defaults pad=0, cover_all=True: Ho = ceil((H-3)/2) + 1, windows clipped
// at the bottom / right border.  blockIdx.y is the image of a batch ([N][H][W][C] -> [N][Ho][Wo][C]).  extents (a canvas
// batch of N images, each at the top-left of its H x W slot, at THIS map's resolution; NULL: H x W each): a window is
// clipped at the image's own border exactly as at the slot's, so no pixel outside the image is ever read, and every output
// pixel outside pool3s2_out(extent) is written as 0.
__global__ void maxpool3x3s2_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl, int H, int W, int C,
                                    int Ho, int Wo, const int* __restrict__ extents, __nv_bfloat16* __restrict__ yh,
                                    __nv_bfloat16* __restrict__ yl) {
    const int C8 = C / 8;
    const long total = (long)Ho * Wo * C8;
    const int img = blockIdx.y;
    xh += (long)img * H * W * C;
    if (xl) xl += (long)img * H * W * C;
    yh += (long)img * Ho * Wo * C;
    if (yl) yl += (long)img * Ho * Wo * C;
    int eh = H, ew = W, oh = Ho, ow = Wo;
    if (extents) {
        eh = canvas_extent(extents, img, 0, 0, H);
        ew = canvas_extent(extents, img, 1, 0, W);
        oh = pool3s2_out(eh);
        ow = pool3s2_out(ew);
    }
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        const long p = i / C8;
        const int wo = (int)(p % Wo), ho = (int)(p / Wo);
        float m[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = 0.f;
        if (ho < oh && wo < ow) {           // the window's first pixel (2ho, 2wo) lies inside the image
            bool first = true;
            for (int dy = 0; dy < 3; ++dy) {
                const int h = ho * 2 + dy;
                if (h >= eh) break;
                for (int dx = 0; dx < 3; ++dx) {
                    const int w = wo * 2 + dx;
                    if (w >= ew) break;
                    float v[8];
                    load8f(xh, xl, ((long)h * W + w) * C + c8 * 8, v);
#pragma unroll
                    for (int j = 0; j < 8; ++j) m[j] = first ? v[j] : fmaxf(m[j], v[j]);
                    first = false;
                }
            }
        }
        store8f(yh, yl, p * C + c8 * 8, m);
    }
}

// pixels (2h, 2w): the input of a stride-2, pad-0 1x1 convolution; blockIdx.y is the image of a batch
__global__ void subsample2x_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl, int H, int W, int C,
                                   int Ho, int Wo, __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl) {
    const int C8 = C / 8;
    const long total = (long)Ho * Wo * C8;
    const long xo = (long)blockIdx.y * H * W * C, yo = (long)blockIdx.y * Ho * Wo * C;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        const long p = i / C8;
        const int wo = (int)(p % Wo), ho = (int)(p / Wo);
        const long src = xo + ((long)(2 * ho) * W + 2 * wo) * C + c8 * 8, dst = yo + p * C + c8 * 8;
        *reinterpret_cast<uint4*>(yh + dst) = *reinterpret_cast<const uint4*>(xh + src);
        if (xl) *reinterpret_cast<uint4*>(yl + dst) = *reinterpret_cast<const uint4*>(xl + src);
    }
}

// The per-level extents of a ResNet canvas batch: out [5][N][2] = conv1, pool1, res3, res4, res5 (res2 keeps pool1's),
// each clamped to that level's canvas size.  One thread per image.
__global__ void resnet_level_extents_kernel(const int* __restrict__ extents, int N, int Hc, int Wc, int* __restrict__ out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    for (int axis = 0; axis < 2; ++axis) {
        int lim = axis ? Wc : Hc;
        int e = canvas_extent(extents, n, axis, 0, lim);
        lim = conv_out(lim, 7, 2, 3);
        e = min(conv_out(e, 7, 2, 3), lim);
        out[(0 * N + n) * 2 + axis] = e;
        lim = pool3s2_out(lim);
        e = min(pool3s2_out(e), lim);
        out[(1 * N + n) * 2 + axis] = e;
        for (int k = 2; k < 5; ++k) {
            lim = (lim + 1) / 2;
            e = min((e + 1) / 2, lim);
            out[(k * N + n) * 2 + axis] = e;
        }
    }
}

// frcnn_preprocess_bgr8_canvas_im2col: the shared memory of one CTA (the K table and the staged window), and the largest
// filter whose one-output-pixel window (4 + 12 bytes per K index and window pixel) fits it
static const size_t PRE_IM2COL_SMEM = 48 * 1024;
static const int PRE_IM2COL_MAX_KSIZE = 45;

static int grid_cover(long total, int block) {
    long g = (total + block - 1) / block;
    const long cap = 132l * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace frcnn

using namespace frcnn;

// the launches behind the one-image, batch and canvas-batch entries
static int im2col_launch(const float* x, int N, int C, int H, int W, int ksize, int stride, int pad, int K_pad, const int* extents,
                         void* y_hi, void* y_lo, void* stream) {
    FRCNN_REQUIRE(x && y_hi && C > 0 && H > 0 && W > 0 && ksize > 0 && stride > 0 && pad >= 0, "pack_image_im2col: bad arguments");
    FRCNN_REQUIRE(K_pad % 8 == 0 && K_pad >= ksize * ksize * C, "pack_image_im2col: K_pad must be a multiple of 8 and >= ksize^2*C");
    const int Ho = conv_out(H, ksize, stride, pad), Wo = conv_out(W, ksize, stride, pad);
    FRCNN_REQUIRE(Ho > 0 && Wo > 0, "pack_image_im2col: image smaller than the filter");
    const long total = (long)Ho * Wo * (K_pad / 8);
    im2col_kernel<<<dim3(grid_cover(total, 256), N), 256, 0, (cudaStream_t)stream>>>(x, C, H, W, ksize, stride, pad, Ho, Wo, K_pad,
                                                                                  extents, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

static int maxpool3x3s2_launch(const void* x_hi, const void* x_lo, int N, int H, int W, int C, const int* extents, void* y_hi,
                               void* y_lo, void* stream) {
    FRCNN_REQUIRE(x_hi && y_hi && H >= 3 && W >= 3 && C > 0 && C % 8 == 0, "maxpool3x3s2_ceil: bad arguments (H=%d W=%d C=%d)", H, W, C);
    FRCNN_REQUIRE((x_lo == nullptr) == (y_lo == nullptr), "maxpool3x3s2_ceil: lo planes must both be given or both NULL");
    const int Ho = pool3s2_out(H), Wo = pool3s2_out(W);
    const long total = (long)Ho * Wo * (C / 8);
    maxpool3x3s2_kernel<<<dim3(grid_cover(total, 256), N), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x_hi, (const __nv_bfloat16*)x_lo, H, W, C, Ho, Wo, extents, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

static int subsample2x_launch(const void* x_hi, const void* x_lo, int N, int H, int W, int C, void* y_hi, void* y_lo, void* stream) {
    FRCNN_REQUIRE(x_hi && y_hi && H > 0 && W > 0 && C > 0 && C % 8 == 0, "subsample2x: bad arguments");
    FRCNN_REQUIRE((x_lo == nullptr) == (y_lo == nullptr), "subsample2x: lo planes must both be given or both NULL");
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    const long total = (long)Ho * Wo * (C / 8);
    subsample2x_kernel<<<dim3(grid_cover(total, 256), N), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x_hi, (const __nv_bfloat16*)x_lo, H, W, C, Ho, Wo, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" {

int frcnn_pack_image_im2col(const float* x_chw, int C, int H, int W, int ksize, int stride, int pad, int K_pad, void* y_hi,
                            void* y_lo, void* stream) {
    FRCNN_ENTRY();
    return im2col_launch(x_chw, 1, C, H, W, ksize, stride, pad, K_pad, nullptr, y_hi, y_lo, stream);
}

int frcnn_pack_image_im2col_batch(const float* x_nchw, int N, int C, int H, int W, int ksize, int stride, int pad, int K_pad,
                                  void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "pack_image_im2col_batch: N must be in [1, 65535] (got %d)", N);
    return im2col_launch(x_nchw, N, C, H, W, ksize, stride, pad, K_pad, nullptr, y_hi, y_lo, stream);
}

int frcnn_pack_image_im2col_batch_ext(const float* x_nchw, int N, int C, int H, int W, int ksize, int stride, int pad, int K_pad,
                                      const int* extents, void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535 && extents, "pack_image_im2col_batch_ext: needs N in [1, 65535] (got %d) and the device extents", N);
    return im2col_launch(x_nchw, N, C, H, W, ksize, stride, pad, K_pad, extents, y_hi, y_lo, stream);
}

}  // extern "C"

// the launch behind frcnn_preprocess_bgr8_canvas_im2col (bilinear), frcnn_preprocess_voc_canvas_im2col (cubic) and
// frcnn_preprocess_voc_canvas_im2col_flip (cubic, mirrored where flip[n] is nonzero; flip NULL for the other two)
static int preprocess_canvas_im2col_launch(const char* fn, bool cubic, const unsigned char* arena, long long arena_bytes,
                                           const long long* src_off, const int* src_hw, const double* inv_scale, const int* extents,
                                           int N, int Hc, int Wc, double mean_b, double mean_g, double mean_r, int ksize, int stride,
                                           int pad, int K_pad, void* y_hi, void* y_lo, void* stream, const int* flip = nullptr) {
    FRCNN_REQUIRE(arena, "%s: arena is NULL", fn);
    FRCNN_REQUIRE(arena_bytes > 0, "%s: arena_bytes must be positive (got %lld)", fn, arena_bytes);
    FRCNN_REQUIRE(src_off, "%s: src_off is NULL", fn);
    FRCNN_REQUIRE(src_hw, "%s: src_hw is NULL", fn);
    FRCNN_REQUIRE(inv_scale, "%s: inv_scale is NULL", fn);
    FRCNN_REQUIRE(extents, "%s: extents is NULL", fn);
    FRCNN_REQUIRE(y_hi, "%s: y_hi is NULL", fn);
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "%s: needs 1 <= N <= 65535 (got N=%d)", fn, N);
    FRCNN_REQUIRE(Hc > 0 && Wc > 0, "%s: the canvas must be positive (got Hc=%d Wc=%d)", fn, Hc, Wc);
    FRCNN_REQUIRE(ksize > 0 && ksize <= PRE_IM2COL_MAX_KSIZE, "%s: needs 1 <= ksize <= %d (got ksize=%d)", fn, PRE_IM2COL_MAX_KSIZE,
                  ksize);
    FRCNN_REQUIRE(stride > 0, "%s: stride must be positive (got stride=%d)", fn, stride);
    FRCNN_REQUIRE(pad >= 0 && 2ll * pad + (Hc > Wc ? Hc : Wc) <= (1ll << 30),
                  "%s: pad must be >= 0 with 2*pad + the canvas side <= 2^30 (got pad=%d)", fn, pad);
    const int kmax = ksize * ksize * 3;
    FRCNN_REQUIRE(K_pad % 8 == 0 && K_pad >= kmax && K_pad <= 65536,
                  "%s: K_pad must be a multiple of 8 in [3*ksize^2 = %d, 65536] (got K_pad=%d)", fn, kmax, K_pad);
    const int Ho = conv_out(Hc, ksize, stride, pad), Wo = conv_out(Wc, ksize, stride, pad);
    FRCNN_REQUIRE(Ho > 0 && Wo > 0, "%s: canvas %dx%d smaller than the filter (ksize=%d pad=%d)", fn, Hc, Wc, ksize, pad);
    PreIm2colArgs a;
    a.arena = arena; a.arena_bytes = arena_bytes;
    a.src_off = src_off; a.src_hw = src_hw; a.inv_scale = inv_scale; a.extents = extents;
    a.Hc = Hc; a.Wc = Wc; a.ks = ksize; a.stride = stride; a.pad = pad; a.Kp = K_pad; a.Ho = Ho; a.Wo = Wo;
    a.m0 = mean_b; a.m1 = mean_g; a.m2 = mean_r;
    a.hi = (__nv_bfloat16*)y_hi; a.lo = (__nv_bfloat16*)y_lo;
    a.flip = flip;
    // the tile: up to 8 output rows, then as many output columns as the window fits PRE_IM2COL_SMEM (the K table comes
    // first); PRE_IM2COL_MAX_KSIZE guarantees one output pixel's window fits
    const int px = (int)((PRE_IM2COL_SMEM - (size_t)kmax * 4) / 12);
    a.band = Ho < 8 ? Ho : 8;
    while (a.band > 1 && ((long)stride * (a.band - 1) + ksize) * ksize > px) --a.band;
    const int rows = stride * (a.band - 1) + ksize;
    const int k8n = K_pad / 8;
    a.tile = (px / rows - ksize) / stride + 1;
    a.tile = a.tile < Wo ? a.tile : Wo;
    const int cap = (int)((0x7fffffffl / a.band) / k8n);         // band * tile * K_pad / 8 thread items stay an int
    a.tile = a.tile < cap ? a.tile : (cap > 1 ? cap : 1);
    a.cols = stride * (a.tile - 1) + ksize;
    a.tiles = cdiv(Wo, a.tile);
    const long blocks = (long)cdiv(Ho, a.band) * a.tiles;
    FRCNN_REQUIRE(blocks <= 0x7fffffffl, "%s: canvas %dx%d needs too many tiles", fn, Hc, Wc);
    const size_t smem = (size_t)kmax * 4 + (size_t)rows * a.cols * 12;
    if (flip)
        preprocess_canvas_im2col_kernel<true, true><<<dim3((unsigned)blocks, N), 256, smem, (cudaStream_t)stream>>>(a);
    else if (cubic)
        preprocess_canvas_im2col_kernel<true><<<dim3((unsigned)blocks, N), 256, smem, (cudaStream_t)stream>>>(a);
    else
        preprocess_canvas_im2col_kernel<false><<<dim3((unsigned)blocks, N), 256, smem, (cudaStream_t)stream>>>(a);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" {

int frcnn_preprocess_bgr8_canvas_im2col(const unsigned char* arena, long long arena_bytes, const long long* src_off,
                                        const int* src_hw, const double* inv_scale, const int* extents, int N, int Hc, int Wc,
                                        double mean_b, double mean_g, double mean_r, int ksize, int stride, int pad, int K_pad,
                                        void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    return preprocess_canvas_im2col_launch("frcnn_preprocess_bgr8_canvas_im2col", false, arena, arena_bytes, src_off, src_hw,
                                           inv_scale, extents, N, Hc, Wc, mean_b, mean_g, mean_r, ksize, stride, pad, K_pad, y_hi,
                                           y_lo, stream);
}

int frcnn_preprocess_voc_canvas_im2col(const unsigned char* arena, long long arena_bytes, const long long* src_off,
                                       const int* src_hw, const double* inv_scale, const int* extents, int N, int Hc, int Wc,
                                       double mean_b, double mean_g, double mean_r, int ksize, int stride, int pad, int K_pad,
                                       void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    return preprocess_canvas_im2col_launch("frcnn_preprocess_voc_canvas_im2col", true, arena, arena_bytes, src_off, src_hw,
                                           inv_scale, extents, N, Hc, Wc, mean_b, mean_g, mean_r, ksize, stride, pad, K_pad, y_hi,
                                           y_lo, stream);
}

int frcnn_preprocess_voc_canvas_im2col_flip(const unsigned char* arena, long long arena_bytes, const long long* src_off,
                                            const int* src_hw, const double* inv_scale, const int* extents, const int* flip, int N,
                                            int Hc, int Wc, double mean_b, double mean_g, double mean_r, int ksize, int stride,
                                            int pad, int K_pad, void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(flip, "frcnn_preprocess_voc_canvas_im2col_flip: flip is NULL");
    return preprocess_canvas_im2col_launch("frcnn_preprocess_voc_canvas_im2col_flip", true, arena, arena_bytes, src_off, src_hw,
                                           inv_scale, extents, N, Hc, Wc, mean_b, mean_g, mean_r, ksize, stride, pad, K_pad, y_hi,
                                           y_lo, stream, flip);
}

}  // extern "C"

// the launch behind frcnn_voc_scale_gt_batch (src_hw and flip NULL) and frcnn_voc_flip_scale_gt_batch
static int voc_scale_gt_launch(const char* fn, const float* scale, const int* count, const float* raw_gt, const int* src_hw,
                               const int* flip, int N, int max_gt, float* gt, int* gt_counts, void* stream) {
    FRCNN_REQUIRE(scale && count && raw_gt && gt && gt_counts, "%s: NULL argument", fn);
    FRCNN_REQUIRE(N >= 1 && N <= 65535 && max_gt >= 1 && max_gt <= (1 << 20),
                  "%s: needs 1 <= N <= 65535 and 1 <= max_gt <= 2^20 (got N=%d max_gt=%d)", fn, N, max_gt);
    const long total = (long)N * max_gt * 5;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (flip)
        voc_scale_gt_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(scale, count, raw_gt, src_hw, flip, N, max_gt, gt, gt_counts);
    else
        voc_scale_gt_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(scale, count, raw_gt, src_hw, flip, N, max_gt, gt, gt_counts);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

extern "C" {

int frcnn_voc_scale_gt_batch(const float* scale, const int* count, const float* raw_gt, int N, int max_gt, float* gt, int* gt_counts,
                             void* stream) {
    FRCNN_ENTRY();
    return voc_scale_gt_launch("frcnn_voc_scale_gt_batch", scale, count, raw_gt, nullptr, nullptr, N, max_gt, gt, gt_counts, stream);
}

int frcnn_voc_flip_scale_gt_batch(const float* scale, const int* count, const float* raw_gt, const int* src_hw, const int* flip,
                                  int N, int max_gt, float* gt, int* gt_counts, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(src_hw && flip, "frcnn_voc_flip_scale_gt_batch: NULL argument");
    return voc_scale_gt_launch("frcnn_voc_flip_scale_gt_batch", scale, count, raw_gt, src_hw, flip, N, max_gt, gt, gt_counts, stream);
}

int frcnn_voc_augment_batch(const unsigned long long* seeds, int N, int S, const int* cand_hw, const double* cand_inv,
                            const float* cand_scale, const int* src_hw, int draw, int* choice, int* flip, int* extents, int* im_info,
                            double* inv_scale, float* scale, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(cand_hw && cand_inv && cand_scale && src_hw && choice && flip && extents && im_info && inv_scale && scale,
                  "frcnn_voc_augment_batch: NULL argument");
    FRCNN_REQUIRE(draw >= 0 && draw <= 2, "frcnn_voc_augment_batch: draw must be 0, 1 or 2 (got %d)", draw);
    FRCNN_REQUIRE(seeds || !draw, "frcnn_voc_augment_batch: a draw needs the seeds");
    FRCNN_REQUIRE(N >= 1 && N <= 65535 && S >= 1 && S <= 8,
                  "frcnn_voc_augment_batch: needs 1 <= N <= 65535 and 1 <= S <= 8 (got N=%d S=%d)", N, S);
    voc_augment_kernel<<<cdiv(N, 128), 128, 0, (cudaStream_t)stream>>>(seeds, N, S, cand_hw, cand_inv, cand_scale, src_hw, draw,
                                                                       choice, flip, extents, im_info, inv_scale, scale);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_pack_conv_weights_im2col(const float* w_oihw, const float* scale, int Cout, int Cin, int ksize, int K_pad, void* w_hi,
                                   void* w_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(w_oihw && w_hi && Cout > 0 && Cin > 0 && ksize > 0 && K_pad % 8 == 0 && K_pad >= ksize * ksize * Cin,
                  "pack_conv_weights_im2col: bad arguments");
    pack_weights_im2col_general_kernel<<<cdiv(Cout * K_pad, 256), 256, 0, (cudaStream_t)stream>>>(
        w_oihw, scale, Cout, Cin, ksize, K_pad, (__nv_bfloat16*)w_hi, (__nv_bfloat16*)w_lo);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_maxpool3x3s2_ceil(const void* x_hi, const void* x_lo, int H, int W, int C, void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    return maxpool3x3s2_launch(x_hi, x_lo, 1, H, W, C, nullptr, y_hi, y_lo, stream);
}

int frcnn_maxpool3x3s2_ceil_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int C, void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "maxpool3x3s2_ceil_batch: N must be in [1, 65535] (got %d)", N);
    return maxpool3x3s2_launch(x_hi, x_lo, N, H, W, C, nullptr, y_hi, y_lo, stream);
}

int frcnn_maxpool3x3s2_ceil_batch_ext(const void* x_hi, const void* x_lo, int N, int H, int W, int C, const int* extents, void* y_hi,
                                      void* y_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535 && extents, "maxpool3x3s2_ceil_batch_ext: needs N in [1, 65535] (got %d) and the device extents", N);
    return maxpool3x3s2_launch(x_hi, x_lo, N, H, W, C, extents, y_hi, y_lo, stream);
}

int frcnn_subsample2x(const void* x_hi, const void* x_lo, int H, int W, int C, void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    return subsample2x_launch(x_hi, x_lo, 1, H, W, C, y_hi, y_lo, stream);
}

int frcnn_subsample2x_batch(const void* x_hi, const void* x_lo, int N, int H, int W, int C, void* y_hi, void* y_lo, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(N >= 1 && N <= 65535, "subsample2x_batch: N must be in [1, 65535] (got %d)", N);
    return subsample2x_launch(x_hi, x_lo, N, H, W, C, y_hi, y_lo, stream);
}

int frcnn_resnet_level_extents(const int* extents, int N, int Hc, int Wc, int* out, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(extents && out, "resnet_level_extents: NULL extents or output");
    FRCNN_REQUIRE(N >= 1 && N <= 65535 && Hc > 0 && Wc > 0, "resnet_level_extents: bad shape N=%d Hc=%d Wc=%d", N, Hc, Wc);
    resnet_level_extents_kernel<<<cdiv(N, 128), 128, 0, (cudaStream_t)stream>>>(extents, N, Hc, Wc, out);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

}  // extern "C"
