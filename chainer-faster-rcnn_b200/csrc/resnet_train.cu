// resnet_train.cu -- what training the ResNet trunk adds to the conv backward of train_backward.cu, with BatchNorm frozen
// (test-mode statistics and affine are constants; DESIGN §2).  A convolution followed by its frozen BN is the folded
// convolution Wf = W * s, bf = beta + (b - mean) * s, s = gamma / sqrt(var + eps) per output channel, so
//   forward and data gradient   run on the folded weights, which frcnn_fold_batchnorm rebuilds from the fp32 masters at
//                               every repack with the float64 arithmetic of resnet_engine.fold_batchnorm;
//   weight / bias gradient      dW = s[co] * sum_pixels dz (x) x and db = s * sum dz: the split-K partials (or the bias
//                               sums) of the folded convolution, reduced in fixed order and scaled per output channel by
//                               frcnn_wgrad_reduce_scaled.
// The 3x3/2 max-pool backward and the stride-2 scatter are modes of the grad_prepare kernel (train_backward.cu), whose
// transposed re-layout they share.
#include "common.cuh"

namespace frcnn {

// dw[m][n][g] = f32(f64(s[m]) * f64(sum over splits of parts[g][s][m][n])), the split sum in fp32 in ascending order
__global__ void wgrad_reduce_scaled_kernel(const float* __restrict__ parts, int groups, int splits, int Mp, int M, int ld, int N,
                                           const double* __restrict__ s, float* __restrict__ dw) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long total = (long)M * N * groups;
    if (t >= total) return;
    const int g = (int)(t % groups);
    const long mn = t / groups;
    const int n = (int)(mn % N), m = (int)(mn / N);
    float acc = 0.f;
    for (int k = 0; k < splits; ++k) acc = __fadd_rn(acc, parts[(((long)g * splits + k) * Mp + m) * ld + n]);
    dw[t] = __double2float_rn(__dmul_rn(s[m], (double)acc));
}

// wf[i] = f32(f64(w[i]) * s[i / per_out]);  bf[c] = f32(f64(beta[c]) + (f64(b[c]) - f64(mean[c])) * s[c]), b = 0 when NULL
__global__ void fold_batchnorm_kernel(const float* __restrict__ w, const double* __restrict__ s, int Cout, long per_out,
                                      const float* __restrict__ b, const float* __restrict__ beta, const float* __restrict__ mean,
                                      float* __restrict__ wf, float* __restrict__ bf) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (long)Cout * per_out) wf[i] = __double2float_rn(__dmul_rn((double)w[i], s[i / per_out]));
    if (bf != nullptr && i < Cout) {
        const double b0 = b != nullptr ? (double)b[i] : 0.0;
        bf[i] = __double2float_rn(__dadd_rn((double)beta[i], __dmul_rn(__dsub_rn(b0, (double)mean[i]), s[i])));
    }
}

}  // namespace frcnn

using namespace frcnn;

extern "C" {

int frcnn_wgrad_reduce_scaled(const float* parts, int groups, int splits, int M_parts, int M, int ld, int N, const double* s,
                              float* dw, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(parts && s && dw, "wgrad_reduce_scaled: NULL parts, scale or output");
    FRCNN_REQUIRE(groups >= 1 && splits >= 1 && M > 0 && M_parts >= M && N > 0 && ld >= N,
                  "wgrad_reduce_scaled: bad shape groups=%d splits=%d M_parts=%d M=%d ld=%d N=%d", groups, splits, M_parts, M, ld, N);
    const long total = (long)M * N * groups;
    FRCNN_REQUIRE(total < (1l << 40), "wgrad_reduce_scaled: too many elements");
    wgrad_reduce_scaled_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(parts, groups, splits, M_parts, M,
                                                                                                 ld, N, s, dw);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

int frcnn_fold_batchnorm(const float* w, const double* s, int Cout, long per_out, const float* b, const float* beta,
                         const float* mean, float* wf, float* bf, void* stream) {
    FRCNN_ENTRY();
    FRCNN_REQUIRE(w && s && wf, "fold_batchnorm: NULL weights, scale or output");
    FRCNN_REQUIRE(Cout > 0 && per_out > 0 && (long)Cout * per_out < (1l << 40), "fold_batchnorm: bad shape Cout=%d per_out=%ld",
                  Cout, per_out);
    FRCNN_REQUIRE(!bf || (beta && mean), "fold_batchnorm: the folded bias needs beta and mean");
    const long total = (long)Cout * per_out > Cout ? (long)Cout * per_out : Cout;
    fold_batchnorm_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, s, Cout, per_out, b, beta, mean, wf,
                                                                                            bf);
    FRCNN_LAUNCH_OK();
    return FRCNN_OK;
}

}  // extern "C"
