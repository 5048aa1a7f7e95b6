// t2_batchnorm.h — the convolution-block batch norm of the Tacotron and CBHG engines and their bias-gradient column sums
// (defined in t2_batchnorm.cu).
//
// tf.layers.batch_normalization after the activation: eps 1e-3, momentum 0.99, biased batch variance. The batch norm works on the
// column slice [c0, c0 + C) of row-pitch-ld matrices, so that the CBHG conv bank can keep its layers side by side in one matrix while
// every layer owns its own gamma / beta / moving tensors. The statistics buffer has four sections of Ct floats, indexed by the
// absolute column: sum of (y - y[0]) | sum of its squares | mean | rstd. Shifting the sums by the column's first row (a sample of the
// column) keeps the variance free of the cancellation that E[y^2] - mean^2 suffers when |mean| >> std.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace t2 {

// inverted dropout after the batch norm: keep probability 1 - p, hash stream `stream` of seed + *step (step nullable). p = 0 is off.
// The hash index is the dense element index r * C + c of the layer, whatever the slice.
struct BnDropout {
  float p;
  unsigned long long seed;
  const unsigned long long* step;
  int stream;
};

// Forward. Training: 64 blocks of stat_threads threads add the shifted sums into stats (the caller zeroes the two sum sections first),
// then mean / rstd are written into stats and the moving statistics updated; inference reads the moving statistics and does not touch
// stats. x = (y - mean) rstd gamma + beta, + add (fp32 [rows][C], nullable), then dropout (training only). Outputs (each nullable):
// xb bf16 at the pitch and slice of y, or with split its rows [hi(ld) | lo(ld)] at pitch 2 ld; xf fp32 [rows][C].
template <typename TY>
void bn_fwd(const TY* y, int ld, int c0, __nv_bfloat16* xb, int split, float* xf, const float* add, float* stats, int Ct, const float* gamma,
            const float* beta, float* mm, float* mv, long long rows, int C, int training, const BnDropout& drop, int stat_threads,
            cudaStream_t st);
// Backward from g (pitch ldg, same column slice; dropout regenerated with the forward's hash): 64 blocks of stat_threads threads add
// sum g | sum g xhat into bsum (two sections of Ct floats, zeroed by the caller), then dpre (bf16, pitch ldd, same column slice) =
// act'(y) gamma rstd (g - mean(g) - xhat mean(g xhat)) with act 0 none, 1 relu, 2 tanh; dgamma / dbeta accumulate.
template <typename T>
void bn_bwd(const T* g, int ldg, const T* y, int ld, int c0, const float* stats, int Ct, float* bsum, const float* gamma, __nv_bfloat16* dpre,
            int ldd, float* dgamma, float* dbeta, long long rows, int C, int act, const BnDropout& drop, int stat_threads, cudaStream_t st);

// dst[c] += sum over rows of src[r * ld + c], c < C (64 blocks of `threads` threads, fp32 atomics)
template <typename TS>
void colsum(const TS* src, long long rows, int C, int ld, float* dst, int threads, cudaStream_t st);

}  // namespace t2
