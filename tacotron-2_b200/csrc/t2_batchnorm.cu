// t2_batchnorm.cu — conv-block batch norm and bias-gradient column sums shared by the Tacotron and CBHG engines (see t2_batchnorm.h).
#include "t2_batchnorm.h"
#include "t2_common.cuh"
#include "t2_params.h"

namespace t2 {
namespace {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ float ldv(const bf16* p, long long i) { return __bfloat162float(p[i]); }
__device__ __forceinline__ float ldv(const float* p, long long i) { return p[i]; }

__device__ __forceinline__ float dropout(float v, const BnDropout& d, uint32_t hs, long long idx) {
  return hash_uniform32(hs, (unsigned long long)idx) >= d.p ? v / (1.f - d.p) : 0.f;
}
__device__ __forceinline__ uint32_t dropout_seed(const BnDropout& d) {
  return hash_seed(d.step ? d.seed + *d.step : d.seed, uint32_t(d.stream));
}

template <typename TY>
__global__ void bn_stats_kernel(const TY* __restrict__ y, int ld, int c0, float* __restrict__ stats, int Ct, long long rows, int C) {
  const long long per = (rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = blockIdx.x * per, r1 = r0 + per < rows ? r0 + per : rows;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float pv = ldv(y, c0 + c);
    float s = 0.f, q = 0.f;
    for (long long r = r0; r < r1; ++r) { const float v = ldv(y, r * ld + c0 + c) - pv; s += v; q += v * v; }
    atomicAdd(stats + c0 + c, s); atomicAdd(stats + Ct + c0 + c, q);
  }
}
// order: affine, + add, dropout
template <typename TY>
__global__ void bn_apply_kernel(const TY* __restrict__ y, int ld, int c0, bf16* __restrict__ xb, int split, float* __restrict__ xf,
                                const float* __restrict__ add, float* __restrict__ stats, int Ct, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float* __restrict__ mm, float* __restrict__ mv, long long rows, int C,
                                int training, BnDropout drop) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= rows * C) return;
  const int c = int(e % C);
  const long long r = e / C;
  float mean, rstd;
  if (training) {
    const float d = stats[c0 + c] / float(rows);
    mean = ldv(y, c0 + c) + d;
    const float var = fmaxf(stats[Ct + c0 + c] / float(rows) - d * d, 0.f);
    rstd = rsqrtf(var + 1e-3f);
    if (e < C) {
      stats[2 * Ct + c0 + c] = mean; stats[3 * Ct + c0 + c] = rstd;
      mm[c] = 0.99f * mm[c] + 0.01f * mean; mv[c] = 0.99f * mv[c] + 0.01f * var;
    }
  } else { mean = mm[c]; rstd = rsqrtf(mv[c] + 1e-3f); }
  float v = (ldv(y, r * ld + c0 + c) - mean) * rstd * gamma[c] + beta[c];
  if (add) v += add[e];
  if (training && drop.p > 0.f) v = dropout(v, drop, dropout_seed(drop), e);
  if (xf) xf[e] = v;
  if (!xb) return;
  const bf16 hi = __float2bfloat16(v);
  if (!split) { xb[r * ld + c0 + c] = hi; return; }
  bf16* row = xb + r * 2 * ld + c0 + c;
  row[0] = hi; row[ld] = __float2bfloat16(v - __bfloat162float(hi));
}
template <typename T>
__global__ void bn_bwd_stats_kernel(const T* __restrict__ g, int ldg, const T* __restrict__ y, int ld, int c0, const float* __restrict__ stats,
                                    int Ct, float* __restrict__ bsum, long long rows, int C, BnDropout drop) {
  const long long per = (rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = blockIdx.x * per, r1 = r0 + per < rows ? r0 + per : rows;
  const uint32_t hs = drop.p > 0.f ? dropout_seed(drop) : 0u;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float mean = stats[2 * Ct + c0 + c], rstd = stats[3 * Ct + c0 + c];
    float s = 0.f, q = 0.f;
    for (long long r = r0; r < r1; ++r) {
      float gv = ldv(g, r * ldg + c0 + c);
      if (drop.p > 0.f) gv = dropout(gv, drop, hs, r * C + c);
      s += gv; q += gv * (ldv(y, r * ld + c0 + c) - mean) * rstd;
    }
    atomicAdd(bsum + c0 + c, s); atomicAdd(bsum + Ct + c0 + c, q);
  }
}
template <typename T>
__global__ void bn_bwd_apply_kernel(const T* __restrict__ g, int ldg, const T* __restrict__ y, int ld, int c0, const float* __restrict__ stats,
                                    int Ct, const float* __restrict__ bsum, const float* __restrict__ gamma, bf16* __restrict__ dpre, int ldd,
                                    float* __restrict__ dgamma, float* __restrict__ dbeta, long long rows, int C, int act, BnDropout drop) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= rows * C) return;
  const int c = int(e % C);
  const long long r = e / C;
  const float mean = stats[2 * Ct + c0 + c], rstd = stats[3 * Ct + c0 + c];
  float gv = ldv(g, r * ldg + c0 + c);
  if (drop.p > 0.f) gv = dropout(gv, drop, dropout_seed(drop), e);
  const float yv = ldv(y, r * ld + c0 + c);
  const float xhat = (yv - mean) * rstd;
  float dy = gamma[c] * rstd * (gv - bsum[c0 + c] / float(rows) - xhat * bsum[Ct + c0 + c] / float(rows));
  if (act == 1) dy = yv > 0.f ? dy : 0.f;
  else if (act == 2) dy *= (1.f - yv * yv);
  dpre[r * ldd + c0 + c] = __float2bfloat16(dy);
  if (e < C) { dgamma[c] += bsum[Ct + c0 + c]; dbeta[c] += bsum[c0 + c]; }
}
template <typename TS>
__global__ void bias_colsum_kernel(const TS* __restrict__ src, long long rows, int C, int ld, float* __restrict__ dst) {
  const long long per = (rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = blockIdx.x * per, r1 = r0 + per < rows ? r0 + per : rows;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (long long r = r0; r < r1; ++r) s += ldv(src, r * ld + c);
    atomicAdd(dst + c, s);
  }
}

}  // namespace

template <typename TY>
void bn_fwd(const TY* y, int ld, int c0, bf16* xb, int split, float* xf, const float* add, float* stats, int Ct, const float* gamma,
            const float* beta, float* mm, float* mv, long long rows, int C, int training, const BnDropout& drop, int stat_threads,
            cudaStream_t st) {
  if (training) { bn_stats_kernel<TY><<<64, stat_threads, 0, st>>>(y, ld, c0, stats, Ct, rows, C); t2_count_launch(); }
  bn_apply_kernel<TY><<<grid1d(rows * C), 256, 0, st>>>(y, ld, c0, xb, split, xf, add, stats, Ct, gamma, beta, mm, mv, rows, C, training, drop);
  t2_count_launch();
}
template <typename T>
void bn_bwd(const T* g, int ldg, const T* y, int ld, int c0, const float* stats, int Ct, float* bsum, const float* gamma, bf16* dpre, int ldd,
            float* dgamma, float* dbeta, long long rows, int C, int act, const BnDropout& drop, int stat_threads, cudaStream_t st) {
  bn_bwd_stats_kernel<T><<<64, stat_threads, 0, st>>>(g, ldg, y, ld, c0, stats, Ct, bsum, rows, C, drop); t2_count_launch();
  bn_bwd_apply_kernel<T><<<grid1d(rows * C), 256, 0, st>>>(g, ldg, y, ld, c0, stats, Ct, bsum, gamma, dpre, ldd, dgamma, dbeta, rows, C, act, drop);
  t2_count_launch();
}
template <typename TS>
void colsum(const TS* src, long long rows, int C, int ld, float* dst, int threads, cudaStream_t st) {
  bias_colsum_kernel<TS><<<64, threads, 0, st>>>(src, rows, C, ld, dst); t2_count_launch();
}

template void bn_fwd<bf16>(const bf16*, int, int, bf16*, int, float*, const float*, float*, int, const float*, const float*, float*, float*,
                           long long, int, int, const BnDropout&, int, cudaStream_t);
template void bn_fwd<float>(const float*, int, int, bf16*, int, float*, const float*, float*, int, const float*, const float*, float*, float*,
                            long long, int, int, const BnDropout&, int, cudaStream_t);
template void bn_bwd<bf16>(const bf16*, int, const bf16*, int, int, const float*, int, float*, const float*, bf16*, int, float*, float*, long long,
                           int, int, const BnDropout&, int, cudaStream_t);
template void bn_bwd<float>(const float*, int, const float*, int, int, const float*, int, float*, const float*, bf16*, int, float*, float*,
                            long long, int, int, const BnDropout&, int, cudaStream_t);
template void colsum<bf16>(const bf16*, long long, int, int, float*, int, cudaStream_t);

}  // namespace t2
