// t2_optim.cu — fused multi-tensor optimizer step over flat fp32 buffers.
// Replaces wavenet_vocoder/models/wavenet.py:586-613 (clip_by_norm(100) + clip_by_value(5) per tensor, Adam, EMA)
// and tacotron/models/tacotron.py:429-437 (clip_by_global_norm(1.0), Adam). Adam follows tf.train.AdamOptimizer:
//   lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t);  theta -= lr_t * m / (sqrt(v) + eps)   (SURVEY.md Appendix A)
#include "../../include/t2b200.h"
#include "t2_common.cuh"

namespace t2 {
namespace {

constexpr long long kChunk = 4096;   // elements per sumsq block

__device__ __forceinline__ int find_tensor(const long long* __restrict__ offs, int n, long long e) {
  int lo = 0, hi = n;  // offs[lo] <= e < offs[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (offs[mid] <= e) lo = mid; else hi = mid;
  }
  return lo;
}

// max(x, c) that keeps a NaN x (fmaxf would return c), so a NaN norm or gradient stays NaN through a clip
__device__ __forceinline__ float nan_max(float x, float c) { return x < c ? c : x; }
__device__ __forceinline__ float nan_min(float x, float c) { return x > c ? c : x; }

// Sum of squares of (grad * grad_scale) per segment: a segment is a tensor cut at the chunk boundaries. One block handles
// chunk c and writes the segment of tensor t to part[t + c] (unique and increasing in memory order, so at most
// n_tensors + n_chunks - 1 slots). No atomics: every partial has one writer and a fixed summation order.
__global__ void sumsq_kernel(const float* __restrict__ g, const long long* __restrict__ offs, int nt, long long n,
                             float gscale, float* __restrict__ part) {
  const long long e0 = blockIdx.x * kChunk;
  const long long e1 = e0 + kChunk < n ? e0 + kChunk : n;
  int t = find_tensor(offs, nt, e0);
  __shared__ float red[8];
  long long e = e0 + threadIdx.x;
  while (true) {
    const long long tend = offs[t + 1] < e1 ? offs[t + 1] : e1;
    float acc = 0.f;
    for (; e < tend; e += blockDim.x) {
      const float v = g[e] * gscale;
      acc += v * v;
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int i = 0; i < (blockDim.x >> 5); ++i) s += red[i];
      part[t + blockIdx.x] = s;
    }
    __syncthreads();
    if (tend >= e1) break;
    ++t;
    // re-align this thread's cursor to the start of the next tensor
    e = offs[t] + threadIdx.x;
  }
}

// norms[t] = sum of tensor t's segment partials (one warp per tensor, lanes strided over the chunks, then a fixed butterfly);
// with `global` (a one-block launch), norms[nt] = the sum of all norms[t] in a fixed order.
__global__ void norms_kernel(const float* __restrict__ part, const long long* __restrict__ offs, int nt, int global,
                             float* __restrict__ norms) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int t = blockIdx.x * nw + w; t < nt; t += gridDim.x * nw) {
    const long long a = offs[t], b = offs[t + 1];
    float s = 0.f;
    if (b > a)
      for (long long c = a / kChunk + lane; c <= (b - 1) / kChunk; c += 32) s += part[t + c];
    s = warp_sum(s);
    if (lane == 0) norms[t] = s;
  }
  if (!global) return;
  __syncthreads();
  if (w != 0) return;
  float s = 0.f;
  for (int i = lane; i < nt; i += 32) s += norms[i];
  s = warp_sum(s);
  if (lane == 0) norms[nt] = s;
}

struct AdamArgs {
  float* p; const float* g; float* m; float* v; float* ema;
  const long long* offs; int nt; long long n;
  float lr_t, b1, b2, eps, gscale, max_norm, max_value, gclip, ema_decay;
  const float* norms;  // per-tensor sumsq; norms[nt] = global sumsq
};
__global__ void adam_kernel(AdamArgs a) {
  // 4 consecutive elements per thread: tensor offsets (and n) are multiples of 4, so they share one tensor
  const long long e = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4;
  if (e >= a.n) return;
  float gs = a.gscale;
  if (a.gclip > 0.f) {
    gs *= a.gclip / nan_max(sqrtf(a.norms[a.nt]), a.gclip);
  } else if (a.max_norm > 0.f) {
    const int t = find_tensor(a.offs, a.nt, e);
    gs *= a.max_norm / nan_max(sqrtf(a.norms[t]), a.max_norm);
  }
  const float4 g4 = *reinterpret_cast<const float4*>(a.g + e);
  float4 m4 = *reinterpret_cast<const float4*>(a.m + e);
  float4 v4 = *reinterpret_cast<const float4*>(a.v + e);
  float4 p4 = *reinterpret_cast<const float4*>(a.p + e);
  float4 e4 = a.ema ? *reinterpret_cast<const float4*>(a.ema + e) : make_float4(0, 0, 0, 0);
  float* gp = const_cast<float*>(reinterpret_cast<const float*>(&g4));
  float* mp = reinterpret_cast<float*>(&m4);
  float* vp = reinterpret_cast<float*>(&v4);
  float* pp = reinterpret_cast<float*>(&p4);
  float* ep = reinterpret_cast<float*>(&e4);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float g = gp[i] * gs;
    if (a.max_value > 0.f) g = nan_min(nan_max(g, -a.max_value), a.max_value);
    mp[i] = a.b1 * mp[i] + (1.f - a.b1) * g;
    vp[i] = a.b2 * vp[i] + (1.f - a.b2) * g * g;
    pp[i] = pp[i] - a.lr_t * mp[i] / (sqrtf(vp[i]) + a.eps);
    ep[i] -= (1.f - a.ema_decay) * (ep[i] - pp[i]);
  }
  *reinterpret_cast<float4*>(a.m + e) = m4;
  *reinterpret_cast<float4*>(a.v + e) = v4;
  *reinterpret_cast<float4*>(a.p + e) = p4;
  if (a.ema) *reinterpret_cast<float4*>(a.ema + e) = e4;
}

}  // namespace
}  // namespace t2

extern "C" int t2_adam_step(float* d_params, const float* d_grads, float* d_m, float* d_v, float* d_ema,
                            const long long* d_offsets, int n_tensors, long long n_total, float lr, float beta1,
                            float beta2, float eps, int step, float grad_scale, float max_norm, float max_value,
                            float global_norm_clip, float ema_decay, float* d_scratch, void* stream) {
  using namespace t2;
  T2_REQUIRE(d_params && d_grads && d_m && d_v && d_offsets && d_scratch, T2_ERR_INVALID_ARG, "adam: null pointer");
  T2_REQUIRE(step >= 1 && n_tensors >= 1 && n_total >= 1, T2_ERR_INVALID_ARG, "adam: bad step / sizes");
  T2_REQUIRE(n_total % 4 == 0, T2_ERR_INVALID_ARG, "adam: flat buffers must hold a multiple of 4 elements (16-byte aligned tensors)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (max_norm > 0.f || global_norm_clip > 0.f) {
    const long long n_chunks = (n_total + kChunk - 1) / kChunk;
    float* part = d_scratch + n_tensors + 1;
    sumsq_kernel<<<(unsigned)n_chunks, 256, 0, st>>>(d_grads, d_offsets, n_tensors, n_total, grad_scale, part); t2_count_launch();
    if (global_norm_clip > 0.f) norms_kernel<<<1, 1024, 0, st>>>(part, d_offsets, n_tensors, 1, d_scratch);
    else norms_kernel<<<(n_tensors + 7) / 8, 256, 0, st>>>(part, d_offsets, n_tensors, 0, d_scratch);   // a warp per tensor
    t2_count_launch();
  }
  AdamArgs a;
  a.p = d_params; a.g = d_grads; a.m = d_m; a.v = d_v; a.ema = d_ema; a.offs = d_offsets; a.nt = n_tensors; a.n = n_total;
  a.lr_t = float(double(lr) * sqrt(1.0 - pow(double(beta2), step)) / (1.0 - pow(double(beta1), step)));
  a.b1 = beta1; a.b2 = beta2; a.eps = eps; a.gscale = grad_scale; a.max_norm = max_norm; a.max_value = max_value;
  a.gclip = global_norm_clip; a.ema_decay = ema_decay; a.norms = d_scratch;
  adam_kernel<<<(unsigned)((n_total / 4 + 255) / 256), 256, 0, st>>>(a); t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}
