// t2_params.cu — host-side parameter plumbing shared by the WaveNet, Tacotron and CBHG engines (see t2_params.h).
#include <stdio.h>
#include <stdlib.h>

#include "t2_common.cuh"
#include "t2_params.h"

namespace t2 {

long long add_param(std::vector<Param>& table, long long& n_params, const std::string& name, std::initializer_list<int> shape,
                    bool trainable) {
  Param p;
  p.name = name;
  p.off = n_params;
  p.ndim = int(shape.size());
  long long n = 1;
  int i = 0;
  for (int s : shape) { p.shape[i++] = s; n *= s; }
  for (; i < 4; ++i) p.shape[i] = 1;
  p.trainable = trainable;
  p.reg = trainable && regularized(name);
  n_params += align_up(n, 4);
  table.push_back(p);
  return p.off;
}

// tacotron.py:343-345: every variable whose name has none of these substrings
bool regularized(const std::string& name) {
  for (const char* s : {"bias", "Bias", "_projection", "inputs_embedding", "RNN", "LSTM"})
    if (name.find(s) != std::string::npos) return false;
  return true;
}

ConvBnParams add_conv_bn_params(std::vector<Param>& table, long long& n_params, const std::string& prefix, int k, int cin, int cout) {
  ConvBnParams p;
  p.kernel = add_param(table, n_params, prefix + "kernel", {k, cin, cout});
  p.bias = add_param(table, n_params, prefix + "bias", {cout});
  p.gamma = add_param(table, n_params, prefix + "gamma", {cout});
  p.beta = add_param(table, n_params, prefix + "beta", {cout});
  p.mm = add_param(table, n_params, prefix + "moving_mean", {cout}, false);
  p.mv = add_param(table, n_params, prefix + "moving_variance", {cout}, false);
  return p;
}

int param_info(const std::vector<Param>& table, int i, char* name, int cap, long long* offset, int* ndim, int* shape4, int* trainable) {
  T2_REQUIRE(i >= 0 && i < int(table.size()), T2_ERR_INVALID_ARG, "tensor index %d out of range", i);
  T2_REQUIRE(name && cap > 0, T2_ERR_INVALID_ARG, "param_info: null name buffer");
  const Param& p = table[i];
  snprintf(name, cap, "%s", p.name.c_str());
  if (offset) *offset = p.off;
  if (ndim) *ndim = p.ndim;
  if (shape4) for (int k = 0; k < 4; ++k) shape4[k] = p.shape[k];
  if (trainable) *trainable = p.trainable ? 1 : 0;
  return T2_OK;
}

void add_pack(std::vector<PackJob>& jobs, long long src, int K, int N, long long dst_bytes, int ld, int transpose, int col0, float scale,
              int perm) {
  PackJob j;
  j.src_off = src; j.K = K; j.N = N; j.dst_off = dst_bytes / 2; j.dst_ld = ld; j.transpose = transpose; j.col0 = col0;
  j.scale = scale; j.perm = perm; j.part = 0;
  jobs.push_back(j);
}

void add_pack_fwd(std::vector<PackJob>& jobs, bool split, long long src, int K, int N, long long dst_bytes, int Kw, int c, int Cp,
                  float scale, int perm, int layer, int layers) {
  const int x = layer * Cp, Ks = layers * Cp;
  if (!split) {
    add_pack(jobs, src, K, N, dst_bytes, Kw, 1, c + x, scale, perm);
    return;
  }
  for (int col : {3 * c + 2 * x, 3 * c + 2 * x + Cp, 3 * c + 2 * Ks + x}) add_pack(jobs, src, K, N, dst_bytes, 3 * Kw, 1, col, scale, perm);
  jobs.back().part = 2;
}

namespace {

typedef __nv_bfloat16 bf16;

// 64x64 tiles through shared memory: float2 reads along the source's fast axis (N), bf16x2 writes along the destination's fast axis
// (K for the transposing jobs); scalar fallbacks when an offset / leading dimension is odd. NG gates of W rows share one row block.
template <int W, int NG>
__global__ void pack_kernel(const float* __restrict__ params, bf16* __restrict__ packed, const PackJob* __restrict__ jobs) {
  __shared__ float tile[64][65];
  const PackJob j = jobs[blockIdx.y];
  const int tiles_n = (j.N + 63) / 64, tiles_k = (j.K + 63) / 64;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const bool vec_src = ((j.N | int(j.src_off)) & 1) == 0;
  const bool vec_dst = ((j.dst_ld | j.col0 | int(j.dst_off)) & 1) == 0;
  for (int ti = blockIdx.x; ti < tiles_n * tiles_k; ti += gridDim.x) {
    const int k0 = (ti / tiles_n) * 64, n0 = (ti % tiles_n) * 64;
    for (int r = ty; r < 64; r += 8) {
      const int k = k0 + r, n = n0 + 2 * tx;
      float a = 0.f, b = 0.f;
      if (k < j.K) {
        const float* src = params + j.src_off + (long long)k * j.N + n;
        if (vec_src && n + 1 < j.N) { const float2 v = *reinterpret_cast<const float2*>(src); a = v.x; b = v.y; }
        else { if (n < j.N) a = src[0]; if (n + 1 < j.N) b = src[1]; }
      }
      a *= j.scale; b *= j.scale;
      if (j.part == 2) { a -= __bfloat162float(__float2bfloat16(a)); b -= __bfloat162float(__float2bfloat16(b)); }
      tile[r][2 * tx] = a; tile[r][2 * tx + 1] = b;
    }
    __syncthreads();
    if (j.transpose) {
      for (int r = ty; r < 64; r += 8) {
        const int n = n0 + r, k = k0 + 2 * tx;
        if (n < j.N && k < j.K) {
          int row = n;
          if (j.perm > 0) {
            const int g = n / j.perm, u = n % j.perm;
            row = (u / W) * (NG * W) + g * W + (u % W);
          }
          bf16* dst = packed + j.dst_off + (long long)row * j.dst_ld + j.col0 + k;
          if (vec_dst && k + 1 < j.K) *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(tile[2 * tx][r], tile[2 * tx + 1][r]);
          else { dst[0] = __float2bfloat16(tile[2 * tx][r]); if (k + 1 < j.K) dst[1] = __float2bfloat16(tile[2 * tx + 1][r]); }
        }
      }
    } else {
      for (int r = ty; r < 64; r += 8) {
        const int k = k0 + r, n = n0 + 2 * tx;
        if (n < j.N && k < j.K) {
          bf16* dst = packed + j.dst_off + (long long)k * j.dst_ld + j.col0 + n;
          if (vec_dst && n + 1 < j.N) *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(tile[r][2 * tx], tile[r][2 * tx + 1]);
          else { dst[0] = __float2bfloat16(tile[r][2 * tx]); if (n + 1 < j.N) dst[1] = __float2bfloat16(tile[r][2 * tx + 1]); }
        }
      }
    }
    __syncthreads();
  }
}

__global__ void reg_loss_kernel(const float* __restrict__ params, const long long* __restrict__ tab, float* __restrict__ dst) {
  const long long off = tab[2 * blockIdx.y], len = tab[2 * blockIdx.y + 1];
  float s = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len; i += (long long)gridDim.x * blockDim.x) {
    const float v = params[off + i]; s += v * v;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0 && s != 0.f) atomicAdd(dst, 0.5f * s);
}

__global__ void reg_grad_kernel(const float* __restrict__ params, float* __restrict__ grads, const long long* __restrict__ tab, float w) {
  const long long off = tab[2 * blockIdx.y], len = tab[2 * blockIdx.y + 1];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len; i += (long long)gridDim.x * blockDim.x)
    grads[off + i] += w * params[off + i];
}

// kSplit: n = rows * Cp elements of the split-bf16 operand rows [hi(Cp) | lo(Cp)] from fp32 [rows][C]; channels C..Cp-1 are zero
template <bool kSplit>
__global__ void f32_to_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, long long n, int C, int Cp) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (!kSplit) {
    if (e < n) out[e] = __float2bfloat16(in[e]);
    return;
  }
  if (e >= n) return;
  const long long r = e / Cp;
  const int c = int(e % Cp);
  const float v = c < C ? in[r * C + c] : 0.f;
  const bf16 hi = __float2bfloat16(v);
  bf16* row = out + r * 2 * Cp + c;
  row[0] = hi; row[Cp] = __float2bfloat16(v - __bfloat162float(hi));
}

}  // namespace

int launch_pack(const float* params, void* packed, const PackJob* jobs_dev, int n_jobs, int W, int grid_x, cudaStream_t st) {
  T2_REQUIRE(W == 128 || W == 32, T2_ERR_INVALID_ARG, "pack: gate block width %d is not 128 or 32", W);
  auto kernel = W == 128 ? pack_kernel<128, 2> : pack_kernel<32, 4>;
  kernel<<<dim3(grid_x, n_jobs), dim3(32, 8), 0, st>>>(params, static_cast<bf16*>(packed), jobs_dev);
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

int upload_reg_table(const std::vector<Param>& table, void* dst, cudaStream_t st) {
  std::vector<long long> tab;
  for (const Param& p : table)
    if (p.reg) {
      long long n = 1;
      for (int k = 0; k < p.ndim; ++k) n *= p.shape[k];
      tab.push_back(p.off); tab.push_back(n);
    }
  if (!tab.empty()) T2_CHECK_CUDA(cudaMemcpyAsync(dst, tab.data(), tab.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
  return T2_OK;
}

void launch_reg_loss(const float* params, const long long* tab, int n_reg, float* dst, cudaStream_t st) {
  if (n_reg <= 0) return;
  reg_loss_kernel<<<dim3(8, n_reg), 256, 0, st>>>(params, tab, dst);
  t2_count_launch();
}

void launch_reg_grad(const float* params, float* grads, const long long* tab, int n_reg, float weight, cudaStream_t st) {
  if (n_reg <= 0) return;
  reg_grad_kernel<<<dim3(8, n_reg), 256, 0, st>>>(params, grads, tab, weight);
  t2_count_launch();
}

void launch_f32_to_bf16(const float* in, __nv_bfloat16* out, long long n, cudaStream_t st) {
  f32_to_bf16_kernel<false><<<grid1d(n), 256, 0, st>>>(in, out, n, 0, 0);
  t2_count_launch();
}

void launch_f32_to_bf16_split(const float* in, __nv_bfloat16* out, long long rows, int C, int Cp, cudaStream_t st) {
  f32_to_bf16_kernel<true><<<grid1d(rows * Cp), 256, 0, st>>>(in, out, rows * Cp, C, Cp);
  t2_count_launch();
}

SideStream* side_stream() {
  static SideStream ss;
  static int state = 0;   // 0 unknown, 1 ready, -1 disabled
  if (state == 0) {
    const char* e = getenv("T2_SIDE_STREAM");
    if (e && e[0] == '0') state = -1;
    else if (cudaStreamCreateWithFlags(&ss.s, cudaStreamNonBlocking) == cudaSuccess &&
             cudaEventCreateWithFlags(&ss.fork, cudaEventDisableTiming) == cudaSuccess &&
             cudaEventCreateWithFlags(&ss.fork2, cudaEventDisableTiming) == cudaSuccess &&
             cudaEventCreateWithFlags(&ss.join, cudaEventDisableTiming) == cudaSuccess) state = 1;
    else state = -1;
  }
  return state == 1 ? &ss : nullptr;
}

}  // namespace t2
