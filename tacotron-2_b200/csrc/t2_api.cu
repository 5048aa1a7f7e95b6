// t2_api.cu — error plumbing of the C-ABI plus the engine-level entry points used by the unit tests.
#include <stdarg.h>
#include <stdio.h>
#include <stddef.h>
#include <string.h>

#include <vector>

#include "../../include/t2b200.h"
#include "t2_common.cuh"
#include "t2_gemm.h"

#include <atomic>
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};
void t2_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" long long t2_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int t2_set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

extern "C" const char* t2_last_error(void) { return g_err; }
extern "C" int t2_abi_version(void) { return T2B200_ABI_VERSION; }

// D[b,t,n] = act( sum_s sum_k A[b, t + shift_s, k] * W[n, s*Kseg + k] + bias[n] ), bf16 in, fp32 accumulate.
extern "C" int t2_dbg_conv_gemm(const void* a, int B, int T, int C, int ld, const int* shifts, int nshift,
                                const void* w, int N, int BN, const float* bias, int relu, void* out_bf16,
                                float* out_f32, void* stream) {
  using namespace t2;
  T2_REQUIRE(nshift >= 1 && nshift <= kMaxSeg, T2_ERR_INVALID_ARG, "nshift out of range");
  T2_REQUIRE(BN == 128 || BN == 256, T2_ERR_UNSUPPORTED_SHAPE, "BN must be 128 or 256");
  const int nkb = (C + kBK - 1) / kBK;
  return launch_bias_act({.a = a, .C = C, .ld = ld, .T = T, .B = B, .ntaps = nshift, .shifts = shifts, .w = w, .N = N, .wK = nshift * nkb * kBK,
                          .BN = BN, .bias = bias, .act = relu, .out_bf16 = out_bf16, .out_f32 = out_f32, .ldo = N, .nvalid = N},
                         static_cast<cudaStream_t>(stream));
}

// dW[m, n] = scale * sum_{b,t} A[b, t + shift_a, m] * Bm[b, t, n]   (fp32 out [Ca, Cb])
extern "C" int t2_dbg_wgrad(const void* a, int Ca, const void* bm, int Cb, int B, int T, int shift_a,
                            float scale, float* out, void* stream) {
  using namespace t2;
  ActT maps[2] = {make_act(a, Ca, T, B), make_act(bm, Cb, T, B)};
  WgradTile proto;
  memset(&proto, 0, sizeof(proto));
  proto.a_map = 0; proto.a_shift = shift_a; proto.b_map = 1; proto.scale = scale;
  std::vector<WgradTile> tiles;
  append_wgrad_tiles(tiles, proto, 0, Ca, 0, Cb, 0, Cb);
  WgradTile* dt = nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  T2_CHECK_CUDA(cudaMallocAsync(&dt, tiles.size() * sizeof(WgradTile), st));
  T2_CHECK_CUDA(cudaMemcpyAsync(dt, tiles.data(), tiles.size() * sizeof(WgradTile), cudaMemcpyHostToDevice, st));
  int rc = launch_wgrad(maps, 2, dt, int(tiles.size()), out, T, B, st);
  cudaStreamSynchronize(st);  // debug entry: tiles is a host temporary
  cudaFreeAsync(dt, st);
  return rc;
}

// the test structs of the header are the engine's own types: the hooks below reinterpret them without copying field by field
#define T2_SAME_FIELD(A, B, f) static_assert(offsetof(A, f) == offsetof(B, f), #A " / " #B ": field " #f)
static_assert(sizeof(t2_dbg_act_t) == sizeof(t2::ActT), "t2_dbg_act_t / ActT");
T2_SAME_FIELD(t2_dbg_act_t, t2::ActT, ptr); T2_SAME_FIELD(t2_dbg_act_t, t2::ActT, C); T2_SAME_FIELD(t2_dbg_act_t, t2::ActT, ld);
static_assert(sizeof(t2_dbg_seg_t) == sizeof(t2::Seg), "t2_dbg_seg_t / Seg");
T2_SAME_FIELD(t2_dbg_seg_t, t2::Seg, map); T2_SAME_FIELD(t2_dbg_seg_t, t2::Seg, nlayers);
static_assert(sizeof(t2_dbg_wgrad_tile_t) == sizeof(t2::WgradTile), "t2_dbg_wgrad_tile_t / WgradTile");
T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, a_map); T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, a_ch0);
T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, a_shift); T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, a_layer);
T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, b_map); T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, b_ch0);
T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, b_shift); T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, b_layer);
T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, out_off); T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, ldc);
T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, m_valid); T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, n_valid);
T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, scale); T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, accumulate);
T2_SAME_FIELD(t2_dbg_wgrad_tile_t, t2::WgradTile, div);
#undef T2_SAME_FIELD

extern "C" int t2_dbg_act_gemm(t2_dbg_gemm_t* call, void* stream) {
  using namespace t2;
  T2_REQUIRE(call != nullptr, T2_ERR_INVALID_ARG, "null call");
  T2_REQUIRE(call->na >= 1 && call->na <= 4 && call->nseg >= 1 && call->nseg <= kMaxSeg, T2_ERR_INVALID_ARG,
             "bad map/segment count (%d, %d)", call->na, call->nseg);
  ActGemmCall c;
  memset(&c, 0, sizeof(c));
  memcpy(c.a, call->a, sizeof(c.a));
  c.na = call->na;
  memcpy(c.seg, call->seg, sizeof(c.seg));
  c.nseg = call->nseg;
  c.w = call->w; c.wN = call->wN; c.wK = call->wK; c.wL = call->wL; c.w_layer = call->w_layer; c.w_k0 = call->w_k0;
  c.T = call->T; c.B = call->B; c.n_tiles = call->n_tiles; c.ksplit = call->ksplit; c.cluster = call->cluster;
  memcpy(c.epi.ptr, call->ptr, sizeof(c.epi.ptr));
  memcpy(c.epi.f, call->f, sizeof(c.epi.f));
  memcpy(c.epi.i, call->i, sizeof(c.epi.i));
  c.epi.seed = call->seed;
  call->cluster_used = 0;
  return launch_act_gemm(call->epi, call->BN, c, static_cast<cudaStream_t>(stream), &call->cluster_used);
}

extern "C" int t2_dbg_wgrad_tiles(const t2_dbg_act_t* maps, int nmaps, const t2_dbg_wgrad_tile_t* tiles, int ntiles, float* d_out, int T,
                                  int B, void* stream) {
  using namespace t2;
  T2_REQUIRE(maps && tiles && nmaps >= 1 && nmaps <= 6 && ntiles >= 1, T2_ERR_INVALID_ARG, "wgrad_tiles: bad map/tile arguments");
  for (int i = 0; i < ntiles; ++i)
    T2_REQUIRE(tiles[i].a_map >= 0 && tiles[i].a_map < nmaps && tiles[i].b_map >= 0 && tiles[i].b_map < nmaps &&
               tiles[i].m_valid >= 1 && tiles[i].m_valid <= 128 && tiles[i].n_valid >= 1 && tiles[i].n_valid <= 256 &&
               tiles[i].accumulate >= 0 && tiles[i].accumulate <= 2,
               T2_ERR_INVALID_ARG, "wgrad_tiles: bad tile %d", i);
  WgradTile* dt = nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  T2_CHECK_CUDA(cudaMallocAsync(&dt, ntiles * sizeof(WgradTile), st));
  const cudaError_t e = cudaMemcpyAsync(dt, tiles, ntiles * sizeof(WgradTile), cudaMemcpyHostToDevice, st);
  int rc = e == cudaSuccess ? launch_wgrad(reinterpret_cast<const ActT*>(maps), nmaps, dt, ntiles, d_out, T, B, st)
                            : t2_set_error(T2_ERR_CUDA, "wgrad_tiles: tile table upload failed: %s", cudaGetErrorString(e));
  cudaStreamSynchronize(st);  // debug entry: the tile table is a temporary
  cudaFreeAsync(dt, st);
  return rc;
}

// each addend goes through fx_add (one thread per addend, so same-column atomics contend as in the epilogues)
__global__ void fx_colsum_kernel(const float* __restrict__ v, long long n, int ncols, long long* acc) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) t2::fx_add(acc + i % ncols, v[i]);
}
extern "C" int t2_dbg_fx_colsum(const float* d_addends, int nrows, int ncols, float* d_out, void* stream) {
  T2_REQUIRE(d_addends && d_out && nrows >= 0 && ncols >= 1, T2_ERR_INVALID_ARG, "fx_colsum: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long* acc = nullptr;
  T2_CHECK_CUDA(cudaMallocAsync(&acc, size_t(ncols) * sizeof(long long), st));
  const long long n = (long long)nrows * ncols;
  cudaError_t e = cudaMemsetAsync(acc, 0, size_t(ncols) * sizeof(long long), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_out, 0, size_t(ncols) * sizeof(float), st);
  if (e == cudaSuccess && n > 0) {
    fx_colsum_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(d_addends, n, ncols, acc);
    t2_count_launch();
    e = cudaGetLastError();
  }
  int rc = e == cudaSuccess ? t2::launch_fx_finalize(acc, d_out, ncols, st)
                            : t2_set_error(T2_ERR_CUDA, "fx_colsum: %s", cudaGetErrorString(e));
  cudaStreamSynchronize(st);  // debug entry: the accumulators are a temporary
  cudaFreeAsync(acc, st);
  return rc;
}

// debug: when non-NULL every act_gemm CTA writes stamps to d_buf[(launch offset + cta) * 16 + slot]: slots 0-6 clock64() at entry,
// setup done, first stage landed, MMAs issued, accumulator ready, epilogue done, teardown; 8-10 %globaltimer (ns) at entry, after the
// programmatic-dependent-launch wait, at exit; 11 = SM id. Each launch advances the offset by its CTA count.
extern "C" int t2_dbg_set_timing_buffer(long long* d_buf) {
  t2::set_timing_buffer(d_buf);
  return T2_OK;
}

// The counter-hash behind every in-kernel dropout / zoneout mask, exported so that a parity test can rebuild the exact
// masks a training step drew and feed them to the CPU oracle: out[i] = hash_uniform32(hash_seed(seed, stream), i0 + i).
// An element is KEPT (dropout) / UPDATED (zoneout) iff out[i] >= rate.
__global__ void rng_uniform_kernel(unsigned long long seed, unsigned int stream, long long i0, long long n, float* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) out[i] = t2::hash_uniform32(t2::hash_seed(seed, stream), (unsigned long long)(i0 + i));
}
extern "C" int t2_rng_uniform_f32(unsigned long long seed, unsigned int stream_id, long long first_index, long long n, float* d_out,
                                  void* stream) {
  T2_REQUIRE(n >= 0 && (n == 0 || d_out != nullptr), T2_ERR_INVALID_ARG, "rng_uniform: bad arguments");
  if (n == 0) return T2_OK;
  rng_uniform_kernel<<<unsigned((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(seed, stream_id, first_index, n, d_out);
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

// sizeof of the POD structs that cross the C-ABI: lets a binding (ctypes, cgo, ...) assert that its mirror matches this build
extern "C" int t2_struct_size(const char* name) {
  if (!name) return -1;
  if (!strcmp(name, "t2_wn_config_t")) return int(sizeof(t2_wn_config_t));
  if (!strcmp(name, "t2_wn_sizes_t")) return int(sizeof(t2_wn_sizes_t));
  if (!strcmp(name, "t2_taco_config_t")) return int(sizeof(t2_taco_config_t));
  if (!strcmp(name, "t2_cbhg_config_t")) return int(sizeof(t2_cbhg_config_t));
  if (!strcmp(name, "t2_audio_config_t")) return int(sizeof(t2_audio_config_t));
  if (!strcmp(name, "t2_dbg_act_t")) return int(sizeof(t2_dbg_act_t));
  if (!strcmp(name, "t2_dbg_gemm_t")) return int(sizeof(t2_dbg_gemm_t));
  if (!strcmp(name, "t2_dbg_wgrad_tile_t")) return int(sizeof(t2_dbg_wgrad_tile_t));
  if (!strcmp(name, "t2_dbg_kernel_t")) return int(sizeof(t2_dbg_kernel_t));
  return -1;
}
