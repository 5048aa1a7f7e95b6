// t2_gemm.h — host-side interface of the wgmma GEMM engine (see t2_gemm.cuh for the kernels).
#pragma once
#include <cuda_runtime.h>
#include <string.h>

#include <vector>

#include "t2_gemm_types.h"

namespace t2 {

// channels-last bf16 activation tensor [L][B][T][ld]; the first C channels of each row are addressable
struct ActT {
  const void* ptr;
  int C, T, B, L, ld;
};
inline ActT make_act(const void* p, int C, int T, int B, int L = 1, int ld = -1) {
  ActT a;
  a.ptr = p; a.C = C; a.T = T; a.B = B; a.L = L; a.ld = ld < 0 ? C : ld;
  return a;
}

struct ActGemmCall {
  ActT a[4];
  int na;
  Seg seg[kMaxSeg];
  int nseg;
  const void* w;   // packed bf16 weights [wL][wN][wK], K contiguous
  int wN, wK, wL, w_layer, w_k0;
  int T, B;
  int n_tiles;     // grid.y
  int ksplit;      // grid.z: CTAs sharing one output tile over slices of K (0/1 = off; epilogue must accumulate atomically)
  int cluster;     // requested weight-multicast cluster size along M: 0 = T2_CLUSTER / default, else 1, 2, 4 or 8
  // split-bf16 ("fp32-class") operands. The call is given in its plain form; make_gemm_args launches its split form: every map
  // becomes rows [hi(Cp) | lo(Cp)] of pitch 2 Cp, with Cp = nkb * kBK of the segments that read it (k0 = 0), every segment one of
  // 2 nkb blocks over both halves and one of nkb blocks over the hi half, wK three times the segments' width (the packing of
  // add_pack_fwd, t2_params.h; w_k0 = 0), and epi.i[11] = 1
  int split;
  EpiArgs epi;
};

void set_timing_buffer(long long* p);
bool pdl_enabled();
int cluster_pref();   // weight-multicast cluster size of the act_gemm launches (T2_CLUSTER; 1 = off)
// launch any kernel with the programmatic-dependent-launch attribute (the kernel must call pdl_wait() before it touches
// global memory; see t2_common.cuh)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
// *cluster_used (nullable) receives the cluster size the kernel was launched with
int launch_act_gemm(int epi, int BN, const ActGemmCall& c, cudaStream_t stream, int* cluster_used = nullptr);
// One EPI_BIAS_ACT launch: a k-tap 'same' convolution or a projection over the [B][T] rows of a channels-last bf16 operand,
//   out[b][t][n] = act(sum_tap sum_k a[b][t + shifts[tap]][k0s[tap] + k] w[n][tap * Cp + k] + bias[n]),   Cp = ceil(C / kBK) * kBK,
// then dropout at rate pdrop with the mask of hash stream `stream` under seed + *step (step nullable), drawn at row hash_row0 + row,
// so a launch over some rows of a larger matrix draws that matrix's mask (Epilogue<EPI_BIAS_ACT>, t2_gemm.cuh). Call sites name the
// fields with designated initialisers, in declaration order.
struct BiasActGemm {
  const void* a; int C;                    // operand A: C channels per tap
  int ld = 0;                              // row pitch (0 = Ctot)
  const int* k0s = nullptr; int Ctot = 0;  // per-tap first channel (null = 0) of rows of Ctot addressable channels (0 = C)
  int T; int B;
  int ntaps = 1; const int* shifts = nullptr;   // tap j reads row t + shifts[j] (null = 0)
  int layers = 1;    // K runs over the [layers][B][T] slabs of the operand, layers outer
  int split = 0;     // split-bf16 ("fp32-class") operand (ActGemmCall::split): rows [hi | lo] of pitch 2 Cp (ld, k0s and Ctot unused)
                     // against weights packed by add_pack_fwd; wK stays the plain one; a bf16 output is written as [hi(ldo) | lo(ldo)]
  const void* w; int N; int wK; int BN;    // packed bf16 weights [N][wK]; BN 128 or 256
  const float* bias = nullptr; int act = 0;
  void* out_bf16 = nullptr; float* out_f32 = nullptr; int ldo; int nvalid;   // columns [0, nvalid) of output rows of pitch ldo
  float pdrop = 0.f; int stream = 0; unsigned long long seed = 0; const unsigned long long* step = nullptr; int hash_row0 = 0;
};
int launch_bias_act(const BiasActGemm& g, cudaStream_t st);
// the checked kernel arguments (tensor maps encoded), grid and cluster size launch_act_gemm launches `c` with
int make_gemm_args(int epi, int BN, const ActGemmCall& c, GemmArgs& g, dim3& grid, int& cs);
// one persistent layer chain (wn_chain_kernel): kind 0 / 1 tiles are EPI_GATE (BN 256) / EPI_RES (BN bn1) when fwd, else
// EPI_GATE_BWD (BN bn0) / EPI_DX (BN bn1); `grid` CTAs take the tickets
int launch_wn_chain(bool fwd, int bn0, int bn1, const ChainArgs& a, int grid, cudaStream_t st);
// the next n_slots int64 stamps of the timing buffer (t2_dbg_set_timing_buffer), or nullptr when it is off
long long* take_timing_slice(long long n_slots);
int launch_wgrad(const ActT* maps, int nmaps, const WgradTile* tiles_dev, int ntiles, float* out,
                 int T, int B, cudaStream_t stream);
// appends the tiles of the dense [Ca x Cb] weight gradient out[out_off + m * ldc + n] of A channels [a_ch0, a_ch0 + Ca) and B channels
// [b_ch0, b_ch0 + Cb), row blocks outer; proto gives the maps, shifts, layers, scale, accumulate and div of every tile
void append_wgrad_tiles(std::vector<WgradTile>& v, const WgradTile& proto, int a_ch0, int Ca, int b_ch0, int Cb, long long out_off,
                        int ldc);
// proto of a plain weight gradient: A map am shifted by a_shift time steps, B map bm, scale 1
WgradTile dense_proto(int am, int bm, int a_shift = 0);
// tap j of a k-tap 'same' convolution reads input row t + conv_tap_shift(k, j) (an even k pads the extra row on the right)
inline int conv_tap_shift(int k, int j) { return j - (k - 1) / 2; }
// the tiles of a conv kernel [k][Ca][Cb] at out_off: per tap, in tap order, the dense weight gradient of map 0 (input, A channels from
// a_ch0, shifted by the tap) x map 1 (output gradient, B channels from b_ch0)
void append_conv_wgrad_tiles(std::vector<WgradTile>& v, int k, int a_ch0, int Ca, int b_ch0, int Cb, long long out_off);

}  // namespace t2
