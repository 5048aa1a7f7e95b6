// t2_gemm_types.h — POD types shared by the GEMM engine's kernels (t2_gemm.cuh) and its host API (t2_gemm.h).
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace t2 {

constexpr int kBM = 128;      // positions per tile (two 64-row wgmma warpgroups)
constexpr int kBK = 64;       // K elements per pipeline stage (= one 128-byte swizzle row of bf16)
constexpr int kMaxSeg = 16;
constexpr int kGemmThreads = 288;   // wgrad_gemm: two consumer warpgroups + producer warp
constexpr int kDbgSlots = 16;  // int64 stamps per CTA in the optional timing buffer (t2_dbg_set_timing_buffer)

struct Seg {
  int map;      // which A tensor map
  int shift;    // time shift applied to the row coordinate (taps of the dilated conv)
  int k0;       // first channel in the A tensor
  int nkb;      // number of 64-wide K blocks
  int layer0;   // first layer coordinate
  int nlayers;  // layers looped (outer) — used when K runs over the layer axis
};

struct EpiArgs {
  void* ptr[12];
  float f[6];
  int i[12];
  unsigned long long seed;
};

struct GemmArgs {
  CUtensorMap amap[4];
  CUtensorMap bmap;
  CUtensorMap omap[3];  // epilogue OUTPUT tensors (TMA stores): dims (C, T, B), box 64 columns x 32 rows, 128-byte swizzle
  Seg seg[kMaxSeg];
  int nseg;
  int T;             // time steps per batch item
  int tiles_per_b;   // ceil(T / 128)
  int b_layer;       // layer coordinate of the weight tensor map (3-D maps), else 0
  int b_k0;          // first K column of the packed weight this GEMM consumes
  long long* dbg;    // optional: kDbgSlots stamps per CTA (see t2_dbg_set_timing_buffer)
  EpiArgs epi;
};

enum EpiKind {
  EPI_GATE = 0,
  EPI_RES = 1,
  EPI_BIAS_ACT = 2,
  EPI_CE = 3,
  EPI_MOL = 4,
  EPI_SCALE_RELUMASK = 5,
  EPI_GATE_BWD = 6,
  EPI_DX = 7,
  EPI_LSTM = 8,   // swapped GEMM (rows = gate units, cols = batch) + LSTM cell + zoneout
  EPI_TOUT = 9,   // swapped GEMM, transposed fp32 output (rows = features, cols = batch)
};


struct WgradTile {
  int a_map, a_ch0, a_shift, a_layer;
  int b_map, b_ch0, b_shift, b_layer;
  long long out_off;   // element offset into the fp32 output buffer
  int ldc;             // row pitch (elements) of the output
  int m_valid, n_valid;
  float scale;
  int accumulate;      // 0: overwrite, 1: add to existing (single writer), 2: atomicAdd (several tiles share an output)
  const float* div;    // optional device scalar: result is divided by max(*div, tiny)
};
struct WgradArgs {
  CUtensorMap map[6];
  const WgradTile* tiles;
  float* out;
  int T, B;
};

// One work item of a persistent layer chain (wn_chain_kernel, t2_gemm.cu; built by build_chain, t2_wavenet.cu): output tile (m, n) of the kind-th GEMM of `layer` (forward: 0 gate,
// 1 out; backward: 0 dz, 1 dx). It may start once the completion counters [dep_lo, dep_hi] have all reached dep_target (dep_hi <
// dep_lo: no dependency inside the kernel) and adds 1 to counter `done` when its stores are complete. Counter of (kind, layer, M
// tile m) = (kind * L + layer) * MT + m, with MT = B * ceil(T / 128) M tiles over all batch items.
struct ChainTicket {
  int kind, layer, m, n;
  int dep_lo, dep_hi, dep_target;
  int done;
};

struct ChainArgs {
  const GemmArgs* args;        // [2][L]: kind-major
  const ChainTicket* tix;
  int n_tix, L;
  int* ctr;                    // [0] ticket counter, [1] stop flag; completion counters from ctr + 16
  int* err;                    // += 1 when a dependency wait of the launch times out (its remaining tickets are then skipped)
  long long* dbg;              // optional: kDbgSlots stamps per ticket (start, dependencies met, end, SM)
  // per-call values the workspace table leaves out (it depends only on the configuration, workspace and packed weights)
  const float* params;         // forward out GEMM: its bias is params + (offset the table stores in epi.ptr[3])
  const unsigned long long* d_step;
  unsigned long long seed;
  int save;                    // forward: write the tanh / sigmoid stashes
};

}  // namespace t2
