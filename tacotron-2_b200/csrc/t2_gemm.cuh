// t2_gemm.cuh — the wgmma GEMM engine all dense contractions of the WaveNet / Tacotron paths run on.
//
//   act_gemm  : D[128 positions, BN] = sum over K-segments A_seg[pos + shift, k] * W[n, k]
//               A = channels-last bf16 activations [L, B, T, C] read by 4-D TMA (negative / past-the-end
//               time coordinates are zero-filled by the TMA unit, which is exactly the causal left pad of
//               wavenet_vocoder/models/modules.py:308-313), B = packed bf16 weights [N, Ktot] (K-major).
//               fp32 accumulators live in the registers of four consumer warpgroups; once the reduction is done they are
//               written to a shared fp32 tile that a fused epilogue (gate / residual / loss / ...) drains, one thread per row.
//   wgrad_gemm: dW[m, n] = sum over positions A[pos + sa, m] * B[pos + sb, n]; both operands are
//               channels-last activations, i.e. MN-major wgmma operands, reduction over positions.
//
// Warp roles of act_gemm (544 threads): warps 0..15 = MMA + epilogue, warp 16 = TMA producer.
#pragma once
#include "t2_common.cuh"
#include "t2_gemm_types.h"

namespace t2 {

// ------------------------------------------------------------------------------------------------
// small vector helpers (one thread = one row, 32 consecutive channels)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_bf16x32(__nv_bfloat16* dst, const float (&v)[32]) {
  uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 u;
    u.x = pack_bf16x2(v[q * 8 + 0], v[q * 8 + 1]);
    u.y = pack_bf16x2(v[q * 8 + 2], v[q * 8 + 3]);
    u.z = pack_bf16x2(v[q * 8 + 4], v[q * 8 + 5]);
    u.w = pack_bf16x2(v[q * 8 + 6], v[q * 8 + 7]);
    d[q] = u;
  }
}
__device__ __forceinline__ void load_bf16x32(const __nv_bfloat16* src, float (&v)[32]) {
  const uint4* s = reinterpret_cast<const uint4*>(src);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 u = __ldg(s + q);
    v[q * 8 + 0] = bf16lo(u.x); v[q * 8 + 1] = bf16hi(u.x);
    v[q * 8 + 2] = bf16lo(u.y); v[q * 8 + 3] = bf16hi(u.y);
    v[q * 8 + 4] = bf16lo(u.z); v[q * 8 + 5] = bf16hi(u.z);
    v[q * 8 + 6] = bf16lo(u.w); v[q * 8 + 7] = bf16hi(u.w);
  }
}
__device__ __forceinline__ void store_f32x32(float* dst, const float (&v)[32]) {
  float4* d = reinterpret_cast<float4*>(dst);
#pragma unroll
  for (int q = 0; q < 8; ++q) d[q] = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
}
// One row of the shared fp32 accumulator tile [128][BN]: the 16-byte chunk c of row r is stored at chunk c ^ (r % 8), so that the
// 8 rows a quarter-warp reads at the same column land in distinct banks. `row + n` addresses column n (a multiple of 4).
struct AccRow {
  const float* row;
  int col;
  int sw;
  __device__ __forceinline__ AccRow operator+(int n) const { return AccRow{row, col + n, sw}; }
};
// 32 consecutive fp32 accumulator columns of this thread's row
__device__ __forceinline__ void acc_ld32f(AccRow a, float (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 f = *reinterpret_cast<const float4*>(a.row + ((((a.col >> 2) + q) ^ a.sw) << 2));
    v[q * 4] = f.x; v[q * 4 + 1] = f.y; v[q * 4 + 2] = f.z; v[q * 4 + 3] = f.w;
  }
}

// Split-bf16 ("fp32-class") mode: an fp32 value travels as hi = bf16(v) and lo = bf16(v - hi) in channels [0,C) and [C,2C) of a row
// of pitch 2C; a GEMM then contracts [hi | lo | hi] against [W_hi | W_hi | W_lo] (the lo x lo term, 2^-18 relative, is dropped).
// These epilogue paths favour clarity over speed (one thread = one row, direct global loads / stores): they exist to show that
// the bf16-mode deviation from the fp32 reference graph is storage rounding and nothing else (tests/test_precision_modes_gpu.py).
__device__ __forceinline__ void store_split32(__nv_bfloat16* dst_hi, __nv_bfloat16* dst_lo, const float (&v)[32]) {
  float hi[32], lo[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    hi[j] = __bfloat162float(__float2bfloat16(v[j]));
    lo[j] = v[j] - hi[j];
  }
  store_bf16x32(dst_hi, hi);
  store_bf16x32(dst_lo, lo);
}
__device__ __forceinline__ void load_split32(const __nv_bfloat16* src_hi, const __nv_bfloat16* src_lo, float (&v)[32]) {
  float lo[32];
  load_bf16x32(src_hi, v);
  load_bf16x32(src_lo, lo);
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] += lo[j];
}

// ------------------------------------------------------------------------------------------------
// Epilogue staging: a thread owns one accumulator ROW, but global memory wants a warp to touch one
// row's contiguous bytes. Every epilogue therefore moves 32-row x 128-column bf16 tiles through shared-memory tiles of its
// row quarter: rows are written / read by their owning lane, global traffic is issued with 16 lanes covering one 256-byte row.
// A staged tile is two 64-column boxes of 32 rows x 128 bytes in the 128-byte swizzle (16-byte chunk index XOR row % 8) the
// output tensor maps are encoded with, so one elected thread per row quarter can hand a finished tile to the TMA engine
// (EPI_GATE / EPI_RES / EPI_GATE_BWD / EPI_DX) instead of 4 warps copying it out through registers.
// Each quarter has three tiles (EpiCtx::tile). Tile 2 is dedicated shared memory: it is the only one an epilogue's prefetch()
// may fill while the mainloop runs. Tiles 0 and 1 are the tail of the pipeline ring, past the fp32 accumulator tile, and exist
// only in run(). The TMA-store epilogues rotate the three: a tile is rewritten two stores after its own (see tile_store).
// ------------------------------------------------------------------------------------------------
constexpr int kSBoxBytes = 32 * 128;
constexpr int kSTileBytes = 2 * kSBoxBytes;
constexpr int kSTiles = 3;

constexpr int kActEpiWarps = 16;                               // 4 row quarters x 4 column groups
constexpr int kActGemmThreads = 32 * kActEpiWarps + 32;        // + producer warp

struct EpiCtx {
  int n_tile, b, t, T;     // output column tile, batch item, this lane's time step, sequence length
  bool valid;              // t < T
  int lane;
  int cg;                  // column group 0..3: this warp owns columns [32*cg, 32*cg+32) of every 128-column group
  int qbar;                // named barrier shared by the 4 warps of this row quarter
  size_t row0;             // b*T + (first time step of this warp)
  int nrows;               // valid rows among this warp's 32
  AccRow trow;             // this thread's row of the accumulator tile, column 0
  uint8_t* stg;            // staging tile 0 of this row quarter; tile k is at stg + k * 4 * kSTileBytes (see tile())
  uint8_t* smem_all;       // CTA-wide scratch that is free after the mainloop (the pipeline ring past the accumulator tile)
  int m_tile;              // index of this CTA's 128-row tile
  const CUtensorMap* omap; // output tensor maps (GemmArgs::omap) of the TMA-store epilogues
  int tq;                  // first time step of this row quarter (row coordinate of its stores)
  mutable int sk;          // stores issued so far by this quarter (tile rotation)
  // staging tile k (0..2) of this row quarter; only tile 2 may be used by prefetch()
  __device__ __forceinline__ uint8_t* tile(int k) const { return stg + k * (4 * kSTileBytes); }
};

__device__ __forceinline__ void quarter_sync(int id) {
  asm volatile("bar.sync %0, 128;\n" ::"r"(id) : "memory");
}
__device__ __forceinline__ void load_f32x32(const float* p, float (&v)[32]) {
  const float4* s = reinterpret_cast<const float4*>(p);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 f = __ldg(s + q);
    v[q * 4] = f.x; v[q * 4 + 1] = f.y; v[q * 4 + 2] = f.z; v[q * 4 + 3] = f.w;
  }
}
// ---- swizzled staging tiles ----------------------------------------------------------------------
__device__ __forceinline__ uint8_t* sw_addr(uint8_t* tile, int row, int chunk) {   // chunk: 16-byte column chunk 0..15 of the 128 columns
  return tile + (chunk >> 3) * kSBoxBytes + row * 128 + (((chunk & 7) ^ (row & 7)) << 4);
}
// smem tile -> global rows g + r*ld (elements), 128 columns each; rows >= nrows are skipped.
// NW warps cooperate (each moves 32/NW rows); with NW == 4 the quarter barrier orders it after every warp's puts.
template <int NW>
__device__ __forceinline__ void tile_flush(uint8_t* tile, __nv_bfloat16* g, size_t ld, int nrows, const EpiCtx& c) {
  if (NW == 4) quarter_sync(c.qbar); else __syncwarp();
  const int ch = c.lane & 15, rh = c.lane >> 4;
  const int it0 = NW == 4 ? c.cg * 4 : 0;
#pragma unroll
  for (int i = 0; i < 16 / NW; ++i) {
    const int r = (it0 + i) * 2 + rh;
    if (r < nrows)
      *reinterpret_cast<uint4*>(g + size_t(r) * ld + ch * 8) = *reinterpret_cast<const uint4*>(sw_addr(tile, r, ch));
  }
  if (NW == 4) quarter_sync(c.qbar); else __syncwarp();
}
__device__ __forceinline__ void stage_put_sw(uint8_t* tile, int lane, int cq, const float (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 u;
    u.x = pack_bf16x2(v[q * 8 + 0], v[q * 8 + 1]);
    u.y = pack_bf16x2(v[q * 8 + 2], v[q * 8 + 3]);
    u.z = pack_bf16x2(v[q * 8 + 4], v[q * 8 + 5]);
    u.w = pack_bf16x2(v[q * 8 + 6], v[q * 8 + 7]);
    *reinterpret_cast<uint4*>(sw_addr(tile, lane, cq * 4 + q)) = u;
  }
}
__device__ __forceinline__ void stage_get_sw(uint8_t* tile, int lane, int cq, float (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint4 u = *reinterpret_cast<const uint4*>(sw_addr(tile, lane, cq * 4 + q));
    v[q * 8 + 0] = bf16lo(u.x); v[q * 8 + 1] = bf16hi(u.x);
    v[q * 8 + 2] = bf16lo(u.y); v[q * 8 + 3] = bf16hi(u.y);
    v[q * 8 + 4] = bf16lo(u.z); v[q * 8 + 5] = bf16hi(u.z);
    v[q * 8 + 6] = bf16lo(u.w); v[q * 8 + 7] = bf16hi(u.w);
  }
}
// global rows -> swizzled tile (rows >= nrows are zero-filled); the 4 warps of the quarter cooperate, then meet on its barrier.
// kCoherent: the rows were written earlier in the same grid by another CTA (the persistent layer chains), so they are read through
// the coherent path instead of the read-only one
template <bool kCoherent = false>
__device__ __forceinline__ void tile_fill_sw(uint8_t* tile, const __nv_bfloat16* g, size_t ld, int nrows, const EpiCtx& c) {
  const int ch = c.lane & 15, rh = c.lane >> 4;
  if constexpr (kCoherent) {
    uint4 u[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {   // all four loads in flight before the first store
      const int r = (c.cg * 4 + i) * 2 + rh;
      u[i] = make_uint4(0, 0, 0, 0);
      if (r < nrows)
        asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(u[i].x), "=r"(u[i].y), "=r"(u[i].z), "=r"(u[i].w) : "l"(g + size_t(r) * ld + ch * 8));
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) *reinterpret_cast<uint4*>(sw_addr(tile, (c.cg * 4 + i) * 2 + rh, ch)) = u[i];
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = (c.cg * 4 + i) * 2 + rh;
      uint4 u = make_uint4(0, 0, 0, 0);
      if (r < nrows) u = __ldg(reinterpret_cast<const uint4*>(g + size_t(r) * ld + ch * 8));
      *reinterpret_cast<uint4*>(sw_addr(tile, r, ch)) = u;
    }
  }
  quarter_sync(c.qbar);
}
// Hand a staged tile (every warp of the quarter has put its 32 columns) to the TMA engine: columns [col0, col0 + 128) of rows
// [tq, tq + 32) of item b in the tensor behind `map`; rows past the sequence end are clipped by the map. ONE fixed thread per quarter
// issues, commits and then waits until all but the newest store have finished reading shared memory. Every warp that has passed the
// barrier of store k therefore knows that stores <= k - 2 have released their tiles: a tile may be rewritten (after that barrier) two
// stores after its own - the three-tile rotation of the epilogues below.
__device__ __forceinline__ void tile_store(uint8_t* tile, const CUtensorMap* map, int col0, const EpiCtx& c) {
  fence_proxy_async_smem();
  quarter_sync(c.qbar);
  if (c.cg == 0 && c.lane == 0) {
    tma_store_3d(map, tile, col0, c.tq, c.b);
    tma_store_3d(map, tile + kSBoxBytes, col0 + 64, c.tq, c.b);
    bulk_commit();
    bulk_wait_read<1>();
  }
  ++c.sk;
}
// all earlier stores of this quarter have released their tiles (needed before tiles are refilled out of rotation order)
__device__ __forceinline__ void tile_guard(const EpiCtx& c) {
  if (c.cg == 0 && c.lane == 0) bulk_wait_read<0>();
  quarter_sync(c.qbar);
}
// end of the epilogue: the issuing thread waits for its stores' global writes before the CTA may exit
__device__ __forceinline__ void tile_store_drain(const EpiCtx& c) {
  if (c.cg == 0 && c.lane == 0) bulk_wait_all();
}

// Column sums across a warp: lane r holds v[0..31] (row r of a 32x32 tile); on return lane j holds sum_r v_r[j].
// Recursive halving: 16 + 8 + 4 + 2 + 1 = 31 shuffles instead of 32 full warp reductions.
__device__ __forceinline__ float warp_colsum32(float (&v)[32], int lane) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const bool up = lane & 16;
    const float send = up ? v[j] : v[j + 16];
    const float keep = up ? v[j + 16] : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const bool up = lane & 8;
    const float send = up ? v[j] : v[j + 8];
    const float keep = up ? v[j + 8] : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const bool up = lane & 4;
    const float send = up ? v[j] : v[j + 4];
    const float keep = up ? v[j + 4] : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const bool up = lane & 2;
    const float send = up ? v[j] : v[j + 2];
    const float keep = up ? v[j + 2] : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  {
    const bool up = lane & 1;
    const float send = up ? v[0] : v[1];
    const float keep = up ? v[1] : v[0];
    v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
  }
  return v[0];   // lane l owns column (bit-reversed mapping resolved below): column index = colsum32_col(lane)
}
// column owned by `lane` after warp_colsum32: at each halving step a lane with the bit set keeps the upper half
__device__ __forceinline__ int colsum32_col(int lane) {
  return ((lane & 16) ? 16 : 0) + ((lane & 8) ? 8 : 0) + ((lane & 4) ? 4 : 0) + ((lane & 2) ? 2 : 0) + ((lane & 1) ? 1 : 0);
}

// ------------------------------------------------------------------------------------------------
// Epilogues (one specialisation per fused op)
// ------------------------------------------------------------------------------------------------
template <int EPI, int BN>
struct Epilogue;

// epilogues whose inputs can be loaded while the mainloop is still running define prefetch(); others do not
template <int EPI>
struct EpiHasPrefetch { static constexpr bool value = EPI == EPI_RES || EPI == EPI_SCALE_RELUMASK || EPI == EPI_GATE_BWD || EPI == EPI_DX; };

// tanh/sigmoid gate of ResidualConv1DGLU (wavenet_vocoder/models/modules.py:494-510).
// tile columns [0,128) = 'a' (tanh) channels cb..cb+127, [128,256) = 'b' (sigmoid) channels.
// ptr: 0 ta_out, 1 sb_out, 2 z_out (bf16 [pos, Gh]), 3 bias fp32 [2*Gh];  i0 = Gh, i2 = bias stride per batch item (0: one bias
// for every item; 2*Gh: per-item gate biases of the speaker conditioning - every M tile lies within one item)
template <>
struct Epilogue<EPI_GATE, 256> {
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    const int Gh = e.i[0];
    const int cb = c.n_tile * 128;
    const float* bias = static_cast<const float*>(e.ptr[3]) + size_t(c.b) * e.i[2];
    __nv_bfloat16* ta_o = static_cast<__nv_bfloat16*>(e.ptr[0]);
    __nv_bfloat16* sb_o = static_cast<__nv_bfloat16*>(e.ptr[1]);
    __nv_bfloat16* z_o = static_cast<__nv_bfloat16*>(e.ptr[2]);
    if (e.i[11]) {   // split-bf16 mode: accurate tanh / sigmoid, z written as hi | lo (row pitch 2 Gh); forward only (no stashes)
      const int cq = c.cg;
      float a[32], g[32], ba[32], bb[32];
      load_f32x32(bias + cb + cq * 32, ba);
      load_f32x32(bias + Gh + cb + cq * 32, bb);
      acc_ld32f(c.trow + cq * 32, a);
      acc_ld32f(c.trow + 128 + cq * 32, g);
#pragma unroll
      for (int j = 0; j < 32; ++j) a[j] = tanhf_(a[j] + ba[j]) * sigmoidf_(g[j] + bb[j]);
      if (c.valid) {
        __nv_bfloat16* zr = z_o + (size_t(c.b) * c.T + c.t) * (2 * Gh) + cb + cq * 32;
        store_split32(zr, zr + Gh, a);
      }
      return;
    }
    {
      const int cq = c.cg;
      float a[32], g[32], ba[32], bb[32];
      load_f32x32(bias + cb + cq * 32, ba);
      load_f32x32(bias + Gh + cb + cq * 32, bb);
      acc_ld32f(c.trow + cq * 32, a);
      acc_ld32f(c.trow + 128 + cq * 32, g);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        a[j] = tanh_approx_(a[j] + ba[j]);
        g[j] = sigmoid_approx_(g[j] + bb[j]);
      }
      // three stores per call through the rotating tiles: tanh stash, z, sigmoid stash (omap 0 / 2 / 1)
      if (ta_o) {
        uint8_t* t = c.tile(c.sk % kSTiles);
        stage_put_sw(t, c.lane, cq, a);
        tile_store(t, c.omap + 0, cb, c);
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) a[j] *= g[j];
      {
        uint8_t* t = c.tile(c.sk % kSTiles);
        stage_put_sw(t, c.lane, cq, a);
        tile_store(t, c.omap + 2, cb, c);
      }
      if (ta_o) {
        uint8_t* t = c.tile(c.sk % kSTiles);
        stage_put_sw(t, c.lane, cq, g);
        tile_store(t, c.omap + 1, cb, c);
      }
    }
  }
};

// residual output of the block (modules.py:512-520): x_out = (W_o z + b_o + x) * res_scale, plus the
// dropped-out copy the NEXT layer's dilated conv consumes (modules.py:483-484).
// ptr: 0 x_in, 1 x_out, 2 xd_out (nullable), 3 bias fp32 [R], 7 device u64 added to the seed (nullable; lets a
// replayed CUDA graph draw fresh masks);  f0 res_scale, f1 dropout p;  i1 = layer
template <int BN>
struct Epilogue<EPI_RES, BN> {
  // the x tile (residual input) of column group 0 does not depend on this kernel's MMAs: load it while the mainloop runs.
  // kCoherent: x was written by another CTA of the same grid (persistent layer chain)
  template <bool kCoherent = false>
  static __device__ __forceinline__ void prefetch(const EpiArgs& e, const EpiCtx& c) {
    if (e.i[11]) return;   // split-bf16 mode reads x directly in run()
    tile_fill_sw<kCoherent>(c.tile(2), static_cast<const __nv_bfloat16*>(e.ptr[0]) + c.row0 * BN, BN, c.nrows, c);
  }
  template <bool kCoherent = false>
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    const int R = BN;
    __nv_bfloat16* x_out = static_cast<__nv_bfloat16*>(e.ptr[1]);
    __nv_bfloat16* xd_out = static_cast<__nv_bfloat16*>(e.ptr[2]);
    const float* bias = static_cast<const float*>(e.ptr[3]);
    const float rs = e.f[0], p = e.f[1];
    if (e.i[11]) {   // split-bf16 mode: x_in / x_out rows are [hi(R) | lo(R)]
      const __nv_bfloat16* x_in = static_cast<const __nv_bfloat16*>(e.ptr[0]);
      const size_t r2 = (size_t(c.b) * c.T + c.t) * (2 * R);
#pragma unroll 1
      for (int gq = 0; gq < BN / 128; ++gq) {
        const int j0 = gq * 128 + c.cg * 32;
        float acc[32], x[32], bv[32];
        load_f32x32(bias + j0, bv);
        acc_ld32f(c.trow + j0, acc);
        if (c.valid) {
          load_split32(x_in + r2 + j0, x_in + r2 + R + j0, x);
#pragma unroll
          for (int j = 0; j < 32; ++j) acc[j] = (acc[j] + bv[j] + x[j]) * rs;
          store_split32(x_out + r2 + j0, x_out + r2 + R + j0, acc);
        }
      }
      return;
    }
    const float keep_inv = 1.f / (1.f - p);
    const unsigned long long seed = e.seed + (e.ptr[7] ? *static_cast<const unsigned long long*>(e.ptr[7]) : 0ull);
    const uint32_t hs = hash_seed(seed, uint32_t(e.i[1]));
    const size_t row = (size_t(c.b) * c.T + c.t) * R;
    if (BN == 256) tile_fill_sw<kCoherent>(c.tile(1), static_cast<const __nv_bfloat16*>(e.ptr[0]) + c.row0 * BN + 128, BN, c.nrows, c);
#pragma unroll 1
    for (int gq = 0; gq < BN / 128; ++gq) {
      // tiles: x of group 0 / 1 arrives in tile 2 / 1 and is replaced in place by x_out; the dropped copies go to tile 0 (group 0)
      // and tile 2 (group 1): store order T2, T0, T1, T2 - never a tile of the two preceding stores (tile_store)
      uint8_t* tile = c.tile(gq == 0 ? 2 : 1);
      uint8_t* tile_d = c.tile(gq == 0 ? 0 : 2);
      const int cq = c.cg;
      const int j0 = gq * 128 + cq * 32;
      float acc[32], x[32], bv[32];
      load_f32x32(bias + j0, bv);
      acc_ld32f(c.trow + j0, acc);
      stage_get_sw(tile, c.lane, cq, x);
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = (acc[j] + bv[j] + x[j]) * rs;
      stage_put_sw(tile, c.lane, cq, acc);      // same rows/columns this lane just read
      tile_store(tile, c.omap + 0, gq * 128, c);
      if (xd_out) {
        const uint32_t thr = uint32_t(p * 65536.f);
#pragma unroll
        for (int j = 0; j < 32; j += 2) {
          const uint32_t h = hash_bits32(hs, (row + j0 + j) >> 1);
          acc[j] = (h & 0xFFFFu) >= thr ? acc[j] * keep_inv : 0.f;
          acc[j + 1] = (h >> 16) >= thr ? acc[j + 1] * keep_inv : 0.f;
        }
        stage_put_sw(tile_d, c.lane, cq, acc);
        tile_store(tile_d, c.omap + 1, gq * 128, c);
      }
    }
  }
};

// out = dropout(act(acc + bias)).  ptr: 0 out bf16 [pos, ldo] (nullable), 1 bias fp32 (nullable), 2 out fp32
// [pos, ldo] (nullable), 7 device u64 seed offset (nullable);  i0 = ldo, i1 = act (0 none, 1 relu, 2 tanh),
// i2 = n_valid columns, i3 = dropout hash stream, i4 = position offset of the dropout hash;  f1 = dropout rate (0 = off;
// mask = hash(seed, stream, (i4 + pos)*ldo + col)): a launch over rows [i4, i4 + T*B) of a larger matrix draws the same mask as
// one launch over the whole matrix
template <int BN>
struct Epilogue<EPI_BIAS_ACT, BN> {
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    const int ldo = e.i[0], act = e.i[1], nvalid = e.i[2];
    __nv_bfloat16* ob = static_cast<__nv_bfloat16*>(e.ptr[0]);
    const float* bias = static_cast<const float*>(e.ptr[1]);
    float* of = static_cast<float*>(e.ptr[2]);
    const size_t row = (size_t(c.b) * c.T + c.t) * ldo;
    const size_t hrow = row + size_t(e.i[4]) * ldo;
    uint8_t* t_o = c.tile(0);
    const float pdrop = e.f[1];
    const float keep_inv = 1.f / (1.f - pdrop);
    const unsigned long long seed = e.seed + (e.ptr[7] ? *static_cast<const unsigned long long*>(e.ptr[7]) : 0ull);
    const uint32_t hs = hash_seed(seed, uint32_t(e.i[3]));
    if (e.i[11]) {   // split-bf16 mode: bf16 output rows are [hi(ldo) | lo(ldo)] (pitch 2 ldo); fp32 output unchanged; the dropout
                     // mask is the bf16 path's draw (same element index), applied before the value is split
#pragma unroll 1
      for (int gq = 0; gq < BN / 128; ++gq) {
        const int c0 = c.n_tile * BN + gq * 128 + c.cg * 32;
        if (c0 >= nvalid) continue;
        float acc[32];
        acc_ld32f(c.trow + gq * 128 + c.cg * 32, acc);
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          float v = acc[j];
          if (bias && c0 + j < nvalid) v += __ldg(bias + c0 + j);
          if (act == 1) v = fmaxf(v, 0.f);
          else if (act == 2) v = tanhf_(v);
          if (pdrop > 0.f) v = (hash_uniform32(hs, hrow + c0 + j) >= pdrop) ? v * keep_inv : 0.f;
          acc[j] = c0 + j < nvalid ? v : 0.f;
        }
        if (!c.valid) continue;
        if (of) for (int j = 0; j < 32 && c0 + j < nvalid; ++j) of[row + c0 + j] = acc[j];
        if (ob) {
          __nv_bfloat16* r2 = ob + (size_t(c.b) * c.T + c.t) * (2 * size_t(ldo)) + c0;
          if (c0 + 32 <= ldo) store_split32(r2, r2 + ldo, acc);
          else for (int j = 0; j < 32 && c0 + j < ldo; ++j) {
            const __nv_bfloat16 h = __float2bfloat16(acc[j]);
            r2[j] = h; r2[ldo + j] = __float2bfloat16(acc[j] - __bfloat162float(h));
          }
        }
      }
      return;
    }
#pragma unroll 1
    for (int gq = 0; gq < BN / 128; ++gq) {
      const int g0 = c.n_tile * BN + gq * 128;
      if (g0 >= nvalid) break;  // warp-uniform
      const bool full = g0 + 128 <= nvalid;
      {
        const int cq = c.cg;
        const int c0 = g0 + cq * 32;
        float acc[32];
        if (c0 < nvalid) acc_ld32f(c.trow + gq * 128 + cq * 32, acc);
        else {
#pragma unroll
          for (int j = 0; j < 32; ++j) acc[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          float v = acc[j];
          if (bias && c0 + j < nvalid) v += __ldg(bias + c0 + j);
          if (act == 1) v = fmaxf(v, 0.f);
          else if (act == 2) v = tanhf_(v);
          if (pdrop > 0.f) v = (hash_uniform32(hs, hrow + c0 + j) >= pdrop) ? v * keep_inv : 0.f;
          acc[j] = v;
        }
        if (ob && full) stage_put_sw(t_o, c.lane, cq, acc);
        if (c.valid && c0 < nvalid) {
          if (of) {
            if (c0 + 32 <= nvalid) store_f32x32(of + row + c0, acc);
            else for (int j = 0; j < 32 && c0 + j < nvalid; ++j) of[row + c0 + j] = acc[j];
          }
          if (ob && !full) for (int j = 0; j < 32 && c0 + j < nvalid; ++j) ob[row + c0 + j] = __float2bfloat16(acc[j]);
        }
      }
      if (ob && full) tile_flush<4>(t_o, ob + c.row0 * ldo + g0, ldo, c.nrows, c);
    }
  }
};

// 256-way softmax cross entropy against the NEXT sample (wavenet.py:488, modules.py:781-798).
// ptr: 0 targets int32 [B,T], 1 lengths int32 [B], 2 bias fp32 [256], 3 loss_sum fp32, 4 nonzero-count fp32,
//      5 dlogits bf16 [pos, ld] (nullable; un-normalised softmax - onehot, stored as an error-compensated bf16 PAIR:
//        columns [0,256) = hi, [256,512) = lo = bf16(v - hi) — the target entry p_y - 1 sits next to 1.0 where a single
//        bf16 has 2^-8 spacing, i.e. it would lose p_y entirely), 6 logits fp32 [pos,256] (nullable);  i1 = ld (>= 512)
template <>
struct Epilogue<EPI_CE, 256> {
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    if (c.cg != 0) return;  // row-wise softmax: one warp per row quarter walks all 256 columns
    const int* tgt = static_cast<const int*>(e.ptr[0]);
    const int* len = static_cast<const int*>(e.ptr[1]);
    const float* bias = static_cast<const float*>(e.ptr[2]);
    __nv_bfloat16* dl = static_cast<__nv_bfloat16*>(e.ptr[5]);
    float* lo_out = static_cast<float*>(e.ptr[6]);
    const size_t ld = size_t(e.i[1]);
    const size_t row = (size_t(c.b) * c.T + c.t) * 256;
    const bool w = c.valid && (c.t + 1 < c.T) && (c.t + 1 < __ldg(len + c.b));
    const int y = w ? __ldg(tgt + size_t(c.b) * c.T + c.t + 1) : -1;
    float mx = -INFINITY, zy = 0.f;
#pragma unroll 1
    for (int j0 = 0; j0 < 256; j0 += 32) {
      float v[32];
      acc_ld32f(c.trow + j0, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        v[j] += __ldg(bias + j0 + j);
        mx = fmaxf(mx, v[j]);
        if (j0 + j == y) zy = v[j];
      }
      if (lo_out && c.valid) store_f32x32(lo_out + row + j0, v);
    }
    float se = 0.f;
#pragma unroll 1
    for (int j0 = 0; j0 < 256; j0 += 32) {
      float v[32];
      acc_ld32f(c.trow + j0, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) se += __expf(v[j] + __ldg(bias + j0 + j) - mx);
    }
    const float lse = mx + __logf(se);
    float loss = w ? (lse - zy) : 0.f;
    float cnt = (loss != 0.f) ? 1.f : 0.f;
    if (dl) {
      const float inv = 1.f / se;
      uint8_t* t_hi = c.tile(0);
      uint8_t* t_lo = c.tile(1);
#pragma unroll 1
      for (int gq = 0; gq < 2; ++gq) {
#pragma unroll 1
        for (int cq = 0; cq < 4; ++cq) {
          const int j0 = gq * 128 + cq * 32;
          float v[32], lo[32];
          acc_ld32f(c.trow + j0, v);
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float pj = __expf(v[j] + __ldg(bias + j0 + j) - mx) * inv;
            const float d = w ? (pj - ((j0 + j == y) ? 1.f : 0.f)) : 0.f;
            const float hi = __bfloat162float(__float2bfloat16(d));
            v[j] = hi;
            lo[j] = d - hi;
          }
          stage_put_sw(t_hi, c.lane, cq, v);
          stage_put_sw(t_lo, c.lane, cq, lo);
        }
        tile_flush<1>(t_hi, dl + c.row0 * ld + gq * 128, ld, c.nrows, c);
        tile_flush<1>(t_lo, dl + c.row0 * ld + 256 + gq * 128, ld, c.nrows, c);
      }
    }
    loss = warp_sum(loss);
    cnt = warp_sum(cnt);
    if (c.lane == 0) {
      atomicAdd(static_cast<float*>(e.ptr[3]), loss);
      atomicAdd(static_cast<float*>(e.ptr[4]), cnt);
    }
  }
};

// Discretised mixture-of-logistics NLL (wavenet_vocoder/models/mixture.py:18-74; masked mean
// modules.py:800-817) with its analytic gradient. Tile has 32 columns: [logit(nm) | mean(nm) | log_scale(nm)].
// ptr: 0 targets f32 [B,T], 1 lengths, 2 bias fp32 [3nm], 3 loss_sum, 4 mask_sum, 5 dyhat bf16 [pos, ld]
//      (nullable, un-normalised; 32 columns written), 6 yhat fp32 [pos,32] (nullable)
// f0 log_scale_min, f1 1/(num_classes-1), f2 log((num_classes-1)/2);  i0 = nr_mix (<= 10), i1 = ld
// i2 != 0: single-Gaussian head instead (wavenet_vocoder/models/gaussian.py:5-37): columns [mean | log_scale], f3 = log_scale_min_gauss,
// i2 = 1 log-density loss, i2 = 2 log(CDF(y + 1/(nc-1)) - CDF(y - 1/(nc-1))) loss
template <>
struct Epilogue<EPI_MOL, 32> {
  static __device__ __forceinline__ float softplus(float x) {
    return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x)));
  }
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    if (c.cg != 0) return;
    const float* tgt = static_cast<const float*>(e.ptr[0]);
    const int* len = static_cast<const int*>(e.ptr[1]);
    const float* bias = static_cast<const float*>(e.ptr[2]);
    __nv_bfloat16* dy = static_cast<__nv_bfloat16*>(e.ptr[5]);
    float* yo = static_cast<float*>(e.ptr[6]);
    const int nm = e.i[0];
    const float lsm = e.f[0], hw = e.f[1], logc = e.f[2];
    const size_t row = (size_t(c.b) * c.T + c.t) * 32;
    const bool w = c.valid && (c.t + 1 < c.T) && (c.t + 1 < __ldg(len + c.b));
    const float y = w ? __ldg(tgt + size_t(c.b) * c.T + c.t + 1) : 0.f;
    float v[32];
    acc_ld32f(c.trow, v);
    if (e.i[2] != 0) {   // ---- single Gaussian ----
      const float lsg = e.f[3];
      const float m = v[0] + __ldg(bias), sraw = v[1] + __ldg(bias + 1);
      if (yo && c.valid) {
        float o[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) o[j] = 0.f;
        o[0] = m; o[1] = sraw;
        store_f32x32(yo + row, o);
      }
      const float ls = fmaxf(sraw, lsg);
      float nll, dm, dls;
      if (e.i[2] == 1) {
        const float iv = __expf(-2.f * ls), d = y - m;
        nll = 0.5f * (1.8378770664093453f + 2.f * ls + d * d * iv);
        dm = -d * iv;
        dls = 1.f - d * d * iv;
      } else {
        const float inv = __expf(-ls);
        const float zp = (y + hw - m) * inv, zn = (y - hw - m) * inv;
        const float P = normcdff(zp) - normcdff(zn);
        nll = -__logf(fmaxf(P, 1e-12f));
        if (P > 1e-12f) {
          const float pp = 0.3989422804014327f * __expf(-0.5f * zp * zp), pn = 0.3989422804014327f * __expf(-0.5f * zn * zn);
          dm = (pp - pn) * inv / P;
          dls = (pp * zp - pn * zn) / P;
        } else { dm = 0.f; dls = 0.f; }
      }
      if (sraw < lsg) dls = 0.f;
      if (dy && c.valid) {
        float g[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) g[j] = 0.f;
        if (w) { g[0] = dm; g[1] = dls; }
        store_bf16x32(dy + (size_t(c.b) * c.T + c.t) * size_t(e.i[1]), g);
      }
      float loss = warp_sum(w ? nll : 0.f);
      float cnt = warp_sum(w ? 1.f : 0.f);
      if (c.lane == 0) {
        atomicAdd(static_cast<float*>(e.ptr[3]), loss);
        atomicAdd(static_cast<float*>(e.ptr[4]), cnt);
      }
      return;
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = (j < 3 * nm) ? v[j] + __ldg(bias + j) : 0.f;
    if (yo && c.valid) store_f32x32(yo + row, v);
    // log-softmax of the mixture logits
    float lmx = -INFINITY;
    for (int k = 0; k < nm; ++k) lmx = fmaxf(lmx, v[k]);
    float lse = 0.f;
    for (int k = 0; k < nm; ++k) lse += __expf(v[k] - lmx);
    lse = lmx + __logf(lse);
    float tot[10], dm[10], ds[10];
    float tmx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 10; ++k) {
      tot[k] = -INFINITY; dm[k] = 0.f; ds[k] = 0.f;
      if (k < nm) {
        const float m = v[nm + k], sraw = v[2 * nm + k];
        const float ls = fmaxf(sraw, lsm);
        const float inv = __expf(-ls);
        const float cy = y - m;
        const float pin = inv * (cy + hw), nin = inv * (cy - hw), mid = inv * cy;
        const float cp = sigmoidf_(pin), cn = sigmoidf_(nin);
        const float delta = cp - cn;
        float lp, dlp_dm, dlp_dls;  // derivatives of log-prob wrt mean and (clamped) log-scale
        if (y < -0.999f) {
          lp = pin - softplus(pin);
          const float g = 1.f - cp;  // d/dpin
          dlp_dm = -inv * g; dlp_dls = -pin * g;
        } else if (y > 0.999f) {
          lp = -softplus(nin);
          const float g = -cn;  // d/dnin
          dlp_dm = -inv * g; dlp_dls = -nin * g;
        } else if (delta > 1e-5f) {
          lp = __logf(fmaxf(delta, 1e-12f));
          const float gp = cp * (1.f - cp) / delta, gn = -cn * (1.f - cn) / delta;
          dlp_dm = -inv * (gp + gn); dlp_dls = -(pin * gp + nin * gn);
        } else {
          const float sm = sigmoidf_(mid);
          lp = mid - ls - 2.f * softplus(mid) - logc;
          const float g = 1.f - 2.f * sm;
          dlp_dm = -inv * g; dlp_dls = -mid * g - 1.f;
        }
        tot[k] = lp + (v[k] - lse);
        tmx = fmaxf(tmx, tot[k]);
        dm[k] = dlp_dm;
        ds[k] = (sraw >= lsm) ? dlp_dls : 0.f;
      }
    }
    float tse = 0.f;
#pragma unroll
    for (int k = 0; k < 10; ++k)
      if (k < nm) tse += __expf(tot[k] - tmx);
    const float nll = -(tmx + __logf(tse));
    if (dy && c.valid) {
      float g[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) g[j] = 0.f;
      if (w) {
#pragma unroll
        for (int k = 0; k < 10; ++k)
          if (k < nm) {
            const float post = __expf(tot[k] - tmx) / tse;   // posterior responsibility
            const float prior = __expf(v[k] - lse);
            g[k] = prior - post;
            g[nm + k] = -post * dm[k];
            g[2 * nm + k] = -post * ds[k];
          }
      }
      store_bf16x32(dy + (size_t(c.b) * c.T + c.t) * size_t(e.i[1]), g);
    }
    float loss = warp_sum(w ? nll : 0.f);
    float cnt = warp_sum(w ? 1.f : 0.f);
    if (c.lane == 0) {
      atomicAdd(static_cast<float*>(e.ptr[3]), loss);
      atomicAdd(static_cast<float*>(e.ptr[4]), cnt);
    }
  }
};

// backward through ReLU: out = acc * scale * (h > 0).
// ptr: 0 out bf16 [pos, ldo], 1 h bf16 [pos, ldo], 2 device scalar fp32* (nullable; multiplies 1/x),
//      3 int64 fixed-point [ldo] column sums of `out` (fx_add; nullable: bias gradient);  f0 const scale; i0 = ldo
template <int BN>
struct Epilogue<EPI_SCALE_RELUMASK, BN> {
  // h of column group 0 is loaded while the mainloop runs, that of group 1 (BN = 256) after it
  static __device__ __forceinline__ void prefetch(const EpiArgs& e, const EpiCtx& c) {
    const int ldo = e.i[0];
    const __nv_bfloat16* h = static_cast<const __nv_bfloat16*>(e.ptr[1]);
    tile_fill_sw(c.tile(2), h + c.row0 * ldo + size_t(c.n_tile) * BN, ldo, c.nrows, c);
  }
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    const int ldo = e.i[0];
    __nv_bfloat16* out = static_cast<__nv_bfloat16*>(e.ptr[0]);
    float s = e.f[0];
    if (e.ptr[2]) s /= fmaxf(__ldg(static_cast<const float*>(e.ptr[2])), 1e-20f);
    if (BN == 256)
      tile_fill_sw(c.tile(1), static_cast<const __nv_bfloat16*>(e.ptr[1]) + c.row0 * ldo + size_t(c.n_tile) * BN + 128, ldo, c.nrows, c);
#pragma unroll 1
    for (int gq = 0; gq < BN / 128; ++gq) {
      const size_t off = c.row0 * ldo + size_t(c.n_tile) * BN + gq * 128;
      uint8_t* tile = c.tile(gq == 0 ? 2 : 1);
      const int cq = c.cg;
      float acc[32], hv[32];
      acc_ld32f(c.trow + gq * 128 + cq * 32, acc);
      stage_get_sw(tile, c.lane, cq, hv);
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = hv[j] > 0.f ? acc[j] * s : 0.f;
      stage_put_sw(tile, c.lane, cq, acc);
      tile_flush<4>(tile, out + off, ldo, c.nrows, c);
      if (e.ptr[3]) {
        const float cs = warp_colsum32(acc, c.lane);
        fx_add(static_cast<long long*>(e.ptr[3]) + c.n_tile * BN + gq * 128 + cq * 32 + colsum32_col(c.lane), cs);
      }
    }
  }
};

// backward of the gate: dz -> (da, db).  ptr: 0 ta, 1 sb (bf16 [pos,Gh]), 2 dg out (bf16 [pos,2Gh]), 3 / 4 int64 fixed-point [2Gh]
// gate-bias gradients (column sums of dg, fx_add; nullable — dilated-conv bias and cin-conv bias get the same sum); i0 = Gh,
// i1 = stride of ptr 3 per batch item (0: one sum over all items; 2*Gh: per-item sums for the speaker conditioning)
template <int BN>
struct Epilogue<EPI_GATE_BWD, BN> {
  // ta of column group 0 is loaded while the mainloop runs; sb of group 0 and both inputs of group 1 after it
  static __device__ __forceinline__ void prefetch(const EpiArgs& e, const EpiCtx& c) {
    const int Gh = e.i[0];
    tile_fill_sw(c.tile(2), static_cast<const __nv_bfloat16*>(e.ptr[0]) + c.row0 * Gh + c.n_tile * BN, Gh, c.nrows, c);
  }
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    const int Gh = e.i[0];
    const __nv_bfloat16* ta = static_cast<const __nv_bfloat16*>(e.ptr[0]);
    const __nv_bfloat16* sb = static_cast<const __nv_bfloat16*>(e.ptr[1]);
    uint8_t* t0 = c.tile(2);
    uint8_t* t1 = c.tile(1);
    tile_fill_sw(t1, sb + c.row0 * Gh + c.n_tile * BN, Gh, c.nrows, c);
#pragma unroll 1
    for (int gq = 0; gq < BN / 128; ++gq) {
      const int cb = c.n_tile * BN + gq * 128;
      const int cq = c.cg;
      float dz[32], a[32], s[32];
      if (gq > 0) {   // the tiles of group 0's stores must be released before group 1's inputs overwrite them
        tile_guard(c);
        tile_fill_sw(t0, ta + c.row0 * Gh + cb, Gh, c.nrows, c);
        tile_fill_sw(t1, sb + c.row0 * Gh + cb, Gh, c.nrows, c);
      }
      stage_get_sw(t0, c.lane, cq, a);
      stage_get_sw(t1, c.lane, cq, s);
      acc_ld32f(c.trow + gq * 128 + cq * 32, dz);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float da = dz[j] * (1.f - a[j] * a[j]) * s[j];
        const float db = dz[j] * a[j] * s[j] * (1.f - s[j]);
        a[j] = da;
        s[j] = db;
      }
      stage_put_sw(t0, c.lane, cq, a);     // in place: this lane's own rows / columns
      stage_put_sw(t1, c.lane, cq, s);
      tile_store(t0, c.omap + 0, cb, c);
      tile_store(t1, c.omap + 0, Gh + cb, c);
      if (e.ptr[3]) {
        const float ca = warp_colsum32(a, c.lane), cb2 = warp_colsum32(s, c.lane);
        const int col = cb + cq * 32 + colsum32_col(c.lane);
        long long* sum = static_cast<long long*>(e.ptr[3]) + size_t(c.b) * e.i[1];
        const FxAdd x0 = fx_issue(sum + col, ca);
        const FxAdd x1 = fx_issue(sum + Gh + col, cb2);
        if (e.ptr[4]) {
          const FxAdd x2 = fx_issue(static_cast<long long*>(e.ptr[4]) + col, ca);
          const FxAdd x3 = fx_issue(static_cast<long long*>(e.ptr[4]) + Gh + col, cb2);
          fx_check(x2);
          fx_check(x3);
        }
        fx_check(x0);
        fx_check(x1);
      }
    }
  }
};

// gradient wrt the block input: dx = dropout_mask/keep * acc + res_scale * dx_out
// ptr: 0 dxo bf16 [pos,R] (nullable), 1 dx_out bf16 [pos,R], 2 int64 fixed-point [R] += f2 * column sums of dx_out (nullable: bias
// gradient of the 1x1 that produced this layer's input), 7 device u64 seed offset (nullable);
// f0 res_scale, f1 dropout p, f2 bias-gradient scale; i1 = layer
template <int BN>
struct Epilogue<EPI_DX, BN> {
  // kCoherent: dxo was written by another CTA of the same grid (persistent layer chain)
  template <bool kCoherent = false>
  static __device__ __forceinline__ void prefetch(const EpiArgs& e, const EpiCtx& c) {
    const __nv_bfloat16* dxo = static_cast<const __nv_bfloat16*>(e.ptr[0]);
    if (dxo) tile_fill_sw<kCoherent>(c.tile(2), dxo + c.row0 * BN, BN, c.nrows, c);   // column group 0; group 1 (BN = 256) is loaded in run()
  }
  template <bool kCoherent = false>
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    const int R = BN;
    const __nv_bfloat16* dxo = static_cast<const __nv_bfloat16*>(e.ptr[0]);
    const float rs = e.f[0], p = e.f[1];
    const float keep_inv = 1.f / (1.f - p);
    const unsigned long long seed = e.seed + (e.ptr[7] ? *static_cast<const unsigned long long*>(e.ptr[7]) : 0ull);
    const uint32_t hs = hash_seed(seed, uint32_t(e.i[1]));
    const size_t row = (size_t(c.b) * c.T + c.t) * R;
    if (BN == 256 && dxo) tile_fill_sw<kCoherent>(c.tile(1), dxo + c.row0 * BN + 128, BN, c.nrows, c);
#pragma unroll 1
    for (int gq = 0; gq < BN / 128; ++gq) {
      uint8_t* tile = c.tile(gq == 0 ? 2 : 1);
      const int cq = c.cg;
      const int j0 = gq * 128 + cq * 32;
      float acc[32], g[32];
      acc_ld32f(c.trow + j0, acc);
      if (p > 0.f) {
        const uint32_t thr = uint32_t(p * 65536.f);
#pragma unroll
        for (int j = 0; j < 32; j += 2) {
          const uint32_t h = hash_bits32(hs, (row + j0 + j) >> 1);
          acc[j] = (h & 0xFFFFu) >= thr ? acc[j] * keep_inv : 0.f;
          acc[j + 1] = (h >> 16) >= thr ? acc[j + 1] * keep_inv : 0.f;
        }
      }
      if (dxo) {
        stage_get_sw(tile, c.lane, cq, g);
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] += rs * g[j];
      }
      stage_put_sw(tile, c.lane, cq, acc);
      tile_store(tile, c.omap + 0, gq * 128, c);
      if (e.ptr[2]) {
        const float cs = warp_colsum32(acc, c.lane);
        fx_add(static_cast<long long*>(e.ptr[2]) + j0 + colsum32_col(c.lane), cs * e.f[2]);
      }
    }
  }
};

// LSTM cell on a SWAPPED GEMM: accumulator rows = gate pre-activations of 32 hidden units (tile row p: gate = p/32
// in i,j,f,o order, unit = 32*m_tile + p%32 — the packed recurrent weight rows are permuted accordingly), columns =
// batch items. Implements tf.nn.rnn_cell.LSTMCell (forget_bias 1) wrapped by ZoneoutLSTMCell
// (tacotron/models/modules.py:81-142): the carried state is zoned, the OUTPUT is the un-zoned new h (:118,142).
// ptr: 0 pre fp32 (row of batch item b = pre + b*i3; gate-major [4H]; nullable), 1 bias fp32 [4H] (nullable),
//      2 c_prev fp32 [B][H], 3 c_out fp32 [B][H], 4 h_prev bf16 (+ b*i4), 5 h_state_out bf16 (+ b*i5),
//      6 h_out bf16 (+ b*i6; un-zoned, zero past the sequence length), 7 gate stash bf16 [B][4H] (nullable),
//      8 tanh(c_new) stash bf16 [B][H] (nullable), 9 lengths int32 [B] (nullable), 10 device u64 seed offset
// i0 = H, i1 = B, i3 = pre stride, i4/i5/i6 = row strides, i7 = time step, i8 = hash stream, i9 = training
// f0 = zoneout rate
// i11 != 0: split-bf16 mode, forward only (the stashes 7 / 8 are not written). h_prev / h_state rows are swapped-GEMM state operands
// [hi | lo | hi]: lo at +i10, the second hi copy at +2 i10. h_out is written as hi at +0 and lo at +i2, plus a second hi copy at +2 i2
// when i11 == 2 (h_out is the next GEMM's state operand) - with i11 == 1 it is a plain [hi | lo] activation row.
template <>
struct Epilogue<EPI_LSTM, 32> {
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    const int H = e.i[0], nb = e.i[1];
    float* ex = reinterpret_cast<float*>(c.smem_all);  // [4 gates][32 units][33]
    const int q = c.qbar - 1;
    if (c.cg == 0) {
      float v[32];
      acc_ld32f(c.trow, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) ex[(q * 32 + c.lane) * 33 + j] = v[j];
    }
    asm volatile("bar.sync 5, 512;\n" ::: "memory");
    const float* pre = static_cast<const float*>(e.ptr[0]);
    const float* bias = static_cast<const float*>(e.ptr[1]);
    const float* c_prev = static_cast<const float*>(e.ptr[2]);
    float* c_out = static_cast<float*>(e.ptr[3]);
    const __nv_bfloat16* h_prev = static_cast<const __nv_bfloat16*>(e.ptr[4]);
    __nv_bfloat16* h_state = static_cast<__nv_bfloat16*>(e.ptr[5]);
    __nv_bfloat16* h_out = static_cast<__nv_bfloat16*>(e.ptr[6]);
    __nv_bfloat16* gst = static_cast<__nv_bfloat16*>(e.ptr[7]);
    __nv_bfloat16* tst = static_cast<__nv_bfloat16*>(e.ptr[8]);
    const int* lens = static_cast<const int*>(e.ptr[9]);
    const unsigned long long seed = e.seed + (e.ptr[10] ? *static_cast<const unsigned long long*>(e.ptr[10]) : 0ull);
    const uint32_t hs_c = hash_seed(seed, uint32_t(e.i[8]) * 2u), hs_h = hash_seed(seed, uint32_t(e.i[8]) * 2u + 1u);
    const float z = e.f[0];
    const int t = e.i[7];
    const int split = e.i[11];
    const int etid = (c.cg * 4 + q) * 32 + c.lane;
    const int u0 = c.m_tile * 32, b0 = c.n_tile * 32;
#pragma unroll 1
    for (int p = etid; p < 1024; p += 512) {
      const int bl = p >> 5, ul = p & 31;
      const int b = b0 + bl, u = u0 + ul;
      if (b >= nb || u >= H) continue;
      float zi = ex[(0 * 32 + ul) * 33 + bl], zj = ex[(1 * 32 + ul) * 33 + bl];
      float zf = ex[(2 * 32 + ul) * 33 + bl], zo = ex[(3 * 32 + ul) * 33 + bl];
      if (pre) {
        const float* pr = pre + size_t(b) * e.i[3];
        zi += pr[u]; zj += pr[H + u]; zf += pr[2 * H + u]; zo += pr[3 * H + u];
      }
      if (bias) { zi += bias[u]; zj += bias[H + u]; zf += bias[2 * H + u]; zo += bias[3 * H + u]; }
      float gi = sigmoidf_(zi), gj = tanhf_(zj), gf = sigmoidf_(zf + 1.f), go = sigmoidf_(zo);
      const float cp = c_prev[size_t(b) * H + u];
      const __nv_bfloat16* hpp = h_prev + size_t(b) * e.i[4] + u;
      const float hp = split ? __bfloat162float(hpp[0]) + __bfloat162float(hpp[e.i[10]]) : __bfloat162float(hpp[0]);
      const float cn = gf * cp + gi * gj;
      const float tc = tanhf_(cn);
      const float hn = go * tc;
      const bool live = lens ? (t < lens[b]) : true;
      float cs, hsv, ho = hn;
      if (e.i[9]) {
        const uint64_t idx = (uint64_t(t) * nb + b) * H + u;
        cs = (z <= 0.f || hash_uniform32(hs_c, idx) >= z) ? cn : cp;
        hsv = (z <= 0.f || hash_uniform32(hs_h, idx) >= z) ? hn : hp;
      } else {
        cs = (1.f - z) * cn + z * cp;
        hsv = (1.f - z) * hn + z * hp;
      }
      float tcs = tc;
      if (!live) { cs = cp; hsv = hp; ho = 0.f; gi = gj = gf = go = 0.f; tcs = 0.f; }
      c_out[size_t(b) * H + u] = cs;
      if (split) {
        const __nv_bfloat16 sh = __float2bfloat16(hsv), oh = __float2bfloat16(ho);
        __nv_bfloat16* hs = h_state + size_t(b) * e.i[5] + u;
        hs[0] = sh; hs[e.i[10]] = __float2bfloat16(hsv - __bfloat162float(sh)); hs[2 * e.i[10]] = sh;
        __nv_bfloat16* hq = h_out + size_t(b) * e.i[6] + u;
        hq[0] = oh; hq[e.i[2]] = __float2bfloat16(ho - __bfloat162float(oh));
        if (split == 2) hq[2 * e.i[2]] = oh;
        continue;
      }
      h_state[size_t(b) * e.i[5] + u] = __float2bfloat16(hsv);
      h_out[size_t(b) * e.i[6] + u] = __float2bfloat16(ho);
      if (gst) {
        __nv_bfloat16* g = gst + size_t(b) * 4 * H;
        g[u] = __float2bfloat16(gi); g[H + u] = __float2bfloat16(gj);
        g[2 * H + u] = __float2bfloat16(gf); g[3 * H + u] = __float2bfloat16(go);
      }
      if (tst) tst[size_t(b) * H + u] = __float2bfloat16(tcs);
    }
  }
};

// transposed fp32 output of a swapped GEMM: accumulator rows = features k, columns = batch items b.
// rows [0, i0) -> ptr0[b*i1 + k], rows [i0, i3) -> ptr1[b*i4 + (k - i0)]; i2 / i5 = 0 overwrite, 1 accumulate (+=), 2 atomic
// accumulate (required with split-K); i6 = B
template <>
struct Epilogue<EPI_TOUT, 32> {
  static __device__ __forceinline__ void run(const EpiArgs& e, const EpiCtx& c) {
    if (c.cg != 0) return;
    const int k = c.t, nb = e.i[6];
    float v[32];
    acc_ld32f(c.trow, v);
    float* dst; int ld, acc, kk;
    if (k < e.i[0]) { dst = static_cast<float*>(e.ptr[0]); ld = e.i[1]; acc = e.i[2]; kk = k; }
    else if (k < e.i[3]) { dst = static_cast<float*>(e.ptr[1]); ld = e.i[4]; acc = e.i[5]; kk = k - e.i[0]; }
    else return;
    if (!dst) return;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int b = c.n_tile * 32 + j;
      if (b < nb) {
        float* d = dst + size_t(b) * ld + kk;
        if (acc == 2) atomicAdd(d, v[j]);      // split-K: several CTAs own slices of the reduction
        else *d = acc ? *d + v[j] : v[j];
      }
    }
  }
};

// ------------------------------------------------------------------------------------------------
// act_gemm kernel
//   Consumer warpgroup w (warps 4w..4w+3) computes rows [64 (w >> 1), +64) x columns [BN/2 (w & 1), +BN/2) of the tile with
//   wgmma, its accumulators in registers. When the reduction is complete the four warpgroups write them to a shared fp32
//   tile that aliases the (then idle) pipeline stages, and the same 16 warps run the epilogue on it: warp e owns rows
//   [32 (e % 4), +32) (one per lane) and column group e / 4.
// ------------------------------------------------------------------------------------------------
template <int BN>
struct ActGemmCfg {
  static constexpr int kABytes = kBM * kBK * 2;   // 16 KB
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccBytes = kBM * BN * 4;
  static constexpr int kEpiBytes = 4 * kSTileBytes;        // staging tile 2 of the 4 row quarters: the only bytes outside the ring
  static constexpr int kTailBytes = 8 * kSTileBytes;       // staging tiles 0 and 1: the ring's last bytes, after the mainloop
  static constexpr int kPipeBudget = 232448 - kEpiBytes - 1024 /*align*/ - 256 /*barriers*/;
  // as many stages as fit (4 at BN = 256, 6 at 128 and for the narrow swapped GEMMs of the recurrences, capped at 6)
  static constexpr int kStages = kPipeBudget / kStageBytes > 6 ? 6 : kPipeBudget / kStageBytes;
  // after the mainloop the ring holds the fp32 accumulator tile at its start and staging tiles 0 and 1 at its end
  static constexpr int kPipeBytes =
      kStages * kStageBytes > kAccBytes + kTailBytes ? kStages * kStageBytes : kAccBytes + kTailBytes;
  static constexpr int kSmemBytes = kPipeBytes + kEpiBytes + 1024 + 256;
  static_assert(kStages >= 2 && kPipeBytes <= kPipeBudget && kSmemBytes <= 232448, "shared memory budget");
  static_assert(kPipeBytes % 1024 == 0, "staging tiles must be aligned to the 1024-byte swizzle atom");

  // `smem` is the 1024-byte aligned base of the dynamic shared memory.
  // the stage barriers follow the dedicated staging tile: kStages full barriers, then kStages empty barriers
  static __device__ __forceinline__ uint64_t* full_bar(uint8_t* smem) {
    return reinterpret_cast<uint64_t*>(smem + kPipeBytes + kEpiBytes);
  }
  static __device__ __forceinline__ uint64_t* empty_bar(uint8_t* smem) { return full_bar(smem) + kStages; }
  // One thread initialises the stage barriers. A full barrier takes the producer's one arrival (plus the stage's TMA bytes), an
  // empty barrier `empty_count` arrivals: one per consumer warp of every CTA that multicasts into the stage.
  static __device__ __forceinline__ void init_barriers(uint8_t* smem, uint32_t empty_count) {
    uint64_t* full = full_bar(smem);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&full[kStages + i], empty_count);
    }
    fence_barrier_init();
  }
};

// One (m_tile, n_tile) output tile of `g`: the body of every act_gemm_kernel CTA and of every ticket of the persistent WaveNet layer
// chains. TMA producer loop, wgmma mainloop over k-blocks [kb_lo, kb_hi), the fp32 accumulator tile, the fused epilogue (on `epi`)
// and the drain of its TMA stores. The caller has initialised the stage barriers (ActGemmCfg<BN>::init_barriers, empty count
// kActEpiWarps * cs) behind a CTA barrier and has made the tile's inputs visible; the tile ends with every store's global writes
// complete in the threads that issued them (no CTA barrier at its end).
// `smem` is the 1024-byte aligned base of the dynamic shared memory; cs / crank / cmask describe the multicast cluster.
// b / t0: the batch item and first time step of m_tile (m_tile = b * g.tiles_per_b + t0 / kBM). The caller divides, so that
// act_gemm_kernel can do it before its PDL wait, off the path from the previous kernel's end to this tile's first TMA load.
// ptxas allocates the 96 registers by how the tile indices and the k-block range reach this body: act_gemm_kernel reads blockIdx.x
// and computes b / t0 and the split-K range at its entry. Reading blockIdx.x / .y in here instead spills the gate GEMM's epilogue to a 72-byte
// stack (24 as it is; DESIGN §4), so check `-Xptxas -v` for every instantiation after changing how the arguments arrive.
// kChain: the tile is a ticket of a persistent layer chain, whose epilogue inputs may come from other CTAs of the same grid
template <int EPI, int BN, bool kChain = false>
__device__ __forceinline__ void act_gemm_tile(const GemmArgs& g, const EpiArgs& epi, uint8_t* smem, int m_tile, int n_tile,
                                              int b, int t0, int kb_lo, int kb_hi, uint32_t cs, uint32_t crank, uint16_t cmask,
                                              long long* dbg) {
  using Cfg = ActGemmCfg<BN>;
  constexpr int WN = BN / 2;          // columns per consumer warpgroup
  float* acc_s = reinterpret_cast<float*>(smem);
  // staging tiles, tile-major over the row quarters: tiles 0 and 1 end the ring, the dedicated tile 2 follows it
  uint8_t* staging = smem + Cfg::kPipeBytes - Cfg::kTailBytes;
  uint64_t* full_bar = Cfg::full_bar(smem);
  uint64_t* empty_bar = Cfg::empty_bar(smem);
  const int warp = threadIdx.x >> 5;
  const int total_kb = kb_hi - kb_lo;

  if (warp == kActEpiWarps) {
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      int kb_global = 0;
      for (int s = 0; s < g.nseg; ++s) {
        const Seg sg = g.seg[s];
        for (int l = 0; l < sg.nlayers; ++l) {
          for (int kb = 0; kb < sg.nkb; ++kb, ++kb_global) {
            if (kb_global < kb_lo || kb_global >= kb_hi) continue;
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
            uint8_t* sa = smem + stage * Cfg::kStageBytes;
            uint8_t* sb = sa + Cfg::kABytes;
            tma_load_4d(sa, &g.amap[sg.map], &full_bar[stage], sg.k0 + kb * kBK, t0 + sg.shift, b, sg.layer0 + l);
            if (cs == 1) {
              tma_load_3d(sb, &g.bmap, &full_bar[stage], g.b_k0 + kb_global * kBK, n_tile * BN, g.b_layer);
            } else {
              const int rows = BN / int(cs);     // this CTA's slice of the weight tile (whole 8-row swizzle atoms: 1024-byte aligned)
              tma_load_3d_mc(sb + crank * rows * (kBK * 2), &g.bmap, &full_bar[stage], g.b_k0 + kb_global * kBK,
                             n_tile * BN + int(crank) * rows, g.b_layer, cmask);
            }
            if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    const int q = warp & 3;  // row quarter of this warp in the epilogue
    const int lane = threadIdx.x & 31;
    EpiCtx c;
    c.lane = lane;
    c.cg = warp >> 2;
    c.qbar = 1 + q;
    c.b = b; c.T = g.T;
    const int tw = t0 + q * 32;          // first time step of this warp
    c.t = tw + c.lane;
    c.valid = c.t < g.T;
    c.row0 = size_t(b) * g.T + tw;
    c.nrows = g.T - tw < 0 ? 0 : (g.T - tw > 32 ? 32 : g.T - tw);
    c.stg = staging + q * kSTileBytes;
    c.smem_all = smem + Cfg::kAccBytes;
    c.m_tile = m_tile;
    c.omap = g.omap; c.tq = tw; c.sk = 0;
    c.n_tile = n_tile;
    constexpr bool kCoh = EPI == EPI_RES || EPI == EPI_DX;   // the epilogues that take a template read-path flag
    if constexpr (kCoh) Epilogue<EPI, BN>::template prefetch<kChain>(epi, c);
    else if constexpr (EpiHasPrefetch<EPI>::value) Epilogue<EPI, BN>::prefetch(epi, c);

    // ---- mainloop: this warpgroup's 64 x WN quarter of the tile
    const int wg = warp >> 2, mh = wg >> 1, nh = wg & 1;
    float d[WN / 2];
#pragma unroll
    for (int i = 0; i < WN / 2; ++i) d[i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < total_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      __syncwarp();                    // wgmma is warp-aligned: reconverge after the spin-wait
      if (dbg && kb == 0 && threadIdx.x == 0) dbg[2] = clock64();
      const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes) + uint32_t(mh * 64 * 128);
      const uint32_t sb = smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kABytes) + uint32_t(nh * WN * 128);
      const uint64_t adesc = make_gdesc_sw128(sa, 16, 1024);
      const uint64_t bdesc = make_gdesc_sw128(sb, 16, 1024);
      wgmma_fence();
      wgmma_fence_regs(d);
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k)
        // advancing K by 16 bf16 = 32 bytes inside the 128-byte swizzle row: +2 in the (addr>>4) field
        Wgmma<WN, 0, 0>::mma(d, adesc + uint64_t(k * 2), bdesc + uint64_t(k * 2), (kb > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_fence_regs(d);
      // the previous k-block's MMAs have finished reading their stage: hand it back to the producer(s)
      wgmma_wait<1>();
      if (kb > 0 && lane == 0) {
        if (cs == 1) mbar_arrive(&empty_bar[prev]);
        else for (uint32_t r = 0; r < cs; ++r) mbar_arrive_cluster(&empty_bar[prev], r);
      }
      prev = stage;
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    if (dbg && threadIdx.x == 0) dbg[3] = clock64();
    // every warpgroup's MMAs are done with the stages: the accumulator tile may overwrite them
    asm volatile("bar.sync 6, 512;\n" ::: "memory");
    {
      const int r0 = mh * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < WN / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = r0 + 8 * i, col = nh * WN + 8 * j + 2 * (lane & 3);
          *reinterpret_cast<float2*>(acc_s + r * BN + ((((col >> 2) ^ (r & 7)) << 2) | (col & 3))) =
              make_float2(d[4 * j + 2 * i], d[4 * j + 2 * i + 1]);
        }
    }
    asm volatile("bar.sync 6, 512;\n" ::: "memory");
    const int row = q * 32 + lane;
    c.trow = AccRow{acc_s + row * BN, 0, row & 7};
    if (dbg && threadIdx.x == 0) dbg[4] = clock64();
    if constexpr (kCoh) Epilogue<EPI, BN>::template run<kChain>(epi, c);
    else Epilogue<EPI, BN>::run(epi, c);
    if (dbg && threadIdx.x == 0) dbg[5] = clock64();
    tile_store_drain(c);
  }
}

template <int EPI, int BN>
__global__ void __launch_bounds__(kActGemmThreads, 1) act_gemm_kernel(const __grid_constant__ GemmArgs g) {
  using Cfg = ActGemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // the M tile, its batch item / first time step and the k-block range are taken here, first: before the PDL wait, and where they
  // are computed decides the tile body's spills (act_gemm_tile)
  const int m_tile = blockIdx.x;
  const int b = m_tile / g.tiles_per_b;
  const int t0 = (m_tile - b * g.tiles_per_b) * kBM;
  int all_kb = 0;
  for (int s = 0; s < g.nseg; ++s) all_kb += g.seg[s].nkb * g.seg[s].nlayers;
  // split-K: gridDim.z CTAs share one output tile, each reducing a contiguous slice of the k-blocks (the epilogue must
  // then accumulate atomically)
  const int kb_lo = int((long long)all_kb * blockIdx.z / gridDim.z), kb_hi = int((long long)all_kb * (blockIdx.z + 1) / gridDim.z);

  // Thread-block cluster along M (launch attribute; 1 = no cluster): the weight tile of a pipeline stage is identical for every M
  // tile, so each CTA of the cluster fetches 1/cs of its rows and MULTICASTS them to all peers (one L2 read feeds cs SMs).
  const uint32_t cs = cluster_nctarank(), crank = cluster_ctarank();
  const uint16_t cmask = uint16_t((1u << cs) - 1u);
  long long* dbg = g.dbg ? g.dbg + ((size_t(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * kDbgSlots : nullptr;
  if (dbg && threadIdx.x == 0) { dbg[0] = clock64(); dbg[8] = globaltimer_ns(); dbg[11] = smid(); }

  if ((threadIdx.x >> 5) == kActEpiWarps && elect_one()) {
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(&g.amap[i]);
    tma_prefetch_desc(&g.bmap);
    // a stage is free once every consumer warp of EVERY CTA of the cluster has consumed it (peers multicast into it)
    Cfg::init_barriers(smem, kActEpiWarps * cs);
  }
  __syncthreads();
  if (cs > 1) cluster_sync_all();      // peers' barriers are initialised before any remote arrive / multicast write
  // everything above is CTA-local set-up and overlaps the previous kernel's tail under PDL; global memory from here on
  pdl_wait();
  pdl_launch_dependents();
  if (dbg && threadIdx.x == 0) { dbg[1] = clock64(); dbg[9] = globaltimer_ns(); }

  act_gemm_tile<EPI, BN>(g, g.epi, smem, m_tile, blockIdx.y, b, t0, kb_lo, kb_hi, cs, crank, cmask, dbg);
  __syncthreads();
  if (dbg && threadIdx.x == 0) { dbg[6] = clock64(); dbg[10] = globaltimer_ns(); }
  // no CTA may leave while a peer can still arrive on its barriers or multicast into its shared memory
  if (cs > 1) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------------
// wgrad_gemm kernel: both operands MN-major (channels contiguous), reduction over positions.
//   Warps 0..7 = two consumer warpgroups (warpgroup w: output rows [64 w, +64), i.e. A channel block w, all N columns),
//   warp 8 = TMA producer. The accumulators go from registers straight to the fp32 output.
// ------------------------------------------------------------------------------------------------
constexpr int kWgBM = 128;      // output rows per tile: one 64-row block per consumer warpgroup
constexpr int kWgBN = 256;      // up to 256 output columns per tile: the A block pair is reused for twice the MMA work
constexpr int kWgStages = 4;
constexpr int kWgStageBytes = 6 * (kBK * 128);  // A: 2 blocks of [64 pos x 128 B] (16 KB), B: up to 4 blocks (32 KB)
constexpr int kWgSmemBytes = kWgStages * kWgStageBytes + 1024 + 256;
static_assert(kWgSmemBytes <= 232448, "shared memory budget");

template <int N>
__device__ __forceinline__ void wgrad_consume(const WgradArgs& g, const WgradTile& tile, uint8_t* smem, uint64_t* full_bar,
                                              uint64_t* empty_bar, int total_kb) {
  constexpr int kBlk = kBK * 128;  // bytes of one [64 pos x 64 ch] block
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  int stage = 0, prev = 0;
  uint32_t phase = 0;
  for (int kb = 0; kb < total_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    __syncwarp();
    const uint32_t sa = smem_u32(smem + stage * kWgStageBytes) + uint32_t(wg * kBlk);
    const uint32_t sb = smem_u32(smem + stage * kWgStageBytes + 2 * kBlk);
    // MN-major SW128: LBO = distance between 64-channel blocks, SBO = distance between 8-position groups
    const uint64_t adesc = make_gdesc_sw128(sa, kBlk, 1024);
    const uint64_t bdesc = make_gdesc_sw128(sb, kBlk, 1024);
    wgmma_fence();
    wgmma_fence_regs(d);
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k)
      // 16 positions = 2 swizzle atoms of 8 rows x 128 B = 2048 bytes -> +128 in the (addr>>4) field
      Wgmma<N, 1, 1>::mma(d, adesc + uint64_t(k * 128), bdesc + uint64_t(k * 128), (kb > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_fence_regs(d);
    wgmma_wait<1>();
    if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == kWgStages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  float sc = tile.scale;
  if (tile.div) sc /= fmaxf(__ldg(tile.div), 1e-20f);
  float* out = g.out + tile.out_off;
  const int m0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int m = m0 + 8 * i, n = 8 * j + 2 * (lane & 3) + e;
        if (m < tile.m_valid && n < tile.n_valid) {
          float* o = out + size_t(m) * tile.ldc + n;
          const float r = d[4 * j + 2 * i + e] * sc;
          if (tile.accumulate == 2) atomicAdd(o, r);
          else if (tile.accumulate == 1) *o += r;
          else *o = r;
        }
      }
}

__global__ void __launch_bounds__(kGemmThreads, 1) wgrad_gemm_kernel(const __grid_constant__ WgradArgs g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kWgStages * kWgStageBytes);
  uint64_t* empty_bar = full_bar + kWgStages;
  const int warp = threadIdx.x >> 5;
  const WgradTile tile = g.tiles[blockIdx.x];
  const int kb_per_b = (g.T + kBK - 1) / kBK;
  const int total_kb = kb_per_b * g.B;
  const int nblk = (tile.n_valid + 63) >> 6;   // 64-channel B blocks this tile needs (1..4)

  if (warp == 8 && elect_one()) {
    for (int i = 0; i < kWgStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }   // 8 consumer warps
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();               // (the tile table read above is written once at init, never by a preceding kernel)
  pdl_launch_dependents();
  constexpr int kBlk = kBK * 128;

  if (warp == 8) {
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int bb = 0; bb < g.B; ++bb)
        for (int kb = 0; kb < kb_per_b; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], uint32_t(2 + nblk) * kBlk);
          uint8_t* sa = smem + stage * kWgStageBytes;
          uint8_t* sb = sa + 2 * kBlk;
          const int tpos = kb * kBK;
          tma_load_4d(sa, &g.map[tile.a_map], &full_bar[stage], tile.a_ch0, tpos + tile.a_shift, bb, tile.a_layer);
          tma_load_4d(sa + kBlk, &g.map[tile.a_map], &full_bar[stage], tile.a_ch0 + 64, tpos + tile.a_shift, bb, tile.a_layer);
          for (int i = 0; i < nblk; ++i)
            tma_load_4d(sb + i * kBlk, &g.map[tile.b_map], &full_bar[stage], tile.b_ch0 + 64 * i, tpos + tile.b_shift, bb, tile.b_layer);
          if (++stage == kWgStages) { stage = 0; phase ^= 1; }
        }
    }
  } else {
    switch (nblk) {
      case 1: wgrad_consume<64>(g, tile, smem, full_bar, empty_bar, total_kb); break;
      case 2: wgrad_consume<128>(g, tile, smem, full_bar, empty_bar, total_kb); break;
      case 3: wgrad_consume<192>(g, tile, smem, full_bar, empty_bar, total_kb); break;
      default: wgrad_consume<256>(g, tile, smem, full_bar, empty_bar, total_kb); break;
    }
  }
}

}  // namespace t2
