// t2_gemm.cu — host side of the wgmma GEMM engine: TMA tensor-map encoding and kernel launches.
#include <stdlib.h>
#include <mutex>

#include "t2_gemm.cuh"
#include "t2_gemm.h"

namespace t2 {

static long long* g_timing_buffer = nullptr;
void set_timing_buffer(long long* p) { g_timing_buffer = p; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// 4-D map over a channels-last bf16 activation tensor: dims (C, T, B, L), box (64, rows, 1, 1), 128B swizzle.
static int encode_act_map(CUtensorMap* m, const ActT& a, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  T2_REQUIRE(fn != nullptr, T2_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  T2_REQUIRE(a.ptr && (reinterpret_cast<uintptr_t>(a.ptr) & 15) == 0, T2_ERR_INVALID_ARG,
             "activation pointer must be non-null and 16-byte aligned");
  T2_REQUIRE(a.ld % 8 == 0 && a.C >= 1 && a.C <= a.ld, T2_ERR_UNSUPPORTED_SHAPE,
             "activation row pitch must be a multiple of 8 elements (ld=%d C=%d)", a.ld, a.C);
  cuuint64_t dims[4] = {cuuint64_t(a.C), cuuint64_t(a.T), cuuint64_t(a.B), cuuint64_t(a.L)};
  cuuint64_t strides[3] = {cuuint64_t(a.ld) * 2, cuuint64_t(a.ld) * 2 * a.T,
                           cuuint64_t(a.ld) * 2 * a.T * a.B};
  cuuint32_t box[4] = {64, cuuint32_t(box_rows), 1, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(a.ptr), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  T2_REQUIRE(r == CUDA_SUCCESS, T2_ERR_CUDA, "cuTensorMapEncodeTiled(act) failed: %d (C=%d T=%d B=%d L=%d ld=%d)",
             int(r), a.C, a.T, a.B, a.L, a.ld);
  return T2_OK;
}

// 3-D map over a channels-last bf16 OUTPUT tensor [B][T][C] for the epilogue's TMA stores: box 64 columns x 32 rows (one epilogue row
// quarter), 128-byte swizzle; rows >= T of an item and columns >= C are clipped by the hardware.
static int encode_out_map(CUtensorMap* m, const void* ptr, int C, int T, int B) {
  EncodeTiledFn fn = get_encode_fn();
  T2_REQUIRE(fn != nullptr, T2_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  T2_REQUIRE(ptr && (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && C % 8 == 0, T2_ERR_INVALID_ARG,
             "epilogue output must be non-null, 16-byte aligned, with a row pitch that is a multiple of 8 elements (C=%d)", C);
  cuuint64_t dims[3] = {cuuint64_t(C), cuuint64_t(T), cuuint64_t(B)};
  cuuint64_t strides[2] = {cuuint64_t(C) * 2, cuuint64_t(C) * 2 * T};
  cuuint32_t box[3] = {64, 32, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  T2_REQUIRE(r == CUDA_SUCCESS, T2_ERR_CUDA, "cuTensorMapEncodeTiled(out) failed: %d (C=%d T=%d B=%d)", int(r), C, T, B);
  return T2_OK;
}

// 3-D map over packed bf16 weights [L][N][K]: dims (K, N, L), box (64, rows, 1)
static int encode_wt_map(CUtensorMap* m, const void* w, int N, int K, int L, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  T2_REQUIRE(fn != nullptr, T2_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  T2_REQUIRE(w && (reinterpret_cast<uintptr_t>(w) & 15) == 0, T2_ERR_INVALID_ARG,
             "weight pointer must be non-null and 16-byte aligned");
  T2_REQUIRE(K % 8 == 0, T2_ERR_UNSUPPORTED_SHAPE, "packed weight K must be a multiple of 8 (K=%d)", K);
  cuuint64_t dims[3] = {cuuint64_t(K), cuuint64_t(N), cuuint64_t(L)};
  cuuint64_t strides[2] = {cuuint64_t(K) * 2, cuuint64_t(K) * 2 * N};
  cuuint32_t box[3] = {64, cuuint32_t(box_rows), 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(w), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  T2_REQUIRE(r == CUDA_SUCCESS, T2_ERR_CUDA, "cuTensorMapEncodeTiled(weight) failed: %d (N=%d K=%d L=%d)", int(r),
             N, K, L);
  return T2_OK;
}

// programmatic dependent launch for the GEMM kernels (T2_PDL=0 in the environment turns it off for A/B measurements)
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("T2_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
  return v != 0;
}

// cluster size along M for the weight-tile multicast (T2_CLUSTER in the environment, for A/B measurements; default 1 = off).
// Multicast stays off by default: with the 4-stage ring, clusters of 2 and 4 made every WaveNet GEMM shape slower on an H100
// (DESIGN §4).
int cluster_pref() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("T2_CLUSTER");
    v = e ? atoi(e) : 1;
    if (v != 1 && v != 2 && v != 4 && v != 8) v = 1;
  }
  return v;
}
static int pick_cluster(int BN, const dim3& grid, int request) {
  int cs = request ? request : cluster_pref();
  if (BN < 128 || grid.z > 1) return 1;                 // the swapped recurrence GEMMs (BN = 32) and split-K keep single CTAs
  while (cs > 1 && (grid.x % cs != 0 || (BN / cs) % 8 != 0)) cs >>= 1;
  return cs;
}

template <int EPI, int BN>
static int launch_one(const GemmArgs& g, dim3 grid, int cs, cudaStream_t stream) {
  using Cfg = ActGemmCfg<BN>;
  static bool configured = false;
  if (!configured) {
    T2_CHECK_CUDA(cudaFuncSetAttribute(act_gemm_kernel<EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       Cfg::kSmemBytes));
    configured = true;
  }
  // every launch gets its own slice of the timing buffer (so a captured graph stamps each of its kernel nodes separately)
  if (g.dbg) g_timing_buffer = g.dbg + size_t(grid.x) * grid.y * grid.z * kDbgSlots;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = dim3(kActGemmThreads); cfg.dynamicSmemBytes = Cfg::kSmemBytes; cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (cs > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cs; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr; cfg.numAttrs = na;
  if (cs > 1) {   // a cluster size the device cannot co-schedule is refused here, not at launch
    static int max_clusters[4] = {-1, -1, -1, -1};
    int& mc = max_clusters[cs == 2 ? 1 : cs == 4 ? 2 : 3];
    if (mc < 0) T2_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&mc, act_gemm_kernel<EPI, BN>, &cfg));
    T2_REQUIRE(mc > 0, T2_ERR_UNSUPPORTED_SHAPE, "act_gemm: clusters of %d CTAs cannot be scheduled on this device", cs);
  }
  T2_CHECK_CUDA(cudaLaunchKernelEx(&cfg, act_gemm_kernel<EPI, BN>, g));
  t2_count_launch();
  return T2_OK;
}

// the split-bf16 form of a plain call (ActGemmCall::split)
static int split_form(ActGemmCall& c) {
  T2_REQUIRE(c.na >= 1 && c.na <= 4 && c.nseg >= 1 && 2 * c.nseg <= kMaxSeg && c.w_k0 == 0, T2_ERR_UNSUPPORTED_SHAPE,
             "split-bf16 GEMM: %d maps and %d segments (at most %d) from K column %d", c.na, c.nseg, kMaxSeg / 2, c.w_k0);
  int nkb[4] = {0, 0, 0, 0}, ktot = 0;
  for (int s = 0; s < c.nseg; ++s) {
    const Seg& p = c.seg[s];
    T2_REQUIRE(p.map >= 0 && p.map < c.na && p.k0 == 0 && p.nkb > 0 && (nkb[p.map] == 0 || nkb[p.map] == p.nkb), T2_ERR_INVALID_ARG,
               "split-bf16 GEMM: segment %d must read its map from channel 0, as wide as the other segments of that map", s);
    nkb[p.map] = p.nkb;
    ktot += p.nkb * p.nlayers * kBK;
  }
  for (int i = 0; i < c.na; ++i) {
    const int Cp = nkb[i] * kBK;
    if (Cp) c.a[i] = make_act(c.a[i].ptr, 2 * Cp, c.a[i].T, c.a[i].B, c.a[i].L, 2 * Cp);
  }
  for (int s = c.nseg - 1; s >= 0; --s) {
    const Seg p = c.seg[s];
    c.seg[2 * s] = Seg{p.map, p.shift, 0, 2 * p.nkb, p.layer0, p.nlayers};
    c.seg[2 * s + 1] = Seg{p.map, p.shift, 0, p.nkb, p.layer0, p.nlayers};
  }
  c.nseg *= 2;
  c.wK = 3 * ktot;
  c.epi.i[11] = 1;
  return T2_OK;
}

int make_gemm_args(int epi, int BN, const ActGemmCall& call, GemmArgs& g, dim3& grid, int& cs) {
  ActGemmCall split;
  if (call.split) {
    split = call;
    const int rc = split_form(split);
    if (rc) return rc;
  }
  const ActGemmCall& c = call.split ? split : call;
  // argument checks first: they touch neither the device nor the driver
  T2_REQUIRE(c.na >= 1 && c.na <= 4 && c.nseg >= 1 && c.nseg <= kMaxSeg, T2_ERR_INVALID_ARG,
             "act_gemm: bad map/segment count (%d, %d)", c.na, c.nseg);
  T2_REQUIRE(c.cluster == 0 || c.cluster == 1 || c.cluster == 2 || c.cluster == 4 || c.cluster == 8, T2_ERR_INVALID_ARG,
             "act_gemm: cluster size must be 0 (default), 1, 2, 4 or 8 (got %d)", c.cluster);
  int ktot = 0;
  for (int s = 0; s < c.nseg; ++s) {
    T2_REQUIRE(c.seg[s].map >= 0 && c.seg[s].map < c.na && c.seg[s].nkb > 0 && c.seg[s].nlayers > 0,
               T2_ERR_INVALID_ARG, "act_gemm: bad segment %d", s);
    ktot += c.seg[s].nkb * c.seg[s].nlayers * kBK;
  }
  T2_REQUIRE(c.w_k0 + ktot <= ((c.wK + kBK - 1) / kBK) * kBK, T2_ERR_INVALID_ARG,
             "act_gemm: segments cover K=%d but packed weight has K=%d", ktot, c.wK);
  if (c.ksplit > 1) {
    T2_REQUIRE(epi == EPI_TOUT && c.ksplit * kBK <= ktot, T2_ERR_INVALID_ARG,
               "act_gemm: split-K needs an atomically accumulating epilogue and at least one k-block per slice");
    // the CTAs of one output tile add their partial sums into the same elements: only the atomic mode (2) is race-free
    const bool use0 = c.epi.ptr[0] && c.epi.i[0] > 0, use1 = c.epi.ptr[1] && c.epi.i[3] > c.epi.i[0];
    T2_REQUIRE((!use0 || c.epi.i[2] == 2) && (!use1 || c.epi.i[5] == 2), T2_ERR_INVALID_ARG,
               "act_gemm: split-K needs atomic accumulation (mode 2) into every destination in use (modes %d, %d)", c.epi.i[2],
               c.epi.i[5]);
  }
  memset(&g, 0, sizeof(g));
  for (int i = 0; i < 4; ++i) {
    int rc = encode_act_map(&g.amap[i], c.a[i < c.na ? i : 0], kBM);
    if (rc) return rc;
  }
  grid = dim3((c.T + kBM - 1) / kBM * c.B, c.n_tiles, c.ksplit > 1 ? c.ksplit : 1);
  cs = pick_cluster(BN, grid, c.cluster);
  // weight-tile rows one TMA box fetches: 1/cs of the tile per CTA of a multicast cluster
  int rc = encode_wt_map(&g.bmap, c.w, c.wN, c.wK, c.wL, BN / cs);
  if (rc) return rc;
  for (int s = 0; s < c.nseg; ++s) g.seg[s] = c.seg[s];
  g.nseg = c.nseg;
  g.T = c.T;
  g.tiles_per_b = (c.T + kBM - 1) / kBM;
  g.b_layer = c.w_layer;
  g.b_k0 = c.w_k0;
  g.dbg = g_timing_buffer;
  g.epi = c.epi;
  // output tensor maps of the epilogues that store through TMA (bf16 mode only; the split-bf16 mode keeps direct stores)
  if (!c.epi.i[11]) {
    const void* outs[3] = {nullptr, nullptr, nullptr};
    int ldo = 0;
    if (epi == EPI_GATE) { outs[0] = c.epi.ptr[0]; outs[1] = c.epi.ptr[1]; outs[2] = c.epi.ptr[2]; ldo = c.epi.i[0]; }
    else if (epi == EPI_RES) { outs[0] = c.epi.ptr[1]; outs[1] = c.epi.ptr[2]; ldo = BN; }
    else if (epi == EPI_GATE_BWD) { outs[0] = c.epi.ptr[2]; ldo = 2 * c.epi.i[0]; }
    else if (epi == EPI_DX) { outs[0] = c.epi.ptr[1]; ldo = BN; }
    for (int i = 0; i < 3; ++i)
      if (outs[i]) {
        rc = encode_out_map(&g.omap[i], outs[i], ldo, c.T, c.B);
        if (rc) return rc;
      }
  }
  return T2_OK;
}

long long* take_timing_slice(long long n_slots) {
  long long* p = g_timing_buffer;
  if (p) g_timing_buffer = p + n_slots;
  return p;
}

int launch_bias_act(const BiasActGemm& g, cudaStream_t st) {
  ActGemmCall c;
  memset(&c, 0, sizeof(c));
  T2_REQUIRE(g.ntaps <= kMaxSeg, T2_ERR_UNSUPPORTED_SHAPE, "bias-act GEMM: %d taps are more than %d segments", g.ntaps, kMaxSeg);
  const int Ctot = g.Ctot > 0 ? g.Ctot : g.C, nkb = (g.C + kBK - 1) / kBK;
  c.a[0] = make_act(g.a, Ctot, g.T, g.B, g.layers, g.ld > 0 ? g.ld : Ctot); c.na = 1;
  for (int s = 0; s < g.ntaps; ++s) c.seg[s] = Seg{0, g.shifts ? g.shifts[s] : 0, g.k0s ? g.k0s[s] : 0, nkb, 0, g.layers};
  c.nseg = g.ntaps;
  c.split = g.split;
  c.w = g.w; c.wN = g.N; c.wK = g.wK; c.wL = 1;
  c.T = g.T; c.B = g.B; c.n_tiles = (g.nvalid + g.BN - 1) / g.BN;
  c.epi.ptr[0] = g.out_bf16; c.epi.ptr[1] = const_cast<float*>(g.bias); c.epi.ptr[2] = g.out_f32;
  c.epi.ptr[7] = const_cast<unsigned long long*>(g.step);
  c.epi.i[0] = g.ldo; c.epi.i[1] = g.act; c.epi.i[2] = g.nvalid; c.epi.i[3] = g.stream; c.epi.i[4] = g.hash_row0; c.epi.f[1] = g.pdrop;
  c.epi.seed = g.seed;
  return launch_act_gemm(EPI_BIAS_ACT, g.BN, c, st);
}

int launch_act_gemm(int epi, int BN, const ActGemmCall& c, cudaStream_t stream, int* cluster_used) {
  GemmArgs g;
  dim3 grid;
  int cs = 1;
  const int rc = make_gemm_args(epi, BN, c, g, grid, cs);
  if (rc) return rc;
  if (cluster_used) *cluster_used = cs;
#define T2_CASE(E, N) \
  if (epi == E && BN == N) return launch_one<E, N>(g, grid, cs, stream);
  T2_CASE(EPI_GATE, 256)
  T2_CASE(EPI_RES, 128)
  T2_CASE(EPI_RES, 256)
  T2_CASE(EPI_BIAS_ACT, 128)
  T2_CASE(EPI_BIAS_ACT, 256)
  T2_CASE(EPI_CE, 256)
  T2_CASE(EPI_SCALE_RELUMASK, 128)
  T2_CASE(EPI_SCALE_RELUMASK, 256)
  T2_CASE(EPI_GATE_BWD, 128)
  T2_CASE(EPI_GATE_BWD, 256)
  T2_CASE(EPI_DX, 128)
  T2_CASE(EPI_DX, 256)
  T2_CASE(EPI_MOL, 32)
  T2_CASE(EPI_LSTM, 32)
  T2_CASE(EPI_TOUT, 32)
#undef T2_CASE
  return t2_set_error(T2_ERR_UNSUPPORTED_SHAPE, "act_gemm: no kernel for epilogue %d with BN=%d", epi, BN);
}

int launch_wgrad(const ActT* maps, int nmaps, const WgradTile* tiles_dev, int ntiles, float* out, int T,
                 int B, cudaStream_t stream) {
  T2_REQUIRE(nmaps >= 1 && nmaps <= 6 && ntiles >= 1, T2_ERR_INVALID_ARG, "wgrad: bad map/tile count");
  WgradArgs g;
  memset(&g, 0, sizeof(g));
  for (int i = 0; i < 6; ++i) {
    int rc = encode_act_map(&g.map[i], maps[i < nmaps ? i : 0], kBK);
    if (rc) return rc;
  }
  g.tiles = tiles_dev;
  g.out = out;
  g.T = T;
  g.B = B;
  static bool configured = false;
  if (!configured) {
    T2_CHECK_CUDA(cudaFuncSetAttribute(wgrad_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmemBytes));
    configured = true;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(ntiles); cfg.blockDim = dim3(kGemmThreads); cfg.dynamicSmemBytes = kWgSmemBytes; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  T2_CHECK_CUDA(cudaLaunchKernelEx(&cfg, wgrad_gemm_kernel, g));
  t2_count_launch();
  return T2_OK;
}

void append_wgrad_tiles(std::vector<WgradTile>& v, const WgradTile& proto, int a_ch0, int Ca, int b_ch0, int Cb, long long out_off,
                        int ldc) {
  for (int m0 = 0; m0 < Ca; m0 += kWgBM)
    for (int n0 = 0; n0 < Cb; n0 += kWgBN) {
      WgradTile t;
      memset(&t, 0, sizeof(t));
      t.a_map = proto.a_map; t.a_ch0 = a_ch0 + m0; t.a_shift = proto.a_shift; t.a_layer = proto.a_layer;
      t.b_map = proto.b_map; t.b_ch0 = b_ch0 + n0; t.b_shift = proto.b_shift; t.b_layer = proto.b_layer;
      t.out_off = out_off + (long long)m0 * ldc + n0; t.ldc = ldc;
      t.m_valid = Ca - m0 < kWgBM ? Ca - m0 : kWgBM;
      t.n_valid = Cb - n0 < kWgBN ? Cb - n0 : kWgBN;
      t.scale = proto.scale; t.accumulate = proto.accumulate; t.div = proto.div;
      v.push_back(t);
    }
}

WgradTile dense_proto(int am, int bm, int a_shift) {
  WgradTile t;
  memset(&t, 0, sizeof(t));
  t.a_map = am; t.a_shift = a_shift; t.b_map = bm; t.scale = 1.f;
  return t;
}

void append_conv_wgrad_tiles(std::vector<WgradTile>& v, int k, int a_ch0, int Ca, int b_ch0, int Cb, long long out_off) {
  for (int j = 0; j < k; ++j)
    append_wgrad_tiles(v, dense_proto(0, 1, conv_tap_shift(k, j)), a_ch0, Ca, b_ch0, Cb, out_off + (long long)j * Ca * Cb, Cb);
}

// ------------------------------------------------------------------------------------------------------
// Persistent layer chains: the gate/out GEMMs of every forward layer (or the dz/dx GEMMs of every backward layer) as ONE launch.
// Each CTA takes tickets (ChainTicket; t2_wavenet.cu build_chain) from a global counter in launch order and runs the same tile body as act_gemm_kernel on
// the GemmArgs of that (kind, layer), so every tile computes exactly what its per-layer launch computes. A ticket waits only for
// the neighbour tiles it reads, not for the whole previous GEMM. Progress does not rely on co-residency: a CTA holds one ticket
// at a time and waits only for tickets handed out before its own, all held by running CTAs, so the lowest unfinished ticket can
// always run.
// ------------------------------------------------------------------------------------------------------
constexpr long long kChainTimeoutNs = 1000000000LL;

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// orders generic-proxy accesses (the counters) with async-proxy (TMA) accesses of global memory
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// the previous ticket's barriers are invalidated before their memory is initialised again (the two GEMMs of a chain may place
// them differently: 4 stages at BN 256, 6 at BN 128)
template <int BN>
__device__ __forceinline__ void chain_inval_barriers(uint8_t* smem) {
  using Cfg = ActGemmCfg<BN>;
  uint64_t* full_bar = Cfg::full_bar(smem);
  for (int i = 0; i < 2 * Cfg::kStages; ++i)
    asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(&full_bar[i])) : "memory");
}

// FWD: kind 0 = EPI_GATE (BN 256), kind 1 = EPI_RES (BN1 = R); backward: kind 0 = EPI_GATE_BWD (BN0), kind 1 = EPI_DX (BN1 = R)
template <bool FWD, int BN0, int BN1>
__global__ void __launch_bounds__(kActGemmThreads, 1) wn_chain_kernel(const __grid_constant__ ChainArgs a) {
  constexpr int E0 = FWD ? EPI_GATE : EPI_GATE_BWD, E1 = FWD ? EPI_RES : EPI_DX;
  using C0 = ActGemmCfg<BN0>;
  using C1 = ActGemmCfg<BN1>;
  static_assert(C0::kPipeBytes == C1::kPipeBytes && C0::kEpiBytes == C1::kEpiBytes && C0::kSmemBytes == C1::kSmemBytes,
                "both GEMMs of a chain share one shared-memory plan");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ EpiArgs s_epi;    // the ticket's epilogue arguments with the per-call values filled in
  __shared__ int s_ticket;
  int* done = a.ctr + 16;
  int* stop = a.ctr + 1;       // set once a wait of this launch timed out: the remaining tickets are skipped
  int prev_kind = -1;          // thread 0: the kind whose barriers are initialised
  for (;;) {
    if (threadIdx.x == 0) {
      int t = atomicAdd(a.ctr, 1);
      if (t < a.n_tix && *reinterpret_cast<volatile int*>(stop) == 0) {
        long long* dbg = a.dbg ? a.dbg + size_t(t) * kDbgSlots : nullptr;
        const long long t_start = globaltimer_ns();
        if (dbg) { dbg[0] = t_start; dbg[3] = smid(); }
        const ChainTicket k = a.tix[t];
        for (int i = k.dep_lo; i <= k.dep_hi && t < a.n_tix; ++i)
          while (ld_acquire_gpu(done + i) < k.dep_target) {
            if (globaltimer_ns() - t_start > kChainTimeoutNs) {
              if (atomicExch(stop, 1) == 0) atomicAdd(a.err, 1);   // one count per failed launch, read by the host
              t = a.n_tix;
              break;
            }
            __nanosleep(32);
          }
        fence_proxy_async_global();
        if (dbg) dbg[1] = globaltimer_ns();
        EpiArgs e = a.args[k.kind * a.L + k.layer].epi;
        if (FWD && k.kind == 0 && !a.save) { e.ptr[0] = nullptr; e.ptr[1] = nullptr; }
        if (FWD && k.kind == 1) e.ptr[3] = const_cast<float*>(a.params) + reinterpret_cast<uintptr_t>(e.ptr[3]);
        if (k.kind == 1) { e.seed = a.seed; e.ptr[7] = const_cast<unsigned long long*>(a.d_step); }
        s_epi = e;
        if (prev_kind == 0) chain_inval_barriers<BN0>(smem);
        else if (prev_kind == 1) chain_inval_barriers<BN1>(smem);
        // one CTA per tile, no multicast: one empty-barrier arrival per consumer warp
        if (k.kind == 0) C0::init_barriers(smem, kActEpiWarps);
        else C1::init_barriers(smem, kActEpiWarps);
        prev_kind = k.kind;
      } else {
        t = a.n_tix;
      }
      s_ticket = t;
    }
    __syncthreads();
    const int t = s_ticket;
    if (t >= a.n_tix) break;
    const ChainTicket k = a.tix[t];
    const GemmArgs& g = a.args[k.kind * a.L + k.layer];
    int all_kb = 0;
    for (int s = 0; s < g.nseg; ++s) all_kb += g.seg[s].nkb * g.seg[s].nlayers;
    // The producer's TMA loads follow the acquire (global), and they overwrite ring bytes the previous ticket's epilogue wrote
    // through the generic proxy (accumulator and staging tiles), observed through the CTA barrier above (shared). Both fences are
    // issued by the one thread that issues the loads: the same fence in all 544 threads cost 0.07 ms per Cfg-2 step.
    if ((threadIdx.x >> 5) == kActEpiWarps) {
      fence_proxy_async_global();
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    const int b = k.m / g.tiles_per_b, t0 = (k.m - b * g.tiles_per_b) * kBM;
    if (k.kind == 0) act_gemm_tile<E0, BN0, true>(g, s_epi, smem, k.m, k.n, b, t0, 0, all_kb, 1, 0, 1, nullptr);
    else act_gemm_tile<E1, BN1, true>(g, s_epi, smem, k.m, k.n, b, t0, 0, all_kb, 1, 0, 1, nullptr);
    // the tile's TMA stores are complete in the threads that issued them: publish them to the tiles that wait for this one
    fence_proxy_async_global();
    __syncthreads();
    if (threadIdx.x == 0) {
      red_release_gpu_add(done + k.done, 1);
      if (a.dbg) a.dbg[size_t(t) * kDbgSlots + 2] = globaltimer_ns();
    }
  }
}

template <bool FWD, int BN0, int BN1>
int launch_chain_kernel(const ChainArgs& a, int grid, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    T2_CHECK_CUDA(cudaFuncSetAttribute(wn_chain_kernel<FWD, BN0, BN1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       ActGemmCfg<BN0>::kSmemBytes));
    configured = true;
  }
  wn_chain_kernel<FWD, BN0, BN1><<<grid, kActGemmThreads, ActGemmCfg<BN0>::kSmemBytes, st>>>(a);
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}


int launch_wn_chain(bool fwd, int bn0, int bn1, const ChainArgs& a, int grid, cudaStream_t st) {
  if (fwd && bn0 == 256) return bn1 == 256 ? launch_chain_kernel<true, 256, 256>(a, grid, st) : launch_chain_kernel<true, 256, 128>(a, grid, st);
  if (!fwd && bn0 == 256) return bn1 == 256 ? launch_chain_kernel<false, 256, 256>(a, grid, st) : launch_chain_kernel<false, 256, 128>(a, grid, st);
  if (!fwd && bn0 == 128) return bn1 == 256 ? launch_chain_kernel<false, 128, 256>(a, grid, st) : launch_chain_kernel<false, 128, 128>(a, grid, st);
  return t2_set_error(T2_ERR_UNSUPPORTED_SHAPE, "layer chain: no kernel for %s with BN %d / %d", fwd ? "forward" : "backward", bn0, bn1);
}

}  // namespace t2
