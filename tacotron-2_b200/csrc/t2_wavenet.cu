// t2_wavenet.cu — WaveNet vocoder (teacher-forced train path) on the wgmma GEMM engine.
//
// Replaces wavenet_vocoder/models/wavenet.py:650-721 (step), :476-519 (add_loss) and the layers in
// wavenet_vocoder/models/modules.py / mixture.py of the reference. HBM data layout (DESIGN.md §3):
//   activations  bf16 channels-last [layer][B][T][channels]  (rows are GEMM-M, channels are GEMM-K / N)
//   parameters   fp32 masters in TensorFlow variable layouts, concatenated (drop-in checkpoint order)
//   packed       bf16 K-major GEMM operand copies of the masters, refreshed after every optimizer step
// Per layer the forward is two GEMM launches:
//   gate : [x(t-(k-1)d) | ... | x(t-d) | x(t) | c(t)] (K = kR + 128, k = kernel_size taps) x Wg -> tanh*sigmoid epilogue -> z (+ stashes)
//   out  : z (K = G/2) x Wo -> (o + b + x) * sqrt(.5) epilogue -> x_next
// the skip 1x1 of ALL layers is deferred into one K = L*G/2 GEMM (skips never round-trip through HBM).
// Global (speaker) conditioning (gin_channels > 0) enters the gate GEMM's epilogue as a per-item bias, not as a GEMM operand.
#include <stdlib.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/t2b200.h"
#include "t2_common.cuh"
#include "t2_gemm.h"
#include "t2_params.h"

namespace t2 {
namespace {

typedef __nv_bfloat16 bf16;

struct ColsumJob {
  long long src_off;  // byte offset in workspace of a bf16 [rows][ld] matrix
  long long rows;
  int C, ld;
  long long dst_off, dst2_off;  // fp32 element offsets in grads (dst2 < 0: none)
  float scale;
  int div_scalar;     // index into ws scalars to divide by (or -1)
};

struct Layout {
  t2_wn_config_t c;
  int L, R, G, Gh, S, C, O, Q, B, T, Tc, Kg, ldo, Op;
  int kw;       // taps of the dilated causal convolution (kernel_size): tap j reads x(t - (kw-1-j) d)
  bool split;   // split-bf16 forward (t2_wn_config_t.split_bf16)
  int xm;       // channel multiplier of the stored activations: 2 in split mode (hi | lo), else 1
  bool scalar_in, mol, gauss;   // mol: scalar-input head (mixture of logistics, or a single Gaussian when gauss)
  int Gi, NS;   // global (speaker) conditioning: embedding width (0 = off) and rows of gc_embedding
  float res_scale;
  std::vector<float> skip_scale;
  // params
  std::vector<Param> params;
  long long n_params;
  long long p_in_k, p_in_b, p_f1_k, p_f1_b, p_f2_k, p_f2_b;
  std::vector<long long> p_dil_k, p_dil_b, p_c_k, p_c_b, p_s_k, p_s_b, p_o_k, p_o_b, p_up_k, p_up_b;
  std::vector<long long> p_g_k, p_g_b;   // residual_block_gin_conv of each layer (Gi > 0)
  long long p_emb;                       // gc_embedding [NS][Gi] (Gi > 0)
  long long layer_stride;                // parameter elements per residual layer (every layer has the same tensors)
  // packed (byte offsets)
  long long k_Wg, k_Wo, k_Ws, k_Wf1, k_Wf2, k_WozT, k_WdT, k_WcT, k_Wf1T, k_Wf2T, k_bias_g, k_bias_skip;
  long long packed_bytes;
  // workspace (byte offsets)
  long long w_cup, w_x, w_xd, w_ta, w_sb, w_z, w_h1, w_h2, w_dlog, w_dh2, w_dskip, w_dxin, w_dg, w_dcup;
  long long w_skipsum;
  long long w_spk;      // Gi > 0: int32 [1 + B]: speaker term on / off, then the ids (t2_wn_set_speakers)
  long long w_gbias;    // Gi > 0: fp32 [L][B][G] per-item gate biases: bias_g + (b_gin + W_gin^T emb[id_b])
  long long w_gsum;     // Gi > 0: int64 fixed-point [L][B][G] per-item column sums of d gate pre-activation
  long long w_gfx;      // int64 fixed-point accumulators of the gradients summed by many blocks (t2_common.cuh fx_add)
  long long w_upgrad[2], w_scalars, w_tiles_main, w_tiles_head, w_packjobs, w_colsum, w_tables;
  std::vector<long long> w_upout;
  std::vector<int> up_w;  // width after each upsample layer
  long long workspace_bytes;
  int n_tiles_main, n_tiles_head, n_packjobs, n_colsum;
  std::vector<PackJob> packjobs;
  std::vector<ColsumJob> colsums;
  std::vector<WgradTile> tiles_main, tiles_head;
  std::vector<int> tile_start;   // [L + 1]: first entry of tiles_main that belongs to layer l (the table is layer-major)
  // persistent layer chains, [0] forward, [1] backward: tickets in launch order, and per direction a workspace block of
  // 16 ints (ticket counter first) + 2 * L * MT completion counters, the tickets and the GemmArgs table ([kind][layer])
  int MT;
  int n_chain[2];   // ticket counts (the tickets themselves are built by build_chain only where a chain is launched or queried)
  long long w_chain_ctr[2], w_chain_tix[2], w_chain_args[2], w_chain_err;
  int dil(int l) const { return 1 << (l % (L / c.stacks)); }
};

// The tickets of both chains, in the order of the per-layer launches they replace: forward, per layer the gate tiles (M fastest, then
// N), then the out tiles (none after the last layer); backward, from the top layer down, the dz tiles then the dx tiles. A ticket
// waits only for the tiles whose outputs its GEMM reads (its A operand through the dilated taps, and its epilogue inputs), all of
// them earlier in the order and inside its batch item (the taps' rows before 0 / past T are zero-filled, not read):
//   gate(l, m) <- out(l-1, m-k..m)   rows [t0 - (kw-1)d, t0 + 128) of xd_l, k = ceil((kw-1)d / 128)   (out(l-1, m) also wrote x_l
//                                     for out(l, m))
//   out(l, m)  <- gate(l, m, every n)   z_l rows [t0, t0 + 128)
//   dz(l, m)   <- dx(l+1, m)         dxin_{l+1} rows [t0, t0 + 128)   (and the dx epilogue's residual input of the same rows)
//   dx(l, m)   <- dz(l, m..m+k, every n)   dg_l rows [t0, t0 + 128 + (kw-1)d)
// Every buffer a chain writes is per layer and read only by later tickets, so no ticket overwrites what an earlier one still reads.
// dir 0: forward, 1: backward.
void build_chain(const Layout& lo, int dir, std::vector<ChainTicket>& v) {
  const int tpb = (lo.T + kBM - 1) / kBM;
  auto idx = [&](int kind, int l, int m) { return (kind * lo.L + l) * lo.MT + m; };
  const int ng = lo.G / 256;                                       // N tiles of the gate GEMM (BN = 256)
  const int nz = lo.Gh / (lo.Gh >= 256 ? 256 : 128);               // N tiles of the dz GEMM
  v.clear();
  v.reserve(lo.n_chain[dir]);
  if (dir == 0) {
    for (int l = 0; l < lo.L; ++l) {
      const int k = ((lo.kw - 1) * lo.dil(l) + kBM - 1) / kBM;
      for (int n = 0; n < ng; ++n)
        for (int m = 0; m < lo.MT; ++m) {
          const int m0 = m / tpb * tpb;                            // first M tile of this batch item
          ChainTicket t{0, l, m, n, 0, -1, 0, idx(0, l, m)};
          if (l > 0) { t.dep_lo = idx(1, l - 1, std::max(m0, m - k)); t.dep_hi = idx(1, l - 1, m); t.dep_target = 1; }
          v.push_back(t);
        }
      if (l + 1 < lo.L)
        for (int m = 0; m < lo.MT; ++m) v.push_back(ChainTicket{1, l, m, 0, idx(0, l, m), idx(0, l, m), ng, idx(1, l, m)});
    }
    return;
  }
  for (int l = lo.L - 1; l >= 0; --l) {
    const int k = ((lo.kw - 1) * lo.dil(l) + kBM - 1) / kBM;
    for (int n = 0; n < nz; ++n)
      for (int m = 0; m < lo.MT; ++m) {
        ChainTicket t{0, l, m, n, 0, -1, 0, idx(0, l, m)};
        if (l + 1 < lo.L) { t.dep_lo = t.dep_hi = idx(1, l + 1, m); t.dep_target = 1; }
        v.push_back(t);
      }
    for (int m = 0; m < lo.MT; ++m) {
      const int m1 = m / tpb * tpb + tpb - 1;                      // last M tile of this batch item
      v.push_back(ChainTicket{1, l, m, 0, idx(0, l, m), idx(0, l, std::min(m1, m + k)), nz, idx(1, l, m)});
    }
  }
}

int build_layout(const t2_wn_config_t* cfg, Layout& lo) {
  T2_REQUIRE(cfg != nullptr, T2_ERR_INVALID_ARG, "null config");
  lo.c = *cfg;
  lo.L = cfg->layers; lo.R = cfg->residual_channels; lo.G = cfg->gate_channels; lo.Gh = lo.G / 2;
  lo.S = cfg->skip_out_channels; lo.C = cfg->cin_channels; lo.O = cfg->out_channels;
  lo.Q = cfg->quantize_channels; lo.B = cfg->B; lo.T = cfg->T; lo.Tc = cfg->Tc;
  lo.split = cfg->split_bf16 != 0;
  lo.xm = lo.split ? 2 : 1;
  T2_REQUIRE(!lo.split || cfg->dropout == 0.f, T2_ERR_INVALID_ARG, "split_bf16 (fp32-class forward) needs dropout = 0");
  lo.scalar_in = cfg->input_type != 2;
  lo.mol = lo.scalar_in;
  T2_REQUIRE(lo.L >= 1 && cfg->stacks >= 1 && lo.L % cfg->stacks == 0, T2_ERR_INVALID_ARG, "layers %% stacks != 0");
  T2_REQUIRE(cfg->kernel_size >= 2 && cfg->kernel_size <= 4, T2_ERR_UNSUPPORTED_SHAPE, "kernel_size must be 2, 3 or 4 (got %d)",
             cfg->kernel_size);
  lo.kw = cfg->kernel_size;
  T2_REQUIRE(lo.R == 128 || lo.R == 256, T2_ERR_UNSUPPORTED_SHAPE, "residual_channels must be 128 or 256 (got %d)", lo.R);
  T2_REQUIRE(lo.S == 128 || lo.S == 256, T2_ERR_UNSUPPORTED_SHAPE, "skip_out_channels must be 128 or 256 (got %d)", lo.S);
  T2_REQUIRE(lo.Gh == 128 || lo.Gh == 256, T2_ERR_UNSUPPORTED_SHAPE, "gate_channels must be 256 or 512 (got %d)", lo.G);
  T2_REQUIRE(lo.C == 0 || (lo.C % 8 == 0 && lo.C <= 128), T2_ERR_UNSUPPORTED_SHAPE, "cin_channels must be 0 or a multiple of 8 <= 128");
  lo.gauss = lo.scalar_in && lo.O == 2;
  if (lo.mol) {
    T2_REQUIRE(lo.gauss || (lo.O % 3 == 0 && lo.O >= 3 && lo.O <= 30), T2_ERR_UNSUPPORTED_SHAPE,
               "scalar input needs out_channels = 2 (Gaussian) or 3 * nr_mix <= 30 (mixture of logistics), got %d", lo.O);
  } else {
    T2_REQUIRE(lo.O == 256 && lo.Q == 256, T2_ERR_UNSUPPORTED_SHAPE, "mulaw-quantize needs out_channels == quantize_channels == 256");
  }
  T2_REQUIRE(lo.B >= 1 && lo.T >= 1, T2_ERR_INVALID_ARG, "bad B/T");
  lo.Gi = cfg->gin_channels; lo.NS = cfg->n_speakers;
  T2_REQUIRE(lo.Gi >= 0 && (lo.Gi == 0 || lo.NS >= 1), T2_ERR_INVALID_ARG,
             "gin_channels must be >= 0, and n_speakers >= 1 when gin_channels > 0 (got %d / %d)", lo.Gi, lo.NS);
  T2_REQUIRE(cfg->upsample_type >= 0 && cfg->upsample_type <= 2, T2_ERR_INVALID_ARG,
             "upsample_type must be 0 (SubPixel), 1 (2D) or 2 (1D), got %d", cfg->upsample_type);
  T2_REQUIRE(cfg->upsample_activation >= 0 && cfg->upsample_activation <= 2, T2_ERR_INVALID_ARG,
             "upsample_activation must be 0 (ReLU), 1 (LeakyReLU) or 2 (none), got %d", cfg->upsample_activation);
  T2_REQUIRE(cfg->leaky_alpha >= 0.f && cfg->leaky_alpha <= 1.f, T2_ERR_INVALID_ARG, "leaky_alpha must be in [0, 1], got %g",
             double(cfg->leaky_alpha));
  lo.Kg = lo.kw * lo.R + (lo.C > 0 ? 128 : 0);
  lo.ldo = lo.mol ? 64 : 512;   // row pitch of dlog (bf16): MoL 32 values (+pad so a 64-wide TMA box fits); CE hi|lo pair
  lo.Op = lo.mol ? 64 : 512;    // K of Wf2T (CE: [Wf2^T | Wf2^T] against the hi|lo split of dlog)
  lo.res_scale = cfg->residual_legacy ? float(sqrt(0.5)) : 1.f;
  lo.skip_scale.resize(lo.L);
  for (int l = 0; l < lo.L; ++l) {
    int e = cfg->legacy ? (l == 0 ? lo.L - 1 : lo.L - l) : 0;
    lo.skip_scale[l] = float(pow(sqrt(0.5), e));
  }
  // upsample widths
  lo.up_w.clear();
  if (lo.C > 0 && !cfg->c_pre_upsampled) {
    T2_REQUIRE(cfg->n_upsample >= 1 && cfg->n_upsample <= 4, T2_ERR_INVALID_ARG, "n_upsample out of range");
    T2_REQUIRE(cfg->upsample_type == 2 || cfg->freq_axis_kernel_size == 3, T2_ERR_UNSUPPORTED_SHAPE,
               "freq_axis_kernel_size must be 3");   // ConvTranspose1D has no frequency axis
    for (int i = 0; i < cfg->n_upsample; ++i)
      T2_REQUIRE(cfg->upsample_scales[i] >= 1, T2_ERR_INVALID_ARG, "upsample_scales[%d] = %d < 1", i, cfg->upsample_scales[i]);
    int w = lo.Tc;
    for (int i = 0; i < cfg->n_upsample; ++i) { w *= cfg->upsample_scales[i]; lo.up_w.push_back(w); }
    T2_REQUIRE(w == lo.T, T2_ERR_INVALID_ARG, "Tc * prod(upsample_scales) = %d != T = %d", w, lo.T);
  }
  // ---- parameters (order == oracle/wavenet.py:param_shapes) ----
  lo.n_params = 0;
  lo.params.clear();
  const int cin = lo.scalar_in ? 1 : lo.Q;
  lo.p_in_k = add_param(lo.params, lo.n_params, "input_convolution/kernel", {1, cin, lo.R});
  lo.p_in_b = add_param(lo.params, lo.n_params, "input_convolution/bias", {lo.R});
  for (int l = 0; l < lo.L; ++l) {
    char p[64];
    snprintf(p, sizeof(p), "ResidualConv1DGLU_%d/", l);
    std::string s(p);
    lo.p_dil_k.push_back(add_param(lo.params, lo.n_params, s + "residual_block_causal_conv/kernel", {lo.kw, lo.R, lo.G}));
    lo.p_dil_b.push_back(add_param(lo.params, lo.n_params, s + "residual_block_causal_conv/bias", {lo.G}));
    if (lo.C > 0) {
      lo.p_c_k.push_back(add_param(lo.params, lo.n_params, s + "residual_block_cin_conv/kernel", {1, lo.C, lo.G}));
      lo.p_c_b.push_back(add_param(lo.params, lo.n_params, s + "residual_block_cin_conv/bias", {lo.G}));
    }
    if (lo.Gi > 0) {
      lo.p_g_k.push_back(add_param(lo.params, lo.n_params, s + "residual_block_gin_conv/kernel", {1, lo.Gi, lo.G}));
      lo.p_g_b.push_back(add_param(lo.params, lo.n_params, s + "residual_block_gin_conv/bias", {lo.G}));
    }
    lo.p_s_k.push_back(add_param(lo.params, lo.n_params, s + "residual_block_skip_conv/kernel", {1, lo.Gh, lo.S}));
    lo.p_s_b.push_back(add_param(lo.params, lo.n_params, s + "residual_block_skip_conv/bias", {lo.S}));
    lo.p_o_k.push_back(add_param(lo.params, lo.n_params, s + "residual_block_out_conv/kernel", {1, lo.Gh, lo.R}));
    lo.p_o_b.push_back(add_param(lo.params, lo.n_params, s + "residual_block_out_conv/bias", {lo.R}));
  }
  lo.p_f1_k = add_param(lo.params, lo.n_params, "final_convolution_1/kernel", {1, lo.S, lo.S});
  lo.p_f1_b = add_param(lo.params, lo.n_params, "final_convolution_1/bias", {lo.S});
  lo.p_f2_k = add_param(lo.params, lo.n_params, "final_convolution_2/kernel", {1, lo.S, lo.O});
  lo.p_f2_b = add_param(lo.params, lo.n_params, "final_convolution_2/bias", {lo.O});
  lo.p_emb = lo.Gi > 0 ? add_param(lo.params, lo.n_params, "gc_embedding", {lo.NS, lo.Gi}) : -1;   // outside the residual stack (modules.py:12-21)
  lo.layer_stride = lo.L > 1 ? lo.p_dil_k[1] - lo.p_dil_k[0] : 0;
  for (size_t i = 0; i < lo.up_w.size(); ++i) {
    char p[64];
    snprintf(p, sizeof(p), "local_conditioning_upsampling_%d/", int(i) + 1);
    std::string s(p);
    const int sc = cfg->upsample_scales[i];
    if (cfg->upsample_type == 0) {
      lo.p_up_k.push_back(add_param(lo.params, lo.n_params, s + "kernel", {3, 3, 1, sc}));
      lo.p_up_b.push_back(add_param(lo.params, lo.n_params, s + "bias", {sc}));
    } else if (cfg->upsample_type == 2) {
      lo.p_up_k.push_back(add_param(lo.params, lo.n_params, s + "kernel", {1, sc, lo.C, lo.C}));
      lo.p_up_b.push_back(add_param(lo.params, lo.n_params, s + "bias", {lo.C}));
    } else {
      lo.p_up_k.push_back(add_param(lo.params, lo.n_params, s + "kernel", {3, sc, 1, 1}));
      lo.p_up_b.push_back(add_param(lo.params, lo.n_params, s + "bias", {1}));
    }
  }
  // ---- packed ----
  Arena pk;
  const long long L = lo.L;
  lo.k_Wg = pk.take(fwd_operand_bytes(L * lo.G, lo.Kg, lo.split));
  lo.k_Wo = pk.take(fwd_operand_bytes(L * lo.R, lo.Gh, lo.split));
  lo.k_Ws = pk.take(fwd_operand_bytes(lo.S, L * lo.Gh, lo.split));
  lo.k_Wf1 = pk.take(fwd_operand_bytes(lo.S, lo.S, lo.split));
  lo.k_Wf2 = pk.take(fwd_operand_bytes(lo.O < 32 ? 32 : lo.O, lo.S, lo.split));
  lo.k_WozT = pk.take(L * lo.Gh * (lo.R + lo.S) * 2);
  lo.k_WdT = pk.take(L * lo.R * lo.kw * lo.G * 2);
  lo.k_WcT = pk.take((long long)(lo.C > 0 ? lo.C : 8) * L * lo.G * 2);
  lo.k_Wf1T = pk.take((long long)lo.S * lo.S * 2);
  lo.k_Wf2T = pk.take((long long)lo.S * lo.Op * 2);
  lo.k_bias_g = pk.take(L * lo.G * 4);
  lo.k_bias_skip = pk.take(lo.S * 4);
  lo.packed_bytes = pk.used;
  // ---- workspace ----
  Arena ws;
  const long long BT = (long long)lo.B * lo.T;
  lo.w_cup = ws.take(BT * (lo.split ? 256 : (lo.C > 0 ? lo.C : 8)) * 2);     // split: [hi(C) pad 128 | lo(C) pad 128]
  lo.w_upout.clear();
  for (size_t i = 0; i < lo.up_w.size(); ++i) lo.w_upout.push_back(ws.take((long long)lo.B * lo.C * lo.up_w[i] * 4));
  lo.w_upgrad[0] = ws.take(BT * (lo.C > 0 ? lo.C : 8) * 4);
  lo.w_upgrad[1] = ws.take(BT * (lo.C > 0 ? lo.C : 8) * 4);
  lo.w_x = ws.take(L * BT * lo.R * 2 * lo.xm);
  lo.w_xd = cfg->dropout > 0.f ? ws.take(L * BT * lo.R * 2) : lo.w_x;
  lo.w_ta = ws.take(L * BT * lo.Gh * 2);
  lo.w_sb = ws.take(L * BT * lo.Gh * 2);
  lo.w_z = ws.take(L * BT * lo.Gh * 2 * lo.xm);
  lo.w_h1 = ws.take(BT * lo.S * 2 * lo.xm);
  lo.w_h2 = ws.take(BT * lo.S * 2 * lo.xm);
  lo.w_dlog = ws.take(BT * lo.ldo * 2);
  lo.w_dh2 = ws.take(BT * lo.S * 2);
  lo.w_dskip = ws.take(BT * lo.S * 2);
  lo.w_dxin = ws.take(L * BT * lo.R * 2);
  lo.w_dg = ws.take(L * BT * lo.G * 2);
  lo.w_dcup = ws.take(BT * (lo.C > 0 ? lo.C : 8) * 4);
  lo.w_scalars = ws.take(64 * 4);
  lo.w_skipsum = ws.take(lo.S * 8);
  lo.w_gfx = ws.take(lo.n_params * 8);

  // ---- pack jobs ----
  lo.packjobs.clear();
  std::vector<PackJob>& pj = lo.packjobs;
  for (int l = 0; l < lo.L; ++l) {
    // gate GEMM: one segment per tap, then the conditioning segment (128 columns wide); the skip GEMM loops K over the layers
    const long long wg = lo.k_Wg + fwd_operand_bytes((long long)l * lo.G, lo.Kg, lo.split);
    for (int j = 0; j < lo.kw; ++j)
      add_pack_fwd(pj, lo.split, lo.p_dil_k[l] + (long long)j * lo.R * lo.G, lo.R, lo.G, wg, lo.Kg, j * lo.R, lo.R, 1.f, lo.Gh);
    if (lo.C > 0) add_pack_fwd(pj, lo.split, lo.p_c_k[l], lo.C, lo.G, wg, lo.Kg, lo.kw * lo.R, 128, 1.f, lo.Gh);
    add_pack_fwd(pj, lo.split, lo.p_o_k[l], lo.Gh, lo.R, lo.k_Wo + fwd_operand_bytes((long long)l * lo.R, lo.Gh, lo.split), lo.Gh, 0, lo.Gh);
    add_pack_fwd(pj, lo.split, lo.p_s_k[l], lo.Gh, lo.S, lo.k_Ws, lo.L * lo.Gh, 0, lo.Gh, lo.skip_scale[l], 0, l, lo.L);
    const long long woz = lo.k_WozT + (long long)l * lo.Gh * (lo.R + lo.S) * 2;
    add_pack(pj, lo.p_o_k[l], lo.Gh, lo.R, woz, lo.R + lo.S, 0, 0, lo.res_scale);
    add_pack(pj, lo.p_s_k[l], lo.Gh, lo.S, woz, lo.R + lo.S, 0, lo.R, lo.skip_scale[l]);
    const long long wd = lo.k_WdT + (long long)l * lo.R * lo.kw * lo.G * 2;
    for (int j = 0; j < lo.kw; ++j) add_pack(pj, lo.p_dil_k[l] + (long long)j * lo.R * lo.G, lo.R, lo.G, wd, lo.kw * lo.G, 0, j * lo.G);
    if (lo.C > 0) add_pack(pj, lo.p_c_k[l], lo.C, lo.G, lo.k_WcT, lo.L * lo.G, 0, l * lo.G);
  }
  add_pack_fwd(pj, lo.split, lo.p_f1_k, lo.S, lo.S, lo.k_Wf1, lo.S, 0, lo.S);
  add_pack_fwd(pj, lo.split, lo.p_f2_k, lo.S, lo.O, lo.k_Wf2, lo.S, 0, lo.S);
  add_pack(pj, lo.p_f1_k, lo.S, lo.S, lo.k_Wf1T, lo.S, 0, 0);
  add_pack(pj, lo.p_f2_k, lo.S, lo.O, lo.k_Wf2T, lo.Op, 0, 0);
  if (!lo.mol) add_pack(pj, lo.p_f2_k, lo.S, lo.O, lo.k_Wf2T, lo.Op, 0, 256);
  lo.n_packjobs = int(lo.packjobs.size());

  // ---- wgrad tiles ----
  // main maps: 0 xd_all, 1 dg_all, 2 c_up, 3 z_all, 4 dxin_all, 5 dskip
  lo.tiles_main.clear();
  auto proto = [](int am, int ash, int al, int bm, int bl, float scale) {
    WgradTile t; memset(&t, 0, sizeof(t));
    t.a_map = am; t.a_shift = ash; t.a_layer = al; t.b_map = bm; t.b_layer = bl; t.scale = scale;
    return t;
  };
  lo.tile_start.assign(lo.L + 1, 0);
  for (int l = 0; l < lo.L; ++l) {
    const int d = lo.dil(l);
    lo.tile_start[l] = int(lo.tiles_main.size());
    for (int j = 0; j < lo.kw; ++j)
      append_wgrad_tiles(lo.tiles_main, proto(0, -(lo.kw - 1 - j) * d, l, 1, l, 1.f), 0, lo.R, 0, lo.G, lo.p_dil_k[l] + (long long)j * lo.R * lo.G, lo.G);
    if (lo.C > 0) append_wgrad_tiles(lo.tiles_main, proto(2, 0, 0, 1, l, 1.f), 0, lo.C, 0, lo.G, lo.p_c_k[l], lo.G);
    for (int m0 = 0; m0 < lo.Gh; m0 += 128) {   // out and skip tiles of one row block side by side
      if (l < lo.L - 1)
        append_wgrad_tiles(lo.tiles_main, proto(3, 0, l, 4, l + 1, lo.res_scale), m0, 128, 0, lo.R, lo.p_o_k[l] + (long long)m0 * lo.R, lo.R);
      append_wgrad_tiles(lo.tiles_main, proto(3, 0, l, 5, 0, lo.skip_scale[l]), m0, 128, 0, lo.S, lo.p_s_k[l] + (long long)m0 * lo.S, lo.S);
    }
  }
  // head maps: 0 h1, 1 dh2, 2 h2, 3 dlog
  lo.tiles_head.clear();
  WgradTile f2 = proto(2, 0, 0, 3, 0, 1.f);
  f2.accumulate = 2;                                   // CE: hi and lo halves of dlog both accumulate (atomics)
  f2.div = reinterpret_cast<const float*>(1);          // patched to scalars[1] at init
  for (int m0 = 0; m0 < lo.S; m0 += 128) {
    append_wgrad_tiles(lo.tiles_head, proto(0, 0, 0, 1, 0, 1.f), m0, 128, 0, lo.S, lo.p_f1_k + (long long)m0 * lo.S, lo.S);
    for (int part = 0; part < (lo.mol ? 1 : 2); ++part)   // O <= 256: one column block per part
      append_wgrad_tiles(lo.tiles_head, f2, m0, 128, part * 256, lo.O, lo.p_f2_k + (long long)m0 * lo.O, lo.O);
  }
  lo.n_tiles_main = int(lo.tiles_main.size());
  lo.tile_start[lo.L] = lo.n_tiles_main;
  lo.n_tiles_head = int(lo.tiles_head.size());

  // ---- column-sum (bias gradient) jobs ----
  lo.colsums.clear();
  auto cs = [&](long long src, long long rows, int C, int ld, long long dst, long long dst2, float scale, int div) {
    ColsumJob j; j.src_off = src; j.rows = rows; j.C = C; j.ld = ld; j.dst_off = dst; j.dst2_off = dst2; j.scale = scale;
    j.div_scalar = div; lo.colsums.push_back(j);
  };
  // (all other bias gradients are column sums fused into the GEMM epilogues that produce dg / dx / dskip / dh2)
  cs(lo.w_dlog, BT, lo.O, lo.ldo, lo.p_f2_b, -1, 1.f, 1);
  if (!lo.mol) cs(lo.w_dlog + 256 * 2, BT, lo.O, lo.ldo, lo.p_f2_b, -1, 1.f, 1);
  lo.n_colsum = int(lo.colsums.size());

  lo.w_tiles_main = ws.take((long long)lo.n_tiles_main * sizeof(WgradTile));
  lo.w_tiles_head = ws.take((long long)lo.n_tiles_head * sizeof(WgradTile));
  lo.w_packjobs = ws.take((long long)lo.n_packjobs * sizeof(PackJob));
  lo.w_colsum = ws.take((long long)lo.n_colsum * sizeof(ColsumJob));
  lo.w_tables = ws.take((long long)lo.L * (3 * sizeof(long long) + sizeof(float)));
  lo.MT = lo.B * ((lo.T + kBM - 1) / kBM);
  lo.n_chain[0] = lo.L * (lo.G / 256) * lo.MT + (lo.L - 1) * lo.MT;
  lo.n_chain[1] = lo.L * (lo.Gh / (lo.Gh >= 256 ? 256 : 128)) * lo.MT + lo.L * lo.MT;
  for (int dir = 0; dir < 2; ++dir) {   // a few MB at most, against the GBs of activations: kept whether the chains run or not
    lo.w_chain_ctr[dir] = ws.take((16 + 2LL * lo.L * lo.MT) * 4);
    lo.w_chain_tix[dir] = ws.take((long long)lo.n_chain[dir] * sizeof(ChainTicket));
    lo.w_chain_args[dir] = ws.take(2LL * lo.L * sizeof(GemmArgs));   // 256-byte aligned: tensor maps in global memory need 64
  }
  lo.w_chain_err = ws.take(4);
  lo.w_spk = lo.w_gbias = lo.w_gsum = -1;
  if (lo.Gi > 0) {
    lo.w_spk = ws.take((1LL + lo.B) * 4);
    lo.w_gbias = ws.take(L * lo.B * lo.G * 4);
    lo.w_gsum = ws.take(L * lo.B * lo.G * 8);
  }
  lo.workspace_bytes = ws.used;
  return T2_OK;
}

// ------------------------------------------------------------------------------------------------------
// small kernels
// ------------------------------------------------------------------------------------------------------
// bias_g[l][g] = b_dil + b_cin ; bias_skip[s] = sum_l scale_l * b_skip_l[s]
struct DerivedArgs {
  const float* params;
  float* bias_g;
  float* bias_skip;
  const long long* offs;  // [3L]: dil_b, c_b (or -1), s_b per layer
  const float* scales;    // [L]
  int L, G, S;
};
__global__ void derived_bias_kernel(DerivedArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < a.L * a.G) {
    const int l = i / a.G, g = i % a.G;
    float v = a.params[a.offs[3 * l] + g];
    if (a.offs[3 * l + 1] >= 0) v += a.params[a.offs[3 * l + 1] + g];
    a.bias_g[i] = v;
  }
  if (i < a.S) {
    float v = 0.f;
    for (int l = 0; l < a.L; ++l) v += a.scales[l] * a.params[a.offs[3 * l + 2] + i];
    a.bias_skip[i] = v;
  }
}

// ---- global (speaker) conditioning (modules.py:10-21,426-433,503-508; wavenet.py:669-678) ----------------------------------
// The speaker term is constant along time, so per layer l and item b it is a gate bias:
//   out[l][b][g] = bias[l][g] + (b_gin[l][g] + sum_k W_gin[l][k][g] * emb[id_b][k])
// kept as its own sum added onto the shared bias, so that zero gin weights give exactly the shared bias. Gate channels are in
// natural order (tanh half, then sigmoid half) like bias_g; the gate epilogue applies the tile permutation.
struct GinArgs {
  const float* params;
  const float* bias;          // shared gate bias of layer l at bias + l * bias_ld
  long long bias_ld;
  const int* on;              // device flag (nullable = on): 0 = no speaker term
  const int* ids;             // [B] (nullable = no speaker term)
  float* out;                 // out + l * out_l + b * out_b + g
  long long out_l, out_b;
  long long p_k, p_b, p_stride, p_emb;   // W_gin / b_gin of layer l at params + p_k / p_b + l * p_stride
  int L, B, G, Gi, NS;
};
__global__ void gin_bias_kernel(GinArgs a) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)a.L * a.B * a.G) return;
  const int g = int(i % a.G), b = int((i / a.G) % a.B), l = int(i / ((long long)a.G * a.B));
  float v = a.bias[l * a.bias_ld + g];
  if (a.ids && (!a.on || *a.on)) {
    const int id = a.ids[b];
    float s = __int_as_float(0x7fffffff);   // an id outside [0, NS) reads nothing and makes the item's gate activations NaN
    if (id >= 0 && id < a.NS) {
      const float* W = a.params + a.p_k + l * a.p_stride + g;
      const float* e = a.params + a.p_emb + (long long)id * a.Gi;
      s = a.params[a.p_b + l * a.p_stride + g];
      for (int k = 0; k < a.Gi; ++k) s += W[(long long)k * a.G] * e[k];
    }
    v += s;
  }
  a.out[l * a.out_l + b * a.out_b + g] = v;
}
// workspace speaker state: spk[0] = 1 if ids are given, spk[1 + b] = id of item b
__global__ void set_speakers_kernel(int* __restrict__ spk, const int* __restrict__ ids, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) spk[0] = ids != nullptr;
  if (ids && i < B) spk[1 + i] = ids[i];
}
// Gradients of the speaker term from the per-item fixed-point column sums S[l][b][g] of d gate pre-activation, one thread per
// (l, g): the gate biases get sum_b S (an integer sum, exact: the same total the shared accumulator would hold), and
// dW_gin[l][k][g] = sum_b emb[id_b][k] * S[l][b][g] in the order of b.
struct GinGradArgs {
  const float* params;
  const int* spk;             // workspace speaker state (see set_speakers_kernel)
  const long long* S;         // [L][B][G]
  long long* gfx;             // fixed-point gradient accumulators (bias gradients)
  float* grads;
  const long long* offs;      // [3L]: dil_b, c_b (or -1), ... (w_tables)
  long long p_k, p_b, p_stride, p_emb;
  int L, B, G, Gi, NS;
};
__global__ void gin_wgrad_kernel(GinGradArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.L * a.G) return;
  const int l = i / a.G, g = i % a.G;
  const long long* S = a.S + (long long)l * a.B * a.G + g;
  long long tot = 0;
  bool poison = false;
  for (int b = 0; b < a.B; ++b) {
    const long long s = S[(long long)b * a.G];
    if (!fx_in_range(s)) poison = true;
    else if (!fx_in_range(tot += s)) poison = true;
  }
  if (poison) tot = kFxPoison;
  a.gfx[a.offs[3 * l] + g] = tot;
  if (a.offs[3 * l + 1] >= 0) a.gfx[a.offs[3 * l + 1] + g] = tot;
  if (!a.spk[0]) return;      // no speaker term: its parameters get no gradient
  a.gfx[a.p_b + l * a.p_stride + g] = tot;
  float* dW = a.grads + a.p_k + l * a.p_stride + g;
  for (int k = 0; k < a.Gi; ++k) {
    float acc = 0.f;
    for (int b = 0; b < a.B; ++b) {
      const int id = a.spk[1 + b];
      const float e = (id >= 0 && id < a.NS) ? a.params[a.p_emb + (long long)id * a.Gi + k] : __int_as_float(0x7fffffff);
      acc += e * fx_value(S[(long long)b * a.G]);
    }
    dW[(long long)k * a.G] = acc;
  }
}
// d gc_embedding[s][k] = sum over items b with id_b == s (in the order of b) of sum_{l,g} W_gin[l][k][g] * S[l][b][g]; one block
// per (speaker, k), a fixed-shape tree per item: no float atomics. Rows no item uses get exactly 0.
constexpr int kGinThreads = 256;
__global__ void __launch_bounds__(kGinThreads) gin_demb_kernel(GinGradArgs a) {
  __shared__ float red[kGinThreads];
  if (!a.spk[0]) return;
  const int s = blockIdx.x, k = blockIdx.y, tid = threadIdx.x;
  {
    float acc = 0.f;
    for (int b = 0; b < a.B; ++b) {
      if (a.spk[1 + b] != s) continue;
      float part = 0.f;
      for (int l = 0; l < a.L; ++l) {
        const float* W = a.params + a.p_k + l * a.p_stride + (long long)k * a.G;
        const long long* S = a.S + ((long long)l * a.B + b) * a.G;
        for (int g = tid; g < a.G; g += kGinThreads) part += W[g] * fx_value(S[g]);
      }
      red[tid] = part;
      __syncthreads();
      for (int h = kGinThreads / 2; h > 0; h >>= 1) {
        if (tid < h) red[tid] += red[tid + h];
        __syncthreads();
      }
      if (tid == 0) acc += red[0];
      __syncthreads();
    }
    if (tid == 0) a.grads[a.p_emb + (long long)s * a.Gi + k] = acc;
  }
}

// first (embedding) 1x1 conv: one-hot input == row gather (wavenet.py:705; SURVEY §8a "embedding in disguise")
__global__ void first_conv_kernel(const void* __restrict__ xin, int scalar_in, const float* __restrict__ W,
                                  const float* __restrict__ bias, bf16* __restrict__ x, bf16* __restrict__ xd,
                                  long long npos, int R, float p, unsigned long long seed,
                                  const unsigned long long* __restrict__ step, int split) {
  // 8 channels per thread (R % 8 == 0): two float4 loads of the embedding row, one 16-byte store per output
  if (step) seed += *step;
  const long long e8 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int R8 = R >> 3;
  if (e8 >= npos * R8) return;
  const long long pos = e8 / R8;
  const int r = int(e8 % R8) * 8;
  float v[8];
  const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + r)), b1 = __ldg(reinterpret_cast<const float4*>(bias + r + 4));
  if (scalar_in) {
    const float xv = static_cast<const float*>(xin)[pos];
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(W + r)), w1 = __ldg(reinterpret_cast<const float4*>(W + r + 4));
    v[0] = xv * w0.x + b0.x; v[1] = xv * w0.y + b0.y; v[2] = xv * w0.z + b0.z; v[3] = xv * w0.w + b0.w;
    v[4] = xv * w1.x + b1.x; v[5] = xv * w1.y + b1.y; v[6] = xv * w1.z + b1.z; v[7] = xv * w1.w + b1.w;
  } else {
    const float* row = W + (long long)static_cast<const int*>(xin)[pos] * R + r;
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(row)), w1 = __ldg(reinterpret_cast<const float4*>(row + 4));
    v[0] = w0.x + b0.x; v[1] = w0.y + b0.y; v[2] = w0.z + b0.z; v[3] = w0.w + b0.w;
    v[4] = w1.x + b1.x; v[5] = w1.y + b1.y; v[6] = w1.z + b1.z; v[7] = w1.w + b1.w;
  }
  const long long e = pos * R + r;
  uint4 o;
  if (split) {   // rows are [hi(R) | lo(R)]
    float hi[8], lo8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { hi[j] = __bfloat162float(__float2bfloat16(v[j])); lo8[j] = v[j] - hi[j]; }
    o.x = pack_bf16x2(hi[0], hi[1]); o.y = pack_bf16x2(hi[2], hi[3]); o.z = pack_bf16x2(hi[4], hi[5]); o.w = pack_bf16x2(hi[6], hi[7]);
    *reinterpret_cast<uint4*>(x + pos * 2 * R + r) = o;
    o.x = pack_bf16x2(lo8[0], lo8[1]); o.y = pack_bf16x2(lo8[2], lo8[3]); o.z = pack_bf16x2(lo8[4], lo8[5]); o.w = pack_bf16x2(lo8[6], lo8[7]);
    *reinterpret_cast<uint4*>(x + pos * 2 * R + R + r) = o;
    return;
  }
  o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]); o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(x + e) = o;
  if (xd != x && xd != nullptr) {
    const float keep_inv = 1.f / (1.f - p);
    const uint32_t hs = hash_seed(seed, 0u), thr = uint32_t(p * 65536.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = hash_keep16(hs, (unsigned long long)(e + j), thr) ? v[j] * keep_inv : 0.f;
    o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]); o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(xd + e) = o;
  }
}
__global__ void first_conv_bwd_kernel(const void* __restrict__ xin, int scalar_in, const bf16* __restrict__ dx0,
                                      long long* __restrict__ dW, long long npos, int R) {
  // one block = 64 positions x R channels; scalar input reduces in registers first
  const int r = threadIdx.x;
  const long long p0 = (long long)blockIdx.x * 64;
  if (scalar_in) {
    float acc = 0.f;
    for (int i = 0; i < 64 && p0 + i < npos; ++i)
      acc += static_cast<const float*>(xin)[p0 + i] * __bfloat162float(dx0[(p0 + i) * R + r]);
    fx_add(dW + r, acc);
  } else {
    const int n = npos - p0 < 64 ? int(npos - p0) : 64;
    for (int i0 = 0; i0 < n; i0 += 8) {
      FxAdd x[8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (i0 + i < n)
          x[i] = fx_issue(dW + (long long)static_cast<const int*>(xin)[p0 + i0 + i] * R + r, __bfloat162float(dx0[(p0 + i0 + i) * R + r]));
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (i0 + i < n) fx_check(x[i]);
    }
  }
}

__global__ void colsum_kernel(const uint8_t* __restrict__ ws, long long* __restrict__ grads, const ColsumJob* __restrict__ jobs,
                              const float* __restrict__ scalars) {
  const ColsumJob j = jobs[blockIdx.y];
  const bf16* src = reinterpret_cast<const bf16*>(ws + j.src_off);
  const long long rows_per = (j.rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = blockIdx.x * rows_per;
  const long long r1 = r0 + rows_per < j.rows ? r0 + rows_per : j.rows;
  float sc = j.scale;
  if (j.div_scalar >= 0) sc /= fmaxf(scalars[j.div_scalar], 1e-20f);
  // one thread = one pair of adjacent columns (C and ld are even); 4 rows in flight per iteration
  for (int c = 2 * threadIdx.x; c < j.C; c += 2 * blockDim.x) {
    float a0 = 0.f, a1 = 0.f;
    long long r = r0;
    for (; r + 4 <= r1; r += 4) {
      uint32_t u[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) u[i] = __ldg(reinterpret_cast<const uint32_t*>(src + (r + i) * j.ld + c));
#pragma unroll
      for (int i = 0; i < 4; ++i) { a0 += bf16lo(u[i]); a1 += bf16hi(u[i]); }
    }
    for (; r < r1; ++r) {
      const uint32_t u = __ldg(reinterpret_cast<const uint32_t*>(src + r * j.ld + c));
      a0 += bf16lo(u); a1 += bf16hi(u);
    }
    a0 *= sc; a1 *= sc;
    const bool two = c + 1 < j.C, dup = j.dst2_off >= 0;
    FxAdd x[4];
    x[0] = fx_issue(grads + j.dst_off + c, a0);
    if (two) x[1] = fx_issue(grads + j.dst_off + c + 1, a1);
    if (dup) {
      x[2] = fx_issue(grads + j.dst2_off + c, a0);
      if (two) x[3] = fx_issue(grads + j.dst2_off + c + 1, a1);
    }
    fx_check(x[0]);
    if (two) fx_check(x[1]);
    if (dup) {
      fx_check(x[2]);
      if (two) fx_check(x[3]);
    }
  }
}

// ---- conditioning upsampling net (modules.py:539-654 SubPixel, :697-733 ConvTranspose1D, :736-770 ConvTranspose2D) + activation ----
// activation after each layer (wavenet.py:197-203): 0 ReLU, 1 LeakyReLU max(alpha x, x) (tf.nn.leaky_relu), 2 none
__device__ __forceinline__ float up_act(float x, int act, float alpha) {
  return act == 0 ? fmaxf(x, 0.f) : act == 1 ? fmaxf(alpha * x, x) : x;
}
// d pre-activation from the stored post-activation output o and d out: ReLU 0 where o <= 0; LeakyReLU alpha there (the gradient of
// tf.nn.leaky_relu for 0 <= alpha <= 1: o <= 0 exactly where x <= 0, up to alpha = 0 where both are 0); none: unchanged
__device__ __forceinline__ float up_dact(float o, float g, int act, float alpha) {
  return act == 2 || o > 0.f ? g : act == 1 ? alpha * g : 0.f;
}
// in [B][H][W] fp32 -> out [B][H][W*s] fp32 (post-activation); optional bf16 channels-last copy [B][W*s][H]
__global__ void upsample_fwd_kernel(const float* __restrict__ in, const float* __restrict__ K, const float* __restrict__ bias,
                                    float* __restrict__ out, bf16* __restrict__ out_cl, int B, int H, int W, int s, int type, int act,
                                    float alpha, int split) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long n = (long long)B * H * W * s;
  if (e >= n) return;
  const int Wo = W * s;
  const int xo = int(e % Wo);
  const int h = int((e / Wo) % H);
  const int b = int(e / ((long long)Wo * H));
  const int w = xo / s, k = xo % s;
  const float* ib = in + (long long)b * H * W;
  float acc;
  if (type == 0) {  // SubPixel: 3x3 'same' conv, 1 -> s channels, then periodic shuffle. K [3][3][1][s]
    acc = bias[k];
#pragma unroll
    for (int dh = 0; dh < 3; ++dh) {
      const int hh = h + dh - 1;
      if (hh < 0 || hh >= H) continue;
#pragma unroll
      for (int dw = 0; dw < 3; ++dw) {
        const int ww = w + dw - 1;
        if (ww < 0 || ww >= W) continue;
        acc += K[(dh * 3 + dw) * s + k] * ib[hh * W + ww];
      }
    }
  } else {  // Conv2DTranspose kernel (3, s), strides (1, s), 'same': out[h, w*s+k] = sum_q in[h+1-q, w] K[q][k]
    acc = bias[0];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const int hh = h + 1 - q;
      if (hh < 0 || hh >= H) continue;
      acc += K[q * s + k] * ib[hh * W + w];
    }
  }
  acc = up_act(acc, act, alpha);
  out[e] = acc;
  if (out_cl && split) {   // rows are [hi(H) zero-padded to 128 | lo(H) zero-padded to 128]
    const bf16 hi = __float2bfloat16(acc);
    bf16* row = out_cl + ((long long)b * Wo + xo) * 256;
    row[h] = hi;
    row[128 + h] = __float2bfloat16(acc - __bfloat162float(hi));
  } else if (out_cl) out_cl[((long long)b * Wo + xo) * H + h] = __float2bfloat16(acc);
}
// channels-last fp32 [B][T][C] -> [B][C][T] (tiled transpose) so the upsampling backward reads contiguously
__global__ void cl_to_chw_kernel(const float* __restrict__ in, float* __restrict__ out, int T, int C) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int t = t0 + r, c = c0 + threadIdx.x;
    tile[r][threadIdx.x] = (t < T && c < C) ? in[((long long)b * T + t) * C + c] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int c = c0 + r, t = t0 + threadIdx.x;
    if (t < T && c < C) out[((long long)b * C + c) * T + t] = tile[threadIdx.x][r];
  }
}
// d_pre = d_out * act'(out); accumulates dK [ntap][s] and dbias. The launch uses gridDim.x * blockDim.x % s == 0, so a
// thread always meets the same sub-pixel phase k = e % s: it sums its taps in registers, the block merges through a
// small shared-memory table (10 atomics per thread, once) and issues one global atomic per table entry.
__global__ void upsample_bwd_param_kernel(const float* __restrict__ in, const float* __restrict__ out, const float* __restrict__ dout,
                                          long long* __restrict__ dK, long long* __restrict__ dbias, int B, int H, int W, int s, int type,
                                          int act, float alpha) {
  __shared__ long long acc[10 * 32];
  const int ntap = type == 0 ? 9 : 3;
  for (int i = threadIdx.x; i < (ntap + 1) * s; i += blockDim.x) acc[i] = 0;
  __syncthreads();
  const int Wo = W * s;
  const long long n = (long long)B * H * Wo;
  const long long e0 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int k = int(e0 % s);
  float r[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) r[i] = 0.f;
  for (long long e = e0; e < n; e += (long long)gridDim.x * blockDim.x) {
    const float o = out[e];
    if (act == 0 && o <= 0.f) continue;   // ReLU: nothing to add (only here may elements be skipped)
    const float g = up_dact(o, dout[e], act, alpha);
    const int xo = int(e % Wo), h = int((e / Wo) % H), b = int(e / ((long long)Wo * H));
    const int w = xo / s;
    r[9] += g;
    const float* ib = in + (long long)b * H * W;
    if (type == 0) {
#pragma unroll
      for (int dh = 0; dh < 3; ++dh) {
        const int hh = h + dh - 1;
        if (hh < 0 || hh >= H) continue;
#pragma unroll
        for (int dw = 0; dw < 3; ++dw) {
          const int ww = w + dw - 1;
          if (ww >= 0 && ww < W) r[dh * 3 + dw] += g * ib[hh * W + ww];
        }
      }
    } else {
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int hh = h + 1 - q;
        if (hh >= 0 && hh < H) r[q] += g * ib[hh * W + w];
      }
    }
  }
  FxAdd x[10];
#pragma unroll
  for (int i = 0; i < 9; ++i)
    if (i < ntap && r[i] != 0.f) x[i] = fx_issue(&acc[i * s + k], r[i]);
  if (r[9] != 0.f) x[9] = fx_issue(&acc[ntap * s + k], r[9]);
#pragma unroll
  for (int i = 0; i < 9; ++i)
    if (i < ntap && r[i] != 0.f) fx_check(x[i]);
  if (r[9] != 0.f) fx_check(x[9]);
  __syncthreads();
  for (int i = threadIdx.x; i < (ntap + 1) * s; i += blockDim.x) {
    const long long v = acc[i];
    if (v == 0) continue;
    // checked merge: two poisoned block totals must not cancel, in-range totals must not wrap
    fx_check(fx_issue_total(i < ntap * s ? dK + i : type == 0 ? dbias + (i - ntap * s) : dbias, v));
  }
}
__global__ void upsample_bwd_input_kernel(const float* __restrict__ out, const float* __restrict__ dout, int cl,
                                          const float* __restrict__ K, float* __restrict__ din, int B, int H, int W, int s, int type,
                                          int act, float alpha) {
  // 4 lanes per input pixel, each walking every 4th sub-pixel phase k; partial sums meet through two shuffles
  const long long e4 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long n = (long long)B * H * W;
  const long long e = e4 >> 2;
  const int part = int(e4 & 3);
  const bool live = e < n;
  const long long ec = live ? e : n - 1;
  const int w = int(ec % W), h = int((ec / W) % H), b = int(ec / ((long long)W * H));
  const int Wo = W * s;
  float acc = 0.f;
  auto dpre = [&](int hh, int xo) -> float {
    const float o = out[((long long)b * H + hh) * Wo + xo];
    if (act == 0 && o <= 0.f) return 0.f;
    return up_dact(o, cl ? dout[((long long)b * Wo + xo) * H + hh] : dout[((long long)b * H + hh) * Wo + xo], act, alpha);
  };
  if (type == 0) {
    for (int dh = 0; dh < 3; ++dh) {
      const int ho = h - dh + 1;
      if (ho < 0 || ho >= H) continue;
      for (int dw = 0; dw < 3; ++dw) {
        const int wo = w - dw + 1;
        if (wo < 0 || wo >= W) continue;
        for (int k = part; k < s; k += 4) acc += dpre(ho, wo * s + k) * K[(dh * 3 + dw) * s + k];
      }
    }
  } else {
    for (int q = 0; q < 3; ++q) {
      const int ho = h - 1 + q;
      if (ho < 0 || ho >= H) continue;
      for (int k = part; k < s; k += 4) acc += dpre(ho, w * s + k) * K[q * s + k];
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  if (live && part == 0) din[e] = acc;
}

// ---- ConvTranspose1D (modules.py:697-733): kernel = stride = s along time, 'same' padding, so the windows never overlap:
//   out[b][co][w*s + j] = act(bias[co] + sum_ci K[j][co][ci] in[b][ci][w])      K = TF [1][s][C(out)][C(in)]
// Per tap j a [B*W, C] x [C, C] product in fp32 (C = 80 does not fill the 64-wide K blocks of the bf16 tensor-core engine, and the
// upsampler is fp32 throughout). Blocks of 32 time positions x 8 rows of threads; a thread owns the channels ty + 8k (k < 16, C <= 128).
// Every output is one thread's sum in a fixed order: no atomics, the same bits on every run.
constexpr int kUp1Tw = 32, kUp1Rows = 8, kUp1MaxK = 16;
inline size_t up1d_smem(int C) { return sizeof(float) * (size_t(C) * C + size_t(C) * kUp1Tw); }
// grid (ceil(W / 32), B, taps per block group): the block stages its 32 input frames once and loops over taps j = z, z + gridDim.z, ...
__global__ void __launch_bounds__(kUp1Tw * kUp1Rows) up1d_fwd_kernel(const float* __restrict__ in, const float* __restrict__ K,
                                                                    const float* __restrict__ bias, float* __restrict__ out,
                                                                    bf16* __restrict__ out_cl, int C, int W, int s, int act, float alpha,
                                                                    int split) {
  extern __shared__ float sm[];
  float* ks = sm;                              // [C][C]: K[j][co][ci]
  float* xs = sm + C * C;                      // [C][32]: in[b][ci][w0 + t]
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kUp1Tw + tx;
  const int w0 = blockIdx.x * kUp1Tw, b = blockIdx.y;
  const int nw = min(kUp1Tw, W - w0);
  const long long Wo = (long long)W * s;
  for (int e = tid; e < C * kUp1Tw; e += kUp1Tw * kUp1Rows) {
    const int ci = e / kUp1Tw, t = e % kUp1Tw;
    xs[e] = t < nw ? in[((long long)b * C + ci) * W + w0 + t] : 0.f;
  }
  for (int j = blockIdx.z; j < s; j += gridDim.z) {
    __syncthreads();                           // xs staged / the previous tap's ks reads are done
    const float* Kj = K + (long long)j * C * C;
    for (int e = tid; e < C * C; e += kUp1Tw * kUp1Rows) ks[e] = Kj[e];
    __syncthreads();
    float acc[kUp1MaxK];
#pragma unroll
    for (int k = 0; k < kUp1MaxK; ++k) acc[k] = 0.f;
    if ((C & 3) == 0) {                        // float4 rows of K; the same sequential order over ci as the scalar loop
      for (int ci = 0; ci < C; ci += 4) {
        const float x0 = xs[ci * kUp1Tw + tx], x1 = xs[(ci + 1) * kUp1Tw + tx], x2 = xs[(ci + 2) * kUp1Tw + tx], x3 = xs[(ci + 3) * kUp1Tw + tx];
#pragma unroll
        for (int k = 0; k < kUp1MaxK; ++k) {
          const int co = ty + kUp1Rows * k;
          if (co < C) {
            const float4 kv = *reinterpret_cast<const float4*>(ks + co * C + ci);
            acc[k] = fmaf(kv.x, x0, acc[k]); acc[k] = fmaf(kv.y, x1, acc[k]); acc[k] = fmaf(kv.z, x2, acc[k]); acc[k] = fmaf(kv.w, x3, acc[k]);
          }
        }
      }
    } else {
      for (int ci = 0; ci < C; ++ci) {
        const float x = xs[ci * kUp1Tw + tx];
#pragma unroll
        for (int k = 0; k < kUp1MaxK; ++k) {
          const int co = ty + kUp1Rows * k;
          if (co < C) acc[k] = fmaf(ks[co * C + ci], x, acc[k]);
        }
      }
    }
    if (tx < nw) {
      const long long xo = (long long)(w0 + tx) * s + j;
#pragma unroll
      for (int k = 0; k < kUp1MaxK; ++k) {
        const int co = ty + kUp1Rows * k;
        if (co >= C) continue;
        const float v = up_act(bias[co] + acc[k], act, alpha);
        out[((long long)b * C + co) * Wo + xo] = v;
        if (out_cl && split) {   // rows are [hi(C) zero-padded to 128 | lo(C) zero-padded to 128]
          const bf16 hi = __float2bfloat16(v);
          bf16* row = out_cl + ((long long)b * Wo + xo) * 256;
          row[co] = hi;
          row[128 + co] = __float2bfloat16(v - __bfloat162float(hi));
        } else if (out_cl) out_cl[((long long)b * Wo + xo) * C + co] = __float2bfloat16(v);
      }
    }
  }
}
// din[b][ci][w] = sum_j sum_co K[j][co][ci] dpre[b][co][w*s + j]; grid (ceil(W / 32), B). Per tap the block stages K[j] transposed
// ([ci][co]) and the 32 positions' dpre; a thread sums its channels ci = ty + 8k over j, then co, in order.
__global__ void __launch_bounds__(kUp1Tw * kUp1Rows) up1d_bwd_input_kernel(const float* __restrict__ out, const float* __restrict__ dout,
                                                                          const float* __restrict__ K, float* __restrict__ din, int C, int W,
                                                                          int s, int act, float alpha) {
  extern __shared__ float sm[];
  float* kt = sm;                              // [C][C]: K[j][co][ci] at kt[ci * C + co]
  float* gs = sm + C * C;                      // [C][32]: dpre[b][co][(w0 + t) * s + j]
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kUp1Tw + tx;
  const int w0 = blockIdx.x * kUp1Tw, b = blockIdx.y;
  const int nw = min(kUp1Tw, W - w0);
  const long long Wo = (long long)W * s;
  float acc[kUp1MaxK];
#pragma unroll
  for (int k = 0; k < kUp1MaxK; ++k) acc[k] = 0.f;
  for (int j = 0; j < s; ++j) {
    __syncthreads();
    const float* Kj = K + (long long)j * C * C;
    for (int e = tid; e < C * C; e += kUp1Tw * kUp1Rows) kt[e] = Kj[(e % C) * C + e / C];   // conflict-free stores; K[j] sits in L1
    for (int e = tid; e < C * kUp1Tw; e += kUp1Tw * kUp1Rows) {
      const int co = e / kUp1Tw, t = e % kUp1Tw;
      float g = 0.f;
      if (t < nw) {
        const long long i = ((long long)b * C + co) * Wo + (long long)(w0 + t) * s + j;
        g = up_dact(out[i], dout[i], act, alpha);
      }
      gs[e] = g;
    }
    __syncthreads();
    if ((C & 3) == 0) {
      for (int co = 0; co < C; co += 4) {
        const float g0 = gs[co * kUp1Tw + tx], g1 = gs[(co + 1) * kUp1Tw + tx], g2 = gs[(co + 2) * kUp1Tw + tx], g3 = gs[(co + 3) * kUp1Tw + tx];
#pragma unroll
        for (int k = 0; k < kUp1MaxK; ++k) {
          const int ci = ty + kUp1Rows * k;
          if (ci < C) {
            const float4 kv = *reinterpret_cast<const float4*>(kt + ci * C + co);
            acc[k] = fmaf(kv.x, g0, acc[k]); acc[k] = fmaf(kv.y, g1, acc[k]); acc[k] = fmaf(kv.z, g2, acc[k]); acc[k] = fmaf(kv.w, g3, acc[k]);
          }
        }
      }
    } else {
      for (int co = 0; co < C; ++co) {
        const float g = gs[co * kUp1Tw + tx];
#pragma unroll
        for (int k = 0; k < kUp1MaxK; ++k) {
          const int ci = ty + kUp1Rows * k;
          if (ci < C) acc[k] = fmaf(kt[ci * C + co], g, acc[k]);
        }
      }
    }
  }
  if (tx < nw) {
#pragma unroll
    for (int k = 0; k < kUp1MaxK; ++k) {
      const int ci = ty + kUp1Rows * k;
      if (ci < C) din[((long long)b * C + ci) * W + w0 + tx] = acc[k];
    }
  }
}
// dK[j][co][ci] = sum_{b,w} dpre[b][co][w*s + j] in[b][ci][w], dbias[co] = sum dpre[b][co][:]. grid (s, G): block (j, y) sums the
// 32-position chunks y, y + G, ... of the flattened (b, w) range in registers (a thread owns ci = tx + 32m, co = ty + 8k) and adds
// its partial tile to the fixed-point accumulators; G depends on the shape only, so every run rounds the same partial sums.
constexpr int kUp1MaxM = 4;
inline size_t up1d_param_smem(int C) { return sizeof(float) * 2 * kUp1Tw * size_t(C + 1); }
__global__ void __launch_bounds__(kUp1Tw * kUp1Rows) up1d_bwd_param_kernel(const float* __restrict__ in, const float* __restrict__ out,
                                                                          const float* __restrict__ dout, long long* __restrict__ dK,
                                                                          long long* __restrict__ dbias, int B, int C, int W, int s, int act,
                                                                          float alpha) {
  extern __shared__ float sm[];
  const int ld = C + 1;
  float* xs = sm;                              // [32][C + 1]: in[b][ci][w] of position t of the chunk
  float* gs = sm + kUp1Tw * ld;                // [32][C + 1]: dpre[b][co][w*s + j]
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kUp1Tw + tx;
  const int j = blockIdx.x;
  const long long npos = (long long)B * W, Wo = (long long)W * s;
  const long long nchunk = (npos + kUp1Tw - 1) / kUp1Tw;
  float acc[kUp1MaxM][kUp1MaxK];
#pragma unroll
  for (int m = 0; m < kUp1MaxM; ++m)
#pragma unroll
    for (int k = 0; k < kUp1MaxK; ++k) acc[m][k] = 0.f;
  float bsum = 0.f;                            // thread tid < C: column tid of gs
  for (long long ch = blockIdx.y; ch < nchunk; ch += gridDim.y) {
    __syncthreads();
    for (int e = tid; e < C * kUp1Tw; e += kUp1Tw * kUp1Rows) {
      const int c = e / kUp1Tw, t = e % kUp1Tw;
      const long long p = ch * kUp1Tw + t;
      float x = 0.f, g = 0.f;
      if (p < npos) {
        const long long b = p / W, w = p % W;
        x = in[(b * C + c) * W + w];
        const long long i = (b * C + c) * Wo + w * s + j;
        g = up_dact(out[i], dout[i], act, alpha);
      }
      xs[t * ld + c] = x;
      gs[t * ld + c] = g;
    }
    __syncthreads();
    if (tid < C)
      for (int t = 0; t < kUp1Tw; ++t) bsum += gs[t * ld + tid];
    for (int t = 0; t < kUp1Tw; ++t) {
      float x[kUp1MaxM];
#pragma unroll
      for (int m = 0; m < kUp1MaxM; ++m) x[m] = tx + kUp1Tw * m < C ? xs[t * ld + tx + kUp1Tw * m] : 0.f;
#pragma unroll
      for (int k = 0; k < kUp1MaxK; ++k) {
        const int co = ty + kUp1Rows * k;
        if (co < C) {
          const float g = gs[t * ld + co];
#pragma unroll
          for (int m = 0; m < kUp1MaxM; ++m) acc[m][k] = fmaf(g, x[m], acc[m][k]);
        }
      }
    }
  }
  long long* dKj = dK + (long long)j * C * C;
#pragma unroll
  for (int k = 0; k < kUp1MaxK; ++k) {
    const int co = ty + kUp1Rows * k;
    if (co >= C) continue;
    FxAdd xa[kUp1MaxM];
#pragma unroll
    for (int m = 0; m < kUp1MaxM; ++m) {
      const int ci = tx + kUp1Tw * m;
      if (ci < C && acc[m][k] != 0.f) xa[m] = fx_issue(dKj + (long long)co * C + ci, acc[m][k]);
    }
#pragma unroll
    for (int m = 0; m < kUp1MaxM; ++m) {
      const int ci = tx + kUp1Tw * m;
      if (ci < C && acc[m][k] != 0.f) fx_check(xa[m]);
    }
  }
  if (tid < C && bsum != 0.f) fx_add(dbias + tid, bsum);
}
// skip-conv bias gradients: db_s[l] = skip_scale[l] * column sums of dskip (table layout: offs[3l+2] = skip bias offset)
__global__ void skip_bias_kernel(const long long* __restrict__ skipsum, float* __restrict__ grads, const long long* __restrict__ offs,
                                 const float* __restrict__ scales, int L, int S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L * S) return;
  const int l = i / S, s = i % S;
  grads[offs[3 * l + 2] + s] = scales[l] * fx_value(skipsum[s]);
}
// grads += the fixed-point totals of the block-summed gradients (first conv, biases, upsampling net)
__global__ void fx_finalize_kernel(const long long* __restrict__ acc, float* __restrict__ grads, long long n) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e < n && acc[e] != 0) grads[e] += fx_value(acc[e]);
}

// the per-layer gate GEMM: [x(t-(kw-1)d) | ... | x(t-d) | x(t) | c(t)] x Wg with the tanh*sigmoid epilogue
ActGemmCall make_gate_call(const Layout& lo, uint8_t* ws, const uint8_t* pk, int l, bool save) {
  const long long BT = (long long)lo.B * lo.T;
  const int d = lo.dil(l);
  ActGemmCall g;
  memset(&g, 0, sizeof(g));
  g.a[0] = make_act(ws + lo.w_xd, lo.R, lo.T, lo.B, lo.L);
  g.a[1] = make_act(ws + lo.w_cup, lo.C > 0 ? lo.C : 8, lo.T, lo.B, 1);
  g.na = lo.C > 0 ? 2 : 1;
  for (int j = 0; j < lo.kw; ++j) g.seg[j] = Seg{0, -(lo.kw - 1 - j) * d, 0, lo.R / kBK, l, 1};
  g.nseg = lo.kw;
  if (lo.C > 0) g.seg[g.nseg++] = Seg{1, 0, 0, 2, 0, 1};
  g.w = pk + lo.k_Wg; g.wN = lo.G; g.wK = lo.Kg; g.wL = lo.L; g.w_layer = l; g.w_k0 = 0;
  g.split = lo.split;
  g.T = lo.T; g.B = lo.B; g.n_tiles = lo.G / 256;
  const long long lofs = (long long)l * BT * lo.Gh;
  g.epi.ptr[0] = save ? reinterpret_cast<bf16*>(ws + lo.w_ta) + lofs : nullptr;
  g.epi.ptr[1] = save ? reinterpret_cast<bf16*>(ws + lo.w_sb) + lofs : nullptr;
  g.epi.ptr[2] = reinterpret_cast<bf16*>(ws + lo.w_z) + lofs * lo.xm;
  g.epi.ptr[3] = const_cast<float*>(reinterpret_cast<const float*>(pk + lo.k_bias_g) + (long long)l * lo.G);
  if (lo.Gi > 0) {   // per-item gate biases (gin_bias_kernel): item b's row at + b * G
    g.epi.ptr[3] = reinterpret_cast<float*>(ws + lo.w_gbias) + (long long)l * lo.B * lo.G;
    g.epi.i[2] = lo.G;
  }
  g.epi.i[0] = lo.Gh;
  return g;
}

ActGemmCall make_out_call(const Layout& lo, uint8_t* ws, const uint8_t* pk, const float* params, int l, float p,
                          unsigned long long seed, const unsigned long long* d_step) {
  const long long BT = (long long)lo.B * lo.T;
  bf16* x_all = reinterpret_cast<bf16*>(ws + lo.w_x);
  bf16* xd_all = reinterpret_cast<bf16*>(ws + lo.w_xd);
  ActGemmCall o;
  memset(&o, 0, sizeof(o));
  o.a[0] = make_act(ws + lo.w_z, lo.Gh, lo.T, lo.B, lo.L); o.na = 1;
  o.seg[0] = Seg{0, 0, 0, lo.Gh / kBK, l, 1}; o.nseg = 1;
  o.w = pk + lo.k_Wo; o.wN = lo.R; o.wK = lo.Gh; o.wL = lo.L; o.w_layer = l;
  o.split = lo.split;
  o.T = lo.T; o.B = lo.B; o.n_tiles = 1;
  o.epi.ptr[0] = x_all + (long long)l * BT * lo.R * lo.xm;
  o.epi.ptr[1] = x_all + (long long)(l + 1) * BT * lo.R * lo.xm;
  o.epi.ptr[2] = p > 0.f ? xd_all + (long long)(l + 1) * BT * lo.R : nullptr;
  o.epi.ptr[3] = const_cast<float*>(params + lo.p_o_b[l]);
  o.epi.f[0] = lo.res_scale; o.epi.f[1] = p; o.epi.i[1] = l + 1; o.epi.seed = seed;
  o.epi.ptr[7] = const_cast<unsigned long long*>(d_step);
  return o;
}

// grads: the int64 fixed-point gradient accumulators (w_gfx), or nullptr for no bias gradients
ActGemmCall make_dz_call(const Layout& lo, uint8_t* ws, const uint8_t* pk, int l, long long* grads) {
  const long long BT = (long long)lo.B * lo.T;
  const bool top = l == lo.L - 1;
  ActGemmCall g;
  memset(&g, 0, sizeof(g));
  g.a[0] = make_act(ws + lo.w_dxin, lo.R, lo.T, lo.B, lo.L);
  g.a[1] = make_act(ws + lo.w_dskip, lo.S, lo.T, lo.B, 1);
  g.na = 2;
  if (top) {
    g.seg[0] = Seg{1, 0, 0, lo.S / kBK, 0, 1}; g.nseg = 1; g.w_k0 = lo.R;
  } else {
    g.seg[0] = Seg{0, 0, 0, lo.R / kBK, l + 1, 1};
    g.seg[1] = Seg{1, 0, 0, lo.S / kBK, 0, 1};
    g.nseg = 2; g.w_k0 = 0;
  }
  const int bn_z = lo.Gh >= 256 ? 256 : 128;
  g.w = pk + lo.k_WozT; g.wN = lo.Gh; g.wK = lo.R + lo.S; g.wL = lo.L; g.w_layer = l;
  g.T = lo.T; g.B = lo.B; g.n_tiles = lo.Gh / bn_z;
  const long long lofs = (long long)l * BT * lo.Gh;
  g.epi.ptr[0] = reinterpret_cast<bf16*>(ws + lo.w_ta) + lofs;
  g.epi.ptr[1] = reinterpret_cast<bf16*>(ws + lo.w_sb) + lofs;
  g.epi.ptr[2] = reinterpret_cast<bf16*>(ws + lo.w_dg) + (long long)l * BT * lo.G;
  g.epi.ptr[3] = grads ? grads + lo.p_dil_b[l] : nullptr;
  g.epi.ptr[4] = (grads && lo.C > 0) ? grads + lo.p_c_b[l] : nullptr;
  if (grads && lo.Gi > 0) {   // per-item sums S[l][b][:], turned into the bias and speaker gradients by gin_wgrad_kernel
    g.epi.ptr[3] = reinterpret_cast<long long*>(ws + lo.w_gsum) + (long long)l * lo.B * lo.G;
    g.epi.ptr[4] = nullptr;
    g.epi.i[1] = lo.G;
  }
  g.epi.i[0] = lo.Gh;
  return g;
}

ActGemmCall make_dx_call(const Layout& lo, uint8_t* ws, const uint8_t* pk, int l, float p, unsigned long long seed,
                         const unsigned long long* d_step, long long* grads) {
  const long long BT = (long long)lo.B * lo.T;
  const int d = lo.dil(l);
  const bool top = l == lo.L - 1;
  bf16* dxin = reinterpret_cast<bf16*>(ws + lo.w_dxin);
  ActGemmCall g;
  memset(&g, 0, sizeof(g));
  g.a[0] = make_act(ws + lo.w_dg, lo.G, lo.T, lo.B, lo.L); g.na = 1;
  for (int j = 0; j < lo.kw; ++j) g.seg[j] = Seg{0, (lo.kw - 1 - j) * d, 0, lo.G / kBK, l, 1};
  g.nseg = lo.kw;
  g.w = pk + lo.k_WdT; g.wN = lo.R; g.wK = lo.kw * lo.G; g.wL = lo.L; g.w_layer = l;
  g.T = lo.T; g.B = lo.B; g.n_tiles = 1;
  g.epi.ptr[0] = top ? nullptr : dxin + (long long)(l + 1) * BT * lo.R;
  g.epi.ptr[1] = dxin + (long long)l * BT * lo.R;
  g.epi.f[0] = lo.res_scale; g.epi.f[1] = p; g.epi.i[1] = l; g.epi.seed = seed;
  g.epi.ptr[7] = const_cast<unsigned long long*>(d_step);
  // dx of layer l is the gradient of x_l = output of layer l-1's out-1x1 (or of the first conv): fused bias gradient
  g.epi.ptr[2] = grads ? grads + (l > 0 ? lo.p_o_b[l - 1] : lo.p_in_b) : nullptr;
  g.epi.f[2] = l > 0 ? lo.res_scale : 1.f;
  return g;
}

// ------------------------------------------------------------------------------------------------------
// Persistent layer chains (wn_chain_kernel in t2_gemm.cu): the tickets come from build_chain, the per-(kind, layer) GemmArgs from
// the same make_*_call as the per-layer launches.
// ------------------------------------------------------------------------------------------------------
// uploaded chain tables per (workspace, direction): the table depends only on the configuration, the workspace and the packed
// weights, so it is written once and stays valid for eager calls and CUDA-graph replays alike (t2_wn_init forgets it)
struct ChainTable {
  const void* key;         // device address of the table (workspace + direction)
  const void* packed;
  t2_wn_config_t cfg;
};
struct ChainCache {
  std::mutex mu;
  std::vector<ChainTable> entries;
};
ChainCache& chain_cache() {
  static ChainCache c;
  return c;
}
void chain_cache_forget(const void* ws, long long bytes) {
  ChainCache& c = chain_cache();
  std::lock_guard<std::mutex> lk(c.mu);
  const uint8_t* lo = static_cast<const uint8_t*>(ws);
  c.entries.erase(std::remove_if(c.entries.begin(), c.entries.end(),
                                 [&](const ChainTable& e) {
                                   const uint8_t* k = static_cast<const uint8_t*>(e.key);
                                   return k >= lo && k < lo + bytes;
                                 }),
                  c.entries.end());
}

int g_chain_mode = 0;   // t2_dbg_wn_per_layer: 0 automatic, 1 per-layer launches (the bit-exact reference), 2 persistent chains

// SM count of the current device (cached per device)
int device_sms() {
  static int sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (sms[dev] == 0 && cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 132;
  return sms[dev];
}

// dir 0: the forward gate / out GEMMs of every layer; dir 1: the backward dz / dx GEMMs. `free_sms` SMs are left to concurrent work.
int launch_chain(const Layout& lo, int dir, uint8_t* ws, const uint8_t* pk, const float* params, int save, unsigned long long seed,
                 const unsigned long long* d_step, int free_sms, cudaStream_t st) {
  const int bn_z = lo.Gh >= 256 ? 256 : 128;
  const void* key = ws + lo.w_chain_tix[dir];
  ChainCache& cache = chain_cache();
  std::lock_guard<std::mutex> lk(cache.mu);
  auto it = std::find_if(cache.entries.begin(), cache.entries.end(), [&](const ChainTable& e) { return e.key == key; });
  if (it == cache.entries.end() || it->packed != pk || memcmp(&it->cfg, &lo.c, sizeof(lo.c)) != 0) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    T2_CHECK_CUDA(cudaStreamIsCapturing(st, &cap));
    T2_REQUIRE(cap == cudaStreamCaptureStatusNone, T2_ERR_INVALID_ARG,
               "the WaveNet layer-chain table of this workspace is not written yet: run one forward / backward before capturing a graph");
    // the table: the tickets, then the GemmArgs [kind][layer] of the per-layer launches (per-call values left out, see ChainArgs)
    std::vector<ChainTicket> tix;
    build_chain(lo, dir, tix);
    std::vector<GemmArgs> args(2 * lo.L);
    memset(args.data(), 0, args.size() * sizeof(GemmArgs));
    long long* gfx = reinterpret_cast<long long*>(ws + lo.w_gfx);
    for (int l = 0; l < lo.L; ++l) {
      ActGemmCall c0, c1;
      int e0, e1, b0, b1;
      const bool has1 = dir == 1 || l + 1 < lo.L;                     // no out GEMM after the top layer
      if (dir == 0) {
        c0 = make_gate_call(lo, ws, pk, l, true); e0 = EPI_GATE; b0 = 256;
        if (has1) {
          c1 = make_out_call(lo, ws, pk, nullptr, l, lo.c.dropout, 0, nullptr);
          c1.epi.ptr[3] = reinterpret_cast<void*>(uintptr_t(lo.p_o_b[l]));   // bias offset in params, resolved by the kernel
        }
        e1 = EPI_RES; b1 = lo.R;
      } else {
        c0 = make_dz_call(lo, ws, pk, l, gfx); e0 = EPI_GATE_BWD; b0 = bn_z;
        c1 = make_dx_call(lo, ws, pk, l, lo.c.dropout, 0, nullptr, gfx); e1 = EPI_DX; b1 = lo.R;
      }
      c0.cluster = c1.cluster = 1;
      dim3 grid;
      int cs = 1;
      int rc = make_gemm_args(e0, b0, c0, args[l], grid, cs);
      if (rc) return rc;
      args[l].dbg = nullptr;
      if (has1) {
        rc = make_gemm_args(e1, b1, c1, args[lo.L + l], grid, cs);
        if (rc) return rc;
        args[lo.L + l].dbg = nullptr;
      }
    }
    T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_chain_tix[dir], tix.data(), tix.size() * sizeof(ChainTicket), cudaMemcpyHostToDevice, st));
    T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_chain_args[dir], args.data(), args.size() * sizeof(GemmArgs), cudaMemcpyHostToDevice, st));
    T2_CHECK_CUDA(cudaStreamSynchronize(st));
    const ChainTable e{key, pk, lo.c};
    if (it == cache.entries.end()) cache.entries.push_back(e);
    else *it = e;
  }
  ChainArgs a;
  a.args = reinterpret_cast<const GemmArgs*>(ws + lo.w_chain_args[dir]);
  a.tix = reinterpret_cast<const ChainTicket*>(ws + lo.w_chain_tix[dir]);
  a.n_tix = lo.n_chain[dir]; a.L = lo.L;
  a.ctr = reinterpret_cast<int*>(ws + lo.w_chain_ctr[dir]);
  a.err = reinterpret_cast<int*>(ws + lo.w_chain_err);
  a.dbg = take_timing_slice((long long)lo.n_chain[dir] * kDbgSlots);
  a.params = params; a.d_step = d_step; a.seed = seed; a.save = save;
  T2_CHECK_CUDA(cudaMemsetAsync(a.ctr, 0, (16 + 2LL * lo.L * lo.MT) * 4, st));
  int grid = device_sms() - free_sms;
  if (grid > a.n_tix) grid = a.n_tix;
  if (grid < 1) grid = 1;
  return launch_wn_chain(dir == 0, dir == 0 ? 256 : bn_z, lo.R, a, grid, st);
}

// the persistent chains run unless the per-layer reference is asked for, or the launch needs what they do not support (split-bf16
// forward, weight multicast clusters). Automatically they run where a layer's gate GEMM is at most two waves of CTAs: there the
// grid-wide drains between launches are a large part of every GEMM. Layers of many waves lose less to the drains than the chains'
// per-tile overheads cost them (wavenet_mol, 1008 M tiles per layer, ran 1.3 % slower on an H100 80GB HBM3 at 700 W).
bool use_chain(const Layout& lo) {
  if (lo.split || cluster_pref() != 1 || g_chain_mode == 1) return false;
  if (g_chain_mode == 2) return true;
  return (long long)lo.MT * (lo.G / 256) <= 2LL * device_sms();
}

// One layer of the conditioning upsampler (type 0 SubPixel, 1 ConvTranspose2D, 2 ConvTranspose1D; in [B][C][W], out [B][C][W*s]):
// the launches of the training forward / backward, AR synthesis and t2_dbg_wn_kernel.
int up1d_smem_limit(const void* fn, size_t smem) {
  if (smem > 48 * 1024) T2_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  return T2_OK;
}
int launch_upsample_fwd(const float* in, const float* K, const float* bias, float* out, bf16* c_up, int B, int C, int W, int s, int type,
                        int act, float alpha, int split, cudaStream_t st) {
  if (type == 2) {
    const size_t smem = up1d_smem(C);
    const int rc = up1d_smem_limit(reinterpret_cast<const void*>(up1d_fwd_kernel), smem);
    if (rc) return rc;
    const long long wt = (W + kUp1Tw - 1) / kUp1Tw;
    const int jz = int(std::max(1LL, std::min<long long>(s, (264 + wt * B - 1) / (wt * B))));   // taps split over blocks: >= ~2 per SM
    up1d_fwd_kernel<<<dim3(unsigned(wt), B, jz), dim3(kUp1Tw, kUp1Rows), smem, st>>>(in, K, bias, out, c_up, C, W, s, act, alpha, split);
  } else {
    upsample_fwd_kernel<<<grid1d((long long)B * C * W * s), 256, 0, st>>>(in, K, bias, out, c_up, B, C, W, s, type, act, alpha, split);
  }
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}
// dK / dbias: int64 fixed-point accumulators (fx_add), turned into gradients by the finalisation
int launch_upsample_bwd_param(const float* in, const float* out, const float* dout, long long* dK, long long* dbias, int B, int C, int W,
                              int s, int type, int act, float alpha, cudaStream_t st) {
  if (type == 2) {
    const long long nchunk = ((long long)B * W + kUp1Tw - 1) / kUp1Tw;
    const int G = int(std::min<long long>(nchunk, (264 + s - 1) / s));
    up1d_bwd_param_kernel<<<dim3(s, G), dim3(kUp1Tw, kUp1Rows), up1d_param_smem(C), st>>>(in, out, dout, dK, dbias, B, C, W, s, act, alpha);
  } else {
    T2_REQUIRE(s <= 32, T2_ERR_UNSUPPORTED_SHAPE, "upsample scale %d > 32, the limit of the SubPixel / 2D weight-gradient kernel", s);
    upsample_bwd_param_kernel<<<s * ((296 + s - 1) / s), 256, 0, st>>>(in, out, dout, dK, dbias, B, C, W, s, type, act, alpha);
  }
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}
int launch_upsample_bwd_input(const float* out, const float* dout, const float* K, float* din, int B, int C, int W, int s, int type, int act,
                              float alpha, cudaStream_t st) {
  if (type == 2) {
    const size_t smem = up1d_smem(C);
    const int rc = up1d_smem_limit(reinterpret_cast<const void*>(up1d_bwd_input_kernel), smem);
    if (rc) return rc;
    up1d_bwd_input_kernel<<<dim3((W + kUp1Tw - 1) / kUp1Tw, B), dim3(kUp1Tw, kUp1Rows), smem, st>>>(out, dout, K, din, C, W, s, act, alpha);
  } else {
    upsample_bwd_input_kernel<<<grid1d(4LL * B * C * W), 256, 0, st>>>(out, dout, 0, K, din, B, C, W, s, type, act, alpha);
  }
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

GinArgs gin_args(const Layout& lo, const float* params) {
  GinArgs a;
  memset(&a, 0, sizeof(a));
  a.params = params;
  a.p_k = lo.p_g_k[0]; a.p_b = lo.p_g_b[0]; a.p_stride = lo.layer_stride; a.p_emb = lo.p_emb;
  a.L = lo.L; a.B = lo.B; a.G = lo.G; a.Gi = lo.Gi; a.NS = lo.NS;
  return a;
}

// Launches of the small kernels, shared by the engine and t2_dbg_wn_kernel (same grid and block). Each counts its launch.
void launch_derived_bias(const DerivedArgs& a, cudaStream_t st) {
  derived_bias_kernel<<<grid1d(std::max((long long)a.L * a.G, (long long)a.S)), 256, 0, st>>>(a); t2_count_launch();
}
void launch_gin_bias(const GinArgs& a, cudaStream_t st) {
  gin_bias_kernel<<<grid1d((long long)a.L * a.B * a.G), 256, 0, st>>>(a); t2_count_launch();
}
void launch_set_speakers(int* spk, const int* ids, int B, cudaStream_t st) {
  set_speakers_kernel<<<grid1d(B), 256, 0, st>>>(spk, ids, B); t2_count_launch();
}
void launch_gin_wgrad(const GinGradArgs& a, cudaStream_t st) {
  gin_wgrad_kernel<<<grid1d((long long)a.L * a.G), 256, 0, st>>>(a); t2_count_launch();
}
void launch_gin_demb(const GinGradArgs& a, cudaStream_t st) {
  gin_demb_kernel<<<dim3(a.NS, a.Gi), kGinThreads, 0, st>>>(a); t2_count_launch();
}
void launch_first_conv(const void* xin, int scalar_in, const float* W, const float* bias, bf16* x, bf16* xd, long long npos, int R,
                       float p, unsigned long long seed, const unsigned long long* step, int split, cudaStream_t st) {
  first_conv_kernel<<<grid1d(npos * (R / 8)), 256, 0, st>>>(xin, scalar_in, W, bias, x, xd, npos, R, p, seed, step, split); t2_count_launch();
}
void launch_first_conv_bwd(const void* xin, int scalar_in, const bf16* dx0, long long* dW, long long npos, int R, cudaStream_t st) {
  first_conv_bwd_kernel<<<dim3((unsigned)((npos + 63) / 64)), R, 0, st>>>(xin, scalar_in, dx0, dW, npos, R); t2_count_launch();
}
void launch_colsum(const uint8_t* ws, long long* acc, const ColsumJob* jobs, int njobs, const float* scalars, cudaStream_t st) {
  colsum_kernel<<<dim3(96, njobs), 256, 0, st>>>(ws, acc, jobs, scalars); t2_count_launch();
}
void launch_skip_bias(const long long* skipsum, float* grads, const long long* offs, const float* scales, int L, int S, cudaStream_t st) {
  skip_bias_kernel<<<grid1d((long long)L * S), 256, 0, st>>>(skipsum, grads, offs, scales, L, S); t2_count_launch();
}
void launch_cl_to_chw(const float* in, float* out, int B, int T, int C, cudaStream_t st) {
  cl_to_chw_kernel<<<dim3((T + 31) / 32, (C + 31) / 32, B), dim3(32, 8), 0, st>>>(in, out, T, C); t2_count_launch();
}

}  // namespace

int launch_fx_finalize(const long long* acc, float* out, long long n, cudaStream_t st) {
  if (n <= 0) return T2_OK;
  fx_finalize_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(acc, out, n);
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}
}  // namespace t2

using namespace t2;

// ----------------------------------------------------------------------------------------------------------
// C-ABI
// ----------------------------------------------------------------------------------------------------------
extern "C" int t2_wn_sizes(const t2_wn_config_t* cfg, t2_wn_sizes_t* out) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  T2_REQUIRE(out != nullptr, T2_ERR_INVALID_ARG, "null out");
  out->n_params = lo.n_params;
  out->packed_bytes = lo.packed_bytes;
  out->workspace_bytes = lo.workspace_bytes;
  out->n_tensors = int(lo.params.size());
  return T2_OK;
}

extern "C" int t2_wn_param_info(const t2_wn_config_t* cfg, int i, char* name, int name_cap, long long* offset,
                                int* ndim, int* shape4) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  return param_info(lo.params, i, name, name_cap, offset, ndim, shape4, nullptr);
}

extern "C" int t2_wn_init(const t2_wn_config_t* cfg, void* d_packed, void* d_workspace, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  T2_CHECK_CUDA(cudaMemsetAsync(d_packed, 0, lo.packed_bytes, st));
  T2_CHECK_CUDA(cudaMemsetAsync(d_workspace, 0, lo.workspace_bytes, st));
  chain_cache_forget(d_workspace, lo.workspace_bytes);   // the chain tables were just cleared with the rest of the workspace
  float* scalars = reinterpret_cast<float*>(ws + lo.w_scalars);
  for (auto& t : lo.tiles_head)
    if (t.div != nullptr) t.div = scalars + 1;
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_tiles_main, lo.tiles_main.data(), lo.tiles_main.size() * sizeof(WgradTile), cudaMemcpyHostToDevice, st));
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_tiles_head, lo.tiles_head.data(), lo.tiles_head.size() * sizeof(WgradTile), cudaMemcpyHostToDevice, st));
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_packjobs, lo.packjobs.data(), lo.packjobs.size() * sizeof(PackJob), cudaMemcpyHostToDevice, st));
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_colsum, lo.colsums.data(), lo.colsums.size() * sizeof(ColsumJob), cudaMemcpyHostToDevice, st));
  std::vector<long long> offs(3 * lo.L);
  for (int l = 0; l < lo.L; ++l) {
    offs[3 * l] = lo.p_dil_b[l];
    offs[3 * l + 1] = lo.C > 0 ? lo.p_c_b[l] : -1;
    offs[3 * l + 2] = lo.p_s_b[l];
  }
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_tables, offs.data(), offs.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_tables + 3 * lo.L * sizeof(long long), lo.skip_scale.data(), lo.L * sizeof(float),
                                cudaMemcpyHostToDevice, st));
  T2_CHECK_CUDA(cudaStreamSynchronize(st));
  return T2_OK;
}

extern "C" int t2_wn_pack_weights(const t2_wn_config_t* cfg, const float* d_params, void* d_packed,
                                  void* d_workspace, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  uint8_t* pk = static_cast<uint8_t*>(d_packed);
  rc = launch_pack(d_params, pk, reinterpret_cast<const PackJob*>(ws + lo.w_packjobs), lo.n_packjobs, 128, 16, st);
  if (rc) return rc;
  long long* d_offs = reinterpret_cast<long long*>(ws + lo.w_tables);
  float* d_scales = reinterpret_cast<float*>(ws + lo.w_tables + 3 * lo.L * sizeof(long long));
  DerivedArgs a;
  a.params = d_params; a.bias_g = reinterpret_cast<float*>(pk + lo.k_bias_g); a.bias_skip = reinterpret_cast<float*>(pk + lo.k_bias_skip);
  a.offs = d_offs; a.scales = d_scales; a.L = lo.L; a.G = lo.G; a.S = lo.S;
  launch_derived_bias(a, st);
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

extern "C" int t2_wn_forward(const t2_wn_config_t* cfg, const float* d_params, const void* d_packed,
                             void* d_workspace, const void* d_x, const float* d_c, const void* d_targets,
                             const int* d_lengths, float* d_loss, float* d_logits, int save_for_backward,
                             unsigned long long seed, const unsigned long long* d_step, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  const uint8_t* pk = static_cast<const uint8_t*>(d_packed);
  const long long BT = (long long)lo.B * lo.T;
  float* scalars = reinterpret_cast<float*>(ws + lo.w_scalars);
  const float p = cfg->dropout;
  T2_CHECK_CUDA(cudaMemsetAsync(scalars, 0, 16 * sizeof(float), st));

  T2_REQUIRE(!lo.split || (!save_for_backward && !cfg->c_pre_upsampled), T2_ERR_INVALID_ARG,
             "split_bf16 (fp32-class) mode is forward / loss only (save_for_backward = 0) and needs the upsampling net");
  if (lo.Gi > 0) {   // 0. per-item gate biases from the speaker ids last set (t2_wn_set_speakers)
    GinArgs a = gin_args(lo, d_params);
    const int* spk = reinterpret_cast<const int*>(ws + lo.w_spk);
    a.bias = reinterpret_cast<const float*>(pk + lo.k_bias_g); a.bias_ld = lo.G;
    a.on = spk; a.ids = spk + 1;
    a.out = reinterpret_cast<float*>(ws + lo.w_gbias); a.out_l = (long long)lo.B * lo.G; a.out_b = lo.G;
    launch_gin_bias(a, st);
    T2_CHECK_CUDA(cudaGetLastError());
  }
  // 1. conditioning -> c_up (bf16 channels-last)
  bf16* c_up = reinterpret_cast<bf16*>(ws + lo.w_cup);
  if (lo.split) T2_CHECK_CUDA(cudaMemsetAsync(c_up, 0, (size_t)BT * 256 * 2, st));     // the channel padding of both halves must read as zero
  if (lo.C > 0) {
    T2_REQUIRE(d_c != nullptr, T2_ERR_INVALID_ARG, "local conditioning enabled but d_c is NULL");
    if (cfg->c_pre_upsampled) {
      launch_f32_to_bf16(d_c, c_up, BT * lo.C, st);
    } else {
      const float* in = d_c;
      int W = lo.Tc;
      for (size_t i = 0; i < lo.up_w.size(); ++i) {
        const int s = cfg->upsample_scales[i];
        float* out = reinterpret_cast<float*>(ws + lo.w_upout[i]);
        const bool last = i + 1 == lo.up_w.size();
        rc = launch_upsample_fwd(in, d_params + lo.p_up_k[i], d_params + lo.p_up_b[i], out, last ? c_up : nullptr, lo.B, lo.C, W, s,
                                 cfg->upsample_type, cfg->upsample_activation, cfg->leaky_alpha, lo.split ? 1 : 0, st);
        if (rc) return rc;
        in = out;
        W *= s;
      }
    }
    T2_CHECK_CUDA(cudaGetLastError());
  }
  // 2. first conv
  bf16* x_all = reinterpret_cast<bf16*>(ws + lo.w_x);
  bf16* xd_all = reinterpret_cast<bf16*>(ws + lo.w_xd);
  launch_first_conv(d_x, lo.scalar_in ? 1 : 0, d_params + lo.p_in_k, d_params + lo.p_in_b, x_all, p > 0.f ? xd_all : x_all, BT, lo.R, p, seed,
                    d_step, lo.split ? 1 : 0, st);
  T2_CHECK_CUDA(cudaGetLastError());
  // 3. residual stack
  bf16* z_all = reinterpret_cast<bf16*>(ws + lo.w_z);
  if (use_chain(lo)) {
    rc = launch_chain(lo, 0, ws, pk, d_params, save_for_backward != 0, seed, d_step, 0, st);
    if (rc) return rc;
  } else {
    for (int l = 0; l < lo.L; ++l) {
      ActGemmCall g = make_gate_call(lo, ws, pk, l, save_for_backward != 0);
      rc = launch_act_gemm(EPI_GATE, 256, g, st);
      if (rc) return rc;
      if (l + 1 < lo.L) {
        ActGemmCall o = make_out_call(lo, ws, pk, d_params, l, p, seed, d_step);
        rc = launch_act_gemm(EPI_RES, lo.R, o, st);
        if (rc) return rc;
      }
    }
  }
  // 4. all skip 1x1s as one K = L*Gh GEMM, + ReLU
  bf16* h1 = reinterpret_cast<bf16*>(ws + lo.w_h1);
  bf16* h2 = reinterpret_cast<bf16*>(ws + lo.w_h2);
  rc = launch_bias_act({.a = z_all, .C = lo.Gh, .T = lo.T, .B = lo.B, .layers = lo.L, .split = lo.split, .w = pk + lo.k_Ws, .N = lo.S,
                        .wK = lo.L * lo.Gh, .BN = lo.S, .bias = reinterpret_cast<const float*>(pk + lo.k_bias_skip), .act = 1, .out_bf16 = h1,
                        .ldo = lo.S, .nvalid = lo.S},
                       st);
  if (rc) return rc;
  rc = launch_bias_act({.a = h1, .C = lo.S, .T = lo.T, .B = lo.B, .split = lo.split, .w = pk + lo.k_Wf1, .N = lo.S, .wK = lo.S, .BN = lo.S,
                        .bias = d_params + lo.p_f1_b, .act = 1, .out_bf16 = h2, .ldo = lo.S, .nvalid = lo.S},
                       st);
  if (rc) return rc;
  // 5. output projection fused with the loss
  {
    ActGemmCall g;
    memset(&g, 0, sizeof(g));
    g.a[0] = make_act(h2, lo.S, lo.T, lo.B); g.na = 1;
    g.seg[0] = Seg{0, 0, 0, lo.S / kBK, 0, 1}; g.nseg = 1;
    g.w = pk + lo.k_Wf2; g.wN = lo.O; g.wK = lo.S; g.wL = 1;
    g.split = lo.split;
    g.T = lo.T; g.B = lo.B; g.n_tiles = 1;
    g.epi.ptr[0] = const_cast<void*>(d_targets);
    g.epi.ptr[1] = const_cast<int*>(d_lengths);
    g.epi.ptr[2] = const_cast<float*>(d_params + lo.p_f2_b);
    g.epi.ptr[3] = scalars + 0; g.epi.ptr[4] = scalars + 1;
    g.epi.ptr[5] = save_for_backward ? ws + lo.w_dlog : nullptr;
    g.epi.ptr[6] = d_logits;
    g.epi.i[1] = lo.ldo;
    if (lo.mol) {
      g.epi.f[0] = cfg->log_scale_min;
      g.epi.f[1] = 1.f / float(lo.Q - 1);
      g.epi.f[2] = logf(float(lo.Q - 1) / 2.f);
      g.epi.i[0] = lo.gauss ? 0 : lo.O / 3;
      g.epi.i[2] = lo.gauss ? (cfg->cdf_loss ? 2 : 1) : 0;     // 0 mixture of logistics, 1 Gaussian log-density, 2 Gaussian CDF difference
      g.epi.f[3] = cfg->log_scale_min_gauss;
      rc = launch_act_gemm(EPI_MOL, 32, g, st);
    } else {
      rc = launch_act_gemm(EPI_CE, 256, g, st);
    }
    if (rc) return rc;
  }
  if (d_loss) T2_CHECK_CUDA(cudaMemcpyAsync(d_loss, scalars, 2 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return T2_OK;
}

extern "C" int t2_wn_backward(const t2_wn_config_t* cfg, const float* d_params, const void* d_packed,
                              void* d_workspace, const void* d_x, const float* d_c, float* d_grads,
                              unsigned long long seed, const unsigned long long* d_step, void* stream) {
  return t2_wn_backward_phased(cfg, d_params, d_packed, d_workspace, d_x, d_c, d_grads, seed, d_step, -1, 1, stream);
}

// Phased form for data-parallel training: the weight gradients of the residual stack are produced by `n_groups` launches (layer
// groups, top of the parameter buffer first) so that the caller can start the gradient all-reduce of a group's contiguous
// parameter range while the next group's GEMM runs. phase -1: everything in one call (== t2_wn_backward); phase 0: the data-gradient
// chain + head + conditioning tails (no stack weight gradients, side stream NOT yet joined); phase 1 + g: weight gradients of layer
// group g (layers [g*L/n, (g+1)*L/n)); phase 100: join the side stream. wavenet.py:561-593 averages tower gradients after backward.
extern "C" int t2_wn_backward_phased(const t2_wn_config_t* cfg, const float* d_params, const void* d_packed,
                                     void* d_workspace, const void* d_x, const float* d_c, float* d_grads,
                                     unsigned long long seed, const unsigned long long* d_step, int phase, int n_groups, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  T2_REQUIRE(!lo.split, T2_ERR_INVALID_ARG, "split_bf16 (fp32-class) mode has no backward pass");
  T2_REQUIRE(n_groups >= 1 && n_groups <= lo.L && (phase == -1 || phase == 100 || (phase >= 0 && phase <= n_groups)), T2_ERR_INVALID_ARG,
             "backward_phased: bad phase %d / n_groups %d", phase, n_groups);
  if (phase >= 1 && phase <= n_groups) {
    uint8_t* ws = static_cast<uint8_t*>(d_workspace);
    const int g = phase - 1;
    const int l0 = int((long long)lo.L * g / n_groups), l1 = int((long long)lo.L * (g + 1) / n_groups);
    const int t0 = lo.tile_start[l0], t1 = lo.tile_start[l1];
    ActT maps[6] = {make_act(ws + lo.w_xd, lo.R, lo.T, lo.B, lo.L), make_act(ws + lo.w_dg, lo.G, lo.T, lo.B, lo.L),
                    make_act(ws + lo.w_cup, lo.C > 0 ? lo.C : 8, lo.T, lo.B, 1),
                    make_act(ws + lo.w_z, lo.Gh, lo.T, lo.B, lo.L), make_act(ws + lo.w_dxin, lo.R, lo.T, lo.B, lo.L),
                    make_act(ws + lo.w_dskip, lo.S, lo.T, lo.B, 1)};
    return launch_wgrad(maps, 6, reinterpret_cast<const WgradTile*>(ws + lo.w_tiles_main) + t0, t1 - t0, d_grads, lo.T, lo.B, st);
  }
  if (phase == 100) {
    SideStream* side = side_stream();
    if (side) {
      T2_CHECK_CUDA(cudaEventRecord(side->join, side->s));
      T2_CHECK_CUDA(cudaStreamWaitEvent(st, side->join, 0));
    }
    return launch_fx_finalize(reinterpret_cast<const long long*>(static_cast<uint8_t*>(d_workspace) + lo.w_gfx), d_grads, lo.n_params, st);
  }
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  const uint8_t* pk = static_cast<const uint8_t*>(d_packed);
  const long long BT = (long long)lo.B * lo.T;
  float* scalars = reinterpret_cast<float*>(ws + lo.w_scalars);
  const float p = cfg->dropout;
  T2_CHECK_CUDA(cudaMemsetAsync(d_grads, 0, lo.n_params * sizeof(float), st));
  T2_CHECK_CUDA(cudaMemsetAsync(ws + lo.w_skipsum, 0, lo.S * sizeof(long long), st));
  T2_CHECK_CUDA(cudaMemsetAsync(ws + lo.w_gfx, 0, lo.n_params * sizeof(long long), st));
  if (lo.Gi > 0) T2_CHECK_CUDA(cudaMemsetAsync(ws + lo.w_gsum, 0, (size_t)lo.L * lo.B * lo.G * sizeof(long long), st));
  long long* gfx = reinterpret_cast<long long*>(ws + lo.w_gfx);
  bf16* h1 = reinterpret_cast<bf16*>(ws + lo.w_h1);
  bf16* h2 = reinterpret_cast<bf16*>(ws + lo.w_h2);
  bf16* dlog = reinterpret_cast<bf16*>(ws + lo.w_dlog);
  bf16* dh2 = reinterpret_cast<bf16*>(ws + lo.w_dh2);
  bf16* dskip = reinterpret_cast<bf16*>(ws + lo.w_dskip);
  bf16* dxin = reinterpret_cast<bf16*>(ws + lo.w_dxin);
  bf16* dg = reinterpret_cast<bf16*>(ws + lo.w_dg);
  bf16* ta_all = reinterpret_cast<bf16*>(ws + lo.w_ta);
  bf16* sb_all = reinterpret_cast<bf16*>(ws + lo.w_sb);
  // head: dh2 = (dlog x Wf2^T) * relu'(h2) / count ; dskip = (dh2 x Wf1^T) * relu'(h1)
  {
    ActGemmCall g;
    memset(&g, 0, sizeof(g));
    g.a[0] = make_act(dlog, lo.ldo, lo.T, lo.B); g.na = 1;
    g.seg[0] = Seg{0, 0, 0, lo.Op / kBK, 0, 1}; g.nseg = 1;
    g.w = pk + lo.k_Wf2T; g.wN = lo.S; g.wK = lo.Op; g.wL = 1;
    g.T = lo.T; g.B = lo.B; g.n_tiles = 1;
    g.epi.ptr[0] = dh2; g.epi.ptr[1] = h2; g.epi.ptr[2] = scalars + 1; g.epi.f[0] = 1.f; g.epi.i[0] = lo.S;
    g.epi.ptr[3] = gfx + lo.p_f1_b;
    rc = launch_act_gemm(EPI_SCALE_RELUMASK, lo.S, g, st);
    if (rc) return rc;
  }
  {
    ActGemmCall g;
    memset(&g, 0, sizeof(g));
    g.a[0] = make_act(dh2, lo.S, lo.T, lo.B); g.na = 1;
    g.seg[0] = Seg{0, 0, 0, lo.S / kBK, 0, 1}; g.nseg = 1;
    g.w = pk + lo.k_Wf1T; g.wN = lo.S; g.wK = lo.S; g.wL = 1;
    g.T = lo.T; g.B = lo.B; g.n_tiles = 1;
    g.epi.ptr[0] = dskip; g.epi.ptr[1] = h1; g.epi.ptr[2] = nullptr; g.epi.f[0] = 1.f; g.epi.i[0] = lo.S;
    g.epi.ptr[3] = ws + lo.w_skipsum;
    rc = launch_act_gemm(EPI_SCALE_RELUMASK, lo.S, g, st);
    if (rc) return rc;
  }
  launch_skip_bias(reinterpret_cast<const long long*>(ws + lo.w_skipsum), d_grads, reinterpret_cast<const long long*>(ws + lo.w_tables),
                   reinterpret_cast<const float*>(ws + lo.w_tables + 3 * lo.L * sizeof(long long)), lo.L, lo.S, st);
  // The head's weight gradients (6 tiles with a 15360-long reduction: ~100 us on 6 SMs) and the bias column sums of dlog
  // depend only on the head backward above: they run on the side stream underneath the whole residual-stack chain below,
  // which leaves SMs idle (120 M tiles).
  SideStream* side = side_stream();
  cudaStream_t sb = st;
  if (side) {
    T2_CHECK_CUDA(cudaEventRecord(side->fork, st));
    T2_CHECK_CUDA(cudaStreamWaitEvent(side->s, side->fork, 0));
    sb = side->s;
  }
  {
    ActT hmaps[4] = {make_act(h1, lo.S, lo.T, lo.B), make_act(dh2, lo.S, lo.T, lo.B), make_act(h2, lo.S, lo.T, lo.B),
                     make_act(dlog, lo.ldo, lo.T, lo.B)};
    rc = launch_wgrad(hmaps, 4, reinterpret_cast<const WgradTile*>(ws + lo.w_tiles_head), lo.n_tiles_head, d_grads, lo.T, lo.B, sb);
    if (rc) return rc;
    launch_colsum(ws, gfx, reinterpret_cast<const ColsumJob*>(ws + lo.w_colsum), lo.n_colsum, scalars, sb);
    T2_CHECK_CUDA(cudaGetLastError());
  }
  // residual stack, top down
  const ActT a_dxin = make_act(dxin, lo.R, lo.T, lo.B, lo.L);
  const ActT a_dskip = make_act(dskip, lo.S, lo.T, lo.B, 1);
  const ActT a_dg = make_act(dg, lo.G, lo.T, lo.B, lo.L);
  const int bn_z = lo.Gh >= 256 ? 256 : 128;
  if (use_chain(lo)) {
    // the head weight-gradient tiles on the side stream keep their SMs (they used to run on the SMs the 120-tile launches left idle)
    rc = launch_chain(lo, 1, ws, pk, d_params, 1, seed, d_step, side ? lo.n_tiles_head : 0, st);
    if (rc) return rc;
  } else {
    for (int l = lo.L - 1; l >= 0; --l) {
      ActGemmCall gz = make_dz_call(lo, ws, pk, l, gfx);
      rc = launch_act_gemm(EPI_GATE_BWD, bn_z, gz, st);
      if (rc) return rc;
      ActGemmCall gx = make_dx_call(lo, ws, pk, l, p, seed, d_step, gfx);
      rc = launch_act_gemm(EPI_DX, lo.R, gx, st);
      if (rc) return rc;
    }
  }
  if (lo.Gi > 0) {   // gate-bias and speaker-term gradients from the per-item sums of the gate backward
    GinGradArgs a;
    a.params = d_params; a.spk = reinterpret_cast<const int*>(ws + lo.w_spk);
    a.S = reinterpret_cast<const long long*>(ws + lo.w_gsum); a.gfx = gfx; a.grads = d_grads;
    a.offs = reinterpret_cast<const long long*>(ws + lo.w_tables);
    a.p_k = lo.p_g_k[0]; a.p_b = lo.p_g_b[0]; a.p_stride = lo.layer_stride; a.p_emb = lo.p_emb;
    a.L = lo.L; a.B = lo.B; a.G = lo.G; a.Gi = lo.Gi; a.NS = lo.NS;
    launch_gin_wgrad(a, st);
    launch_gin_demb(a, st);
    T2_CHECK_CUDA(cudaGetLastError());
  }
  // From here on two independent tails: (A) the batched weight-gradient GEMM of the stack (fills the machine), (B) the
  // conditioning path (K = L*G data-gradient GEMM, transposes, upsampling-net backward) + first-conv gradient: latency-bound
  // small kernels. (B) continues on the side stream (fork/join through events, capturable into the caller's CUDA graph).
  if (side) {
    T2_CHECK_CUDA(cudaEventRecord(side->fork2, st));
    T2_CHECK_CUDA(cudaStreamWaitEvent(side->s, side->fork2, 0));
  }
  // weight gradients of the stack: one batched launch
  if (phase == -1) {
    ActT maps[6] = {make_act(ws + lo.w_xd, lo.R, lo.T, lo.B, lo.L), a_dg,
                    make_act(ws + lo.w_cup, lo.C > 0 ? lo.C : 8, lo.T, lo.B, 1),
                    make_act(ws + lo.w_z, lo.Gh, lo.T, lo.B, lo.L), a_dxin, a_dskip};
    rc = launch_wgrad(maps, 6, reinterpret_cast<const WgradTile*>(ws + lo.w_tiles_main), lo.n_tiles_main, d_grads, lo.T, lo.B, st);
    if (rc) return rc;
  }
  // first conv
  launch_first_conv_bwd(d_x, lo.scalar_in ? 1 : 0, dxin, gfx + lo.p_in_k, BT, lo.R, sb);
  T2_CHECK_CUDA(cudaGetLastError());
  // conditioning path
  if (lo.C > 0 && !cfg->c_pre_upsampled) {
    float* dcup = reinterpret_cast<float*>(ws + lo.w_dcup);
    rc = launch_bias_act({.a = dg, .C = lo.G, .T = lo.T, .B = lo.B, .layers = lo.L, .w = pk + lo.k_WcT, .N = lo.C, .wK = lo.L * lo.G, .BN = 128,
                          .out_f32 = dcup, .ldo = lo.C, .nvalid = lo.C},
                         sb);
    if (rc) return rc;
    // dc_up arrives channels-last from the GEMM: transpose once into [B][C][T]
    float* dchw = reinterpret_cast<float*>(ws + lo.w_upgrad[1]);
    launch_cl_to_chw(dcup, dchw, lo.B, lo.T, lo.C, sb);
    const float* dout = dchw;
    int pp = 0;
    for (int i = int(lo.up_w.size()) - 1; i >= 0; --i) {
      const int s = cfg->upsample_scales[i];
      const int W = lo.up_w[i] / s;
      const float* layer_in = i == 0 ? d_c : reinterpret_cast<const float*>(ws + lo.w_upout[i - 1]);
      const float* out = reinterpret_cast<const float*>(ws + lo.w_upout[i]);
      rc = launch_upsample_bwd_param(layer_in, out, dout, gfx + lo.p_up_k[i], gfx + lo.p_up_b[i], lo.B, lo.C, W, s, cfg->upsample_type,
                                     cfg->upsample_activation, cfg->leaky_alpha, sb);
      if (rc) return rc;
      if (i > 0) {
        float* din = reinterpret_cast<float*>(ws + lo.w_upgrad[pp]);
        rc = launch_upsample_bwd_input(out, dout, d_params + lo.p_up_k[i], din, lo.B, lo.C, W, s, cfg->upsample_type, cfg->upsample_activation,
                                       cfg->leaky_alpha, sb);
        if (rc) return rc;
        dout = din;
        pp ^= 1;
      }
    }
  }
  if (side && phase == -1) {
    T2_CHECK_CUDA(cudaEventRecord(side->join, sb));
    T2_CHECK_CUDA(cudaStreamWaitEvent(st, side->join, 0));
  }
  if (phase == -1) {   // (phased: once the side stream has joined, in phase 100)
    const int rc = launch_fx_finalize(gfx, d_grads, lo.n_params, st);
    if (rc) return rc;
  }
  return T2_OK;
}

extern "C" int t2_dbg_wn_per_layer(int mode) {
  T2_REQUIRE(mode >= 0 && mode <= 2, T2_ERR_INVALID_ARG, "dbg_wn_per_layer: mode must be 0, 1 or 2 (got %d)", mode);
  g_chain_mode = mode;
  return T2_OK;
}

extern "C" int t2_dbg_wn_chain(const t2_wn_config_t* cfg, int dir, int* out, int cap) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  T2_REQUIRE(dir == 0 || dir == 1, T2_ERR_INVALID_ARG, "dbg_wn_chain: dir must be 0 (forward) or 1 (backward), got %d", dir);
  std::vector<ChainTicket> v;
  build_chain(lo, dir, v);
  T2_REQUIRE(int(v.size()) == lo.n_chain[dir], T2_ERR_INVALID_ARG, "dbg_wn_chain: %d tickets built, %d reserved", int(v.size()),
             lo.n_chain[dir]);
  T2_REQUIRE(out == nullptr || cap >= int(v.size()), T2_ERR_INVALID_ARG, "dbg_wn_chain: %d tickets do not fit in %d", int(v.size()), cap);
  if (out)
    for (size_t i = 0; i < v.size(); ++i) {
      const ChainTicket& t = v[i];
      const int row[8] = {t.kind, t.layer, t.m, t.n, t.dep_lo, t.dep_hi, t.dep_target, t.done};
      memcpy(out + 8 * i, row, sizeof(row));
    }
  return int(v.size());
}

extern "C" int t2_wn_set_speakers(const t2_wn_config_t* cfg, void* d_workspace, const int* d_speaker_ids, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  T2_REQUIRE(lo.Gi > 0, T2_ERR_INVALID_ARG, "speaker ids need gin_channels > 0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  launch_set_speakers(reinterpret_cast<int*>(static_cast<uint8_t*>(d_workspace) + lo.w_spk), d_speaker_ids, lo.B, st);
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

extern "C" int t2_wn_workspace_tensor(const t2_wn_config_t* cfg, void* d_workspace, const char* name, void** ptr,
                                      long long* count, int* elem_bytes) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  const long long BT = (long long)lo.B * lo.T;
  struct E { const char* n; long long off; long long cnt; int eb; };
  const E table[] = {
      {"c_up", lo.w_cup, BT * lo.C, 2},       {"x", lo.w_x, lo.L * BT * lo.R, 2},    {"xd", lo.w_xd, lo.L * BT * lo.R, 2},
      {"ta", lo.w_ta, lo.L * BT * lo.Gh, 2},  {"sb", lo.w_sb, lo.L * BT * lo.Gh, 2}, {"z", lo.w_z, lo.L * BT * lo.Gh, 2},
      {"h1", lo.w_h1, BT * lo.S, 2},          {"h2", lo.w_h2, BT * lo.S, 2},         {"dlog", lo.w_dlog, BT * lo.ldo, 2},
      {"dh2", lo.w_dh2, BT * lo.S, 2},        {"dskip", lo.w_dskip, BT * lo.S, 2},   {"dxin", lo.w_dxin, lo.L * BT * lo.R, 2},
      {"dg", lo.w_dg, lo.L * BT * lo.G, 2},   {"dc_up", lo.w_dcup, BT * lo.C, 4},    {"scalars", lo.w_scalars, 16, 4},
      {"chain_err", lo.w_chain_err, 1, 4},
  };
  for (const E& e : table)
    if (strcmp(e.n, name) == 0) {
      *ptr = ws + e.off; *count = e.cnt; *elem_bytes = e.eb;
      return T2_OK;
    }
  return t2_set_error(T2_ERR_INVALID_ARG, "unknown workspace tensor '%s'", name);
}

// test hook: one launch of a conditioning-upsampler kernel or of a small kernel on caller buffers (include/t2b200.h, T2_DBG_WN_*)
namespace {
int dbg_wn_upsample(const t2_dbg_kernel_t* call, cudaStream_t st) {
  void* const* p = call->p;
  const long long* i = call->i;
  const long long B = i[0], C = i[1], W = i[2], s = i[3], type = i[4], act = i[5];
  const float alpha = call->f[0];
  T2_REQUIRE(B >= 1 && B <= 65535 && C >= 1 && C <= 128 && W >= 1 && s >= 1 && W * s <= (1LL << 28) && B * C * W * s <= (1LL << 31) &&
                 type >= 0 && type <= 2 && act >= 0 && act <= 2 && alpha >= 0.f && alpha <= 1.f,
             T2_ERR_INVALID_ARG, "dbg_wn_kernel: bad shape, type, activation or alpha");
  const int b = int(B), c = int(C), w = int(W), sc = int(s), ty = int(type), ac = int(act);
  switch (call->kernel) {
    case T2_DBG_WN_UP_FWD:
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && (i[6] == 0 || i[6] == 1), T2_ERR_INVALID_ARG, "dbg_wn_kernel UP_FWD: bad arguments");
      return launch_upsample_fwd(static_cast<const float*>(p[0]), static_cast<const float*>(p[1]), static_cast<const float*>(p[2]),
                                 static_cast<float*>(p[3]), static_cast<bf16*>(p[4]), b, c, w, sc, ty, ac, alpha, int(i[6]), st);
    case T2_DBG_WN_UP_BWD_PARAM: {
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && p[4] && p[5], T2_ERR_INVALID_ARG, "dbg_wn_kernel UP_BWD_PARAM: null pointer argument");
      T2_REQUIRE(ty == 2 || sc <= 32, T2_ERR_UNSUPPORTED_SHAPE, "dbg_wn_kernel UP_BWD_PARAM: upsample scale %d > 32 (SubPixel / 2D)", sc);
      const long long nK = ty == 0 ? 9LL * sc : ty == 1 ? 3LL * sc : s * C * C, nb = ty == 0 ? sc : ty == 1 ? 1 : C;
      long long* acc = static_cast<long long*>(p[5]);
      float* dK = static_cast<float*>(p[3]);
      float* db = static_cast<float*>(p[4]);
      T2_CHECK_CUDA(cudaMemsetAsync(acc, 0, size_t(nK + nb) * sizeof(long long), st));
      int rc = launch_upsample_bwd_param(static_cast<const float*>(p[0]), static_cast<const float*>(p[1]), static_cast<const float*>(p[2]),
                                         acc, acc + nK, b, c, w, sc, ty, ac, alpha, st);
      if (rc) return rc;
      T2_CHECK_CUDA(cudaMemsetAsync(dK, 0, size_t(nK) * sizeof(float), st));
      T2_CHECK_CUDA(cudaMemsetAsync(db, 0, size_t(nb) * sizeof(float), st));
      rc = launch_fx_finalize(acc, dK, nK, st);
      return rc ? rc : launch_fx_finalize(acc + nK, db, nb, st);
    }
    default:  // T2_DBG_WN_UP_BWD_INPUT
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3], T2_ERR_INVALID_ARG, "dbg_wn_kernel UP_BWD_INPUT: null pointer argument");
      return launch_upsample_bwd_input(static_cast<const float*>(p[0]), static_cast<const float*>(p[1]), static_cast<const float*>(p[2]),
                                       static_cast<float*>(p[3]), b, c, w, sc, ty, ac, alpha, st);
  }
}

bool in_range(long long v, long long lo, long long hi) { return v >= lo && v <= hi; }

// the speaker kernels' integer arguments i[0..11]: L, B, G, Gi, NS, then (per id) offsets; shapes in [1, 2^20] with L*B*G < 2^31
int dbg_gin_shape(const long long* i, const char* what) {
  for (int k = 0; k < 5; ++k)
    T2_REQUIRE(in_range(i[k], 1, 1 << 20), T2_ERR_UNSUPPORTED_SHAPE, "dbg_wn_kernel %s: L, B, G, Gi, NS must be in [1, 2^20] (i[%d] = %lld)",
               what, k, i[k]);
  T2_REQUIRE(i[0] * i[1] * i[2] < (1LL << 31) && i[3] <= 65535, T2_ERR_UNSUPPORTED_SHAPE, "dbg_wn_kernel %s: L*B*G >= 2^31 or Gi > 65535",
             what);
  return T2_OK;
}
}  // namespace

extern "C" int t2_dbg_wn_kernel(const t2_dbg_kernel_t* call, void* stream) {
  T2_REQUIRE(call != nullptr, T2_ERR_INVALID_ARG, "dbg_wn_kernel: null call");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  void* const* p = call->p;
  const long long* i = call->i;
  switch (call->kernel) {
    case T2_DBG_WN_UP_FWD:
    case T2_DBG_WN_UP_BWD_PARAM:
    case T2_DBG_WN_UP_BWD_INPUT:
      return dbg_wn_upsample(call, st);
    case T2_DBG_WN_FIRST_CONV: {
      const long long npos = i[0], R = i[1];
      const float pd = call->f[0];
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3], T2_ERR_INVALID_ARG, "dbg_wn_kernel FIRST_CONV: null pointer argument");
      T2_REQUIRE(in_range(npos, 1, 1LL << 28) && in_range(R, 8, 1024) && R % 8 == 0, T2_ERR_UNSUPPORTED_SHAPE,
                 "dbg_wn_kernel FIRST_CONV: npos must be in [1, 2^28], R a multiple of 8 in [8, 1024]");
      T2_REQUIRE(in_range(i[2], 0, 1) && in_range(i[3], 0, 1) && (i[3] == 0 || p[4] == nullptr) && pd >= 0.f && pd < 1.f, T2_ERR_INVALID_ARG,
                 "dbg_wn_kernel FIRST_CONV: scalar_in and split are 0 / 1, split has no dropout copy, dropout p in [0, 1)");
      launch_first_conv(p[0], int(i[2]), static_cast<const float*>(p[1]), static_cast<const float*>(p[2]), static_cast<bf16*>(p[3]),
                        static_cast<bf16*>(p[4]), npos, int(R), pd, call->seed, call->step, int(i[3]), st);
      break;
    }
    case T2_DBG_WN_FIRST_CONV_BWD: {
      const long long npos = i[0], R = i[1], Q = i[3];
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3], T2_ERR_INVALID_ARG, "dbg_wn_kernel FIRST_CONV_BWD: null pointer argument");
      T2_REQUIRE(in_range(npos, 1, 1LL << 28) && in_range(R, 1, 1024) && in_range(i[2], 0, 1) && in_range(Q, 1, 1 << 20) &&
                     (i[2] == 0 || Q == 1),
                 T2_ERR_UNSUPPORTED_SHAPE, "dbg_wn_kernel FIRST_CONV_BWD: npos in [1, 2^28], R in [1, 1024], scalar_in 0 / 1, Q in [1, 2^20] (1 for scalar input)");
      long long* acc = static_cast<long long*>(p[2]);
      T2_CHECK_CUDA(cudaMemsetAsync(acc, 0, size_t(Q * R) * sizeof(long long), st));
      launch_first_conv_bwd(p[0], int(i[2]), static_cast<const bf16*>(p[1]), acc, npos, int(R), st);
      T2_CHECK_CUDA(cudaGetLastError());
      return launch_fx_finalize(acc, static_cast<float*>(p[3]), Q * R, st);
    }
    case T2_DBG_WN_COLSUM: {
      const long long njobs = i[0], n_acc = i[1], ws_bytes = i[2], n_scalars = i[3];
      T2_REQUIRE(p[0] && p[1] && p[2] && p[4] && p[5] && p[6], T2_ERR_INVALID_ARG, "dbg_wn_kernel COLSUM: null pointer argument");
      T2_REQUIRE(in_range(njobs, 1, 65535) && in_range(n_acc, 1, 1LL << 40) && ws_bytes >= 0 && in_range(n_scalars, 0, 1 << 20) &&
                     (n_scalars == 0 || p[3]),
                 T2_ERR_INVALID_ARG, "dbg_wn_kernel COLSUM: bad job count, accumulator count, workspace size or scalars");
      static_assert(sizeof(ColsumJob) <= 64, "T2_DBG_WN_COLSUM documents 64 bytes of table per job");
      const long long* ji = static_cast<const long long*>(p[5]);
      const float* jf = static_cast<const float*>(p[6]);
      std::vector<ColsumJob> jobs(static_cast<size_t>(njobs));
      for (long long k = 0; k < njobs; ++k) {
        const long long* r = ji + 7 * k;
        ColsumJob& j = jobs[size_t(k)];
        T2_REQUIRE(in_range(r[1], 1, 1LL << 31) && in_range(r[2], 2, 1 << 20) && r[2] % 2 == 0 && in_range(r[3], r[2], 1 << 20) && r[3] % 2 == 0,
                   T2_ERR_UNSUPPORTED_SHAPE, "dbg_wn_kernel COLSUM job %lld: rows in [1, 2^31], C and ld even with 2 <= C <= ld <= 2^20", k);
        T2_REQUIRE(r[0] >= 0 && r[0] % 4 == 0 && r[0] + r[1] * r[3] * 2 <= ws_bytes && in_range(r[4], 0, n_acc - r[2]) &&
                       (r[5] == -1 || in_range(r[5], 0, n_acc - r[2])) && in_range(r[6], -1, n_scalars - 1) && std::isfinite(jf[k]),
                   T2_ERR_INVALID_ARG, "dbg_wn_kernel COLSUM job %lld: source outside the workspace, destination outside the accumulators, "
                   "bad scalar index or non-finite scale", k);
        j.src_off = r[0]; j.rows = r[1]; j.C = int(r[2]); j.ld = int(r[3]); j.dst_off = r[4]; j.dst2_off = r[5]; j.scale = jf[k];
        j.div_scalar = int(r[6]);
      }
      long long* acc = static_cast<long long*>(p[1]);
      ColsumJob* table = static_cast<ColsumJob*>(p[4]);
      T2_CHECK_CUDA(cudaMemsetAsync(acc, 0, size_t(n_acc) * sizeof(long long), st));
      // from pageable memory: returns once the table is staged, so it may go out of scope
      T2_CHECK_CUDA(cudaMemcpyAsync(table, jobs.data(), jobs.size() * sizeof(ColsumJob), cudaMemcpyHostToDevice, st));
      launch_colsum(static_cast<const uint8_t*>(p[0]), acc, table, int(njobs), static_cast<const float*>(p[3]), st);
      T2_CHECK_CUDA(cudaGetLastError());
      return launch_fx_finalize(acc, static_cast<float*>(p[2]), n_acc, st);
    }
    case T2_DBG_WN_DERIVED_BIAS: {
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && p[4], T2_ERR_INVALID_ARG, "dbg_wn_kernel DERIVED_BIAS: null pointer argument");
      T2_REQUIRE(in_range(i[0], 1, 1 << 20) && in_range(i[1], 1, 1 << 20) && in_range(i[2], 1, 1 << 20) && i[0] * i[1] < (1LL << 31),
                 T2_ERR_UNSUPPORTED_SHAPE, "dbg_wn_kernel DERIVED_BIAS: L, G, S in [1, 2^20] with L*G < 2^31");
      DerivedArgs a;
      a.params = static_cast<const float*>(p[0]); a.bias_g = static_cast<float*>(p[1]); a.bias_skip = static_cast<float*>(p[2]);
      a.offs = static_cast<const long long*>(p[3]); a.scales = static_cast<const float*>(p[4]);
      a.L = int(i[0]); a.G = int(i[1]); a.S = int(i[2]);
      launch_derived_bias(a, st);
      break;
    }
    case T2_DBG_WN_SKIP_BIAS:
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3], T2_ERR_INVALID_ARG, "dbg_wn_kernel SKIP_BIAS: null pointer argument");
      T2_REQUIRE(in_range(i[0], 1, 1 << 20) && in_range(i[1], 1, 1 << 20) && i[0] * i[1] < (1LL << 31), T2_ERR_UNSUPPORTED_SHAPE,
                 "dbg_wn_kernel SKIP_BIAS: L, S in [1, 2^20] with L*S < 2^31");
      launch_skip_bias(static_cast<const long long*>(p[0]), static_cast<float*>(p[1]), static_cast<const long long*>(p[2]),
                       static_cast<const float*>(p[3]), int(i[0]), int(i[1]), st);
      break;
    case T2_DBG_WN_FX_FINALIZE:
      T2_REQUIRE(p[0] && p[1] && in_range(i[0], 1, 1LL << 40), T2_ERR_INVALID_ARG, "dbg_wn_kernel FX_FINALIZE: null pointer or n outside [1, 2^40]");
      return launch_fx_finalize(static_cast<const long long*>(p[0]), static_cast<float*>(p[1]), i[0], st);
    case T2_DBG_WN_CL_TO_CHW:
      T2_REQUIRE(p[0] && p[1], T2_ERR_INVALID_ARG, "dbg_wn_kernel CL_TO_CHW: null pointer argument");
      T2_REQUIRE(in_range(i[0], 1, 65535) && in_range(i[1], 1, 1 << 26) && in_range(i[2], 1, 1 << 20), T2_ERR_UNSUPPORTED_SHAPE,
                 "dbg_wn_kernel CL_TO_CHW: B in [1, 65535], T in [1, 2^26], C in [1, 2^20]");
      launch_cl_to_chw(static_cast<const float*>(p[0]), static_cast<float*>(p[1]), int(i[0]), int(i[1]), int(i[2]), st);
      break;
    case T2_DBG_WN_GIN_BIAS: {
      T2_REQUIRE(p[0] && p[1] && p[4], T2_ERR_INVALID_ARG, "dbg_wn_kernel GIN_BIAS: null pointer argument");
      int rc = dbg_gin_shape(i, "GIN_BIAS");
      if (rc) return rc;
      for (int k = 5; k < 12; ++k)
        T2_REQUIRE(in_range(i[k], 0, 1LL << 40), T2_ERR_INVALID_ARG, "dbg_wn_kernel GIN_BIAS: strides / offsets must be in [0, 2^40] (i[%d])", k);
      GinArgs a;
      a.params = static_cast<const float*>(p[0]); a.bias = static_cast<const float*>(p[1]); a.on = static_cast<const int*>(p[2]);
      a.ids = static_cast<const int*>(p[3]); a.out = static_cast<float*>(p[4]);
      a.L = int(i[0]); a.B = int(i[1]); a.G = int(i[2]); a.Gi = int(i[3]); a.NS = int(i[4]);
      a.bias_ld = i[5]; a.out_l = i[6]; a.out_b = i[7]; a.p_k = i[8]; a.p_b = i[9]; a.p_stride = i[10]; a.p_emb = i[11];
      launch_gin_bias(a, st);
      break;
    }
    case T2_DBG_WN_SET_SPEAKERS:
      T2_REQUIRE(p[0] && in_range(i[0], 1, 1 << 20), T2_ERR_INVALID_ARG, "dbg_wn_kernel SET_SPEAKERS: null spk or B outside [1, 2^20]");
      launch_set_speakers(static_cast<int*>(p[0]), static_cast<const int*>(p[1]), int(i[0]), st);
      break;
    case T2_DBG_WN_GIN_WGRAD:
    case T2_DBG_WN_GIN_DEMB: {
      const char* what = call->kernel == T2_DBG_WN_GIN_WGRAD ? "GIN_WGRAD" : "GIN_DEMB";
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && p[4] && p[5], T2_ERR_INVALID_ARG, "dbg_wn_kernel %s: null pointer argument", what);
      int rc = dbg_gin_shape(i, what);
      if (rc) return rc;
      for (int k = 5; k < 9; ++k)
        T2_REQUIRE(in_range(i[k], 0, 1LL << 40), T2_ERR_INVALID_ARG, "dbg_wn_kernel %s: offsets must be in [0, 2^40] (i[%d])", what, k);
      GinGradArgs a;
      a.params = static_cast<const float*>(p[0]); a.spk = static_cast<const int*>(p[1]); a.S = static_cast<const long long*>(p[2]);
      a.gfx = static_cast<long long*>(p[3]); a.grads = static_cast<float*>(p[4]); a.offs = static_cast<const long long*>(p[5]);
      a.L = int(i[0]); a.B = int(i[1]); a.G = int(i[2]); a.Gi = int(i[3]); a.NS = int(i[4]);
      a.p_k = i[5]; a.p_b = i[6]; a.p_stride = i[7]; a.p_emb = i[8];
      if (call->kernel == T2_DBG_WN_GIN_WGRAD) launch_gin_wgrad(a, st);
      else launch_gin_demb(a, st);
      break;
    }
    default:
      return t2_set_error(T2_ERR_INVALID_ARG, "dbg_wn_kernel: unknown kernel id %d", call->kernel);
  }
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

// Times `reps` back-to-back launches of one per-layer GEMM of the residual stack with CUDA events on the launching
// stream: which = 0 gate (dilated conv + cin + tanh*sigmoid), 1 out 1x1 + residual, 2 dz + gate backward, 3 dx (data
// gradient of the dilated conv). The workspace must hold the state of a previous forward (+ backward). Synchronises.
extern "C" int t2_wn_time_kernel(const t2_wn_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                                 int which, int layer, int reps, float* ms_per_launch, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  T2_REQUIRE(layer >= 0 && layer < lo.L && reps >= 1 && ms_per_launch && which >= 0 && which <= 4, T2_ERR_INVALID_ARG,
             "time_kernel: bad arguments");
  T2_REQUIRE(which != 1 || layer + 1 < lo.L, T2_ERR_INVALID_ARG, "the last layer has no out GEMM");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  const uint8_t* pk = static_cast<const uint8_t*>(d_packed);
  ActGemmCall g;
  int epi, bn;
  if (which == 0 || which == 4) { g = make_gate_call(lo, ws, pk, layer, which == 0); epi = EPI_GATE; bn = 256; }   // 4: without the tanh / sigmoid stashes
  else if (which == 1) { g = make_out_call(lo, ws, pk, d_params, layer, cfg->dropout, 1, nullptr); epi = EPI_RES; bn = lo.R; }
  else if (which == 2) { g = make_dz_call(lo, ws, pk, layer, nullptr); epi = EPI_GATE_BWD; bn = lo.Gh >= 256 ? 256 : 128; }
  else { g = make_dx_call(lo, ws, pk, layer, cfg->dropout, 1, nullptr, nullptr); epi = EPI_DX; bn = lo.R; }
  // `reps` back-to-back launches captured into ONE CUDA graph on a private stream and replayed, so that the figure is the
  // device-side time per launch (as in the captured training step) and not the host's launch rate
  T2_CHECK_CUDA(cudaStreamSynchronize(st));
  cudaStream_t ps;
  T2_CHECK_CUDA(cudaStreamCreateWithFlags(&ps, cudaStreamNonBlocking));
  cudaEvent_t e0, e1;
  T2_CHECK_CUDA(cudaEventCreate(&e0));
  T2_CHECK_CUDA(cudaEventCreate(&e1));
  rc = launch_act_gemm(epi, bn, g, ps);  // warm-up (also sets the kernel attributes outside the capture)
  if (rc) return rc;
  T2_CHECK_CUDA(cudaStreamSynchronize(ps));
  cudaGraph_t graph;
  cudaGraphExec_t exec;
  T2_CHECK_CUDA(cudaStreamBeginCapture(ps, cudaStreamCaptureModeThreadLocal));
  for (int i = 0; i < reps && rc == 0; ++i) rc = launch_act_gemm(epi, bn, g, ps);
  cudaError_t ce = cudaStreamEndCapture(ps, &graph);
  if (rc) return rc;
  T2_CHECK_CUDA(ce);
  T2_CHECK_CUDA(cudaGraphInstantiate(&exec, graph, 0));
  T2_CHECK_CUDA(cudaGraphLaunch(exec, ps));   // warm replay
  T2_CHECK_CUDA(cudaEventRecord(e0, ps));
  T2_CHECK_CUDA(cudaGraphLaunch(exec, ps));
  T2_CHECK_CUDA(cudaEventRecord(e1, ps));
  T2_CHECK_CUDA(cudaEventSynchronize(e1));
  float ms = 0.f;
  T2_CHECK_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  *ms_per_launch = ms / reps;
  cudaGraphExecDestroy(exec);
  cudaGraphDestroy(graph);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaStreamDestroy(ps);
  return T2_OK;
}

// =========================================================================================================
// Fast-WaveNet autoregressive synthesis (wavenet_vocoder/models/wavenet.py:724-911, modules.py:273-303)
// =========================================================================================================
// One persistent kernel generates the whole utterance. A thread-block CLUSTER of CS CTAs owns `NI` batch items;
// every layer's output channels are split across the cluster's CTAs, bf16 weights stream from L2 (the 27.6 MB of
// the paper-width model stay L2-resident), activations live in shared memory as fp32 and are exchanged between
// CTAs through distributed shared memory + one cluster barrier per stage (2 per layer). The reference's
// convolution queues (O(d) concat shift per step, modules.py:285-288) become ring buffers in global memory.
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace t2 {
namespace {

constexpr int kArThreads = 512;
__device__ long long* g_ar_dbg = nullptr;   // tools only: clock64 stamps of (t = 64, l = 7) in CTA 0
#define AR_STAMP(i) do { if (g_ar_dbg && blockIdx.x == 0 && threadIdx.x == 0 && t == 64 && l == 7) g_ar_dbg[i] = clock64(); } while (0)
constexpr int kArMaxItems = 4;

struct ArLayout {
  int CS, ZC, RC, SC, FC, OC, K1;
  int esize;                       // bytes per stored weight: 2 (bf16), or 4 (fp32) in the fp32-class mode (split_bf16)
  long long per_rank_layer;        // weight elements per (layer, rank): 2*ZC*K1 + (RC+SC)*Gh
  long long o_head1, o_head2;      // element offsets of the head blocks (after all layers)
  long long n_weights;             // weight elements
  long long o_bias;                // byte offset of the fp32 bias block
  long long packed_bytes;
  long long ring_slots_total;      // sum over layers of slots
  long long workspace_bytes, w_cup, w_upout_base, w_ring, w_ringoff;   // w_cup: bf16 mode only (-1 in the fp32-class mode)
  long long w_gbias;               // Gi > 0: fp32 [B][L][G] per-item gate biases (t2_wn_ar_set_speakers), else -1
  std::vector<int> ring_slots, ring_off;
};

int build_ar_layout(const Layout& lo, int CS, ArLayout& a) {
  T2_REQUIRE(CS == 1 || CS == 2 || CS == 4 || CS == 8 || CS == 16, T2_ERR_INVALID_ARG, "cluster size must be 1,2,4,8,16");
  a.CS = CS;
  a.ZC = lo.Gh / CS; a.RC = lo.R / CS; a.SC = lo.S / CS; a.FC = lo.S / CS; a.OC = (lo.O + CS - 1) / CS;
  a.K1 = lo.kw * lo.R + lo.C;
  a.per_rank_layer = 2LL * a.ZC * a.K1 + (long long)(a.RC + a.SC) * lo.Gh;
  a.o_head1 = a.per_rank_layer * CS * lo.L;
  a.o_head2 = a.o_head1 + (long long)CS * a.FC * lo.S;
  a.n_weights = a.o_head2 + (long long)CS * a.OC * lo.S;
  a.esize = lo.split ? 4 : 2;
  a.o_bias = align_up(a.n_weights * a.esize, 256);
  // biases fp32: per layer [G gate | R out], then skip_total [S], f1 [S], f2 [O padded to CS*OC]
  a.packed_bytes = a.o_bias + 4LL * ((long long)lo.L * (lo.G + lo.R) + 2 * lo.S + CS * a.OC);
  a.ring_slots.clear(); a.ring_off.clear();
  long long off = 0;
  for (int l = 0; l < lo.L; ++l) {
    int need = (lo.kw - 1) * lo.dil(l) + 1, s = 1;   // x(t - (kw-1)d) .. x(t)
    while (s < need) s <<= 1;
    a.ring_slots.push_back(s);
    a.ring_off.push_back(int(off));
    off += s;
  }
  a.ring_slots_total = off;
  Arena ws;
  const long long BT = (long long)lo.B * lo.T;
  // the fp32-class mode reads the fp32 conditioning where it lies (d_c, or the last upsampling layer's output): no c_up copy
  a.w_cup = lo.split ? -1 : ws.take(BT * (lo.C > 0 ? lo.C : 8) * 2);
  a.w_upout_base = ws.used;
  for (size_t i = 0; i < lo.up_w.size(); ++i) ws.take((long long)lo.B * lo.C * lo.up_w[i] * 4);
  a.w_ring = ws.take((long long)lo.B * off * lo.R * 4);
  a.w_ringoff = ws.take(2LL * lo.L * 4);
  a.w_gbias = lo.Gi > 0 ? ws.take((long long)lo.B * lo.L * lo.G * 4) : -1;
  a.workspace_bytes = ws.used;
  return T2_OK;
}

struct ArPackArgs {
  const float* params;
  void* w;                 // WT (bf16, or fp32 in the fp32-class mode) [n_weights], slice-major
  float* bias;
  const long long* offs;   // per layer: dil_k, dil_b, c_k, c_b, s_k, s_b, o_k, o_b  (8 per layer); then f1_k,f1_b,f2_k,f2_b
  const float* skip_scale;
  int L, R, G, Gh, S, C, O, CS, ZC, RC, SC, FC, OC, K1;
  long long per_rank_layer, o_head1, o_head2, n_weights;
};
__device__ __forceinline__ void ar_store(bf16* p, float v) { *p = __float2bfloat16(v); }
__device__ __forceinline__ void ar_store(float* p, float v) { *p = v; }

template <typename WT>
__global__ void ar_pack_kernel(ArPackArgs a) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e < a.n_weights) {
    float v = 0.f;
    if (e < a.o_head1) {
      const int lr = int(e / a.per_rank_layer);
      const int l = lr / a.CS, r = lr % a.CS;
      long long i = e % a.per_rank_layer;
      const long long* o = a.offs + 8 * l;
      if (i < 2LL * a.ZC * a.K1) {
        const int row = int(i / a.K1), k = int(i % a.K1);
        const int ch = (row < a.ZC) ? r * a.ZC + row : a.Gh + r * a.ZC + (row - a.ZC);
        const int kR = a.K1 - a.C;   // kernel_size taps of R
        if (k < kR) v = a.params[o[0] + (long long)(k / a.R) * a.R * a.G + (long long)(k % a.R) * a.G + ch];
        else v = a.params[o[2] + (long long)(k - kR) * a.G + ch];
      } else {
        i -= 2LL * a.ZC * a.K1;
        const int row = int(i / a.Gh), k = int(i % a.Gh);
        if (row < a.RC) v = a.params[o[6] + (long long)k * a.R + r * a.RC + row];
        else v = a.params[o[4] + (long long)k * a.S + r * a.SC + (row - a.RC)] * a.skip_scale[l];
      }
    } else if (e < a.o_head2) {
      const long long i = e - a.o_head1;
      const int row = int(i / a.S), k = int(i % a.S);   // row = r*FC + j == output channel
      v = a.params[a.offs[8 * a.L + 0] + (long long)k * a.S + row];
    } else {
      const long long i = e - a.o_head2;
      const int row = int(i / a.S), k = int(i % a.S);
      if (row < a.O) v = a.params[a.offs[8 * a.L + 2] + (long long)k * a.O + row];
    }
    ar_store(static_cast<WT*>(a.w) + e, v);
  }
  // biases
  const long long nb = (long long)a.L * (a.G + a.R) + 2 * a.S + a.CS * a.OC;
  if (e < nb) {
    float v = 0.f;
    const long long lg = (long long)a.L * (a.G + a.R);
    if (e < lg) {
      const int l = int(e / (a.G + a.R)), j = int(e % (a.G + a.R));
      const long long* o = a.offs + 8 * l;
      if (j < a.G) v = a.params[o[1] + j] + (a.C > 0 ? a.params[o[3] + j] : 0.f);
      else v = a.params[o[7] + (j - a.G)];
    } else if (e < lg + a.S) {
      const int s = int(e - lg);
      for (int l = 0; l < a.L; ++l) v += a.skip_scale[l] * a.params[a.offs[8 * l + 5] + s];
    } else if (e < lg + 2 * a.S) {
      v = a.params[a.offs[8 * a.L + 1] + (e - lg - a.S)];
    } else {
      const int j = int(e - lg - 2 * a.S);
      if (j < a.O) v = a.params[a.offs[8 * a.L + 3] + j];
    }
    a.bias[e] = v;
  }
}

struct ArArgs {
  const void* w;            // slice-major weights, WT (bf16, or fp32 in the fp32-class mode)
  const float* bias;
  const float* gbias;       // nullable: per-item gate biases [B][L][G] replacing the shared gate rows of `bias` (speaker conditioning)
  const float* in_k;        // input_convolution kernel fp32 [cin][R]
  const float* in_b;
  const void* c_up;         // bf16 mode: bf16 [B][T][C]; fp32-class mode: fp32, element (b, t, ch) at b*c_sb + t*c_st + ch*c_sc
  float* ring;              // [B][ring_slots_total][R]
  const int* ring_off;      // [L] then ring_slots [L]
  const void* initial;      // int32 [B] or f32 [B]
  const void* test_inputs;  // nullable: int32 / f32 [B][T]
  const float* u_a;         // MoL: [B][T][nm] mixture-selection uniforms; categorical: [B][T]; nullable
  const float* u_b;         // MoL: [B][T] logistic uniforms; nullable
  void* out_samples;        // int32 / f32 [B][T]
  float* out_raw;           // nullable [B][T][O]
  unsigned long long seed;
  int B, T, L, R, G, Gh, S, C, O, Q, scalar_in, layers_per_stack;
  int CS, ZC, RC, SC, FC, OC, K1;
  long long per_rank_layer, o_head1, o_head2;
  float res_scale, log_scale_min, log_scale_min_gauss;
  int items_per_cluster;
  int prefetch;             // 1: this CTA's per-layer weight slice is double-buffered in shared memory (bulk async copies)
  long long c_sb, c_st, c_sc;   // fp32-class mode: element strides of the fp32 conditioning (item, time, channel)
};

// y[it][o] = sum_k W[o][k] * x[it][k] for o in [0, nout): all outputs of a pass run side by side - a group of GS lanes
// (GS = 512 / nout rounded down to a power of two, <= 32) owns one output row and strides its 16-byte chunks, the partial
// sums meet in log2(GS) shuffles. (The warp-per-output form serialised 2 rows x 5 shuffle levels x NI per warp.)
// WT: stored weight type; a 16-byte chunk holds 8 bf16 weights or 4 fp32 weights (the fp32-class mode: exact fp32 products).
template <int NI, typename WT>
__device__ __forceinline__ void ar_matvec(const WT* __restrict__ W, int nout, int K, const float* __restrict__ x /*[NI][ldx]*/,
                                          int ldx, float* __restrict__ y /*[NI][ldy]*/, int ldy, int ni) {
  int gs = 32;
  while (gs > 1 && gs * nout > kArThreads) gs >>= 1;
  const int per_pass = kArThreads / gs;
  const int sub = threadIdx.x % gs;
  if constexpr (sizeof(WT) == 4) {
    const int nchunk = K >> 2;
    for (int o0 = 0; o0 < nout; o0 += per_pass) {
      const int o = o0 + threadIdx.x / gs;
      const bool live = o < nout;
      float acc[NI];
#pragma unroll
      for (int it = 0; it < NI; ++it) acc[it] = 0.f;
      if (live) {
        const float4* wr = reinterpret_cast<const float4*>(W + (size_t)o * K);
#pragma unroll 2
        for (int c = sub; c < nchunk; c += gs) {
          const float4 w = wr[c];
#pragma unroll
          for (int it = 0; it < NI; ++it) {
            if (it < ni) {
              const float4 p = *reinterpret_cast<const float4*>(x + it * ldx + c * 4);
              acc[it] += w.x * p.x + w.y * p.y + w.z * p.z + w.w * p.w;
            }
          }
        }
      }
#pragma unroll
      for (int it = 0; it < NI; ++it) {
        if (it < ni) {
          float v = acc[it];
          for (int m = gs >> 1; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
          if (live && sub == 0) y[it * ldy + o] = v;
        }
      }
    }
    return;
  }
  const int nchunk = K >> 3;
  for (int o0 = 0; o0 < nout; o0 += per_pass) {
    const int o = o0 + threadIdx.x / gs;
    const bool live = o < nout;
    float acc[NI];
#pragma unroll
    for (int it = 0; it < NI; ++it) acc[it] = 0.f;
    if (live) {
      const uint4* wr = reinterpret_cast<const uint4*>(W + (size_t)o * K);
#pragma unroll 2
      for (int c = sub; c < nchunk; c += gs) {
        const uint4 u = wr[c];          // generic load: the slice is either in L2 (global) or prefetched into shared memory
        const float w0 = bf16lo(u.x), w1 = bf16hi(u.x), w2 = bf16lo(u.y), w3 = bf16hi(u.y);
        const float w4 = bf16lo(u.z), w5 = bf16hi(u.z), w6 = bf16lo(u.w), w7 = bf16hi(u.w);
#pragma unroll
        for (int it = 0; it < NI; ++it) {
          if (it < ni) {
            const float4 p = *reinterpret_cast<const float4*>(x + it * ldx + c * 8);
            const float4 q = *reinterpret_cast<const float4*>(x + it * ldx + c * 8 + 4);
            acc[it] += w0 * p.x + w1 * p.y + w2 * p.z + w3 * p.w + w4 * q.x + w5 * q.y + w6 * q.z + w7 * q.w;
          }
        }
      }
    }
#pragma unroll
    for (int it = 0; it < NI; ++it) {
      if (it < ni) {      // block-uniform
        float v = acc[it];
        for (int m = gs >> 1; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
        if (live && sub == 0) y[it * ldy + o] = v;
      }
    }
  }
}

// NT: past taps of the dilated convolution (kernel_size - 1), read from the ring; the last tap is the current x.
// WT: stored weight type, bf16 or fp32 (the fp32-class mode, which also reads its conditioning in fp32).
template <int NI, int NT, typename WT>
__global__ void __launch_bounds__(kArThreads, 1) wn_ar_kernel(ArArgs a) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = int(cluster.block_rank());
  const int cid = blockIdx.x / a.CS;
  const int item0 = cid * a.items_per_cluster;
  int ni = a.B - item0;
  if (ni > a.items_per_cluster) ni = a.items_per_cluster;
  if (ni < 0) ni = 0;   // surplus clusters still take part in no barriers of other clusters; they just idle through
  extern __shared__ __align__(16) float sm[];
  const int ld1 = (a.K1 + 3) & ~3;
  const int nbs = 2 * a.ZC + a.RC;                  // bias slice per layer: a rows | b rows | residual-out rows
  float* in1 = sm;                                  // [NI][ld1]  : x(t-NT*d) | ... | x(t-d) | x(t) | c(t)
  float* zbuf = in1 + NI * ld1;                     // [NI][Gh]   : full z vector (pulled from the cluster)
  float* xbuf = zbuf + NI * a.Gh;                   // [NI][R]    : current layer input (full vector)
  float* zsl = xbuf + NI * a.R;                     // [NI][ZC]   : this CTA's z slice, read remotely by the cluster
  float* xsl = zsl + NI * a.ZC;                     // [NI][RC]   : this CTA's slice of the next layer input, read remotely
  float* loc = xsl + NI * a.RC;                     // [NI][2*ZC] : this CTA's gate pre-activations / stage-2 outputs
  float* skip = loc + NI * (2 * a.ZC > a.RC + a.SC ? 2 * a.ZC : a.RC + a.SC);   // [NI][SC] running skip sum (slice)
  float* hbuf = skip + NI * a.SC;                   // [NI][S]    : head activations (full vector)
  float* obuf = hbuf + NI * a.S;                    // [NI][CS*OC]: network output (full vector)
  float* bsl = obuf + NI * a.CS * a.OC;             // [L][nbs]   : this CTA's bias slices (cluster.sync flushes L1: keep them here)
  float* cvec = bsl + a.L * nbs;                    // [NI][C]    : conditioning frame of the current step
  int* rofs = reinterpret_cast<int*>(cvec + NI * ((a.C + 3) & ~3));   // [2L+1] ring offsets / slots / total
  float* cur = reinterpret_cast<float*>(rofs + ((2 * a.L + 1 + 3) & ~3));   // [NI] current input sample (scalar) or index
  // weight prefetch: two slots of per_rank_layer WT + two mbarriers behind the activation buffers (16-byte aligned)
  uint64_t* wbar = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(cur + NI) + 15) & ~uintptr_t(15));
  WT* wslot = reinterpret_cast<WT*>(wbar + 2);
  const uint32_t wbytes = uint32_t(a.per_rank_layer * (long long)sizeof(WT));
  const int tid = threadIdx.x;
  if (a.prefetch && tid == 0) {
    mbar_init(&wbar[0], 1); mbar_init(&wbar[1], 1);
    fence_barrier_init();
  }
  const float* bias_all = a.bias;
  const float* b_skip = bias_all + (long long)a.L * (a.G + a.R);
  const float* b_f1 = b_skip + a.S;
  const float* b_f2 = b_f1 + a.S;
  const int nm = a.O / 3;

  for (int i = tid; i < a.L * nbs; i += kArThreads) {
    const int l = i / nbs, j = i % nbs;
    const float* bgl = bias_all + (long long)l * (a.G + a.R);
    bsl[i] = j < a.ZC ? bgl[rank * a.ZC + j] : (j < 2 * a.ZC ? bgl[a.Gh + rank * a.ZC + (j - a.ZC)] : bgl[a.G + rank * a.RC + (j - 2 * a.ZC)]);
  }
  for (int i = tid; i < 2 * a.L + 1; i += kArThreads) rofs[i] = a.ring_off[i];
  for (int i = tid; i < NI; i += kArThreads)
    if (i < ni) cur[i] = a.scalar_in ? static_cast<const float*>(a.initial)[item0 + i]
                                     : float(static_cast<const int*>(a.initial)[item0 + i]);
  __syncthreads();
  if (a.prefetch && tid == 0) {   // slice of layer 0 -> slot 0
    mbar_expect_tx(&wbar[0], wbytes);
    bulk_load_1d(wslot, static_cast<const WT*>(a.w) + (long long)rank * a.per_rank_layer, wbytes, &wbar[0]);
  }
  uint32_t wphase = 0;            // bit s = parity to wait for on slot s
  long long seq = 0;              // (t, l) sequence number: slot = seq & 1
  // ring taps of the NEXT layer are fetched into registers one layer ahead (their producers ran >= one time step ago)
  constexpr int kTapRegs = (NI * NT * 512 + kArThreads - 1) / kArThreads;   // R <= 512
  float tapv[kTapRegs];
  auto fetch_taps = [&](int tt0, int l) {
    const int d = 1 << (l % a.layers_per_stack);
    const int slots = rofs[a.L + l];
    const long long roff = rofs[l];
#pragma unroll
    for (int j = 0; j < kTapRegs; ++j) {
      const int i = tid + j * kArThreads;
      float v = 0.f;
      if (i < ni * NT * a.R) {
        const int it = i / (NT * a.R), k = i % (NT * a.R);
        const int tap = k / a.R, r = k % a.R;
        const int tt = tt0 - (NT - tap) * d;
        if (tt >= 0) v = __ldcg(a.ring + ((long long)(item0 + it) * rofs[2 * a.L] + roff + (tt & (slots - 1))) * a.R + r);
      }
      tapv[j] = v;
    }
  };
  fetch_taps(0, 0);

  for (int t = 0; t < a.T; ++t) {
    // ---- first conv: x0 = W_in[idx] + b (one-hot) or x * w + b (scalar); every CTA builds the full vector ----
    for (int i = tid; i < ni * a.R; i += kArThreads) {
      const int it = i / a.R, r = i % a.R;
      float v;
      if (a.scalar_in) v = cur[it] * a.in_k[r] + a.in_b[r];
      else v = a.in_k[(long long)int(cur[it]) * a.R + r] + a.in_b[r];
      xbuf[it * a.R + r] = v;
    }
    for (int i = tid; i < ni * a.SC; i += kArThreads) skip[i] = 0.f;
    for (int i = tid; i < ni * a.C; i += kArThreads) {   // conditioning frame of this step, once (not once per layer)
      if constexpr (sizeof(WT) == 4)
        cvec[(i / a.C) * ((a.C + 3) & ~3) + i % a.C] =
            static_cast<const float*>(a.c_up)[(item0 + i / a.C) * a.c_sb + t * a.c_st + (i % a.C) * a.c_sc];
      else
        cvec[(i / a.C) * ((a.C + 3) & ~3) + i % a.C] =
            __bfloat162float(static_cast<const bf16*>(a.c_up)[((long long)(item0 + i / a.C) * a.T + t) * a.C + i % a.C]);
    }
    __syncthreads();
    for (int l = 0; l < a.L; ++l) {
      const int slots = rofs[a.L + l];
      const long long roff = rofs[l];
      AR_STAMP(0);
      // ---- gather the stage-1 input: taps (prefetched registers), current x, conditioning ----
#pragma unroll
      for (int j = 0; j < kTapRegs; ++j) {
        const int i = tid + j * kArThreads;
        if (i < ni * NT * a.R) in1[(i / (NT * a.R)) * ld1 + i % (NT * a.R)] = tapv[j];
      }
      for (int i = tid; i < ni * (ld1 - NT * a.R); i += kArThreads) {
        const int it = i / (ld1 - NT * a.R), k = NT * a.R + i % (ld1 - NT * a.R);
        float v = 0.f;
        if (k < (NT + 1) * a.R) v = xbuf[it * a.R + (k - NT * a.R)];
        else if (k < a.K1) v = cvec[it * ((a.C + 3) & ~3) + (k - (NT + 1) * a.R)];
        in1[it * ld1 + k] = v;
      }
      __syncthreads();
      AR_STAMP(1);
      // rank 0 publishes x_l(t) into the ring for later steps (read back no earlier than step t + d)
      if (rank == 0)
        for (int i = tid; i < ni * a.R; i += kArThreads) {
          const int it = i / a.R, r = i % a.R;
          a.ring[((long long)(item0 + it) * rofs[2 * a.L] + roff + (t & (slots - 1))) * a.R + r] = xbuf[i];
        }
      // ---- stage 1: gate pre-activations for this CTA's ZC z-channels (a rows then b rows) ----
      const WT* w1 = static_cast<const WT*>(a.w) + ((long long)l * a.CS + rank) * a.per_rank_layer;
      if (a.prefetch) {
        const int slot = int(seq & 1);
        mbar_wait(&wbar[slot], (wphase >> slot) & 1u);       // this layer's slice has landed
        wphase ^= 1u << slot;
        w1 = wslot + (long long)slot * a.per_rank_layer;
        if (tid == 0 && (t + 1 < a.T || l + 1 < a.L)) {      // next layer's slice -> the other slot (free since the last cluster.sync)
          const int ln = l + 1 < a.L ? l + 1 : 0;
          mbar_expect_tx(&wbar[slot ^ 1], wbytes);
          bulk_load_1d(wslot + (long long)(slot ^ 1) * a.per_rank_layer, static_cast<const WT*>(a.w) + ((long long)ln * a.CS + rank) * a.per_rank_layer, wbytes,
                       &wbar[slot ^ 1]);
        }
      }
      ++seq;
      AR_STAMP(2);
      ar_matvec<NI>(w1, 2 * a.ZC, a.K1, in1, ld1, loc, 2 * a.ZC, ni);
      __syncthreads();
      AR_STAMP(3);
      // taps of the next layer (or of layer 0 at the next time step): issued now, consumed after two cluster barriers
      if (l + 1 < a.L) fetch_taps(t, l + 1);
      else if (t + 1 < a.T) fetch_taps(t + 1, 0);
      const float* bg = bsl + l * nbs;
      for (int i = tid; i < ni * a.ZC; i += kArThreads) {
        const int it = i / a.ZC, j = i % a.ZC;
        float ba = bg[j], bb = bg[a.ZC + j];
        if (a.gbias) {
          const float* gb = a.gbias + ((long long)(item0 + it) * a.L + l) * a.G + rank * a.ZC + j;
          ba = __ldg(gb);
          bb = __ldg(gb + a.Gh);
        }
        const float av = loc[it * 2 * a.ZC + j] + ba;
        const float bv = loc[it * 2 * a.ZC + a.ZC + j] + bb;
        zsl[it * a.ZC + j] = tanhf_(av) * sigmoidf_(bv);      // local slice; the cluster PULLS it after the barrier
      }
      AR_STAMP(4);
      cluster.sync();
      AR_STAMP(5);
      // pull the full z vector: 16-byte pieces from the owners' slices through distributed shared memory
      for (int i = tid; i < ni * (a.Gh >> 2); i += kArThreads) {
        const int it = i / (a.Gh >> 2), ch = (i % (a.Gh >> 2)) << 2;
        const int r = ch / a.ZC, j = ch % a.ZC;
        *reinterpret_cast<float4*>(zbuf + it * a.Gh + ch) = *reinterpret_cast<const float4*>(cluster.map_shared_rank(zsl, r) + it * a.ZC + j);
      }
      __syncthreads();
      // ---- stage 2: this CTA's RC residual-out channels and SC skip channels ----
      const WT* w2 = w1 + 2LL * a.ZC * a.K1;
      ar_matvec<NI>(w2, a.RC + a.SC, a.Gh, zbuf, a.Gh, loc, a.RC + a.SC, ni);
      __syncthreads();
      AR_STAMP(6);
      for (int i = tid; i < ni * (a.RC + a.SC); i += kArThreads) {
        const int it = i / (a.RC + a.SC), j = i % (a.RC + a.SC);
        const float v = loc[it * (a.RC + a.SC) + j];
        if (j < a.RC) xsl[it * a.RC + j] = (v + bg[2 * a.ZC + j] + xbuf[it * a.R + rank * a.RC + j]) * a.res_scale;
        else skip[it * a.SC + (j - a.RC)] += v;   // scale_l folded into the packed skip weights
      }
      AR_STAMP(7);
      cluster.sync();
      AR_STAMP(8);
      if (l + 1 < a.L) {
        for (int i = tid; i < ni * (a.R >> 2); i += kArThreads) {
          const int it = i / (a.R >> 2), ch = (i % (a.R >> 2)) << 2;
          const int r = ch / a.RC, j = ch % a.RC;
          *reinterpret_cast<float4*>(xbuf + it * a.R + ch) = *reinterpret_cast<const float4*>(cluster.map_shared_rank(xsl, r) + it * a.RC + j);
        }
        __syncthreads();
      }
      AR_STAMP(9);
    }
    // ---- head: relu(skips + b) -> f1 -> relu -> f2 ----
    for (int i = tid; i < ni * a.SC; i += kArThreads) {
      const int it = i / a.SC, j = i % a.SC, ch = rank * a.SC + j;
      const float v = fmaxf(skip[i] + b_skip[ch], 0.f);
      for (int r = 0; r < a.CS; ++r) cluster.map_shared_rank(hbuf, r)[it * a.S + ch] = v;
    }
    cluster.sync();
    ar_matvec<NI>(static_cast<const WT*>(a.w) + a.o_head1 + (long long)rank * a.FC * a.S, a.FC, a.S, hbuf, a.S, loc, a.FC, ni);
    __syncthreads();
    cluster.sync();   // every CTA has finished reading hbuf (h1) before it is overwritten with h2
    for (int i = tid; i < ni * a.FC; i += kArThreads) {
      const int it = i / a.FC, j = i % a.FC, ch = rank * a.FC + j;
      const float v = fmaxf(loc[it * a.FC + j] + b_f1[ch], 0.f);
      for (int r = 0; r < a.CS; ++r) cluster.map_shared_rank(hbuf, r)[it * a.S + ch] = v;
    }
    cluster.sync();
    ar_matvec<NI>(static_cast<const WT*>(a.w) + a.o_head2 + (long long)rank * a.OC * a.S, a.OC, a.S, hbuf, a.S, loc, a.OC, ni);
    __syncthreads();
    for (int i = tid; i < ni * a.OC; i += kArThreads) {
      const int it = i / a.OC, j = i % a.OC, ch = rank * a.OC + j;
      const float v = loc[it * a.OC + j] + b_f2[ch];
      for (int r = 0; r < a.CS; ++r) cluster.map_shared_rank(obuf, r)[it * a.CS * a.OC + ch] = v;
    }
    cluster.sync();
    // ---- sample (identically in every CTA: same inputs, same uniforms) ----
    if (tid < 32 * NI) {
      const int it = tid >> 5, lane = tid & 31;
      if (it < ni) {
        const int bi = item0 + it;
        const float* y = obuf + it * a.CS * a.OC;
        if (rank == 0 && a.out_raw)
          for (int j = lane; j < a.O; j += 32) a.out_raw[((long long)bi * a.T + t) * a.O + j] = y[j];
        float nxt;
        if (a.scalar_in && a.O == 2) {
          // sample_from_gaussian (gaussian.py:39-52): x = mean + exp(max(log_scale, min)) * n, clipped to [-1, 1]; the standard-normal
          // draw n is injected through u_b or made by Box-Muller from two counter-hash uniforms
          float n;
          if (a.u_b) n = a.u_b[(long long)bi * a.T + t];
          else {
            const float u1 = 1e-7f + (1.f - 2e-7f) * hash_uniform(a.seed, ((unsigned long long)bi * a.T + t) * 16 + 14);
            const float u2 = hash_uniform(a.seed, ((unsigned long long)bi * a.T + t) * 16 + 15);
            n = sqrtf(-2.f * __logf(u1)) * __cosf(6.28318530718f * u2);
          }
          const float x = y[0] + __expf(fmaxf(y[1], a.log_scale_min_gauss)) * n;
          nxt = fminf(fmaxf(x, -1.f), 1.f);
          if (rank == 0 && lane == 0) static_cast<float*>(a.out_samples)[(long long)bi * a.T + t] = nxt;
        } else if (a.scalar_in) {
          // sample_from_discretized_mix_logistic (mixture.py:76-107): Gumbel-max over the mixture logits
          float best = -INFINITY;
          int bk = 0;
          for (int k = 0; k < nm; ++k) {
            float u = a.u_a ? a.u_a[((long long)bi * a.T + t) * nm + k]
                            : 1e-5f + (1.f - 2e-5f) * hash_uniform(a.seed, ((unsigned long long)bi * a.T + t) * 16 + k);
            const float g = y[k] - __logf(-__logf(u));
            if (g > best) { best = g; bk = k; }
          }
          const float mean = y[nm + bk];
          const float ls = fmaxf(y[2 * nm + bk], a.log_scale_min);
          const float u = a.u_b ? a.u_b[(long long)bi * a.T + t]
                                : 1e-5f + (1.f - 2e-5f) * hash_uniform(a.seed, ((unsigned long long)bi * a.T + t) * 16 + 15);
          float x = mean + __expf(ls) * (__logf(u) - __logf(1.f - u));
          nxt = fminf(fmaxf(x, -1.f), 1.f);
          if (rank == 0 && lane == 0) static_cast<float*>(a.out_samples)[(long long)bi * a.T + t] = nxt;
        } else {
          // categorical sample from softmax(logits) by inverse CDF (tf.multinomial on raw logits, wavenet.py:865)
          float mx = -INFINITY;
          for (int j = lane; j < a.O; j += 32) mx = fmaxf(mx, y[j]);
          mx = warp_max(mx);
          float se = 0.f;
          for (int j = lane; j < a.O; j += 32) se += __expf(y[j] - mx);
          se = warp_sum(se);
          const float u = (a.u_a ? a.u_a[(long long)bi * a.T + t]
                                 : hash_uniform(a.seed, (unsigned long long)bi * a.T + t)) * se;
          // lane-blocked scan: each lane owns O/32 consecutive classes
          const int per = (a.O + 31) / 32;
          float part = 0.f;
          for (int j = lane * per; j < (lane + 1) * per && j < a.O; ++j) part += __expf(y[j] - mx);
          float incl = part;
          for (int o = 1; o < 32; o <<= 1) {
            const float nb = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += nb;
          }
          const float excl = incl - part;
          int pick = -1;
          if (u >= excl && u < incl) {
            float c = excl;
            pick = lane * per;
            for (int j = lane * per; j < (lane + 1) * per && j < a.O; ++j) { c += __expf(y[j] - mx); pick = j; if (c > u) break; }
          }
          pick = __reduce_max_sync(0xffffffffu, pick);
          if (pick < 0) pick = a.O - 1;
          nxt = float(pick);
          if (rank == 0 && lane == 0) static_cast<int*>(a.out_samples)[(long long)bi * a.T + t] = pick;
        }
        if (a.test_inputs)
          nxt = a.scalar_in ? static_cast<const float*>(a.test_inputs)[(long long)bi * a.T + t]
                            : float(static_cast<const int*>(a.test_inputs)[(long long)bi * a.T + t]);
        if (lane == 0) cur[it] = nxt;
      }
    }
    __syncthreads();
  }
}

// the instantiation for NIt items per cluster pass, NT past taps and stored weight type WT
template <int NT, typename WT>
void (*ar_kernel(int NIt))(ArArgs) {
  return NIt == 1 ? wn_ar_kernel<1, NT, WT> : (NIt == 2 ? wn_ar_kernel<2, NT, WT> : wn_ar_kernel<kArMaxItems, NT, WT>);
}
template <typename WT>
void (*ar_kernel_kw(int kw, int NIt))(ArArgs) {
  return kw == 2 ? ar_kernel<1, WT>(NIt) : kw == 3 ? ar_kernel<2, WT>(NIt) : ar_kernel<3, WT>(NIt);
}

}  // namespace
}  // namespace t2

typedef struct {
  long long packed_bytes, workspace_bytes;
} t2_wn_ar_sizes_t_;

// tools only: device buffer of 16 int64 receiving clock64() stamps of one AR layer pass (NULL = off)
extern "C" int t2_dbg_ar_stamps(long long* d_buf) {
  T2_CHECK_CUDA(cudaMemcpyToSymbol(t2::g_ar_dbg, &d_buf, sizeof(d_buf)));
  return T2_OK;
}

extern "C" int t2_wn_ar_sizes(const t2_wn_config_t* cfg, int cluster_size, long long* packed_bytes, long long* workspace_bytes) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  ArLayout a;
  rc = build_ar_layout(lo, cluster_size, a);
  if (rc) return rc;
  T2_REQUIRE(lo.Gh % cluster_size == 0 && lo.R % cluster_size == 0 && lo.S % cluster_size == 0 && lo.R <= lo.S + 0,
             T2_ERR_UNSUPPORTED_SHAPE, "channel counts must divide by the cluster size and R <= S");
  *packed_bytes = a.packed_bytes;
  *workspace_bytes = a.workspace_bytes;
  return T2_OK;
}

extern "C" int t2_wn_ar_pack(const t2_wn_config_t* cfg, int cluster_size, const float* d_params, void* d_packed_ar,
                             void* d_workspace, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  ArLayout a;
  rc = build_ar_layout(lo, cluster_size, a);
  if (rc) return rc;
  T2_REQUIRE(d_params && d_packed_ar && d_workspace, T2_ERR_INVALID_ARG, "t2_wn_ar_pack: null buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<long long> offs(8 * lo.L + 4);
  for (int l = 0; l < lo.L; ++l) {
    long long* o = &offs[8 * l];
    o[0] = lo.p_dil_k[l]; o[1] = lo.p_dil_b[l]; o[2] = lo.C > 0 ? lo.p_c_k[l] : 0; o[3] = lo.C > 0 ? lo.p_c_b[l] : 0;
    o[4] = lo.p_s_k[l]; o[5] = lo.p_s_b[l]; o[6] = lo.p_o_k[l]; o[7] = lo.p_o_b[l];
  }
  offs[8 * lo.L] = lo.p_f1_k; offs[8 * lo.L + 1] = lo.p_f1_b; offs[8 * lo.L + 2] = lo.p_f2_k; offs[8 * lo.L + 3] = lo.p_f2_b;
  // tables go through a temporary device allocation (this entry point synchronises; it runs once per checkpoint)
  long long* d_offs = nullptr;
  float* d_scale = nullptr;
  T2_CHECK_CUDA(cudaMallocAsync(&d_offs, offs.size() * sizeof(long long), st));
  T2_CHECK_CUDA(cudaMallocAsync(&d_scale, lo.L * sizeof(float), st));
  T2_CHECK_CUDA(cudaMemcpyAsync(d_offs, offs.data(), offs.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
  T2_CHECK_CUDA(cudaMemcpyAsync(d_scale, lo.skip_scale.data(), lo.L * sizeof(float), cudaMemcpyHostToDevice, st));
  ArPackArgs p;
  p.params = d_params; p.w = d_packed_ar;
  p.bias = reinterpret_cast<float*>(static_cast<uint8_t*>(d_packed_ar) + a.o_bias);
  p.offs = d_offs; p.skip_scale = d_scale;
  p.L = lo.L; p.R = lo.R; p.G = lo.G; p.Gh = lo.Gh; p.S = lo.S; p.C = lo.C; p.O = lo.O; p.CS = a.CS; p.ZC = a.ZC; p.RC = a.RC;
  p.SC = a.SC; p.FC = a.FC; p.OC = a.OC; p.K1 = a.K1; p.per_rank_layer = a.per_rank_layer; p.o_head1 = a.o_head1;
  p.o_head2 = a.o_head2; p.n_weights = a.n_weights;
  if (lo.split) ar_pack_kernel<float><<<grid1d(a.n_weights), 256, 0, st>>>(p);
  else ar_pack_kernel<bf16><<<grid1d(a.n_weights), 256, 0, st>>>(p);
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  // ring tables
  std::vector<int> rt(2 * lo.L + 1);
  for (int l = 0; l < lo.L; ++l) { rt[l] = a.ring_off[l]; rt[lo.L + l] = a.ring_slots[l]; }
  rt[2 * lo.L] = int(a.ring_slots_total);
  T2_CHECK_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(d_workspace) + a.w_ringoff, rt.data(), rt.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  if (lo.Gi > 0) {   // per-item gate biases start without a speaker term
    rc = t2_wn_ar_set_speakers(cfg, cluster_size, d_params, d_packed_ar, d_workspace, nullptr, stream);
    if (rc) return rc;
  }
  T2_CHECK_CUDA(cudaStreamSynchronize(st));
  cudaFreeAsync(d_offs, st);
  cudaFreeAsync(d_scale, st);
  return T2_OK;
}

extern "C" int t2_wn_ar_set_speakers(const t2_wn_config_t* cfg, int cluster_size, const float* d_params, const void* d_packed_ar,
                                     void* d_workspace, const int* d_speaker_ids, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  ArLayout al;
  rc = build_ar_layout(lo, cluster_size, al);
  if (rc) return rc;
  T2_REQUIRE(lo.Gi > 0, T2_ERR_INVALID_ARG, "speaker ids need gin_channels > 0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GinArgs a = gin_args(lo, d_params);
  a.bias = reinterpret_cast<const float*>(static_cast<const uint8_t*>(d_packed_ar) + al.o_bias); a.bias_ld = lo.G + lo.R;
  a.on = nullptr; a.ids = d_speaker_ids;
  a.out = reinterpret_cast<float*>(static_cast<uint8_t*>(d_workspace) + al.w_gbias); a.out_l = lo.G; a.out_b = (long long)lo.L * lo.G;
  launch_gin_bias(a, st);
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

extern "C" int t2_wn_ar_generate(const t2_wn_config_t* cfg, int cluster_size, const float* d_params, const void* d_packed_ar,
                                 void* d_workspace, const float* d_c, const void* d_initial, const void* d_test_inputs,
                                 const float* d_u_a, const float* d_u_b, unsigned long long seed, void* d_out_samples,
                                 float* d_out_raw, void* stream) {
  Layout lo;
  int rc = build_layout(cfg, lo);
  if (rc) return rc;
  ArLayout al;
  rc = build_ar_layout(lo, cluster_size, al);
  if (rc) return rc;
  T2_REQUIRE(lo.C > 0, T2_ERR_UNSUPPORTED_SHAPE, "AR synthesis needs local conditioning");
  T2_REQUIRE(lo.R <= lo.S, T2_ERR_UNSUPPORTED_SHAPE, "AR synthesis needs residual_channels <= skip_out_channels");
  T2_REQUIRE(d_params && d_packed_ar && d_workspace && d_c && d_initial && d_out_samples, T2_ERR_INVALID_ARG,
             "t2_wn_ar_generate: null buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  const uint8_t* pk = static_cast<const uint8_t*>(d_packed_ar);
  const long long BT = (long long)lo.B * lo.T;
  // conditioning -> c_up (bf16 channels-last), same kernels as the training path. The fp32-class mode reads the fp32 conditioning
  // in place instead: d_c [B][T][C] when pre-upsampled, else the last upsampling layer's output [B][C][T]
  bf16* c_up = lo.split ? nullptr : reinterpret_cast<bf16*>(ws + al.w_cup);
  const float* c32 = d_c;
  if (cfg->c_pre_upsampled) {
    if (!lo.split) launch_f32_to_bf16(d_c, c_up, BT * lo.C, st);
  } else {
    const float* in = d_c;
    int W = lo.Tc;
    long long o = al.w_upout_base;
    for (size_t i = 0; i < lo.up_w.size(); ++i) {
      const int s = cfg->upsample_scales[i];
      float* out = reinterpret_cast<float*>(ws + o);
      o = align_up(o + (long long)lo.B * lo.C * lo.up_w[i] * 4, 256);
      const bool last = i + 1 == lo.up_w.size();
      rc = launch_upsample_fwd(in, d_params + lo.p_up_k[i], d_params + lo.p_up_b[i], out, last ? c_up : nullptr, lo.B, lo.C, W, s,
                               cfg->upsample_type, cfg->upsample_activation, cfg->leaky_alpha, 0, st);
      if (rc) return rc;
      in = out;
      W *= s;
    }
    c32 = in;
  }
  T2_CHECK_CUDA(cudaGetLastError());
  ArArgs a;
  memset(&a, 0, sizeof(a));
  a.w = pk;
  a.bias = reinterpret_cast<const float*>(pk + al.o_bias);
  a.gbias = lo.Gi > 0 ? reinterpret_cast<const float*>(ws + al.w_gbias) : nullptr;
  a.in_k = d_params + lo.p_in_k; a.in_b = d_params + lo.p_in_b;
  if (lo.split) {
    a.c_up = c32;
    const bool cl = cfg->c_pre_upsampled != 0;
    a.c_sb = (long long)lo.T * lo.C; a.c_st = cl ? lo.C : 1; a.c_sc = cl ? 1 : lo.T;
  } else {
    a.c_up = c_up;
  }
  a.ring = reinterpret_cast<float*>(ws + al.w_ring);
  a.ring_off = reinterpret_cast<const int*>(ws + al.w_ringoff);
  a.initial = d_initial; a.test_inputs = d_test_inputs; a.u_a = d_u_a; a.u_b = d_u_b;
  a.out_samples = d_out_samples; a.out_raw = d_out_raw; a.seed = seed;
  a.B = lo.B; a.T = lo.T; a.L = lo.L; a.R = lo.R; a.G = lo.G; a.Gh = lo.Gh; a.S = lo.S; a.C = lo.C; a.O = lo.O; a.Q = lo.Q;
  a.scalar_in = lo.scalar_in ? 1 : 0; a.layers_per_stack = lo.L / cfg->stacks;
  a.CS = al.CS; a.ZC = al.ZC; a.RC = al.RC; a.SC = al.SC; a.FC = al.FC; a.OC = al.OC; a.K1 = al.K1;
  a.per_rank_layer = al.per_rank_layer; a.o_head1 = al.o_head1; a.o_head2 = al.o_head2;
  a.res_scale = lo.res_scale; a.log_scale_min = cfg->log_scale_min; a.log_scale_min_gauss = cfg->log_scale_min_gauss;
  // clusters: as many as fit on the device, but never more than batch items
  int dev = 0, sms = 148;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int n_clusters = sms / al.CS;
  if (n_clusters > lo.B) n_clusters = lo.B;
  if (n_clusters < 1) n_clusters = 1;
  int ipc = (lo.B + n_clusters - 1) / n_clusters;
  while (ipc > kArMaxItems) { ++n_clusters; ipc = (lo.B + n_clusters - 1) / n_clusters; }  // more clusters than fit run in waves
  n_clusters = (lo.B + ipc - 1) / ipc;
  a.items_per_cluster = ipc;
  const int ld1 = (al.K1 + 3) & ~3;
  const int locw = 2 * al.ZC > al.RC + al.SC ? 2 * al.ZC : al.RC + al.SC;
  T2_REQUIRE(al.ZC % 4 == 0 && al.RC % 4 == 0, T2_ERR_UNSUPPORTED_SHAPE, "AR synthesis: channel slices per CTA must be multiples of 4");
  const int NIt = ipc <= 1 ? 1 : (ipc <= 2 ? 2 : kArMaxItems);     // kernel instantiation: items per cluster pass
  size_t smem = sizeof(float) * (size_t(NIt) * (ld1 + lo.Gh + lo.R + al.ZC + al.RC + locw + al.SC + lo.S + al.CS * al.OC + ((lo.C + 3) & ~3) + 1) +
                                 size_t(lo.L) * (2 * al.ZC + al.RC) + ((2 * lo.L + 1 + 3) & ~3)) + 64;
  // double-buffered shared-memory copy of this CTA's per-layer weight slice when it fits next to the activations
  // (paper widths at cluster size 16: 70.6 KB per bf16 slice; the fp32 slices, 141 KB, do not fit twice); otherwise the slices
  // stream from L2 as before
  const size_t wslots = 2 * size_t(al.per_rank_layer) * al.esize + 64;
  a.prefetch = ((al.per_rank_layer * al.esize) % 16 == 0 && smem + wslots <= 232448 - 1024) ? 1 : 0;
  if (const char* e = getenv("T2_AR_PREFETCH")) { if (e[0] == '0') a.prefetch = 0; }
  if (a.prefetch) smem += wslots;
  void (*kern)(ArArgs) = lo.split ? ar_kernel_kw<float>(lo.kw, NIt) : ar_kernel_kw<bf16>(lo.kw, NIt);
  T2_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  if (al.CS > 8) T2_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  T2_CHECK_CUDA(cudaMemsetAsync(ws + al.w_ring, 0, (size_t)lo.B * al.ring_slots_total * lo.R * 4, st));
  cudaLaunchConfig_t lc;
  memset(&lc, 0, sizeof(lc));
  lc.gridDim = dim3(n_clusters * al.CS);
  lc.blockDim = dim3(kArThreads);
  lc.dynamicSmemBytes = smem;
  lc.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = al.CS; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  lc.attrs = at; lc.numAttrs = 1;
  T2_CHECK_CUDA(cudaLaunchKernelEx(&lc, kern, a));
  t2_count_launch();
  return T2_OK;
}
