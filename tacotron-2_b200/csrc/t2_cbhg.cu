// t2_cbhg.cu — the CBHG post-processing network + linear-spectrogram head of the Tacotron graph (predict_linear = True,
// the reference's DEFAULT: hparams.py:175).
//
// Replaces tacotron/models/tacotron.py:203-219 (CBHG_postnet -> cbhg_linear_specs_projection -> clip), :323-330 (linear loss) and
// tacotron/models/modules.py:4-16 (HighwayNet), :19-78 (CBHG), :457-485 (MaskedLinearLoss). Forward and backward.
//
// Dataflow (rows = b * T + t, batch-major; N = B * T):
//   mel_outputs fp32 [N][M] -> bf16
//   conv bank: k = 1..K convolutions M -> CC ('same' padding, the extra pad of an even kernel on the right) + bias + ReLU, each one a
//     tap-shifted GEMM on the wgmma engine writing its 128-column slice of Y [N][K*CC]; every layer's batch norm runs on its slice
//   max-pool (2, stride 1, 'same': max(x[t], x[t+1]))
//   proj1 (k = 3, K*CC -> PJ, ReLU, BN), proj2 (k = 3, PJ -> M, linear, BN), + mel_outputs, dense M -> HU
//   NH highway layers: one GEMM with N = 2 HU ([H | T] pre-activations) + an elementwise kernel
//   bidirectional GRU (HU -> RU per direction, whole padded sequence): the input projections of all steps are ONE GEMM (N = 6 RU);
//     the recurrence runs in a persistent kernel - one CTA per (4 batch items, direction) keeps the recurrent weights (bf16) and the
//     state (fp32) in shared memory for all T steps
//   linear projection 2 RU -> num_freq (GEMM), clip, L1 loss with half of the weight on the bins below 2 kHz
// Backward mirrors it: elementwise / batch-norm backward kernels, data-gradient GEMMs with reversed taps, a persistent BPTT kernel
// for the GRU, and the weight gradients of every layer as tiles of the batched wgrad GEMM (reduction over positions).
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/t2b200.h"
#include "t2_batchnorm.h"
#include "t2_common.cuh"
#include "t2_gemm.h"
#include "t2_params.h"

namespace t2 {
namespace {

typedef __nv_bfloat16 bf16;
constexpr int kMaxBank = 16, kMaxHw = 8;
constexpr int kGruItems = 4;          // batch items per CTA of the recurrent kernels
constexpr int kGruThreads = 256;

struct CConv {
  int cin, cout, k, act;               // act: 1 relu, 0 none
  ConvBnParams p;
  int cinp, coutp;                     // channels rounded up to 64 (K slots of the packed operands)
  long long k_w, k_wT;                 // packed forward [cout][k * cinp], packed dgrad [cin rows][k * coutp]
};

struct CL {
  t2_cbhg_config_t c;
  int B, T, M, K, CC, KC, PJc, PK, NH, HU, RU, NF, NFP, NFR;
  long long N;
  std::vector<Param> params;
  long long n_params;
  std::vector<CConv> bank;
  CConv proj1, proj2;
  bool has_dense;
  long long p_dk, p_db, p_hk[kMaxHw][2], p_hb[kMaxHw][2], p_gk[2], p_gb[2], p_ck[2], p_cb[2], p_lk, p_lb;
  // packed operands (bytes)
  long long k_dense, k_denseT, k_hw[kMaxHw], k_hwT[kMaxHw], k_gx, k_gxT, k_lin, k_linT, k_bankT[3], packed_bytes;
  int grp_first[4], grp_taps[3], n_grp;   // bank layers [grp_first[g], grp_first[g+1]) share one data-gradient GEMM (<= 16 taps)
  // workspace (bytes)
  long long w_x0, w_Y, w_Xb, w_P, w_stb, w_Y1, w_X1, w_st1, w_Y2, w_st2, w_hin, w_hf[kMaxHw + 1], w_hb[kMaxHw + 1], w_HT[kMaxHw];
  long long w_XP, w_out, w_gr[2], w_gu[2], w_gc[2], w_grh[2], w_lin, w_scal, w_tlen;
  long long w_dlin, w_dout, w_dXP, w_dh, w_dhb, w_dHT, w_dhin, w_dY2b, w_d1, w_d2, w_dP, w_dbank, w_dx0[3], w_bsum, w_tiles, w_jobs, w_regtab;
  long long workspace_bytes;
  int n_jobs, n_reg;
};

int build(const t2_cbhg_config_t* cfg, CL& lo, std::vector<PackJob>* jobs_out) {
  T2_REQUIRE(cfg != nullptr, T2_ERR_INVALID_ARG, "null CBHG config");
  T2_REQUIRE(cfg->split_bf16 == 0 || cfg->split_bf16 == 1, T2_ERR_INVALID_ARG, "split_bf16 %d is not 0 or 1", cfg->split_bf16);
  lo.c = *cfg;
  lo.B = cfg->B; lo.T = cfg->T; lo.M = cfg->num_mels; lo.K = cfg->kernels; lo.CC = cfg->conv_channels; lo.KC = lo.K * lo.CC;
  lo.PJc = cfg->projection; lo.PK = cfg->projection_kernel_size; lo.NH = cfg->highwaynet_layers; lo.HU = cfg->highway_units;
  lo.RU = cfg->rnn_units; lo.NF = cfg->num_freq;
  lo.NFP = (lo.NF + 7) / 8 * 8;                 // row pitch of the bf16 gradient of the linear outputs
  lo.NFR = (lo.NF + 127) / 128 * 128;           // rows of the packed projection (whole 128-column output tiles)
  lo.N = (long long)lo.B * lo.T;
  T2_REQUIRE(lo.B >= 1 && lo.T >= 2, T2_ERR_UNSUPPORTED_SHAPE, "CBHG: B >= 1, T >= 2");
  T2_REQUIRE(lo.M % 8 == 0 && lo.M <= 128, T2_ERR_UNSUPPORTED_SHAPE, "CBHG: num_mels must be a multiple of 8, <= 128");
  T2_REQUIRE(lo.K >= 1 && lo.K <= 8 && lo.CC == 128, T2_ERR_UNSUPPORTED_SHAPE, "CBHG: 1..8 bank kernels of 128 channels");
  T2_REQUIRE(cfg->pool_size == 2, T2_ERR_UNSUPPORTED_SHAPE, "CBHG: pool_size must be 2");
  T2_REQUIRE(lo.PJc % 128 == 0 && lo.PJc <= 512 && lo.PK >= 1 && lo.PK <= 7 && lo.PK % 2 == 1, T2_ERR_UNSUPPORTED_SHAPE, "CBHG: projection sizes");
  T2_REQUIRE(lo.NH >= 1 && lo.NH <= kMaxHw && lo.HU == 128 && lo.RU == 128, T2_ERR_UNSUPPORTED_SHAPE,
             "CBHG: 1..8 highway layers, 128 highway / GRU units");
  T2_REQUIRE(lo.NF >= 8 && lo.NF <= 4096, T2_ERR_UNSUPPORTED_SHAPE, "CBHG: num_freq");
  lo.n_params = 0; lo.params.clear(); lo.bank.clear();
  const std::string P = "CBHG_postnet/";
  auto conv_params = [&](CConv& L, const std::string& pre) {
    L.p = add_conv_bn_params(lo.params, lo.n_params, pre, L.k, L.cin, L.cout);
    L.cinp = (L.cin + 63) / 64 * 64; L.coutp = (L.cout + 63) / 64 * 64;
  };
  for (int k = 1; k <= lo.K; ++k) {
    CConv L; L.cin = lo.M; L.cout = lo.CC; L.k = k; L.act = 1;
    char b[64]; snprintf(b, sizeof(b), "conv_bank/conv1d_%d/", k);
    conv_params(L, P + b); lo.bank.push_back(L);
  }
  lo.proj1.cin = lo.KC; lo.proj1.cout = lo.PJc; lo.proj1.k = lo.PK; lo.proj1.act = 1; conv_params(lo.proj1, P + "proj1/");
  lo.proj2.cin = lo.PJc; lo.proj2.cout = lo.M; lo.proj2.k = lo.PK; lo.proj2.act = 0; conv_params(lo.proj2, P + "proj2/");
  lo.has_dense = lo.M != lo.HU;
  T2_REQUIRE(lo.has_dense, T2_ERR_UNSUPPORTED_SHAPE, "CBHG: num_mels == highway_units (no dense layer) is not implemented");
  lo.p_dk = add_param(lo.params, lo.n_params, P + "dense/kernel", {lo.M, lo.HU}); lo.p_db = add_param(lo.params, lo.n_params, P + "dense/bias", {lo.HU});
  for (int i = 0; i < lo.NH; ++i) {
    char b[64];
    for (int j = 0; j < 2; ++j) {
      snprintf(b, sizeof(b), "highwaynet_%d/%s/", i + 1, j == 0 ? "H" : "T");
      lo.p_hk[i][j] = add_param(lo.params, lo.n_params, P + b + "kernel", {lo.HU, lo.HU}); lo.p_hb[i][j] = add_param(lo.params, lo.n_params, P + b + "bias", {lo.HU});
    }
  }
  const char* dn[2] = {"forward_RNN/", "backward_RNN/"};
  for (int d = 0; d < 2; ++d) {
    lo.p_gk[d] = add_param(lo.params, lo.n_params, P + dn[d] + "gates/kernel", {lo.HU + lo.RU, 2 * lo.RU}); lo.p_gb[d] = add_param(lo.params, lo.n_params, P + dn[d] + "gates/bias", {2 * lo.RU});
    lo.p_ck[d] = add_param(lo.params, lo.n_params, P + dn[d] + "candidate/kernel", {lo.HU + lo.RU, lo.RU}); lo.p_cb[d] = add_param(lo.params, lo.n_params, P + dn[d] + "candidate/bias", {lo.RU});
  }
  lo.p_lk = add_param(lo.params, lo.n_params, "cbhg_linear_specs_projection/kernel", {2 * lo.RU, lo.NF}); lo.p_lb = add_param(lo.params, lo.n_params, "cbhg_linear_specs_projection/bias", {lo.NF});

  // ---- packed operands ----
  // split_bf16: the forward operands take the split-bf16 layout (add_pack_fwd); the data-gradient operands of the backward pass keep
  // their bf16 layout
  const bool split = cfg->split_bf16 != 0;
  std::vector<PackJob> jobs;
  Arena pk;
  auto conv_pack = [&](CConv& L, bool with_t) {
    const int rows_f = (L.cout + 127) / 128 * 128, rows_t = (L.cin + 127) / 128 * 128;
    L.k_w = pk.take(fwd_operand_bytes(rows_f, L.k * L.cinp, split));
    L.k_wT = with_t ? pk.take(2LL * rows_t * L.k * L.coutp) : 0;
    for (int j = 0; j < L.k; ++j) {
      add_pack_fwd(jobs, split, L.p.kernel + (long long)j * L.cin * L.cout, L.cin, L.cout, L.k_w, L.k * L.cinp, j * L.cinp, L.cinp);   // fwd [cout][tap j | cin]
      if (with_t) add_pack(jobs, L.p.kernel + (long long)j * L.cin * L.cout, L.cin, L.cout, L.k_wT, L.k * L.coutp, 0, j * L.coutp);   // dgrad [cin][tap j | cout]
    }
  };
  for (auto& L : lo.bank) conv_pack(L, false);
  conv_pack(lo.proj1, true); conv_pack(lo.proj2, true);
  // data gradient of the bank: layers grouped greedily so that one GEMM holds <= 16 (layer, tap) segments; operand [M rows][taps * CC]
  lo.n_grp = 0; lo.grp_first[0] = 0;
  for (int l = 0, taps = 0; l < lo.K; ++l) {
    if (taps + (l + 1) > kMaxSeg) { lo.grp_taps[lo.n_grp++] = taps; lo.grp_first[lo.n_grp] = l; taps = 0; }
    taps += l + 1;
    if (l == lo.K - 1) { lo.grp_taps[lo.n_grp++] = taps; lo.grp_first[lo.n_grp] = lo.K; }
  }
  T2_REQUIRE(lo.n_grp <= 3, T2_ERR_UNSUPPORTED_SHAPE, "CBHG: conv bank too large for three data-gradient groups");
  for (int g = 0; g < lo.n_grp; ++g) {
    lo.k_bankT[g] = pk.take(2LL * 128 * lo.grp_taps[g] * lo.CC);
    int slot = 0;
    for (int l = lo.grp_first[g]; l < lo.grp_first[g + 1]; ++l)
      for (int j = 0; j < lo.bank[l].k; ++j, ++slot)
        add_pack(jobs, lo.bank[l].p.kernel + (long long)j * lo.M * lo.CC, lo.M, lo.CC, lo.k_bankT[g], lo.grp_taps[g] * lo.CC, 0, slot * lo.CC);
  }
  const int Ms = (lo.M + 63) / 64 * 64;     // the K slot of num_mels: the half width of the split mel rows
  lo.k_dense = pk.take(fwd_operand_bytes(lo.HU, Ms, split));
  add_pack_fwd(jobs, split, lo.p_dk, lo.M, lo.HU, lo.k_dense, Ms, 0, Ms);
  lo.k_denseT = pk.take(2LL * 128 * lo.HU); add_pack(jobs, lo.p_dk, lo.M, lo.HU, lo.k_denseT, lo.HU, 0, 0);
  for (int i = 0; i < lo.NH; ++i) {
    lo.k_hw[i] = pk.take(fwd_operand_bytes(2 * lo.HU, lo.HU, split));        // rows [H units | T units][K = HU]
    add_pack_fwd(jobs, split, lo.p_hk[i][0], lo.HU, lo.HU, lo.k_hw[i], lo.HU, 0, lo.HU);
    add_pack_fwd(jobs, split, lo.p_hk[i][1], lo.HU, lo.HU, lo.k_hw[i] + fwd_operand_bytes(lo.HU, lo.HU, split), lo.HU, 0, lo.HU);
    lo.k_hwT[i] = pk.take(2LL * lo.HU * 2 * lo.HU);            // [HU in][H units | T units]
    add_pack(jobs, lo.p_hk[i][0], lo.HU, lo.HU, lo.k_hwT[i], 2 * lo.HU, 0, 0);
    add_pack(jobs, lo.p_hk[i][1], lo.HU, lo.HU, lo.k_hwT[i], 2 * lo.HU, 0, lo.HU);
  }
  // GRU input projections: output columns [fw gates 2RU | fw cand RU | bw gates 2RU | bw cand RU], K = HU (the first HU kernel rows)
  const int XPW = 6 * lo.RU;
  lo.k_gx = pk.take(fwd_operand_bytes(XPW, lo.HU, split));
  lo.k_gxT = pk.take(2LL * lo.HU * XPW);
  for (int d = 0; d < 2; ++d) {
    add_pack_fwd(jobs, split, lo.p_gk[d], lo.HU, 2 * lo.RU, lo.k_gx + fwd_operand_bytes(d * 3 * lo.RU, lo.HU, split), lo.HU, 0, lo.HU);
    add_pack_fwd(jobs, split, lo.p_ck[d], lo.HU, lo.RU, lo.k_gx + fwd_operand_bytes(d * 3 * lo.RU + 2 * lo.RU, lo.HU, split), lo.HU, 0, lo.HU);
    add_pack(jobs, lo.p_gk[d], lo.HU, 2 * lo.RU, lo.k_gxT, XPW, 0, d * 3 * lo.RU);
    add_pack(jobs, lo.p_ck[d], lo.HU, lo.RU, lo.k_gxT, XPW, 0, d * 3 * lo.RU + 2 * lo.RU);
  }
  lo.k_lin = pk.take(fwd_operand_bytes(lo.NFR, 2 * lo.RU, split));
  add_pack_fwd(jobs, split, lo.p_lk, 2 * lo.RU, lo.NF, lo.k_lin, 2 * lo.RU, 0, 2 * lo.RU);
  const int NFK = (lo.NF + 63) / 64 * 64;
  lo.k_linT = pk.take(2LL * 2 * lo.RU * NFK); add_pack(jobs, lo.p_lk, 2 * lo.RU, lo.NF, lo.k_linT, NFK, 0, 0);
  lo.packed_bytes = pk.used;
  lo.n_jobs = int(jobs.size());

  // ---- workspace ----
  Arena ws;
  const long long N = lo.N;
  // split_bf16: the bf16 operands become [hi | lo] rows (num_mels padded to Ms per half), the pre-batch-norm activations fp32
  const long long xm = split ? 2 : 1, ym = split ? 4 : 2, mw = split ? 2LL * Ms : lo.M;
  lo.w_x0 = ws.take(N * mw * 2);
  lo.w_Y = ws.take(N * lo.KC * ym); lo.w_Xb = ws.take(N * lo.KC * 2 * xm); lo.w_P = ws.take(N * lo.KC * 2 * xm); lo.w_stb = ws.take(8LL * lo.KC * 4);
  lo.w_Y1 = ws.take(N * lo.PJc * ym); lo.w_X1 = ws.take(N * lo.PJc * 2 * xm); lo.w_st1 = ws.take(8LL * lo.PJc * 4);
  lo.w_Y2 = ws.take(N * lo.M * 4); lo.w_st2 = ws.take(8LL * 128 * 4);
  lo.w_hin = ws.take(N * mw * 2);
  for (int i = 0; i <= lo.NH; ++i) { lo.w_hf[i] = ws.take(N * lo.HU * 4); lo.w_hb[i] = ws.take(N * lo.HU * 2 * xm); }
  for (int i = 0; i < lo.NH; ++i) lo.w_HT[i] = ws.take(N * 2 * lo.HU * 2);
  lo.w_XP = ws.take(N * XPW * 4);
  lo.w_out = ws.take(N * 2 * lo.RU * 2 * xm);
  for (int d = 0; d < 2; ++d) { lo.w_gr[d] = ws.take(N * lo.RU * 2); lo.w_gu[d] = ws.take(N * lo.RU * 2); lo.w_gc[d] = ws.take(N * lo.RU * 2); lo.w_grh[d] = ws.take(N * lo.RU * 2); }
  lo.w_lin = ws.take(N * lo.NFP * 4);            // fp32 [N][NFP]: padded pitch (the epilogue stores whole float4s)
  lo.w_scal = ws.take(64 * 4);
  lo.w_tlen = ws.take(lo.B * 4);
  // backward
  lo.w_dlin = ws.take(N * lo.NFP * 2);
  lo.w_dout = ws.take(N * 2 * lo.RU * 4);
  lo.w_dXP = ws.take(N * XPW * 2);
  lo.w_dh = ws.take(N * lo.HU * 4); lo.w_dhb = ws.take(N * lo.HU * 2);
  lo.w_dHT = ws.take(N * 2 * lo.HU * 2);
  lo.w_dhin = ws.take(N * lo.M * 4);
  lo.w_dY2b = ws.take(N * 128 * 2);
  lo.w_d1 = ws.take(N * lo.PJc * 2); lo.w_d2 = ws.take(N * lo.PJc * 2);
  lo.w_dP = ws.take(N * lo.KC * 2); lo.w_dbank = ws.take(N * lo.KC * 2);
  for (int i = 0; i < 3; ++i) lo.w_dx0[i] = ws.take(N * 128 * 4);
  lo.w_bsum = ws.take(2LL * lo.KC * 4);
  lo.w_tiles = ws.take(4096 * sizeof(WgradTile));
  lo.w_jobs = ws.take((long long)jobs.size() * sizeof(PackJob));
  lo.n_reg = 0;
  for (auto& p : lo.params) lo.n_reg += p.reg ? 1 : 0;
  lo.w_regtab = ws.take((long long)lo.n_reg * 2 * sizeof(long long));
  lo.workspace_bytes = ws.used;
  if (jobs_out) jobs_out->swap(jobs);
  return T2_OK;
}

// ------------------------------------------------------------------------------------------------------
// small kernels
// ------------------------------------------------------------------------------------------------------
// tf.layers.max_pooling1d(pool 2, stride 1, 'same'): out[t] = max(x[t], x[t + 1]) (last step: x[t])
// kSplit: x / out rows are [hi(C) | lo(C)]; the recombined values hi + lo are compared and the winning pair is copied (exact)
template <bool kSplit>
__global__ void maxpool_fwd_k(const bf16* __restrict__ x, bf16* __restrict__ out, long long N, int T, int C) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= N * C) return;
  const long long r = e / C;
  const int t = int(r % T);
  if (kSplit) {
    const long long o = r * 2 * C + e % C;
    bf16 h = x[o], l = x[o + C];
    if (t + 1 < T) {
      const bf16 h2 = x[o + 2 * C], l2 = x[o + 3 * C];
      if (__bfloat162float(h2) + __bfloat162float(l2) > __bfloat162float(h) + __bfloat162float(l)) { h = h2; l = l2; }
    }
    out[o] = h; out[o + C] = l;
    return;
  }
  float v = __bfloat162float(x[e]);
  if (t + 1 < T) v = fmaxf(v, __bfloat162float(x[e + C]));
  out[e] = __float2bfloat16(v);
}
// gradient routing: x[t] receives dout[t] when it is the (first) maximum of window t and dout[t - 1] when it beats x[t - 1]
__global__ void maxpool_bwd_k(const bf16* __restrict__ x, const bf16* __restrict__ dout, bf16* __restrict__ dx, long long N, int T, int C) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= N * C) return;
  const long long r = e / C;
  const int t = int(r % T);
  const float v = __bfloat162float(x[e]);
  float g = 0.f;
  if (t + 1 >= T || v >= __bfloat162float(x[e + C])) g += __bfloat162float(dout[e]);
  if (t > 0 && v > __bfloat162float(x[e - C])) g += __bfloat162float(dout[e - C]);
  dx[e] = __float2bfloat16(g);
}
// highway layer (modules.py:12-16): pre [N][2HU] = [H pre-activation | T pre-activation] (biases added here);
// h' = relu(H) sigmoid(T) + h (1 - sigmoid(T)). Stashes relu(H) | sigmoid(T) in bf16 for the backward pass.
// kSplit: hb rows are [hi(HU) | lo(HU)] (the split operand of the next GEMM); hf stays the fp32 carry.
template <bool kSplit>
__global__ void highway_fwd_k(const float* __restrict__ pre, const float* __restrict__ bh, const float* __restrict__ bt, const float* __restrict__ h,
                              float* __restrict__ hf, bf16* __restrict__ hb, bf16* __restrict__ HT, long long N, int HU) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= N * HU) return;
  const long long r = e / HU; const int c = int(e % HU);
  const float Hh = fmaxf(pre[r * 2 * HU + c] + bh[c], 0.f);
  const float Tt = 1.f / (1.f + __expf(-(pre[r * 2 * HU + HU + c] + bt[c])));
  const float v = Hh * Tt + h[e] * (1.f - Tt);
  hf[e] = v;
  if (kSplit) {
    const bf16 hi = __float2bfloat16(v);
    hb[r * 2 * HU + c] = hi; hb[r * 2 * HU + HU + c] = __float2bfloat16(v - __bfloat162float(hi));
  } else {
    hb[e] = __float2bfloat16(v);
  }
  if (HT) { HT[r * 2 * HU + c] = __float2bfloat16(Hh); HT[r * 2 * HU + HU + c] = __float2bfloat16(Tt); }
}
// dh' -> d[H pre | T pre] (bf16, GEMM operand) and the carry part dh * (1 - T) written to dcarry (fp32)
__global__ void highway_bwd_k(const float* __restrict__ dh, const bf16* __restrict__ HT, const float* __restrict__ h, bf16* __restrict__ dHT,
                              float* __restrict__ dcarry, long long N, int HU) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= N * HU) return;
  const long long r = e / HU; const int c = int(e % HU);
  const float Hh = __bfloat162float(HT[r * 2 * HU + c]), Tt = __bfloat162float(HT[r * 2 * HU + HU + c]);
  const float g = dh[e];
  dHT[r * 2 * HU + c] = __float2bfloat16(Hh > 0.f ? g * Tt : 0.f);
  dHT[r * 2 * HU + HU + c] = __float2bfloat16(g * (Hh - h[e]) * Tt * (1.f - Tt));
  dcarry[e] = g * (1.f - Tt);
}
void maxpool_fwd(const bf16* x, bf16* out, long long N, int T, int C, int split, cudaStream_t st) {
  (split ? maxpool_fwd_k<true> : maxpool_fwd_k<false>)<<<grid1d(N * C), 256, 0, st>>>(x, out, N, T, C); t2_count_launch();
}
void maxpool_bwd(const bf16* x, const bf16* dout, bf16* dx, long long N, int T, int C, cudaStream_t st) {
  maxpool_bwd_k<<<grid1d(N * C), 256, 0, st>>>(x, dout, dx, N, T, C); t2_count_launch();
}
void highway_fwd(const float* pre, const float* bh, const float* bt, const float* h, float* hf, bf16* hb, bf16* HT, long long N, int HU, int split,
                 cudaStream_t st) {
  (split ? highway_fwd_k<true> : highway_fwd_k<false>)<<<grid1d(N * HU), 256, 0, st>>>(pre, bh, bt, h, hf, hb, HT, N, HU); t2_count_launch();
}
void highway_bwd(const float* dh, const bf16* HT, const float* h, bf16* dHT, float* dcarry, long long N, int HU, cudaStream_t st) {
  highway_bwd_k<<<grid1d(N * HU), 256, 0, st>>>(dh, HT, h, dHT, dcarry, N, HU); t2_count_launch();
}
// out fp32 += a (fp32) ; optional bf16 copy
__global__ void add_k(float* __restrict__ acc, const float* __restrict__ a, bf16* __restrict__ outb, long long n) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float v = acc[e] + a[e];
  acc[e] = v;
  if (outb) outb[e] = __float2bfloat16(v);
}
// linear outputs: clip (tacotron.py:218-219), L1 loss with priority on the low bins (:323-330 / MaskedLinearLoss), gradient seed.
// scal[0] += sum |t - o| * w over all bins, scal[1] += the same over bins < n_prio; normalisers are applied by the caller-side kernel.
__global__ void lin_finish_k(float* __restrict__ lin, const float* __restrict__ tgt, bf16* __restrict__ dlin, float* __restrict__ scal, long long N,
                             int T, int NF, int NFP, int n_prio, int clip, float lo, float hi, const int* __restrict__ tlen) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  float l_all = 0.f, l_low = 0.f;
  const float n_all = scal[8], n_low = scal[9];
  if (e < N * NFP) {
    const long long r = e / NFP; const int f = int(e % NFP);
    float g = 0.f;
    if (f < NF) {
      const long long o = r * NF + f;           // targets are dense [N][NF]; the outputs have pitch NFP
      const float raw = lin[e];
      const float v = clip ? fminf(fmaxf(raw, lo), hi) : raw;
      lin[e] = v;
      if (tgt) {
        const bool live = !tlen || int(r % T) < tlen[r / T];
        if (live) {
          const float d = v - tgt[o];
          l_all = fabsf(d);
          if (f < n_prio) l_low = l_all;
          const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
          g = sg * (0.5f / n_all + (f < n_prio ? 0.5f / n_low : 0.f));
          if (clip && (raw < lo || raw > hi)) g = 0.f;
        }
      }
    }
    if (dlin) dlin[e] = __float2bfloat16(g);
  }
  l_all = warp_sum(l_all); l_low = warp_sum(l_low);
  if ((threadIdx.x & 31) == 0 && tgt) { atomicAdd(scal + 0, l_all); atomicAdd(scal + 1, l_low); }
}
// normalisers of the two L1 means: plain = (N NF, N n_prio); masked (MaskedLinearLoss) = sum(mask) for BOTH terms
__global__ void lin_norm_k(float* __restrict__ scal, const int* __restrict__ tlen, int B, int T, int NF, int n_prio) {
  if (!tlen) { scal[8] = float((long long)B * T) * NF; scal[9] = float((long long)B * T) * n_prio; return; }
  long long n = 0;
  for (int b = 0; b < B; ++b) n += tlen[b] < T ? tlen[b] : T;
  scal[8] = scal[9] = fmaxf(float(n) * NF, 1.f);
}
__global__ void loss_out_k(const float* __restrict__ scal, float* __restrict__ out, float regw) {
  out[0] = 0.5f * scal[0] / scal[8] + 0.5f * scal[1] / scal[9];
  out[1] = scal[2] * regw;
}
// dmel_out[r][m] = sum of the three partial data gradients of the conv bank + the residual path (d highway_in) ; rows of 128
__global__ void dmel_k(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c, const float* __restrict__ dhin,
                       float* __restrict__ out, long long N, int M) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= N * M) return;
  const long long r = e / M; const int m = int(e % M);
  out[e] = a[r * 128 + m] + b[r * 128 + m] + c[r * 128 + m] + dhin[e];
}

// ------------------------------------------------------------------------------------------------------
// GRU recurrence (tf.nn.rnn_cell.GRUCell inside bidirectional_dynamic_rnn, modules.py:34-35,69-75)
//   r, u = sigmoid(xg + h Wg_h) ; c = tanh(xc + (r h) Wc_h) ; h' = u h + (1 - u) c        (xg, xc: input projections incl. biases)
// One CTA = kGruItems batch items of one direction for all T steps; recurrent weights live in shared memory as bf16 PAIRS along k
// ([k/2][col] of bf16x2) so that a 4-byte load feeds two FMAs; state in fp32.
// kSplit (split_bf16): the lo halves W - bf16(W) of the recurrent weights are staged behind the hi halves in the same layouts and every
// product is h W_hi + h W_lo; out rows are [hi(2RU) | lo(2RU)] and the backward stashes are not written.
// ------------------------------------------------------------------------------------------------------
struct GruArgs {
  const float* params; long long p_gk[2], p_ck[2], p_gb[2], p_cb[2];
  const float* XP;          // [N][6RU] fp32
  bf16* out;                // [N][2RU]: h of direction d in columns [d RU, (d+1) RU); split: [N][4RU], the lo halves at +2RU
  bf16 *r[2], *u[2], *c[2], *rh[2];   // stashes [N][RU] (nullable)
  int B, T, HU, RU;
};
constexpr int kRU = 128;
// the lo halves w - bf16(w) of a k pair (pack_bf16x2 layout)
__device__ __forceinline__ uint32_t pack_lo_bf16x2(float w0, float w1) {
  return pack_bf16x2(w0 - __bfloat162float(__float2bfloat16(w0)), w1 - __bfloat162float(__float2bfloat16(w1)));
}
template <bool kSplit>
__global__ void __launch_bounds__(kGruThreads, 1) gru_fwd_kernel(GruArgs a) {
  extern __shared__ __align__(16) uint8_t gsm[];
  uint32_t* Wg = reinterpret_cast<uint32_t*>(gsm);                 // [64][256] bf16x2 (k pairs)
  uint32_t* Wc = Wg + 64 * 256;                                    // [64][128]
  uint32_t* Wgl = Wc + 64 * 128;                                   // kSplit: lo halves, [64][256] then [64][128]
  uint32_t* Wcl = Wgl + 64 * 256;
  float* h = reinterpret_cast<float*>(kSplit ? Wcl + 64 * 128 : Wgl);   // [4][128]
  float* rhs = h + kGruItems * kRU;                                // [4][128]
  float* us = rhs + kGruItems * kRU;                               // [4][128]
  const int d = blockIdx.y, b0 = blockIdx.x * kGruItems, tid = threadIdx.x;
  const float* gk = a.params + a.p_gk[d] + (long long)a.HU * 2 * kRU;     // recurrent rows of the gates kernel [RU][2RU]
  const float* ck = a.params + a.p_ck[d] + (long long)a.HU * kRU;          // recurrent rows of the candidate kernel [RU][RU]
  for (int i = tid; i < 64 * 256; i += kGruThreads) {
    const int kp = i / 256, col = i % 256;
    Wg[i] = pack_bf16x2(gk[(2 * kp) * 256 + col], gk[(2 * kp + 1) * 256 + col]);
    if (kSplit) Wgl[i] = pack_lo_bf16x2(gk[(2 * kp) * 256 + col], gk[(2 * kp + 1) * 256 + col]);
  }
  for (int i = tid; i < 64 * 128; i += kGruThreads) {
    const int kp = i / 128, col = i % 128;
    Wc[i] = pack_bf16x2(ck[(2 * kp) * 128 + col], ck[(2 * kp + 1) * 128 + col]);
    if (kSplit) Wcl[i] = pack_lo_bf16x2(ck[(2 * kp) * 128 + col], ck[(2 * kp + 1) * 128 + col]);
  }
  for (int i = tid; i < kGruItems * kRU; i += kGruThreads) h[i] = 0.f;
  __syncthreads();
  const int XPW = 6 * kRU;
  const int j2 = tid & 127, half = tid >> 7;     // phase 2: column j2 of items {2 half, 2 half + 1}
  const float bg = a.params[a.p_gb[d] + tid], bc = a.params[a.p_cb[d] + j2];
  for (int s = 0; s < a.T; ++s) {
    const int t = d == 0 ? s : a.T - 1 - s;
    // phase 1: gate column `tid` (r: 0..127, u: 128..255) of all items
    float acc[kGruItems];
#pragma unroll
    for (int i = 0; i < kGruItems; ++i) acc[i] = b0 + i < a.B ? a.XP[((long long)(b0 + i) * a.T + t) * XPW + d * 3 * kRU + tid] + bg : 0.f;
#pragma unroll 4
    for (int kp = 0; kp < 64; ++kp) {
      const uint32_t w = Wg[kp * 256 + tid];
      const float w0 = bf16lo(w), w1 = bf16hi(w);
      if (kSplit) {
        const uint32_t wl = Wgl[kp * 256 + tid];
        const float l0 = bf16lo(wl), l1 = bf16hi(wl);
#pragma unroll
        for (int i = 0; i < kGruItems; ++i) {
          const float2 hv = *reinterpret_cast<const float2*>(h + i * kRU + 2 * kp);
          acc[i] += hv.x * w0 + hv.y * w1 + (hv.x * l0 + hv.y * l1);
        }
        continue;
      }
#pragma unroll
      for (int i = 0; i < kGruItems; ++i) {
        const float2 hv = *reinterpret_cast<const float2*>(h + i * kRU + 2 * kp);
        acc[i] += hv.x * w0 + hv.y * w1;
      }
    }
#pragma unroll
    for (int i = 0; i < kGruItems; ++i) {
      const float g = 1.f / (1.f + __expf(-acc[i]));
      if (tid < kRU) {
        const float rhv = g * h[i * kRU + tid];
        rhs[i * kRU + tid] = rhv;
        if (!kSplit && a.r[d] && b0 + i < a.B) {
          const long long o = ((long long)(b0 + i) * a.T + t) * kRU + tid;
          a.r[d][o] = __float2bfloat16(g); a.rh[d][o] = __float2bfloat16(rhv);
        }
      } else {
        us[i * kRU + tid - kRU] = g;
        if (!kSplit && a.u[d] && b0 + i < a.B) a.u[d][((long long)(b0 + i) * a.T + t) * kRU + tid - kRU] = __float2bfloat16(g);
      }
    }
    __syncthreads();
    // phase 2: candidate column j2 for two items, then the state update
    float cc[2];
#pragma unroll
    for (int q = 0; q < 2; ++q)
      cc[q] = b0 + 2 * half + q < a.B ? a.XP[((long long)(b0 + 2 * half + q) * a.T + t) * XPW + d * 3 * kRU + 2 * kRU + j2] + bc : 0.f;
#pragma unroll 4
    for (int kp = 0; kp < 64; ++kp) {
      const uint32_t w = Wc[kp * 128 + j2];
      const float w0 = bf16lo(w), w1 = bf16hi(w);
      if (kSplit) {
        const uint32_t wl = Wcl[kp * 128 + j2];
        const float l0 = bf16lo(wl), l1 = bf16hi(wl);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const float2 v = *reinterpret_cast<const float2*>(rhs + (2 * half + q) * kRU + 2 * kp);
          cc[q] += v.x * w0 + v.y * w1 + (v.x * l0 + v.y * l1);
        }
        continue;
      }
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float2 v = *reinterpret_cast<const float2*>(rhs + (2 * half + q) * kRU + 2 * kp);
        cc[q] += v.x * w0 + v.y * w1;
      }
    }
    float hn[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = 2 * half + q;
      const float cv = tanhf(cc[q]);
      const float uv = us[i * kRU + j2];
      hn[q] = uv * h[i * kRU + j2] + (1.f - uv) * cv;
      const long long row = (long long)(b0 + i) * a.T + t;
      if (b0 + i < a.B && kSplit) {
        const bf16 hi = __float2bfloat16(hn[q]);
        a.out[row * 4 * kRU + d * kRU + j2] = hi;
        a.out[row * 4 * kRU + 2 * kRU + d * kRU + j2] = __float2bfloat16(hn[q] - __bfloat162float(hi));
      } else if (b0 + i < a.B) {
        a.out[row * 2 * kRU + d * kRU + j2] = __float2bfloat16(hn[q]);
        if (a.c[d]) a.c[d][row * kRU + j2] = __float2bfloat16(cv);
      }
    }
    __syncthreads();          // every thread has read h / us / rhs of this step
#pragma unroll
    for (int q = 0; q < 2; ++q) h[(2 * half + q) * kRU + j2] = hn[q];
    __syncthreads();
  }
}

// BPTT of the recurrence: walks the steps in reverse processing order, carries dh in shared memory, writes the gradients of the
// pre-activations [dr_pre | du_pre | dc_pre] (bf16) into dXP (the operand of the input-projection dgrad / wgrad GEMMs).
struct GruBwdArgs {
  const float* params; long long p_gk[2], p_ck[2];
  const float* dout;        // [N][2RU] fp32: upstream gradient of the outputs
  const bf16* out;          // [N][2RU] forward outputs (h_prev of a step = the output of the previously processed step)
  const bf16 *r[2], *u[2], *c[2];
  bf16* dXP;                // [N][6RU]
  int B, T, HU, RU;
};
__global__ void __launch_bounds__(kGruThreads, 1) gru_bwd_kernel(GruBwdArgs a) {
  extern __shared__ __align__(16) uint8_t gsm[];
  uint32_t* WgT = reinterpret_cast<uint32_t*>(gsm);                // [128 (j pairs of 256 gate cols)][128 k] : bf16x2 over gate columns j
  uint32_t* WcT = WgT + 128 * 128;                                 // [64 (j pairs of 128 cand cols)][128 k]
  float* dh = reinterpret_cast<float*>(WcT + 64 * 128);            // [4][128] carried gradient
  float* dcp = dh + kGruItems * kRU;                               // [4][128]
  float* dgp = dcp + kGruItems * kRU;                              // [4][256]: dr_pre | du_pre
  const int d = blockIdx.y, b0 = blockIdx.x * kGruItems, tid = threadIdx.x;
  const float* gk = a.params + a.p_gk[d] + (long long)a.HU * 2 * kRU;
  const float* ck = a.params + a.p_ck[d] + (long long)a.HU * kRU;
  for (int i = tid; i < 128 * 128; i += kGruThreads) {
    const int jp = i / 128, k = i % 128;
    WgT[i] = pack_bf16x2(gk[k * 256 + 2 * jp], gk[k * 256 + 2 * jp + 1]);
  }
  for (int i = tid; i < 64 * 128; i += kGruThreads) {
    const int jp = i / 128, k = i % 128;
    WcT[i] = pack_bf16x2(ck[k * 128 + 2 * jp], ck[k * 128 + 2 * jp + 1]);
  }
  for (int i = tid; i < kGruItems * kRU; i += kGruThreads) dh[i] = 0.f;
  __syncthreads();
  const int XPW = 6 * kRU;
  const int k2 = tid & 127, half = tid >> 7;     // thread owns unit k2 of items {2 half, 2 half + 1}
  for (int s = a.T - 1; s >= 0; --s) {
    const int t = d == 0 ? s : a.T - 1 - s;
    const int tp = d == 0 ? t - 1 : t + 1;       // time index of the previously processed step (h_prev)
    float g[2], hp[2], uv[2], rv[2], du[2], part[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = 2 * half + q;
      const bool live = b0 + i < a.B;               // a batch that is not a multiple of the CTA's item count: idle lanes carry zeros
      const long long row = live ? (long long)(b0 + i) * a.T + t : 0;
      g[q] = live ? dh[i * kRU + k2] + a.dout[row * 2 * kRU + d * kRU + k2] : 0.f;
      hp[q] = (live && s > 0) ? __bfloat162float(a.out[((long long)(b0 + i) * a.T + tp) * 2 * kRU + d * kRU + k2]) : 0.f;
      uv[q] = live ? __bfloat162float(a.u[d][row * kRU + k2]) : 0.f;
      rv[q] = live ? __bfloat162float(a.r[d][row * kRU + k2]) : 0.f;
      const float cv = live ? __bfloat162float(a.c[d][row * kRU + k2]) : 0.f;
      du[q] = g[q] * (hp[q] - cv);
      const float dc = g[q] * (1.f - uv[q]);
      const float dcpv = dc * (1.f - cv * cv);
      dcp[i * kRU + k2] = dcpv;
      if (live) a.dXP[row * XPW + d * 3 * kRU + 2 * kRU + k2] = __float2bfloat16(dcpv);
      part[q] = g[q] * uv[q];
    }
    __syncthreads();
    // d(r h)[k2] = sum_j dc_pre[j] Wc_h[k2][j]
    float drh[2] = {0.f, 0.f};
#pragma unroll 4
    for (int jp = 0; jp < 64; ++jp) {
      const uint32_t w = WcT[jp * 128 + k2];
      const float w0 = bf16lo(w), w1 = bf16hi(w);
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float2 v = *reinterpret_cast<const float2*>(dcp + (2 * half + q) * kRU + 2 * jp);
        drh[q] += v.x * w0 + v.y * w1;
      }
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = 2 * half + q;
      const long long row = (long long)(b0 + i) * a.T + t;
      const float drp = drh[q] * hp[q] * rv[q] * (1.f - rv[q]);
      const float dup = du[q] * uv[q] * (1.f - uv[q]);
      dgp[i * 2 * kRU + k2] = drp; dgp[i * 2 * kRU + kRU + k2] = dup;
      if (b0 + i < a.B) {
        a.dXP[row * XPW + d * 3 * kRU + k2] = __float2bfloat16(drp);
        a.dXP[row * XPW + d * 3 * kRU + kRU + k2] = __float2bfloat16(dup);
      }
      part[q] += drh[q] * rv[q];
    }
    __syncthreads();
    // dh_prev[k2] += sum_j [dr_pre | du_pre][j] Wg_h[k2][j]
#pragma unroll 4
    for (int jp = 0; jp < 128; ++jp) {
      const uint32_t w = WgT[jp * 128 + k2];
      const float w0 = bf16lo(w), w1 = bf16hi(w);
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float2 v = *reinterpret_cast<const float2*>(dgp + (2 * half + q) * 2 * kRU + 2 * jp);
        part[q] += v.x * w0 + v.y * w1;
      }
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) dh[(2 * half + q) * kRU + k2] = part[q];   // only this thread reads / writes dh[i][k2]
    __syncthreads();          // dcp / dgp are rewritten by the next step
  }
}

// ------------------------------------------------------------------------------------------------------
// host helpers
// ------------------------------------------------------------------------------------------------------
// wgrad launches, in the order t2_cbhg_backward issues them
enum { WG_LIN = 0, WG_GRU = 1, WG_HW0 = 2 /* NH launches, last highway layer first */ };
void build_tiles(const CL& lo, std::vector<std::vector<WgradTile>>& L) {
  L.clear();
  const int RU = lo.RU, HU = lo.HU;
  { std::vector<WgradTile> w; append_wgrad_tiles(w, dense_proto(0, 1), 0, 2 * RU, 0, lo.NF, lo.p_lk, lo.NF); L.push_back(w); }      // maps: 0 rnn out, 1 dlin
  { std::vector<WgradTile> w;     // maps: 0 h_last (bf16 [N][HU]), 1 dXP, 2 rnn out, 3 rh fw, 4 rh bw
    for (int d = 0; d < 2; ++d) {
      append_wgrad_tiles(w, dense_proto(0, 1), 0, HU, d * 3 * RU, 2 * RU, lo.p_gk[d], 2 * RU);                                       // input rows of the gates kernel
      append_wgrad_tiles(w, dense_proto(0, 1), 0, HU, d * 3 * RU + 2 * RU, RU, lo.p_ck[d], RU);                                      // input rows of the candidate kernel
      append_wgrad_tiles(w, dense_proto(2, 1, d == 0 ? -1 : 1), d * RU, RU, d * 3 * RU, 2 * RU, lo.p_gk[d] + (long long)HU * 2 * RU, 2 * RU);   // h_prev x d gates
      append_wgrad_tiles(w, dense_proto(3 + d, 1), 0, RU, d * 3 * RU + 2 * RU, RU, lo.p_ck[d] + (long long)HU * RU, RU);             // (r h_prev) x d cand
    }
    L.push_back(w); }
  for (int i = lo.NH - 1; i >= 0; --i) {   // maps: 0 h_i (bf16), 1 dHT
    std::vector<WgradTile> w;
    append_wgrad_tiles(w, dense_proto(0, 1), 0, HU, 0, HU, lo.p_hk[i][0], HU);
    append_wgrad_tiles(w, dense_proto(0, 1), 0, HU, HU, HU, lo.p_hk[i][1], HU);
    L.push_back(w);
  }
  { std::vector<WgradTile> w; append_wgrad_tiles(w, dense_proto(0, 1), 0, lo.M, 0, HU, lo.p_dk, HU); L.push_back(w); }               // dense: hin x dh0
  for (const CConv* c : {&lo.proj2, &lo.proj1}) {   // maps: 0 X1, 1 dY2b / 0 P, 1 d1
    std::vector<WgradTile> w; append_conv_wgrad_tiles(w, c->k, 0, c->cin, 0, c->cout, c->p.kernel); L.push_back(w);
  }
  { std::vector<WgradTile> w;  // bank: maps 0 x0, 1 dbank (channel block k-1)
    for (int k = 1; k <= lo.K; ++k) append_conv_wgrad_tiles(w, k, 0, lo.M, (k - 1) * lo.CC, lo.CC, lo.bank[k - 1].p.kernel);
    L.push_back(w); }
}

// bf16 104,448 B; split 202,752 B (the lo halves of both weight blocks), under the 232,448 B opt-in limit of sm_90
size_t gru_fwd_smem(int split) { return (64 * 256 + 64 * 128) * 4 * (split ? 2 : 1) + 3 * kGruItems * kRU * 4; }
size_t gru_bwd_smem() { return (128 * 128 + 64 * 128) * 4 + (2 * kGruItems * kRU + kGruItems * 2 * kRU) * 4; }

// launch helpers shared by t2_cbhg_forward / t2_cbhg_backward and t2_dbg_cbhg_kernel: one grid (B / 4 items x 2 directions), block and
// shared-memory size. The checks run before any driver call.
int gru_setup() {
  T2_CHECK_CUDA(cudaFuncSetAttribute(gru_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(gru_fwd_smem(0))));
  T2_CHECK_CUDA(cudaFuncSetAttribute(gru_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(gru_fwd_smem(1))));
  T2_CHECK_CUDA(cudaFuncSetAttribute(gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(gru_bwd_smem())));
  return T2_OK;
}
int check_gru_shape(int B, int T, int HU, int RU, const char* what) {
  T2_REQUIRE(B >= 1 && T >= 1 && HU >= 1, T2_ERR_UNSUPPORTED_SHAPE, "%s: B >= 1, T >= 1, HU >= 1 (B %d, T %d, HU %d)", what, B, T, HU);
  T2_REQUIRE(RU == kRU, T2_ERR_UNSUPPORTED_SHAPE, "%s: RU must be %d (got %d)", what, kRU, RU);
  return T2_OK;
}
int check_gru_fwd(const GruArgs& a, int split) {
  T2_REQUIRE(a.params && a.XP && a.out, T2_ERR_INVALID_ARG, "gru_fwd: null params / XP / out");
  T2_REQUIRE(split == 0 || split == 1, T2_ERR_INVALID_ARG, "gru_fwd: split %d is not 0 or 1", split);
  int n = 0;
  for (int d = 0; d < 2; ++d) n += (a.r[d] != nullptr) + (a.u[d] != nullptr) + (a.c[d] != nullptr) + (a.rh[d] != nullptr);
  T2_REQUIRE(!split || n == 0, T2_ERR_INVALID_ARG, "gru_fwd: the split mode writes no stashes (%d of 8 given)", n);
  T2_REQUIRE(n == 0 || n == 8, T2_ERR_INVALID_ARG, "gru_fwd: the r / u / c / rh stashes of both directions are all present or all null (%d of 8)", n);
  for (int d = 0; d < 2; ++d)
    T2_REQUIRE(a.p_gk[d] >= 0 && a.p_ck[d] >= 0 && a.p_gb[d] >= 0 && a.p_cb[d] >= 0, T2_ERR_INVALID_ARG, "gru_fwd: negative parameter offset");
  return check_gru_shape(a.B, a.T, a.HU, a.RU, "gru_fwd");
}
int check_gru_bwd(const GruBwdArgs& a) {
  T2_REQUIRE(a.params && a.dout && a.out && a.dXP, T2_ERR_INVALID_ARG, "gru_bwd: null params / dout / out / dXP");
  for (int d = 0; d < 2; ++d) {
    T2_REQUIRE(a.r[d] && a.u[d] && a.c[d], T2_ERR_INVALID_ARG, "gru_bwd: null stash of direction %d", d);
    T2_REQUIRE(a.p_gk[d] >= 0 && a.p_ck[d] >= 0, T2_ERR_INVALID_ARG, "gru_bwd: negative parameter offset");
  }
  return check_gru_shape(a.B, a.T, a.HU, a.RU, "gru_bwd");
}
int launch_gru_fwd(const GruArgs& a, int split, cudaStream_t st) {
  int rc = check_gru_fwd(a, split);
  if (rc) return rc;
  (split ? gru_fwd_kernel<true> : gru_fwd_kernel<false>)<<<dim3((a.B + kGruItems - 1) / kGruItems, 2), kGruThreads, gru_fwd_smem(split), st>>>(a);
  t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}
int launch_gru_bwd(const GruBwdArgs& a, cudaStream_t st) {
  int rc = check_gru_bwd(a);
  if (rc) return rc;
  gru_bwd_kernel<<<dim3((a.B + kGruItems - 1) / kGruItems, 2), kGruThreads, gru_bwd_smem(), st>>>(a); t2_count_launch();
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

}  // namespace
}  // namespace t2

using namespace t2;

extern "C" int t2_cbhg_sizes(const t2_cbhg_config_t* cfg, long long* n_params, long long* packed_bytes, long long* workspace_bytes, int* n_tensors) {
  CL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  if (n_params) *n_params = lo.n_params;
  if (packed_bytes) *packed_bytes = lo.packed_bytes;
  if (workspace_bytes) *workspace_bytes = lo.workspace_bytes;
  if (n_tensors) *n_tensors = int(lo.params.size());
  return T2_OK;
}

extern "C" int t2_cbhg_param_info(const t2_cbhg_config_t* cfg, int i, char* name, int cap, long long* offset, int* ndim, int* shape4, int* trainable) {
  CL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  return param_info(lo.params, i, name, cap, offset, ndim, shape4, trainable);
}

extern "C" int t2_cbhg_init(const t2_cbhg_config_t* cfg, void* d_packed, void* d_workspace, void* stream) {
  CL lo;
  std::vector<PackJob> jobs;
  int rc = build(cfg, lo, &jobs);
  if (rc) return rc;
  T2_REQUIRE(d_packed && d_workspace, T2_ERR_INVALID_ARG, "cbhg_init: null buffers");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  T2_CHECK_CUDA(cudaMemsetAsync(d_packed, 0, lo.packed_bytes, st));
  T2_CHECK_CUDA(cudaMemsetAsync(d_workspace, 0, lo.workspace_bytes, st));
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_jobs, jobs.data(), jobs.size() * sizeof(PackJob), cudaMemcpyHostToDevice, st));
  std::vector<std::vector<WgradTile>> wl;
  build_tiles(lo, wl);
  std::vector<WgradTile> all;
  for (auto& w : wl) all.insert(all.end(), w.begin(), w.end());
  T2_REQUIRE(all.size() <= 4096, T2_ERR_UNSUPPORTED_SHAPE, "cbhg: too many wgrad tiles (%d)", int(all.size()));
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_tiles, all.data(), all.size() * sizeof(WgradTile), cudaMemcpyHostToDevice, st));
  rc = upload_reg_table(lo.params, ws + lo.w_regtab, st);
  if (rc) return rc;
  rc = gru_setup();
  if (rc) return rc;
  T2_CHECK_CUDA(cudaStreamSynchronize(st));
  return T2_OK;
}

extern "C" int t2_cbhg_pack_weights(const t2_cbhg_config_t* cfg, const float* d_params, void* d_packed, void* d_workspace, void* stream) {
  CL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  return launch_pack(d_params, d_packed, reinterpret_cast<const PackJob*>(static_cast<uint8_t*>(d_workspace) + lo.w_jobs), lo.n_jobs, 32, 32,
                     static_cast<cudaStream_t>(stream));
}

extern "C" int t2_cbhg_set_target_lengths(const t2_cbhg_config_t* cfg, void* d_workspace, const int* d_target_lengths, void* stream) {
  CL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  T2_REQUIRE(d_workspace && d_target_lengths, T2_ERR_INVALID_ARG, "cbhg_set_target_lengths: null pointer");
  T2_CHECK_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(d_workspace) + lo.w_tlen, d_target_lengths, lo.B * sizeof(int), cudaMemcpyDeviceToDevice,
                                static_cast<cudaStream_t>(stream)));
  return T2_OK;
}

namespace {
struct Ctx { const CL* lo; uint8_t* ws; const uint8_t* pk; float* params; cudaStream_t st; int training; };
template <typename T> T* W(const Ctx& s, long long off) { return reinterpret_cast<T*>(s.ws + off); }

// conv (+ bias, activation) into `y` (bf16 [N][ldo] column slice or fp32), batch-norm statistics are taken by the caller
int conv_fwd(const Ctx& s, const CConv& L, const void* x, int ld_x, bf16* y_b, float* y_f, int ldo) {
  int shifts[16];
  for (int j = 0; j < L.k; ++j) shifts[j] = conv_tap_shift(L.k, j);
  const int BN = L.cout % 256 == 0 ? 256 : 128;
  const int sp = s.lo->c.split_bf16;
  return launch_bias_act({.a = x, .C = L.cin, .ld = ld_x, .T = s.lo->T, .B = s.lo->B, .ntaps = L.k, .shifts = shifts, .split = sp, .w = s.pk + L.k_w,
                          .N = (L.cout + 127) / 128 * 128, .wK = L.k * L.cinp, .BN = BN, .bias = s.params + L.p.bias, .act = L.act,
                          .out_bf16 = y_b, .out_f32 = y_f, .ldo = ldo, .nvalid = L.cout},
                         s.st);
}
}  // namespace

extern "C" int t2_cbhg_forward(const t2_cbhg_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace, const float* d_mel,
                               const float* d_linear_targets, float* d_loss, int training, void* stream) {
  CL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  T2_REQUIRE(d_params && d_packed && d_workspace && d_mel, T2_ERR_INVALID_ARG, "cbhg_forward: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ctx s{&lo, static_cast<uint8_t*>(d_workspace), static_cast<const uint8_t*>(d_packed), d_params, st, training};
  const long long N = lo.N;
  const int T = lo.T, B = lo.B, M = lo.M, HU = lo.HU, RU = lo.RU, KC = lo.KC, PJc = lo.PJc;
  float* scal = W<float>(s, lo.w_scal);
  T2_CHECK_CUDA(cudaMemsetAsync(scal, 0, 16 * sizeof(float), st));
  // split_bf16: every bf16 operand below is a [hi | lo] row pair, every contraction a split GEMM (launch_bias_act), and the
  // pre-batch-norm activations of the bank and of proj1 are fp32
  const int sp = lo.c.split_bf16, Ms = (M + 63) / 64 * 64;
  bf16* x0 = W<bf16>(s, lo.w_x0);
  if (sp) launch_f32_to_bf16_split(d_mel, x0, N, M, Ms, st);
  else launch_f32_to_bf16(d_mel, x0, N * M, st);
  // ---- conv bank (each layer writes its 128-column slice) + per-layer batch norm ----
  bf16* Y = W<bf16>(s, lo.w_Y);
  float* Yf = W<float>(s, lo.w_Y);
  bf16* Xb = W<bf16>(s, lo.w_Xb);
  float* stb = W<float>(s, lo.w_stb);
  if (training) T2_CHECK_CUDA(cudaMemsetAsync(stb, 0, 2LL * KC * sizeof(float), st));
  for (int k = 1; k <= lo.K; ++k) {
    const CConv& L = lo.bank[k - 1];
    const int c0 = (k - 1) * lo.CC;
    rc = conv_fwd(s, L, x0, M, sp ? nullptr : Y + c0, sp ? Yf + c0 : nullptr, KC);
    if (rc) return rc;
    if (sp)
      bn_fwd(Yf, KC, c0, Xb, 1, nullptr, nullptr, stb, KC, d_params + L.p.gamma, d_params + L.p.beta, d_params + L.p.mm, d_params + L.p.mv, N, lo.CC,
             training, BnDropout{}, 128, st);
    else
      bn_fwd(Y, KC, c0, Xb, 0, nullptr, nullptr, stb, KC, d_params + L.p.gamma, d_params + L.p.beta, d_params + L.p.mm, d_params + L.p.mv, N, lo.CC,
             training, BnDropout{}, 128, st);
  }
  bf16* P = W<bf16>(s, lo.w_P);
  maxpool_fwd(Xb, P, N, T, KC, sp, st);
  // ---- projections ----
  bf16* Y1 = W<bf16>(s, lo.w_Y1); float* Y1f = W<float>(s, lo.w_Y1); bf16* X1 = W<bf16>(s, lo.w_X1); float* st1 = W<float>(s, lo.w_st1);
  rc = conv_fwd(s, lo.proj1, P, KC, sp ? nullptr : Y1, sp ? Y1f : nullptr, PJc);
  if (rc) return rc;
  if (training) T2_CHECK_CUDA(cudaMemsetAsync(st1, 0, 2LL * PJc * sizeof(float), st));
  if (sp)
    bn_fwd(Y1f, PJc, 0, X1, 1, nullptr, nullptr, st1, PJc, d_params + lo.proj1.p.gamma, d_params + lo.proj1.p.beta, d_params + lo.proj1.p.mm,
           d_params + lo.proj1.p.mv, N, PJc, training, BnDropout{}, 256, st);
  else
    bn_fwd(Y1, PJc, 0, X1, 0, nullptr, nullptr, st1, PJc, d_params + lo.proj1.p.gamma, d_params + lo.proj1.p.beta, d_params + lo.proj1.p.mm,
           d_params + lo.proj1.p.mv, N, PJc, training, BnDropout{}, 256, st);
  float* Y2 = W<float>(s, lo.w_Y2); float* st2 = W<float>(s, lo.w_st2);
  rc = conv_fwd(s, lo.proj2, X1, PJc, nullptr, Y2, M);
  if (rc) return rc;
  if (training) T2_CHECK_CUDA(cudaMemsetAsync(st2, 0, 2LL * M * sizeof(float), st));
  // highway input = BN(proj2) + mel_outputs (modules.py:59); the fp32 sum goes through w_dhin (free until the backward pass)
  float* hin_f = W<float>(s, lo.w_dhin);
  bf16* hin = W<bf16>(s, lo.w_hin);
  bn_fwd(Y2, M, 0, nullptr, 0, hin_f, d_mel, st2, M, d_params + lo.proj2.p.gamma, d_params + lo.proj2.p.beta, d_params + lo.proj2.p.mm,
         d_params + lo.proj2.p.mv, N, M, training, BnDropout{}, 128, st);
  if (sp) launch_f32_to_bf16_split(hin_f, hin, N, M, Ms, st);
  else launch_f32_to_bf16(hin_f, hin, N * M, st);
  // ---- dense to the highway width, highway layers ----
  rc = launch_bias_act({.a = hin, .C = M, .T = T, .B = B, .split = sp, .w = s.pk + lo.k_dense, .N = HU, .wK = Ms, .BN = 128,
                        .bias = d_params + lo.p_db, .out_bf16 = W<bf16>(s, lo.w_hb[0]), .out_f32 = W<float>(s, lo.w_hf[0]), .ldo = HU, .nvalid = HU},
                       st);
  if (rc) return rc;
  float* pre = W<float>(s, lo.w_XP);       // [N][2HU] scratch (the GRU input projections overwrite it afterwards)
  for (int i = 0; i < lo.NH; ++i) {
    rc = launch_bias_act({.a = W<bf16>(s, lo.w_hb[i]), .C = HU, .T = T, .B = B, .split = sp, .w = s.pk + lo.k_hw[i], .N = 2 * HU, .wK = HU,
                          .BN = 256, .out_f32 = pre, .ldo = 2 * HU, .nvalid = 2 * HU},
                         st);
    if (rc) return rc;
    highway_fwd(pre, d_params + lo.p_hb[i][0], d_params + lo.p_hb[i][1], W<float>(s, lo.w_hf[i]), W<float>(s, lo.w_hf[i + 1]), W<bf16>(s, lo.w_hb[i + 1]),
                (training && !sp) ? W<bf16>(s, lo.w_HT[i]) : nullptr, N, HU, sp, st);
  }
  // ---- bidirectional GRU ----
  const int XPW = 6 * RU;
  float* XP = W<float>(s, lo.w_XP);
  rc = launch_bias_act({.a = W<bf16>(s, lo.w_hb[lo.NH]), .C = HU, .T = T, .B = B, .split = sp, .w = s.pk + lo.k_gx, .N = XPW, .wK = HU, .BN = 256,
                        .out_f32 = XP, .ldo = XPW, .nvalid = XPW},
                       st);
  if (rc) return rc;
  {
    GruArgs a;
    memset(&a, 0, sizeof(a));
    a.params = d_params;
    for (int d = 0; d < 2; ++d) {
      a.p_gk[d] = lo.p_gk[d]; a.p_ck[d] = lo.p_ck[d]; a.p_gb[d] = lo.p_gb[d]; a.p_cb[d] = lo.p_cb[d];
      if (training && !sp) { a.r[d] = W<bf16>(s, lo.w_gr[d]); a.u[d] = W<bf16>(s, lo.w_gu[d]); a.c[d] = W<bf16>(s, lo.w_gc[d]); a.rh[d] = W<bf16>(s, lo.w_grh[d]); }
    }
    a.XP = XP; a.out = W<bf16>(s, lo.w_out); a.B = B; a.T = T; a.HU = HU; a.RU = RU;
    rc = launch_gru_fwd(a, sp, st);
    if (rc) return rc;
  }
  // ---- linear projection, clip, loss ----
  float* lin = W<float>(s, lo.w_lin);
  rc = launch_bias_act({.a = W<bf16>(s, lo.w_out), .C = 2 * RU, .T = T, .B = B, .split = sp, .w = s.pk + lo.k_lin, .N = lo.NFR, .wK = 2 * RU,
                        .BN = 128, .bias = d_params + lo.p_lb, .out_f32 = lin, .ldo = lo.NFP, .nvalid = lo.NF},
                       st);
  if (rc) return rc;
  const int* tlen = lo.c.mask_decoder ? W<int>(s, lo.w_tlen) : nullptr;
  const float lo_c = -lo.c.max_abs_value - lo.c.lower_bound_decay, hi_c = lo.c.max_abs_value;
  lin_norm_k<<<1, 1, 0, st>>>(scal, tlen, B, T, lo.NF, lo.c.n_priority_freq); t2_count_launch();
  lin_finish_k<<<grid1d(N * lo.NFP), 256, 0, st>>>(lin, d_linear_targets, (training && d_linear_targets) ? W<bf16>(s, lo.w_dlin) : nullptr, scal, N, T, lo.NF,
                                               lo.NFP, lo.c.n_priority_freq, lo.c.clip_outputs, lo_c, hi_c, tlen); t2_count_launch();
  if (d_loss) {
    launch_reg_loss(d_params, W<long long>(s, lo.w_regtab), lo.n_reg, scal + 2, st);
    loss_out_k<<<1, 1, 0, st>>>(scal, d_loss, lo.c.reg_weight); t2_count_launch();
  }
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

extern "C" int t2_cbhg_backward(const t2_cbhg_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace, const float* d_mel,
                                float* d_grads, float* d_mel_grad, void* stream) {
  CL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  T2_REQUIRE(!lo.c.split_bf16, T2_ERR_INVALID_ARG, "split_bf16 (fp32-class) CBHG mode has no backward pass");
  T2_REQUIRE(d_params && d_packed && d_workspace && d_mel && d_grads && d_mel_grad, T2_ERR_INVALID_ARG, "cbhg_backward: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ctx s{&lo, static_cast<uint8_t*>(d_workspace), static_cast<const uint8_t*>(d_packed), const_cast<float*>(d_params), st, 1};
  const long long N = lo.N;
  const int T = lo.T, B = lo.B, M = lo.M, HU = lo.HU, RU = lo.RU, KC = lo.KC, PJc = lo.PJc, XPW = 6 * lo.RU;
  std::vector<std::vector<WgradTile>> wl;
  build_tiles(lo, wl);
  std::vector<int> toff(wl.size());
  { int o = 0; for (size_t i = 0; i < wl.size(); ++i) { toff[i] = o; o += int(wl[i].size()); } }
  const WgradTile* tiles = W<WgradTile>(s, lo.w_tiles);
  int li = 0;
  auto wgrad = [&](const ActT* maps, int nmaps) {
    int r = launch_wgrad(maps, nmaps, tiles + toff[li], int(wl[li].size()), d_grads, T, B, st);
    ++li;
    return r;
  };
  T2_CHECK_CUDA(cudaMemsetAsync(d_grads, 0, lo.n_params * sizeof(float), st));
  // ---- linear projection ----
  bf16* dlin = W<bf16>(s, lo.w_dlin);
  bf16* out = W<bf16>(s, lo.w_out);
  float* dout = W<float>(s, lo.w_dout);
  const int NFK = (lo.NF + 63) / 64 * 64;
  rc = launch_bias_act({.a = dlin, .C = lo.NF, .ld = lo.NFP, .T = T, .B = B, .w = s.pk + lo.k_linT, .N = 2 * RU, .wK = NFK, .BN = 256, .out_f32 = dout,
                        .ldo = 2 * RU, .nvalid = 2 * RU},
                       st);
  if (rc) return rc;
  { ActT maps[2] = {make_act(out, 2 * RU, T, B), make_act(dlin, lo.NF, T, B, 1, lo.NFP)}; rc = wgrad(maps, 2); if (rc) return rc; }
  colsum(dlin, N, lo.NF, lo.NFP, d_grads + lo.p_lb, 256, st);
  // ---- GRU ----
  bf16* dXP = W<bf16>(s, lo.w_dXP);
  {
    GruBwdArgs a;
    memset(&a, 0, sizeof(a));
    a.params = d_params;
    for (int d = 0; d < 2; ++d) {
      a.p_gk[d] = lo.p_gk[d]; a.p_ck[d] = lo.p_ck[d];
      a.r[d] = W<bf16>(s, lo.w_gr[d]); a.u[d] = W<bf16>(s, lo.w_gu[d]); a.c[d] = W<bf16>(s, lo.w_gc[d]);
    }
    a.dout = dout; a.out = out; a.dXP = dXP; a.B = B; a.T = T; a.HU = HU; a.RU = RU;
    rc = launch_gru_bwd(a, st);
    if (rc) return rc;
  }
  {
    ActT maps[5] = {make_act(W<bf16>(s, lo.w_hb[lo.NH]), HU, T, B), make_act(dXP, XPW, T, B), make_act(out, 2 * RU, T, B),
                    make_act(W<bf16>(s, lo.w_grh[0]), RU, T, B), make_act(W<bf16>(s, lo.w_grh[1]), RU, T, B)};
    rc = wgrad(maps, 5); if (rc) return rc;
  }
  for (int d = 0; d < 2; ++d) {
    colsum(dXP + d * 3 * RU, N, 2 * RU, XPW, d_grads + lo.p_gb[d], 256, st);
    colsum(dXP + d * 3 * RU + 2 * RU, N, RU, XPW, d_grads + lo.p_cb[d], 128, st);
  }
  float* dh = W<float>(s, lo.w_dh);
  rc = launch_bias_act({.a = dXP, .C = XPW, .T = T, .B = B, .w = s.pk + lo.k_gxT, .N = HU, .wK = XPW, .BN = 128, .out_f32 = dh, .ldo = HU, .nvalid = HU}, st);
  if (rc) return rc;
  // ---- highway layers (last first) ----
  bf16* dHT = W<bf16>(s, lo.w_dHT);
  float* dcar = W<float>(s, lo.w_XP);        // [N][HU] fp32 scratch (the forward input projections are no longer needed)
  for (int i = lo.NH - 1; i >= 0; --i) {
    highway_bwd(dh, W<bf16>(s, lo.w_HT[i]), W<float>(s, lo.w_hf[i]), dHT, dcar, N, HU, st);
    rc = launch_bias_act({.a = dHT, .C = 2 * HU, .T = T, .B = B, .w = s.pk + lo.k_hwT[i], .N = HU, .wK = 2 * HU, .BN = 128, .out_f32 = dh, .ldo = HU,
                          .nvalid = HU},
                         st);
    if (rc) return rc;
    add_k<<<grid1d(N * HU), 256, 0, st>>>(dh, dcar, i == 0 ? W<bf16>(s, lo.w_dhb) : nullptr, N * HU); t2_count_launch();
    { ActT maps[2] = {make_act(W<bf16>(s, lo.w_hb[i]), HU, T, B), make_act(dHT, 2 * HU, T, B)}; rc = wgrad(maps, 2); if (rc) return rc; }
    colsum(dHT, N, HU, 2 * HU, d_grads + lo.p_hb[i][0], 128, st);
    colsum(dHT + HU, N, HU, 2 * HU, d_grads + lo.p_hb[i][1], 128, st);
  }
  // ---- dense ----
  bf16* dhb = W<bf16>(s, lo.w_dhb);
  float* dhin = W<float>(s, lo.w_dhin);
  rc = launch_bias_act({.a = dhb, .C = HU, .T = T, .B = B, .w = s.pk + lo.k_denseT, .N = 128, .wK = HU, .BN = 128, .out_f32 = dhin, .ldo = M, .nvalid = M}, st);
  if (rc) return rc;
  { ActT maps[2] = {make_act(W<bf16>(s, lo.w_hin), M, T, B), make_act(dhb, HU, T, B)}; rc = wgrad(maps, 2); if (rc) return rc; }
  colsum(dhb, N, HU, HU, d_grads + lo.p_db, 128, st);
  // ---- proj2 (BN, linear) ----
  float* bsum = W<float>(s, lo.w_bsum);
  bf16* dY2b = W<bf16>(s, lo.w_dY2b);
  T2_CHECK_CUDA(cudaMemsetAsync(bsum, 0, 2LL * KC * sizeof(float), st));
  bn_bwd(dhin, M, W<float>(s, lo.w_Y2), M, 0, W<float>(s, lo.w_st2), M, bsum, d_params + lo.proj2.p.gamma, dY2b, 128, d_grads + lo.proj2.p.gamma,
         d_grads + lo.proj2.p.beta, N, M, 0, BnDropout{}, 128, st);
  int sh[16];
  bf16* d2 = W<bf16>(s, lo.w_d2);
  for (int j = 0; j < lo.PK; ++j) sh[j] = -conv_tap_shift(lo.PK, j);
  rc = launch_bias_act({.a = dY2b, .C = lo.proj2.coutp, .ld = 128, .T = T, .B = B, .ntaps = lo.PK, .shifts = sh, .w = s.pk + lo.proj2.k_wT,
                        .N = (PJc + 127) / 128 * 128, .wK = lo.PK * lo.proj2.coutp, .BN = 256, .out_bf16 = d2, .ldo = PJc, .nvalid = PJc},
                       st);
  if (rc) return rc;
  { ActT maps[2] = {make_act(W<bf16>(s, lo.w_X1), PJc, T, B), make_act(dY2b, M, T, B, 1, 128)}; rc = wgrad(maps, 2); if (rc) return rc; }
  colsum(dY2b, N, M, 128, d_grads + lo.proj2.p.bias, 128, st);
  // ---- proj1 (ReLU, BN) ----
  bf16* d1 = W<bf16>(s, lo.w_d1);
  T2_CHECK_CUDA(cudaMemsetAsync(bsum, 0, 2LL * KC * sizeof(float), st));
  bn_bwd(d2, PJc, W<bf16>(s, lo.w_Y1), PJc, 0, W<float>(s, lo.w_st1), PJc, bsum, d_params + lo.proj1.p.gamma, d1, PJc, d_grads + lo.proj1.p.gamma,
         d_grads + lo.proj1.p.beta, N, PJc, 1, BnDropout{}, 256, st);
  bf16* dP = W<bf16>(s, lo.w_dP);
  rc = launch_bias_act({.a = d1, .C = PJc, .T = T, .B = B, .ntaps = lo.PK, .shifts = sh, .w = s.pk + lo.proj1.k_wT, .N = KC, .wK = lo.PK * lo.proj1.coutp,
                        .BN = 256, .out_bf16 = dP, .ldo = KC, .nvalid = KC},
                       st);
  if (rc) return rc;
  { ActT maps[2] = {make_act(W<bf16>(s, lo.w_P), KC, T, B), make_act(d1, PJc, T, B)}; rc = wgrad(maps, 2); if (rc) return rc; }
  colsum(d1, N, PJc, PJc, d_grads + lo.proj1.p.bias, 256, st);
  // ---- max-pool, conv bank ----
  bf16* dbank = W<bf16>(s, lo.w_dbank);
  maxpool_bwd(W<bf16>(s, lo.w_Xb), dP, dbank, N, T, KC, st);
  T2_CHECK_CUDA(cudaMemsetAsync(bsum, 0, 2LL * KC * sizeof(float), st));
  bf16* dpre = dP;                              // pre-activation gradients of the bank reuse the (consumed) dP buffer
  for (int k = 1; k <= lo.K; ++k) {
    const CConv& L = lo.bank[k - 1];
    const int c0 = (k - 1) * lo.CC;
    bn_bwd(dbank, KC, W<bf16>(s, lo.w_Y), KC, c0, W<float>(s, lo.w_stb), KC, bsum, d_params + L.p.gamma, dpre, KC, d_grads + L.p.gamma,
           d_grads + L.p.beta, N, lo.CC, 1, BnDropout{}, 128, st);
    colsum(dpre + c0, N, lo.CC, KC, d_grads + L.p.bias, 128, st);
  }
  { ActT maps[2] = {make_act(W<bf16>(s, lo.w_x0), M, T, B), make_act(dpre, KC, T, B)}; rc = wgrad(maps, 2); if (rc) return rc; }
  for (int g = 0; g < 3; ++g) {
    float* dx = W<float>(s, lo.w_dx0[g]);
    if (g >= lo.n_grp) { T2_CHECK_CUDA(cudaMemsetAsync(dx, 0, N * 128 * sizeof(float), st)); continue; }
    int shifts[16], k0s[16], n = 0;
    for (int l = lo.grp_first[g]; l < lo.grp_first[g + 1]; ++l)
      for (int j = 0; j < lo.bank[l].k; ++j, ++n) { shifts[n] = -conv_tap_shift(lo.bank[l].k, j); k0s[n] = l * lo.CC; }
    rc = launch_bias_act({.a = dpre, .C = lo.CC, .k0s = k0s, .Ctot = KC, .T = T, .B = B, .ntaps = n, .shifts = shifts, .w = s.pk + lo.k_bankT[g], .N = 128,
                          .wK = n * lo.CC, .BN = 128, .out_f32 = dx, .ldo = 128, .nvalid = M},
                         st);
    if (rc) return rc;
  }
  dmel_k<<<grid1d(N * M), 256, 0, st>>>(W<float>(s, lo.w_dx0[0]), W<float>(s, lo.w_dx0[1]), W<float>(s, lo.w_dx0[2]), dhin, d_mel_grad, N, M); t2_count_launch();
  if (lo.c.reg_weight != 0.f) launch_reg_grad(d_params, d_grads, W<long long>(s, lo.w_regtab), lo.n_reg, lo.c.reg_weight, st);
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

extern "C" int t2_cbhg_workspace_tensor(const t2_cbhg_config_t* cfg, void* d_workspace, const char* name, void** ptr, long long* count) {
  CL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  T2_REQUIRE(d_workspace && name && ptr, T2_ERR_INVALID_ARG, "cbhg_workspace_tensor: null pointer");
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  const std::string n(name);
  long long off = -1, cnt = 0;
  // split_bf16 doubles the rows of the bf16 tensors below to [hi | lo] (include/t2b200.h); highway_input pads M to a multiple of 64 per half
  const long long xm = lo.c.split_bf16 ? 2 : 1, mw = lo.c.split_bf16 ? 2LL * ((lo.M + 63) / 64 * 64) : lo.M;
  if (n == "linear_outputs") { off = lo.w_lin; cnt = lo.N * lo.NFP; }           // fp32 [B][T][num_freq rounded up to 8] (row pitch!)
  else if (n == "rnn_outputs") { off = lo.w_out; cnt = lo.N * 2 * lo.RU * xm; } // bf16 [B][T][2 RU]
  else if (n == "highway_input") { off = lo.w_hin; cnt = lo.N * mw; }          // bf16 [B][T][M]
  else if (n == "bank_outputs") { off = lo.w_Xb; cnt = lo.N * lo.KC * xm; }    // bf16 [B][T][K CC] (after batch norm)
  else if (n == "pooled_outputs") { off = lo.w_P; cnt = lo.N * lo.KC * xm; }   // bf16 [B][T][K CC] (after the max-pool)
  else if (n == "gru_input") { off = lo.w_hb[lo.NH]; cnt = lo.N * lo.HU * xm; } // bf16 [B][T][HU]: the last highway output
  // fp32 [B][T][6 RU] input projections [fw gates | fw cand | bw gates | bw cand] (no biases); valid between the forward and the
  // backward pass only: the highway backward reuses the buffer
  else if (n == "gru_xp") { off = lo.w_XP; cnt = lo.N * 6 * lo.RU; }
  else if (n == "gru_dout") { off = lo.w_dout; cnt = lo.N * 2 * lo.RU; }       // fp32 [B][T][2 RU]: d loss / d rnn_outputs
  else if (n == "gru_dxp") { off = lo.w_dXP; cnt = lo.N * 6 * lo.RU; }         // bf16 [B][T][6 RU]: [dr_pre | du_pre | dc_pre] per direction
  else {
    // training stashes, bf16 [B][T][RU]: gru_{r,u,c,rh}_{fw,bw} (reset gate, update gate, candidate, r * h_prev)
    const char* dn[2] = {"fw", "bw"};
    for (int d = 0; d < 2 && off < 0; ++d) {
      const std::string sfx = std::string("_") + dn[d];
      if (n == "gru_r" + sfx) off = lo.w_gr[d];
      else if (n == "gru_u" + sfx) off = lo.w_gu[d];
      else if (n == "gru_c" + sfx) off = lo.w_gc[d];
      else if (n == "gru_rh" + sfx) off = lo.w_grh[d];
    }
    cnt = lo.N * lo.RU;
  }
  T2_REQUIRE(off >= 0, T2_ERR_INVALID_ARG, "cbhg_workspace_tensor: unknown tensor '%s'", name);
  *ptr = ws + off;
  if (count) *count = cnt;
  return T2_OK;
}

// test hook: one production kernel on caller buffers (include/t2b200.h, T2_DBG_CBHG_*)
extern "C" int t2_dbg_cbhg_kernel(const t2_dbg_kernel_t* call, void* stream) {
  T2_REQUIRE(call != nullptr, T2_ERR_INVALID_ARG, "dbg_cbhg_kernel: null call");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  void* const* p = call->p;
  const long long* i = call->i;
  switch (call->kernel) {
    case T2_DBG_CBHG_BN_FWD: {
      const long long rows = i[0];
      const int C = int(i[1]), ld = int(i[2]), c0 = int(i[3]), Ct = int(i[4]), thr = int(i[7]);
      T2_REQUIRE(rows >= 1 && C >= 1 && c0 >= 0 && c0 + C <= ld && c0 + C <= Ct && (thr == 128 || thr == 256) && p[0] && (p[1] || p[2]) && p[4] &&
                     p[5] && p[6] && p[7] && p[8],
                 T2_ERR_INVALID_ARG, "dbg_cbhg_kernel BN_FWD: bad arguments");
      T2_REQUIRE(i[8] == 0 || i[8] == 1, T2_ERR_INVALID_ARG, "dbg_cbhg_kernel BN_FWD: split i[8] = %lld is not 0 or 1", i[8]);
      if (i[6])
        bn_fwd(static_cast<const float*>(p[0]), ld, c0, static_cast<bf16*>(p[1]), int(i[8]), static_cast<float*>(p[2]), static_cast<const float*>(p[3]),
               static_cast<float*>(p[4]), Ct, static_cast<const float*>(p[5]), static_cast<const float*>(p[6]), static_cast<float*>(p[7]),
               static_cast<float*>(p[8]), rows, C, int(i[5]), BnDropout{}, thr, st);
      else
        bn_fwd(static_cast<const bf16*>(p[0]), ld, c0, static_cast<bf16*>(p[1]), int(i[8]), static_cast<float*>(p[2]), static_cast<const float*>(p[3]),
               static_cast<float*>(p[4]), Ct, static_cast<const float*>(p[5]), static_cast<const float*>(p[6]), static_cast<float*>(p[7]),
               static_cast<float*>(p[8]), rows, C, int(i[5]), BnDropout{}, thr, st);
      break;
    }
    case T2_DBG_CBHG_BN_BWD: {
      const long long rows = i[0];
      const int C = int(i[1]), ldg = int(i[2]), ld = int(i[3]), c0 = int(i[4]), Ct = int(i[5]), ldd = int(i[6]), act = int(i[7]), thr = int(i[8]);
      T2_REQUIRE(rows >= 1 && C >= 1 && c0 >= 0 && c0 + C <= ld && c0 + C <= ldg && c0 + C <= ldd && c0 + C <= Ct && (act == 0 || act == 1) &&
                     (thr == 128 || thr == 256) && p[0] && p[1] && p[2] && p[3] && p[4] && p[5] && p[6] && p[7],
                 T2_ERR_INVALID_ARG, "dbg_cbhg_kernel BN_BWD: bad arguments");
      if (i[9])
        bn_bwd(static_cast<const float*>(p[0]), ldg, static_cast<const float*>(p[1]), ld, c0, static_cast<const float*>(p[2]), Ct,
               static_cast<float*>(p[3]), static_cast<const float*>(p[4]), static_cast<bf16*>(p[5]), ldd, static_cast<float*>(p[6]),
               static_cast<float*>(p[7]), rows, C, act, BnDropout{}, thr, st);
      else
        bn_bwd(static_cast<const bf16*>(p[0]), ldg, static_cast<const bf16*>(p[1]), ld, c0, static_cast<const float*>(p[2]), Ct,
               static_cast<float*>(p[3]), static_cast<const float*>(p[4]), static_cast<bf16*>(p[5]), ldd, static_cast<float*>(p[6]),
               static_cast<float*>(p[7]), rows, C, act, BnDropout{}, thr, st);
      break;
    }
    case T2_DBG_CBHG_POOL_FWD:
    case T2_DBG_CBHG_POOL_BWD: {
      const bool fwd = call->kernel == T2_DBG_CBHG_POOL_FWD;
      T2_REQUIRE(i[0] >= 1 && i[1] >= 1 && i[0] % i[1] == 0 && i[2] >= 1 && p[0] && p[1] && (fwd || p[2]), T2_ERR_INVALID_ARG,
                 "dbg_cbhg_kernel POOL: bad arguments");
      T2_REQUIRE(!fwd || i[3] == 0 || i[3] == 1, T2_ERR_INVALID_ARG, "dbg_cbhg_kernel POOL_FWD: split i[3] = %lld is not 0 or 1", i[3]);
      if (fwd) maxpool_fwd(static_cast<const bf16*>(p[0]), static_cast<bf16*>(p[1]), i[0], int(i[1]), int(i[2]), int(i[3]), st);
      else maxpool_bwd(static_cast<const bf16*>(p[0]), static_cast<const bf16*>(p[1]), static_cast<bf16*>(p[2]), i[0], int(i[1]), int(i[2]), st);
      break;
    }
    case T2_DBG_CBHG_HIGHWAY_FWD:
      T2_REQUIRE(i[0] >= 1 && i[1] >= 1 && p[0] && p[1] && p[2] && p[3] && p[4] && p[5], T2_ERR_INVALID_ARG, "dbg_cbhg_kernel HIGHWAY_FWD: bad arguments");
      T2_REQUIRE(i[2] == 0 || i[2] == 1, T2_ERR_INVALID_ARG, "dbg_cbhg_kernel HIGHWAY_FWD: split i[2] = %lld is not 0 or 1", i[2]);
      highway_fwd(static_cast<const float*>(p[0]), static_cast<const float*>(p[1]), static_cast<const float*>(p[2]), static_cast<const float*>(p[3]),
                  static_cast<float*>(p[4]), static_cast<bf16*>(p[5]), static_cast<bf16*>(p[6]), i[0], int(i[1]), int(i[2]), st);
      break;
    case T2_DBG_CBHG_HIGHWAY_BWD:
      T2_REQUIRE(i[0] >= 1 && i[1] >= 1 && p[0] && p[1] && p[2] && p[3] && p[4], T2_ERR_INVALID_ARG, "dbg_cbhg_kernel HIGHWAY_BWD: bad arguments");
      highway_bwd(static_cast<const float*>(p[0]), static_cast<const bf16*>(p[1]), static_cast<const float*>(p[2]), static_cast<bf16*>(p[3]),
                  static_cast<float*>(p[4]), i[0], int(i[1]), st);
      break;
    case T2_DBG_CBHG_GRU_FWD: {
      GruArgs a;
      memset(&a, 0, sizeof(a));
      a.params = static_cast<const float*>(p[0]); a.XP = static_cast<const float*>(p[1]); a.out = static_cast<bf16*>(p[2]);
      for (int d = 0; d < 2; ++d) {
        a.r[d] = static_cast<bf16*>(p[3 + 4 * d]); a.u[d] = static_cast<bf16*>(p[4 + 4 * d]);
        a.c[d] = static_cast<bf16*>(p[5 + 4 * d]); a.rh[d] = static_cast<bf16*>(p[6 + 4 * d]);
        a.p_gk[d] = i[4 + 4 * d]; a.p_ck[d] = i[5 + 4 * d]; a.p_gb[d] = i[6 + 4 * d]; a.p_cb[d] = i[7 + 4 * d];
      }
      for (int k = 0; k < 4; ++k)   // B, T, HU, RU: in int range before the narrowing below
        T2_REQUIRE(i[k] >= 1 && i[k] <= (1 << 20), T2_ERR_UNSUPPORTED_SHAPE, "dbg_cbhg_kernel GRU_FWD: B, T, HU, RU must be in [1, 2^20] (i[%d] = %lld)", k, i[k]);
      a.B = int(i[0]); a.T = int(i[1]); a.HU = int(i[2]); a.RU = int(i[3]);
      T2_REQUIRE(i[12] == 0 || i[12] == 1, T2_ERR_INVALID_ARG, "dbg_cbhg_kernel GRU_FWD: split i[12] = %lld is not 0 or 1", i[12]);
      int rc = check_gru_fwd(a, int(i[12]));
      if (!rc) rc = gru_setup();
      return rc ? rc : launch_gru_fwd(a, int(i[12]), st);
    }
    case T2_DBG_CBHG_GRU_BWD: {
      GruBwdArgs a;
      memset(&a, 0, sizeof(a));
      a.params = static_cast<const float*>(p[0]); a.dout = static_cast<const float*>(p[1]); a.out = static_cast<const bf16*>(p[2]);
      for (int d = 0; d < 2; ++d) {
        a.r[d] = static_cast<const bf16*>(p[3 + 3 * d]); a.u[d] = static_cast<const bf16*>(p[4 + 3 * d]); a.c[d] = static_cast<const bf16*>(p[5 + 3 * d]);
        a.p_gk[d] = i[4 + 2 * d]; a.p_ck[d] = i[5 + 2 * d];
      }
      a.dXP = static_cast<bf16*>(p[9]);
      for (int k = 0; k < 4; ++k)   // B, T, HU, RU: in int range before the narrowing below
        T2_REQUIRE(i[k] >= 1 && i[k] <= (1 << 20), T2_ERR_UNSUPPORTED_SHAPE, "dbg_cbhg_kernel GRU_BWD: B, T, HU, RU must be in [1, 2^20] (i[%d] = %lld)", k, i[k]);
      a.B = int(i[0]); a.T = int(i[1]); a.HU = int(i[2]); a.RU = int(i[3]);
      int rc = check_gru_bwd(a);
      if (!rc) rc = gru_setup();
      return rc ? rc : launch_gru_bwd(a, st);
    }
    case T2_DBG_CBHG_LINEAR: {
      const long long B = i[0], T = i[1];
      const int NF = int(i[2]), NFP = int(i[3]), n_prio = int(i[4]), clip = int(i[5]);
      T2_REQUIRE(p[0] && p[3] && B >= 1 && B <= 65535 && T >= 1 && T <= 65535 && NF >= 1 && NFP >= NF && n_prio >= 1 && n_prio <= NF &&
                     (clip == 0 || clip == 1),
                 T2_ERR_INVALID_ARG, "dbg_cbhg_kernel LINEAR: bad arguments");
      float* scal = static_cast<float*>(p[3]);
      const float* tgt = static_cast<const float*>(p[1]);
      const long long N = B * T;
      lin_norm_k<<<1, 1, 0, st>>>(scal, static_cast<const int*>(p[5]), int(B), int(T), NF, n_prio); t2_count_launch();
      lin_finish_k<<<grid1d(N * NFP), 256, 0, st>>>(static_cast<float*>(p[0]), tgt, tgt ? static_cast<bf16*>(p[2]) : nullptr, scal, N, int(T), NF, NFP,
                                                    n_prio, clip, call->f[0], call->f[1], static_cast<const int*>(p[5]));
      t2_count_launch();
      if (p[4]) { loss_out_k<<<1, 1, 0, st>>>(scal, static_cast<float*>(p[4]), call->f[2]); t2_count_launch(); }
      break;
    }
    case T2_DBG_CBHG_ADD: {
      T2_REQUIRE(i[0] == 0 || i[0] == 1, T2_ERR_INVALID_ARG, "dbg_cbhg_kernel ADD: bad kernel selector %lld", i[0]);
      if (i[0] == 0) {
        T2_REQUIRE(p[0] && p[1] && i[1] >= 1, T2_ERR_INVALID_ARG, "dbg_cbhg_kernel ADD add_k: bad arguments");
        add_k<<<grid1d(i[1]), 256, 0, st>>>(static_cast<float*>(p[0]), static_cast<const float*>(p[1]), static_cast<bf16*>(p[2]), i[1]);
      } else {
        T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && p[4] && i[1] >= 1 && i[2] >= 1 && i[2] <= 128, T2_ERR_INVALID_ARG,
                   "dbg_cbhg_kernel ADD dmel_k: bad arguments");
        dmel_k<<<grid1d(i[1] * i[2]), 256, 0, st>>>(static_cast<const float*>(p[0]), static_cast<const float*>(p[1]), static_cast<const float*>(p[2]),
                                                  static_cast<const float*>(p[3]), static_cast<float*>(p[4]), i[1], int(i[2]));
      }
      t2_count_launch();
      break;
    }
    default:
      return t2_set_error(T2_ERR_INVALID_ARG, "dbg_cbhg_kernel: unknown kernel id %d", call->kernel);
  }
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}
