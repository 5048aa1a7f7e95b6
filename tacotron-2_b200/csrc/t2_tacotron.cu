// t2_tacotron.cu — Tacotron-2 mel-spectrogram predictor (training graph, teacher forcing, r = 1) on the GEMM engine.
//
// Replaces tacotron/models/tacotron.py:104-200 (graph assembly), :315-354 (losses), modules.py (conv1d / BN blocks,
// ZoneoutLSTMCell, Prenet, projections, Postnet), attention.py (location-sensitive attention) and
// Architecture_wrappers.py:169-213 (decoder step order) of the reference.
//
// Mapping onto the H100:
//   * everything that is batched over time runs on act_gemm_kernel: the k=5 'same' convolutions are 5 row-shifted
//     K-segments (zero padding = TMA out-of-bounds fill), prenet / LSTM input projections / frame+stop projections /
//     attention keys are plain 1x1 GEMMs; weight gradients of all of them go through wgrad_gemm_kernel.
//   * the recurrences (BiLSTM encoder, 2-layer decoder LSTM) use the SWAPPED GEMM: the permuted recurrent weight
//     matrix is the 128-row M operand, the batch is N = 32, and the LSTM cell + zoneout is the epilogue (EPI_LSTM).
//     Backward-through-time uses the transposed weights the same way (EPI_TOUT) and stashes gate gradients so that
//     every recurrent weight gradient is ONE wgrad GEMM over all time steps afterwards.
//   * one attention CTA per batch item per step (query projection, location conv, energies, masked softmax, context).
#include <stdlib.h>
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

struct ConvL {   // one conv + BN block
  int cin, cout, k, act;   // act: 1 relu, 2 tanh, 0 none
  ConvBnParams p;
  long long k_w, k_wT;     // packed forward [cout][k*cinp], packed dgrad [cinp][k*cout]
  int cinp;                // cin rounded up to 64
  long long w_y, w_x;      // workspace: y (post-activation, pre-BN) bf16 [B][T][cout], x = block output bf16
  long long w_stats;       // fp32 [4][cout]: sums of (y - y[0]) / (y - y[0])^2 (fwd) then mean / rstd ; [2][cout] bwd sums
  int stream;              // dropout hash stream
};

struct TL {  // layout
  t2_taco_config_t c;
  int B, Ti, To, E, C, H, D, A, F, KA, P1, P2, M, PC, NS;
  std::vector<Param> params;
  long long n_params;
  long long p_emb, p_elk[2], p_elb[2], p_mem, p_qry, p_lck, p_lcb, p_lfl, p_v, p_ba, p_p1k, p_p1b, p_p2k, p_p2b;
  long long p_l1k, p_l1b, p_l2k, p_l2b, p_fk, p_fb, p_sk, p_sb, p_ppk, p_ppb;
  std::vector<ConvL> enc, post;
  // packed (bytes)
  long long k_encWx[2], k_encWr[2], k_encWrT[2], k_encWxT, k_mem, k_memT, k_p1, k_p1T, k_p2, k_p2T, k_l1x, k_l1xT, k_l1r, k_l1rT;
  long long k_l2, k_l2T, k_proj, k_projT, k_pp, k_ppT, k_qT, packed_bytes;
  // workspace (bytes)
  long long w_emb, w_encpre[2], w_ench[2], w_encc[2], w_encg[2], w_enct[2], w_memory, w_values, w_keys, w_decin, w_pn1, w_pn2;
  long long w_pre1, w_S1, w_S2, w_PI, w_c1, w_c2, w_g1, w_g2, w_t1, w_t2, w_cum, w_alpha, w_projo, w_decbm, w_decf, w_stop;
  long long w_resid, w_mel, w_scal, w_zero, w_tlen;
  // backward
  long long w_dmel, w_dY, w_ddec_tm, w_dPI, w_dh1ext, w_dh2ext, w_dhs1, w_dhs2, w_dcs1, w_dcs2, w_dg1, w_dg2, w_dgstep;
  long long w_dctxl, w_dctx_all, w_dq_all, w_dcum, w_cumrun, w_dkeys, w_dvalues, w_attacc, w_dpn2, w_dpn1;
  long long w_dencpre[2], w_dx3, w_encdh[2], w_encdc[2], w_encdg, w_demb, w_tiles, w_packjobs, w_regtab;
  long long w_ddecf, w_encdgall[2], w_dkeysb, w_dz, w_attU;
  long long w_tfsel, w_dfb;   // teacher_forcing_ratio < 1: per-step choices int32 [To], d(fed-back frame) fp32 [B][M]
  // row pitches (elements) of the decoder-side bf16 rows; split_bf16 widens them (see build)
  int ld_decin, ld_pn1, ld_pn2, ld_S1, ld_S2, ld_PI, ld_mem;
  std::vector<int> tile_off, tile_cnt;  // per wgrad launch (fixed order, see build_tiles)
  long long workspace_bytes;
  int n_packjobs, n_reg;
};

int build(const t2_taco_config_t* cfg, TL& lo, std::vector<PackJob>* jobs_out) {
  T2_REQUIRE(cfg != nullptr, T2_ERR_INVALID_ARG, "null config");
  lo.c = *cfg;
  lo.B = cfg->B; lo.Ti = cfg->T_in; lo.To = cfg->T_out; lo.E = cfg->embedding_dim; lo.C = cfg->enc_conv_channels;
  lo.H = cfg->encoder_lstm_units; lo.D = cfg->decoder_lstm_units; lo.A = cfg->attention_dim; lo.F = cfg->attention_filters;
  lo.KA = cfg->attention_kernel; lo.P1 = cfg->prenet1; lo.P2 = cfg->prenet2; lo.M = cfg->num_mels; lo.PC = cfg->postnet_channels;
  lo.NS = cfg->n_symbols;
  T2_REQUIRE(lo.B >= 1 && lo.B <= 256 && lo.Ti >= 1 && lo.To >= 1, T2_ERR_INVALID_ARG, "bad B / T_in / T_out");
  T2_REQUIRE(lo.E % 64 == 0 && lo.C % 64 == 0 && lo.PC % 64 == 0 && lo.P1 % 64 == 0 && lo.P2 % 64 == 0, T2_ERR_UNSUPPORTED_SHAPE,
             "channel counts must be multiples of 64");
  T2_REQUIRE(lo.H % 32 == 0 && lo.D % 32 == 0 && (4 * lo.H) % 128 == 0 && (2 * lo.H) % 64 == 0, T2_ERR_UNSUPPORTED_SHAPE, "LSTM sizes");
  T2_REQUIRE(lo.A % 64 == 0 && lo.A <= 128 && lo.F <= 32 && lo.KA % 2 == 1 && lo.KA <= 31, T2_ERR_UNSUPPORTED_SHAPE, "attention sizes");
  T2_REQUIRE(lo.M % 8 == 0 && lo.M + 1 <= 128 && lo.Ti <= 1024, T2_ERR_UNSUPPORTED_SHAPE, "num_mels / T_in");
  T2_REQUIRE(cfg->enc_conv_layers >= 1 && cfg->enc_conv_layers <= 8 && cfg->postnet_layers >= 1 && cfg->postnet_layers <= 8,
             T2_ERR_INVALID_ARG, "layer counts");
  T2_REQUIRE(cfg->teacher_forcing_ratio >= 0.f && cfg->teacher_forcing_ratio <= 1.f, T2_ERR_INVALID_ARG,
             "teacher_forcing_ratio %g outside [0, 1]", double(cfg->teacher_forcing_ratio));
  T2_REQUIRE(cfg->unmasked_encoder == 0 || cfg->unmasked_encoder == 1, T2_ERR_INVALID_ARG, "unmasked_encoder %d is not 0 or 1",
             cfg->unmasked_encoder);
  T2_REQUIRE(cfg->noncumulative_weights == 0 || cfg->noncumulative_weights == 1, T2_ERR_INVALID_ARG, "noncumulative_weights %d is not 0 or 1",
             cfg->noncumulative_weights);
  T2_REQUIRE(!cfg->split_bf16 || (lo.H % 64 == 0 && lo.D % 64 == 0), T2_ERR_UNSUPPORTED_SHAPE,
             "split_bf16: the LSTM sizes must be multiples of 64 (the hi / lo halves of a state row are whole 64-wide K blocks)");
  // ---- parameters (order == oracle/tacotron.py:param_shapes) ----
  lo.n_params = 0; lo.params.clear(); lo.enc.clear(); lo.post.clear();
  lo.p_emb = add_param(lo.params, lo.n_params, "inputs_embedding", {lo.NS, lo.E});
  int cin = lo.E;
  for (int i = 0; i < cfg->enc_conv_layers; ++i) {
    ConvL L; L.cin = cin; L.cout = lo.C; L.k = cfg->enc_conv_kernel; L.act = 1; L.stream = 10 + i;
    char b[64]; snprintf(b, sizeof(b), "encoder_convolutions/conv_layer_%d/", i + 1);
    L.p = add_conv_bn_params(lo.params, lo.n_params, b, L.k, L.cin, L.cout); lo.enc.push_back(L); cin = lo.C;
  }
  const char* dn[2] = {"fw", "bw"};
  for (int d = 0; d < 2; ++d) {
    lo.p_elk[d] = add_param(lo.params, lo.n_params, std::string("encoder_LSTM/") + dn[d] + "/kernel", {lo.C + lo.H, 4 * lo.H});
    lo.p_elb[d] = add_param(lo.params, lo.n_params, std::string("encoder_LSTM/") + dn[d] + "/bias", {4 * lo.H});
  }
  lo.p_mem = add_param(lo.params, lo.n_params, "attention/memory_layer/kernel", {2 * lo.H, lo.A});
  lo.p_qry = add_param(lo.params, lo.n_params, "attention/query_layer/kernel", {lo.D, lo.A});
  lo.p_lck = add_param(lo.params, lo.n_params, "attention/location_features_convolution/kernel", {lo.KA, 1, lo.F});
  lo.p_lcb = add_param(lo.params, lo.n_params, "attention/location_features_convolution/bias", {lo.F});
  lo.p_lfl = add_param(lo.params, lo.n_params, "attention/location_features_layer/kernel", {lo.F, lo.A});
  lo.p_v = add_param(lo.params, lo.n_params, "attention/attention_variable_projection", {lo.A});
  lo.p_ba = add_param(lo.params, lo.n_params, "attention/attention_bias", {lo.A});
  lo.p_p1k = add_param(lo.params, lo.n_params, "decoder_prenet/dense_1/kernel", {lo.M, lo.P1}); lo.p_p1b = add_param(lo.params, lo.n_params, "decoder_prenet/dense_1/bias", {lo.P1});
  lo.p_p2k = add_param(lo.params, lo.n_params, "decoder_prenet/dense_2/kernel", {lo.P1, lo.P2}); lo.p_p2b = add_param(lo.params, lo.n_params, "decoder_prenet/dense_2/bias", {lo.P2});
  const int K1 = lo.P2 + 2 * lo.H + lo.D, K2 = 2 * lo.D;
  lo.p_l1k = add_param(lo.params, lo.n_params, "decoder_LSTM/cell_1/kernel", {K1, 4 * lo.D}); lo.p_l1b = add_param(lo.params, lo.n_params, "decoder_LSTM/cell_1/bias", {4 * lo.D});
  lo.p_l2k = add_param(lo.params, lo.n_params, "decoder_LSTM/cell_2/kernel", {K2, 4 * lo.D}); lo.p_l2b = add_param(lo.params, lo.n_params, "decoder_LSTM/cell_2/bias", {4 * lo.D});
  const int PIK = lo.D + 2 * lo.H;
  lo.p_fk = add_param(lo.params, lo.n_params, "linear_transform_projection/kernel", {PIK, lo.M}); lo.p_fb = add_param(lo.params, lo.n_params, "linear_transform_projection/bias", {lo.M});
  lo.p_sk = add_param(lo.params, lo.n_params, "stop_token_projection/kernel", {PIK, 1}); lo.p_sb = add_param(lo.params, lo.n_params, "stop_token_projection/bias", {1});
  cin = lo.M;
  for (int i = 0; i < cfg->postnet_layers; ++i) {
    ConvL L; L.cin = cin; L.cout = lo.PC; L.k = cfg->postnet_kernel; L.act = (i + 1 < cfg->postnet_layers) ? 2 : 0; L.stream = 30 + i;
    char b[64]; snprintf(b, sizeof(b), "postnet_convolutions/conv_layer_%d/", i + 1);
    L.p = add_conv_bn_params(lo.params, lo.n_params, b, L.k, L.cin, L.cout); lo.post.push_back(L); cin = lo.PC;
  }
  lo.p_ppk = add_param(lo.params, lo.n_params, "postnet_projection/kernel", {lo.PC, lo.M}); lo.p_ppb = add_param(lo.params, lo.n_params, "postnet_projection/bias", {lo.M});

  // ---- packed operands + pack jobs ----
  std::vector<PackJob> jobs;
  Arena pk;
  const bool split = cfg->split_bf16 != 0;
  auto conv_pack = [&](ConvL& L) {
    L.cinp = (L.cin + 63) / 64 * 64;
    L.k_w = pk.take(fwd_operand_bytes(L.cout, L.k * L.cinp, split));
    L.k_wT = pk.take(2LL * L.cinp * L.k * L.cout);
    for (int j = 0; j < L.k; ++j) {
      add_pack_fwd(jobs, split, L.p.kernel + (long long)j * L.cin * L.cout, L.cin, L.cout, L.k_w, L.k * L.cinp, j * L.cinp, L.cinp);   // fwd: [cout][tap j | cin]
      add_pack(jobs, L.p.kernel + (long long)j * L.cin * L.cout, L.cin, L.cout, L.k_wT, L.k * L.cout, 0, j * L.cout);     // dgrad: [cin][tap j | cout]
    }
  };
  for (auto& L : lo.enc) conv_pack(L);
  for (auto& L : lo.post) conv_pack(L);
  for (int d = 0; d < 2; ++d) {
    lo.k_encWx[d] = pk.take(fwd_operand_bytes(4 * lo.H, lo.C, split));            // [4H][C]  input projection (natural gate order)
    add_pack_fwd(jobs, split, lo.p_elk[d], lo.C, 4 * lo.H, lo.k_encWx[d], lo.C, 0, lo.C);
    lo.k_encWr[d] = pk.take(fwd_operand_bytes(4 * lo.H, lo.H, split));   // [4H perm][H] recurrent, rows permuted for EPI_LSTM
    add_pack_fwd(jobs, split, lo.p_elk[d] + (long long)lo.C * 4 * lo.H, lo.H, 4 * lo.H, lo.k_encWr[d], lo.H, 0, lo.H, 1.f, lo.H);
    lo.k_encWrT[d] = pk.take(2LL * lo.H * 4 * lo.H);           // [H][4H] for the backward step
    add_pack(jobs, lo.p_elk[d] + (long long)lo.C * 4 * lo.H, lo.H, 4 * lo.H, lo.k_encWrT[d], 4 * lo.H, 0, 0);
  }
  lo.k_encWxT = pk.take(2LL * lo.C * 8 * lo.H);                // [C][fw 4H | bw 4H]
  for (int d = 0; d < 2; ++d) add_pack(jobs, lo.p_elk[d], lo.C, 4 * lo.H, lo.k_encWxT, 8 * lo.H, 0, d * 4 * lo.H);
  lo.k_mem = pk.take(fwd_operand_bytes(lo.A, 2 * lo.H, split));
  add_pack_fwd(jobs, split, lo.p_mem, 2 * lo.H, lo.A, lo.k_mem, 2 * lo.H, 0, 2 * lo.H);
  lo.k_memT = pk.take(2LL * 2 * lo.H * lo.A); add_pack(jobs, lo.p_mem, 2 * lo.H, lo.A, lo.k_memT, lo.A, 0, 0);
  const int Mc = (lo.M + 63) / 64 * 64;   // the K slot of num_mels: the half width of the split mel rows
  lo.k_p1 = pk.take(fwd_operand_bytes(lo.P1, Mc, split));
  add_pack_fwd(jobs, split, lo.p_p1k, lo.M, lo.P1, lo.k_p1, Mc, 0, Mc);
  lo.k_p1T = pk.take(2LL * lo.M * lo.P1); add_pack(jobs, lo.p_p1k, lo.M, lo.P1, lo.k_p1T, lo.P1, 0, 0);
  lo.k_p2 = pk.take(fwd_operand_bytes(lo.P2, lo.P1, split));
  add_pack_fwd(jobs, split, lo.p_p2k, lo.P1, lo.P2, lo.k_p2, lo.P1, 0, lo.P1);
  lo.k_p2T = pk.take(2LL * lo.P1 * lo.P2); add_pack(jobs, lo.p_p2k, lo.P1, lo.P2, lo.k_p2T, lo.P2, 0, 0);
  lo.k_l1x = pk.take(fwd_operand_bytes(4 * lo.D, lo.P2, split));
  add_pack_fwd(jobs, split, lo.p_l1k, lo.P2, 4 * lo.D, lo.k_l1x, lo.P2, 0, lo.P2);
  lo.k_l1xT = pk.take(2LL * lo.P2 * 4 * lo.D); add_pack(jobs, lo.p_l1k, lo.P2, 4 * lo.D, lo.k_l1xT, 4 * lo.D, 0, 0);
  const int K1r = 2 * lo.H + lo.D;
  lo.k_l1r = pk.take(fwd_operand_bytes(4 * lo.D, K1r, split));
  add_pack_fwd(jobs, split, lo.p_l1k + (long long)lo.P2 * 4 * lo.D, K1r, 4 * lo.D, lo.k_l1r, K1r, 0, K1r, 1.f, lo.D);
  lo.k_l1rT = pk.take(2LL * K1r * 4 * lo.D); add_pack(jobs, lo.p_l1k + (long long)lo.P2 * 4 * lo.D, K1r, 4 * lo.D, lo.k_l1rT, 4 * lo.D, 0, 0);
  lo.k_l2 = pk.take(fwd_operand_bytes(4 * lo.D, K2, split));
  add_pack_fwd(jobs, split, lo.p_l2k, K2, 4 * lo.D, lo.k_l2, K2, 0, K2, 1.f, lo.D);
  lo.k_l2T = pk.take(2LL * K2 * 4 * lo.D); add_pack(jobs, lo.p_l2k, K2, 4 * lo.D, lo.k_l2T, 4 * lo.D, 0, 0);
  lo.k_proj = pk.take(fwd_operand_bytes(128, PIK, split));      // rows 0..M-1 frame projection, row M stop projection
  add_pack_fwd(jobs, split, lo.p_fk, PIK, lo.M, lo.k_proj, PIK, 0, PIK);
  add_pack_fwd(jobs, split, lo.p_sk, PIK, 1, lo.k_proj + fwd_operand_bytes(lo.M, PIK, split), PIK, 0, PIK);
  lo.k_projT = pk.take(2LL * PIK * 128);                        // [PIK][128]: cols 0..M-1 Wf, col M Ws
  add_pack(jobs, lo.p_fk, PIK, lo.M, lo.k_projT, 128, 0, 0);
  add_pack(jobs, lo.p_sk, PIK, 1, lo.k_projT, 128, 0, lo.M);
  lo.k_pp = pk.take(fwd_operand_bytes(128, lo.PC, split));
  add_pack_fwd(jobs, split, lo.p_ppk, lo.PC, lo.M, lo.k_pp, lo.PC, 0, lo.PC);
  lo.k_ppT = pk.take(2LL * lo.PC * 128); add_pack(jobs, lo.p_ppk, lo.PC, lo.M, lo.k_ppT, 128, 0, 0);
  lo.k_qT = pk.take(2LL * lo.A * lo.D * (split ? 2 : 1));     // [A][D] for the attention kernel; split: [A][hi(D) | lo(D)]
  add_pack(jobs, lo.p_qry, lo.D, lo.A, lo.k_qT, split ? 2 * lo.D : lo.D, 1, 0);
  if (split) { add_pack(jobs, lo.p_qry, lo.D, lo.A, lo.k_qT, 2 * lo.D, 1, lo.D); jobs.back().part = 2; }
  lo.packed_bytes = pk.used;
  lo.n_packjobs = int(jobs.size());

  // ---- workspace ----
  Arena ws;
  const long long B = lo.B, Ti = lo.Ti, To = lo.To;
  const long long xm = split ? 2 : 1;       // split-bf16: stored conv-stack activations are [hi | lo]; pre-batch-norm activations fp32
  const long long sm = split ? 3 : 1;       // split-bf16: recurrent state rows (the N operand of the swapped GEMMs) are [hi | lo | hi]
  lo.ld_decin = split ? 2 * Mc : lo.M; lo.ld_pn1 = lo.P1 * int(xm); lo.ld_pn2 = lo.P2 * int(xm);
  lo.ld_S1 = K1r * int(sm); lo.ld_S2 = K2 * int(sm); lo.ld_PI = PIK * int(xm); lo.ld_mem = 2 * lo.H * int(xm);
  lo.w_emb = ws.take(B * Ti * lo.E * 2 * xm);
  auto conv_ws = [&](ConvL& L, long long T) {
    L.w_y = ws.take(B * T * L.cout * (split ? 4 : 2)); L.w_x = ws.take(B * T * L.cout * 2 * xm); L.w_stats = ws.take(8LL * L.cout * 4);
  };
  for (auto& L : lo.enc) conv_ws(L, Ti);
  for (int d = 0; d < 2; ++d) {
    lo.w_encpre[d] = ws.take(B * Ti * 4 * lo.H * 4);
    lo.w_ench[d] = ws.take((Ti + 1) * B * lo.H * 2 * sm);   // h_state history, slot s = state after s processed steps
    lo.w_encc[d] = ws.take((Ti + 1) * B * lo.H * 4);
    lo.w_encg[d] = ws.take(Ti * B * 4 * lo.H * 2);
    lo.w_enct[d] = ws.take(Ti * B * lo.H * 2);
  }
  lo.w_memory = ws.take(B * Ti * lo.ld_mem * 2);
  lo.w_values = ws.take(B * Ti * lo.ld_mem * 2);
  lo.w_keys = ws.take(B * Ti * lo.A * 4);
  lo.w_decin = ws.take(B * To * lo.ld_decin * 2);           // time-major [To][B][M]; split: [hi(M) padded to Mc | lo(M) padded to Mc]
  lo.w_pn1 = ws.take(To * B * lo.ld_pn1 * 2);
  lo.w_pn2 = ws.take(To * B * lo.ld_pn2 * 2);
  lo.w_pre1 = ws.take(To * B * 4 * lo.D * 4);
  lo.w_S1 = ws.take((To + 1) * B * lo.ld_S1 * 2);
  lo.w_S2 = ws.take((To + 1) * B * lo.ld_S2 * 2);
  lo.w_PI = ws.take(To * B * lo.ld_PI * 2);
  lo.w_c1 = ws.take((To + 1) * B * lo.D * 4); lo.w_c2 = ws.take((To + 1) * B * lo.D * 4);
  lo.w_g1 = ws.take(To * B * 4 * lo.D * 2); lo.w_g2 = ws.take(To * B * 4 * lo.D * 2);
  lo.w_t1 = ws.take(To * B * lo.D * 2); lo.w_t2 = ws.take(To * B * lo.D * 2);
  lo.w_cum = ws.take(B * Ti * 4);
  lo.w_alpha = ws.take(To * B * Ti * 4);
  lo.w_projo = ws.take(To * B * 128 * 4);
  lo.w_decbm = ws.take(B * To * lo.ld_decin * 2);     /* split: [hi(M) padded to Mc | lo(M) padded to Mc] */ lo.w_decf = ws.take(B * To * lo.M * 4); lo.w_stop = ws.take(B * To * 4);
  for (auto& L : lo.post) conv_ws(L, To);
  lo.w_tlen = ws.take(B * 4);
  lo.w_resid = ws.take(B * To * 128 * 4); lo.w_mel = ws.take(B * To * lo.M * 4);
  lo.w_scal = ws.take(64 * 4);
  // backward
  lo.w_dmel = ws.take(B * To * 128 * 2);                    // bf16 [B][To][128] (cols >= M zero)
  lo.w_dY = ws.take(2 * B * (To > Ti ? To : Ti) * (lo.PC > lo.C ? lo.PC : lo.C) * 2);   // ping-pong activation grads bf16
  lo.w_ddec_tm = ws.take(To * B * 128 * 2);
  lo.w_dPI = ws.take(To * B * PIK * 4);
  lo.w_dh1ext = ws.take(B * lo.D * 4); lo.w_dh2ext = ws.take(B * lo.D * 4);
  lo.w_dhs1 = ws.take(B * lo.D * 4); lo.w_dhs2 = ws.take(B * lo.D * 4); lo.w_dcs1 = ws.take(B * lo.D * 4); lo.w_dcs2 = ws.take(B * lo.D * 4);
  lo.w_dg1 = ws.take(To * B * 4 * lo.D * 2); lo.w_dg2 = ws.take(To * B * 4 * lo.D * 2);
  lo.w_dgstep = 0;
  lo.w_dctxl = ws.take(B * 2 * lo.H * 4);
  lo.w_dctx_all = ws.take(To * B * 2 * lo.H * 2);
  lo.w_dq_all = ws.take(To * B * lo.A * 2);
  lo.w_dcum = ws.take(B * Ti * 4); lo.w_cumrun = ws.take(B * Ti * 4);
  lo.w_dkeys = ws.take(B * Ti * lo.A * 4);
  lo.w_dvalues = ws.take(B * Ti * 2 * lo.H * 4);
  lo.w_attacc = ws.take(B * (lo.KA + 2) * lo.A * 4);
  lo.w_attU = ws.take((2 * lo.KA + 4) * lo.A * 4);
  lo.w_dpn2 = ws.take(To * B * lo.P2 * 2); lo.w_dpn1 = ws.take(To * B * lo.P1 * 2);
  for (int d = 0; d < 2; ++d) {
    lo.w_dencpre[d] = ws.take(B * Ti * 4 * lo.H * 2);       // bf16 gate grads [B][Ti][4H] (batch-major, = dpre)
    lo.w_encdh[d] = ws.take(B * lo.H * 4); lo.w_encdc[d] = ws.take(B * lo.H * 4);
  }
  lo.w_encdg = ws.take(B * 4 * lo.H * 2);
  lo.w_ddecf = ws.take(B * To * lo.M * 4);
  for (int d = 0; d < 2; ++d) lo.w_encdgall[d] = ws.take(Ti * B * 4 * lo.H * 2);
  lo.w_dkeysb = ws.take(B * Ti * lo.A * 2);
  lo.w_dz = ws.take(To * B * (lo.P1 > lo.P2 ? lo.P1 : lo.P2) * 2);
  lo.w_dx3 = ws.take(B * Ti * lo.C * 2);
  lo.w_demb = ws.take(B * Ti * lo.E * 2);
  lo.w_tiles = ws.take(16384 * sizeof(WgradTile));
  lo.w_packjobs = ws.take((long long)jobs.size() * sizeof(PackJob));
  lo.n_reg = 0;
  for (auto& p : lo.params) lo.n_reg += p.reg ? 1 : 0;
  lo.w_regtab = ws.take((long long)lo.n_reg * 2 * sizeof(long long));
  lo.w_zero = ws.take(B * 4096 * 4);
  lo.w_tfsel = ws.take(To * 4);
  lo.w_dfb = ws.take(B * lo.M * 4);
  lo.workspace_bytes = ws.used;
  if (jobs_out) jobs_out->swap(jobs);
  return T2_OK;
}

// ------------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------------
__global__ void embed_fwd_kernel(const int* __restrict__ idx, const float* __restrict__ table, bf16* __restrict__ out, long long npos, int E,
                                 int split) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= npos * E) return;
  const float v = table[(long long)idx[e / E] * E + e % E];
  if (!split) { out[e] = __float2bfloat16(v); return; }
  const bf16 hi = __float2bfloat16(v);
  bf16* row = out + (e / E) * 2 * E + e % E;       // rows [hi(E) | lo(E)]
  row[0] = hi; row[E] = __float2bfloat16(v - __bfloat162float(hi));
}
__global__ void embed_bwd_kernel(const int* __restrict__ idx, const bf16* __restrict__ dx, float* __restrict__ dtable, long long npos, int E) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= npos * E) return;
  atomicAdd(dtable + (long long)idx[e / E] * E + e % E, __bfloat162float(dx[e]));
}

// memory [B][Ti][2H] -> values = memory * mask (BahdanauAttention memory masking)
__global__ void mask_values_kernel(const bf16* __restrict__ mem, const int* __restrict__ lens, bf16* __restrict__ vals, int B, int Ti, int C2) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)B * Ti * C2) return;
  const int t = int((e / C2) % Ti), b = int(e / ((long long)C2 * Ti));
  vals[e] = t < lens[b] ? mem[e] : __float2bfloat16(0.f);
}
// decoder inputs, time-major: dec_in[t][b][:] = t == 0 ? 0 : target[b][t-1][:]   (helpers.py:62-128, r = 1)
// split: rows [hi(M) | pad | lo(M) | pad] of pitch 2 Cp, Cp = ceil(M / 64) * 64 (the padding stays zero from t2_taco_init)
__global__ void decin_kernel(const float* __restrict__ tgt, bf16* __restrict__ out, int B, int To, int M, int split) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)To * B * M) return;
  const int m = int(e % M), b = int((e / M) % B), t = int(e / ((long long)M * B));
  const float v = t == 0 ? 0.f : tgt[((long long)b * To + t - 1) * M + m];
  if (!split) { out[e] = __float2bfloat16(v); return; }
  const int Cp = (M + 63) / 64 * 64;
  const bf16 hi = __float2bfloat16(v);
  bf16* row = out + (e / M) * 2 * Cp + m;
  row[0] = hi; row[Cp] = __float2bfloat16(v - __bfloat162float(hi));
}

// ---- location-sensitive attention, one CTA per batch item per decoder step (attention.py:169-226) -------------
// The location branch conv1d(k=31, 1 -> F) followed by dense(F -> A) is linear in the cumulative alignments, so it is
// evaluated as ONE 31-tap filter bank U[k][a] = sum_f K[k][f] Wl[f][a] with offset u0[a] = sum_f bK[f] Wl[f][a] + b_a[a]
// (built once per forward by att_prep_kernel); the backward pass differentiates through the same factorisation.
constexpr int kAttThreads = 512;
__device__ long long* g_att_dbg = nullptr;   // optional phase stamps (tools only): [0..15] forward, [16..31] backward
#define ATT_STAMP(i) do { if (g_att_dbg && blockIdx.x == 0 && threadIdx.x == 0) g_att_dbg[i] = clock64(); } while (0)
__global__ void att_prep_kernel(const float* __restrict__ K, const float* __restrict__ bK, const float* __restrict__ Wl,
                                const float* __restrict__ ba, float* __restrict__ U, int KA, int F, int A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (KA + 1) * A) return;
  const int k = i / A, a = i % A;
  float acc = 0.f;
  if (k < KA) { for (int f = 0; f < F; ++f) acc += K[k * F + f] * Wl[f * A + a]; }
  else { acc = ba[a]; for (int f = 0; f < F; ++f) acc += bK[f] * Wl[f * A + a]; }
  U[i] = acc;   // rows 0..KA-1: U, row KA: u0
}
struct AttArgs {
  const bf16* h2out; int ld_h2;            // query source: PI_all[t][b][0:D]
  const bf16* WqT;                          // [A][D] bf16
  const float* U;                           // [KA + 1][A]
  const float* v;
  const float* keys;                        // [B][Ti][A] fp32
  const bf16* values;                       // [B][Ti][C2]
  const int* lens;
  float* cum;                               // [B][Ti] running cumulative alignments (in/out)
  float* alpha;                             // [B][Ti] output for this step
  bf16* ctx_a; int ld_a;                    // context -> S1_all[t+1][b][0:C2]
  bf16* ctx_b; int ld_b;                    // context -> PI_all[t][b][D:]
  int B, Ti, D, A, KA, C2;
  int unmasked, noncumulative;              // t2_taco_config_t flags: pick the att_fwd_kernel instantiation (host side only)
  // split (t2_taco_config_t.split_bf16): h2out / values / the context outputs are hi + lo pairs. The lo half of h2out sits at +lo_h2,
  // of a values row at +C2 (row pitch 2 C2), of ctx_b at +lo_b; ctx_a is a swapped-GEMM state row: lo at +lo_a, hi again at +2 lo_a.
  // WqT rows are [hi(D) | lo(D)].
  int split = 0, lo_h2 = 0, lo_a = 0, lo_b = 0;
};
// q[a] = sum_k h[k] WqT[a][k]: one warp per output row (two rows in flight), lanes stride the row in 16-byte pieces so
// that every load instruction reads 512 contiguous bytes (the 4-threads-per-output form touched 32 sectors per load)
// A length-D fp32 vector that is dotted against 16-byte bf16 pieces lives in shared memory in a SPLIT layout: element
// 8p + x of the vector sits at xs[(x >> 2) * (D/2) + 4p + (x & 3)], so lane p reads two float4 at a 16-byte lane stride
// (conflict-free); the natural layout (32-byte lane stride) made every one of these loads an 8-way bank conflict.
__device__ __forceinline__ int split8(int i, int D) { return ((i >> 2) & 1) * (D >> 1) + ((i >> 3) << 2) + (i & 3); }
__device__ __forceinline__ float dot8s(const uint4 u, const float* __restrict__ xs, int p, int D) {
  const float4 lo = *reinterpret_cast<const float4*>(xs + 4 * p), hi = *reinterpret_cast<const float4*>(xs + (D >> 1) + 4 * p);
  return bf16lo(u.x) * lo.x + bf16hi(u.x) * lo.y + bf16lo(u.y) * lo.z + bf16hi(u.y) * lo.w + bf16lo(u.z) * hi.x +
         bf16hi(u.z) * hi.y + bf16lo(u.w) * hi.z + bf16hi(u.w) * hi.w;
}
// q[a] = sum_k h[k] WqT[a][k]: one warp per output row (two rows in flight), lanes stride the row in 16-byte pieces so
// that every load instruction reads 512 contiguous bytes; hs is in the split layout above
// kSplit: WqT rows are [hi(D) | lo(D)] and q = sum_k h[k] (hi + lo)[a][k]
template <bool kSplit>
__device__ __forceinline__ void att_query(const bf16* __restrict__ WqT, const float* __restrict__ hs, float* __restrict__ q, int A, int D) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, NW = kAttThreads / 32;
  const int n16 = D >> 3;   // 16-byte pieces per row
  const long long ldw = kSplit ? 2LL * D : D;
  for (int o = warp; o < A; o += 2 * NW) {
    const int o2 = o + NW;
    const uint4* w0 = reinterpret_cast<const uint4*>(WqT + (long long)o * ldw);
    const uint4* w1 = reinterpret_cast<const uint4*>(WqT + (long long)(o2 < A ? o2 : o) * ldw);
    float a0 = 0.f, a1 = 0.f;
#pragma unroll 4
    for (int i = lane; i < n16; i += 32) {
      const uint4 u0 = __ldg(w0 + i), u1 = __ldg(w1 + i);
      a0 += dot8s(u0, hs, i, D);
      a1 += dot8s(u1, hs, i, D);
      if (kSplit) {
        const uint4 l0 = __ldg(w0 + n16 + i), l1 = __ldg(w1 + n16 + i);
        a0 += dot8s(l0, hs, i, D);
        a1 += dot8s(l1, hs, i, D);
      }
    }
    a0 = warp_sum(a0); a1 = warp_sum(a1);
    if (lane == 0) { q[o] = a0; if (o2 < A) q[o2] = a1; }
  }
}
// ---- the location filter bank on tensor cores -------------------------------------------------------------------
// pl[j][n] = u0[n] + sum_k cum[j + k - half] U[k][n] is a [T_in x 32] Toeplitz matrix times the [32 x A] filter bank
// (row KA of the bank is the offset u0, matched by a column of ones): per batch item 160 x 32 x 128 - far too small for a
// wgmma tile pipeline, so it runs as warp-level mma.sync.m16n8k8 TF32 (fp32 accumulate) straight out of shared memory;
// the Toeplitz operand is never materialised (fragments read cum[j + k]). The same instruction computes the three
// products of the backward pass (dU = T^T dE, P = dE U^T for dcum). The scalar FMA form was issue/shared-memory bound:
// 20 k (forward) / 55 k (backward) cycles per step at T_in = 160 (tools/att_phases.py).
__device__ __forceinline__ uint32_t f2tf32(float f) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(f));
  return r;
}
// D(16x8) += A(16x8, row) * B(8x8, col); g = lane >> 2, t = lane & 3:
//   a0 (g, t) a1 (g+8, t) a2 (g, t+4) a3 (g+8, t+4) | b0 (k=t, n=g) b1 (k=t+4, n=g) | c0 (g, 2t) c1 (g, 2t+1) c2 (g+8, 2t) c3 (g+8, 2t+1)
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__host__ __device__ inline int att_ti16(int Ti) { return (Ti + 15) & ~15; }
__host__ __device__ inline int att_cumlen(int Ti, int KA) { return (att_ti16(Ti) + KA + 16 + 3) & ~3; }   // zero-padded cum window
__host__ __device__ inline int att_erows(int Ti, int KA) { return (att_ti16(Ti) + 2 * (KA / 2) + 15) & ~15; } // rows of dE (backward)
constexpr int kAttPad = 8;   // row padding (floats) of the filter bank / dE tiles in shared memory: conflict-free fragments
// Toeplitz element T[j][k]: cum window for the taps, a column of ones for the offset row, zero beyond
__device__ __forceinline__ float toep(const float* __restrict__ cum, int j, int k, int KA) {
  return k < KA ? cum[j + k] : (k == KA ? 1.f : 0.f);
}
// the TF32 remainder of x: tf32(x - tf32(x)) (the subtraction is exact in fp32)
__device__ __forceinline__ uint32_t tf32_rest(float x, uint32_t big) { return f2tf32(x - __uint_as_float(big)); }
// pl for the 16 rows j0.. and the 64 channels n0..: acc[nt] = C fragment of n-tile nt (8 channels each)
// kSplit (split_bf16): 3xTF32. Both operands are split as big = tf32(x), small = tf32(x - big) and the three products
// small.big + big.small + big.big are accumulated; the dropped small.small and the remainders past small are <= ~2^-21 of |cum| |U|,
// where one TF32 product alone rounds each operand by up to 2^-11.
template <bool kSplit>
__device__ __forceinline__ void loc_tile(const float* __restrict__ Us, int AP, const float* __restrict__ cum, int KA, int j0, int n0,
                                         float (&acc)[8][4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const int k = ks * 8 + t;
    uint32_t af[4];
    af[0] = f2tf32(toep(cum, j0 + g, k, KA)); af[1] = f2tf32(toep(cum, j0 + g + 8, k, KA));
    af[2] = f2tf32(toep(cum, j0 + g, k + 4, KA)); af[3] = f2tf32(toep(cum, j0 + g + 8, k + 4, KA));
    uint32_t as[4];
    if (kSplit) {
      as[0] = tf32_rest(toep(cum, j0 + g, k, KA), af[0]); as[1] = tf32_rest(toep(cum, j0 + g + 8, k, KA), af[1]);
      as[2] = tf32_rest(toep(cum, j0 + g, k + 4, KA), af[2]); as[3] = tf32_rest(toep(cum, j0 + g + 8, k + 4, KA), af[3]);
    }
    const bool v0 = k <= KA, v1 = k + 4 <= KA;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int n = n0 + nt * 8 + g;
      const uint32_t b0 = v0 ? f2tf32(Us[k * AP + n]) : 0u, b1 = v1 ? f2tf32(Us[(k + 4) * AP + n]) : 0u;
      if (kSplit) {
        mma_tf32(acc[nt], as, b0, b1);
        mma_tf32(acc[nt], af, v0 ? tf32_rest(Us[k * AP + n], b0) : 0u, v1 ? tf32_rest(Us[(k + 4) * AP + n], b1) : 0u);
      }
      mma_tf32(acc[nt], af, b0, b1);
    }
  }
}
inline size_t att_fwd_smem(int Ti, int KA, int A, int D, int C2) {
  return sizeof(float) * (size_t)((KA + 1) * (A + kAttPad) + att_cumlen(Ti, KA) + A + ((Ti + 3) & ~3) + D + 8 * C2 + 32) + 64;
}
// kMasked: the scores of positions past lens[b] are -inf (mask_encoder); otherwise the energies and the softmax cover all T_in
// positions. The context sum stays bounded by lens[b] either way: the values rows past it are zero. kCumulative: the state after
// the step is cum + alpha (cumulative_weights); otherwise alpha itself. kSplit: the split_bf16 operands (see AttArgs).
template <bool kMasked, bool kCumulative, bool kSplit>
__global__ void __launch_bounds__(kAttThreads) att_fwd_kernel(AttArgs a) {
  extern __shared__ __align__(16) float sm[];
  pdl_wait();
  pdl_launch_dependents();
  ATT_STAMP(0);
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Ti = a.Ti, A = a.A, AP = A + kAttPad, half = a.KA / 2, NW = kAttThreads / 32;
  const int Tip = (Ti + 3) & ~3, cumlen = att_cumlen(Ti, a.KA);
  float* Us = sm;                       // [(KA+1)][AP] filter bank, row KA = offset u0
  float* cum = Us + (a.KA + 1) * AP;    // [cumlen] zero-padded halo
  float* q = cum + cumlen;              // [A]
  float* e = q + A;                     // [Ti]
  float* hs = e + Tip;                  // [D] query source as fp32
  float* part = hs + a.D;               // [8][C2] context partials
  float* red = part + 8 * a.C2;         // [32]
  for (int i = tid; i < (a.KA + 1) * A; i += kAttThreads) Us[(i / A) * AP + (i % A)] = a.U[i];
  for (int i = tid; i < cumlen; i += kAttThreads) {
    const int j = i - half;
    cum[i] = (j >= 0 && j < Ti) ? a.cum[(long long)b * Ti + j] : 0.f;
  }
  for (int i = tid; i < a.D; i += kAttThreads) {
    const bf16* hp = a.h2out + (long long)b * a.ld_h2 + i;
    hs[split8(i, a.D)] = kSplit ? __bfloat162float(hp[0]) + __bfloat162float(hp[a.lo_h2]) : __bfloat162float(hp[0]);
  }
  for (int i = tid; i < Tip; i += kAttThreads) e[i] = 0.f;
  __syncthreads();
  ATT_STAMP(1);
  att_query<kSplit>(a.WqT, hs, q, A, a.D);
  __syncthreads();
  ATT_STAMP(2);
  const int len = a.lens[b];
  const int el = kMasked ? len : Ti;    // positions that get an energy
  {
    // energies: units of 16 memory rows x 64 channels; e[j] += sum over the unit's channels of v tanh(keys + q + pl)
    const int g = lane >> 2, t = lane & 3;
    const int n_nh = A >> 6, n_units = ((el + 15) >> 4) * n_nh;
    for (int u = warp; u < n_units; u += NW) {
      const int j0 = (u / n_nh) * 16, n0 = (u % n_nh) * 64;
      float acc[8][4];
      loc_tile<kSplit>(Us, AP, cum, a.KA, j0, n0, acc);
      const int r0 = j0 + g, r1 = r0 + 8;
      const float* k0p = a.keys + ((long long)b * Ti + (r0 < el ? r0 : 0)) * A + n0 + 2 * t;
      const float* k1p = a.keys + ((long long)b * Ti + (r1 < el ? r1 : 0)) * A + n0 + 2 * t;
      float2 ky0[8], ky1[8];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) { ky0[nt] = __ldg(reinterpret_cast<const float2*>(k0p + nt * 8)); ky1[nt] = __ldg(reinterpret_cast<const float2*>(k1p + nt * 8)); }
      float e0 = 0.f, e1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int c = n0 + nt * 8 + 2 * t;
        const float2 qq = *reinterpret_cast<const float2*>(q + c);
        const float2 vv = __ldg(reinterpret_cast<const float2*>(a.v + c));
        e0 += vv.x * tanhf_(ky0[nt].x + qq.x + acc[nt][0]) + vv.y * tanhf_(ky0[nt].y + qq.y + acc[nt][1]);
        e1 += vv.x * tanhf_(ky1[nt].x + qq.x + acc[nt][2]) + vv.y * tanhf_(ky1[nt].y + qq.y + acc[nt][3]);
      }
      e0 += __shfl_xor_sync(0xffffffffu, e0, 1); e0 += __shfl_xor_sync(0xffffffffu, e0, 2);
      e1 += __shfl_xor_sync(0xffffffffu, e1, 1); e1 += __shfl_xor_sync(0xffffffffu, e1, 2);
      if (t == 0) {
        if (r0 < el) atomicAdd(&e[r0], e0);
        if (r1 < el) atomicAdd(&e[r1], e1);
      }
    }
  }
  __syncthreads();
  ATT_STAMP(3);
  float mx = -INFINITY;
  for (int j = tid; j < el; j += kAttThreads) mx = fmaxf(mx, e[j]);
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < kAttThreads / 32; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float s = 0.f;
  for (int j = tid; j < Ti; j += kAttThreads) { const float p = j < el ? __expf(e[j] - mx) : 0.f; e[j] = p; s += p; }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  s = 0.f;
  for (int w = 0; w < kAttThreads / 32; ++w) s += red[w];
  const float inv = 1.f / s;
  for (int j = tid; j < Ti; j += kAttThreads) {
    const float al = e[j] * inv;
    e[j] = al;
    a.alpha[(long long)b * Ti + j] = al;
    a.cum[(long long)b * Ti + j] = kCumulative ? cum[j + half] + al : al;
  }
  __syncthreads();
  ATT_STAMP(4);
  // context = alpha . values: 8 row groups x (C2/8) column chunks of 8 channels; one work item per thread up to C2 = 512,
  // strided over the CTA beyond that so that every row group of part[] is written
  {
    const int nch = a.C2 >> 3;                 // uint4 chunks per row
    for (int w = tid; w < 8 * nch; w += kAttThreads) {
      const int rg = w / nch, ch = w % nch;
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      const int ldv = kSplit ? 2 * nch : nch;  // uint4 chunks per values row ([hi | lo] in split mode)
      const uint4* vp = reinterpret_cast<const uint4*>(a.values + (long long)b * Ti * ldv * 8) + ch;
#pragma unroll 4
      for (int j = rg; j < len; j += 8) {
        const uint4 u = __ldg(vp + (long long)j * ldv);
        const float al = e[j];
        acc[0] += al * bf16lo(u.x); acc[1] += al * bf16hi(u.x); acc[2] += al * bf16lo(u.y); acc[3] += al * bf16hi(u.y);
        acc[4] += al * bf16lo(u.z); acc[5] += al * bf16hi(u.z); acc[6] += al * bf16lo(u.w); acc[7] += al * bf16hi(u.w);
        if (kSplit) {
          const uint4 w = __ldg(vp + (long long)j * ldv + nch);
          acc[0] += al * bf16lo(w.x); acc[1] += al * bf16hi(w.x); acc[2] += al * bf16lo(w.y); acc[3] += al * bf16hi(w.y);
          acc[4] += al * bf16lo(w.z); acc[5] += al * bf16hi(w.z); acc[6] += al * bf16lo(w.w); acc[7] += al * bf16hi(w.w);
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) part[rg * a.C2 + ch * 8 + i] = acc[i];
    }
  }
  __syncthreads();
  ATT_STAMP(5);
  for (int c = tid; c < a.C2; c += kAttThreads) {
    float acc = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) acc += part[r * a.C2 + c];
    const bf16 r16 = __float2bfloat16(acc);
    if (kSplit) {
      const bf16 l16 = __float2bfloat16(acc - __bfloat162float(r16));
      if (a.ctx_a) {
        bf16* ca = a.ctx_a + (long long)b * a.ld_a + c;
        ca[0] = r16; ca[a.lo_a] = l16; ca[2 * a.lo_a] = r16;
      }
      bf16* cb = a.ctx_b + (long long)b * a.ld_b + c;
      cb[0] = r16; cb[a.lo_b] = l16;
      continue;
    }
    if (a.ctx_a) a.ctx_a[(long long)b * a.ld_a + c] = r16;
    a.ctx_b[(long long)b * a.ld_b + c] = r16;
  }
  ATT_STAMP(6);
}
// once per forward: the merged location filter bank U (from the conv kernel K [KA][F], its bias bK, the dense Wl [F][A] and the
// attention bias) and the kernel's shared-memory opt-in
using AttFwdFn = void (*)(AttArgs);
template <bool kSplit>
AttFwdFn att_fwd_fn_t(int unmasked, int noncumulative) {
  return unmasked ? (noncumulative ? att_fwd_kernel<false, false, kSplit> : att_fwd_kernel<false, true, kSplit>)
                  : (noncumulative ? att_fwd_kernel<true, false, kSplit> : att_fwd_kernel<true, true, kSplit>);
}
AttFwdFn att_fwd_fn(int unmasked, int noncumulative, int split) {
  return split ? att_fwd_fn_t<true>(unmasked, noncumulative) : att_fwd_fn_t<false>(unmasked, noncumulative);
}
int att_fwd_setup(const float* K, const float* bK, const float* Wl, const float* ba, float* U, int KA, int F, int A, size_t smem, int unmasked,
                  int noncumulative, int split, cudaStream_t st) {
  att_prep_kernel<<<grid1d((KA + 1) * A), 256, 0, st>>>(K, bK, Wl, ba, U, KA, F, A); t2_count_launch();
  T2_CHECK_CUDA(cudaFuncSetAttribute(att_fwd_fn(unmasked, noncumulative, split), cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}
int launch_att_fwd(const AttArgs& a, size_t smem, cudaStream_t st) {
  T2_CHECK_CUDA(launch_pdl(att_fwd_fn(a.unmasked, a.noncumulative, a.split), dim3(a.B), dim3(kAttThreads), smem, st, a)); t2_count_launch();
  return T2_OK;
}

// ---- output heads / losses ---------------------------------------------------------------------------------------
// projo [To][B][128] fp32 (cols 0..M-1 frames, col M stop logit) -> clipped decoder output (batch-major), stop logits,
// loss sums: scal[0] += sum (dec - tgt)^2, scal[2] += sum BCE(stop)
__global__ void dec_finish_kernel(const float* __restrict__ projo, const float* __restrict__ tgt, const float* __restrict__ stop_tgt,
                                  bf16* __restrict__ dec_bm, float* __restrict__ dec_f, float* __restrict__ stop, float* __restrict__ scal,
                                  int B, int To, int M, int clip, float lo, float hi, int split, const int* __restrict__ tlen, float pos_w) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  float l0 = 0.f, l2 = 0.f, nz = 0.f;
  if (e < (long long)B * To * (M + 1)) {
    const int m = int(e % (M + 1)), t = int((e / (M + 1)) % To), b = int(e / ((long long)(M + 1) * To));
    const bool live = !tlen || t < tlen[b];     // mask_decoder: frames past the target length do not count
    const float v = projo[((long long)t * B + b) * 128 + m];
    if (m < M) {
      const float d = clip ? fminf(fmaxf(v, lo), hi) : v;
      const long long o = ((long long)b * To + t) * M + m;
      dec_f[o] = d;
      if (!split) dec_bm[o] = __float2bfloat16(d);
      else {   // rows [hi(M) zero-padded to Cp | lo(M) zero-padded to Cp], Cp = ceil(M / 64) * 64 (the buffer is cleared once at init)
        const int Cp = (M + 63) / 64 * 64;
        const bf16 h = __float2bfloat16(d);
        bf16* row = dec_bm + ((long long)b * To + t) * 2 * Cp + m;
        row[0] = h; row[Cp] = __float2bfloat16(d - __bfloat162float(h));
      }
      if (tgt && live) { const float df = d - tgt[o]; l0 = df * df; }
    } else {
      stop[(long long)b * To + t] = v;
      if (stop_tgt) {
        const float z = stop_tgt[(long long)b * To + t];
        if (!tlen) l2 = fmaxf(v, 0.f) - v * z + log1pf(__expf(-fabsf(v)));
        else if (live) {   // tf.nn.weighted_cross_entropy_with_logits, then / count_nonzero(masked loss) (modules.py:450-455)
          l2 = (1.f - z) * v + (1.f + (pos_w - 1.f) * z) * (log1pf(__expf(-fabsf(v))) + fmaxf(-v, 0.f));
          nz = l2 != 0.f ? 1.f : 0.f;
        }
      }
    }
  }
  l0 = warp_sum(l0); l2 = warp_sum(l2); nz = warp_sum(nz);
  if ((threadIdx.x & 31) == 0) {
    if (l0 != 0.f) atomicAdd(scal + 0, l0);
    if (l2 != 0.f) atomicAdd(scal + 2, l2);
    if (nz != 0.f) atomicAdd(scal + 4, nz);
  }
}
// mel = clip(dec + residual); scal[1] += sum (mel - tgt)^2
__global__ void mel_finish_kernel(const float* __restrict__ dec_f, const float* __restrict__ resid, const float* __restrict__ tgt,
                                  float* __restrict__ mel, float* __restrict__ scal, long long npos, int M, int clip, float lo, float hi,
                                  const int* __restrict__ tlen, int To) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  float l = 0.f;
  if (e < npos * M) {
    const long long pos = e / M; const int m = int(e % M);
    float v = dec_f[e] + resid[pos * 128 + m];
    if (clip) v = fminf(fmaxf(v, lo), hi);
    mel[e] = v;
    if (tgt && (!tlen || int(pos % To) < tlen[pos / To])) { const float d = v - tgt[e]; l = d * d; }
  }
  l = warp_sum(l);
  if ((threadIdx.x & 31) == 0 && l != 0.f) atomicAdd(scal + 1, l);
}
__global__ void proj_bias_kernel(float* p, const float* fb, const float* sb, long long rows, int M) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= rows * (M + 1)) return;
  const int m = int(e % (M + 1));
  p[(e / (M + 1)) * 128 + m] += m < M ? fb[m] : sb[0];
}
constexpr uint32_t kTfStream = 40;   // hash stream of the per-step teacher-forcing draw (include/t2b200.h)
// projo[t] += bias; next decoder input = the raw (un-clipped) frame just predicted (helpers.py:56). With tgt (TacoTrainingHelper at a
// teacher-forcing ratio < 1, helpers.py:115-128): ONE draw u_t for the whole batch (stream kTfStream, element t, under seed + *step);
// u_t < ratio feeds the target frame tgt[b][t] instead, and choice[t] records which of the two step t + 1 consumed.
// split: next_in rows are the split decoder-input rows [hi(M) | pad | lo(M) | pad] of pitch 2 Cp (decin_kernel)
__global__ void proj_bias_feedback_kernel(float* __restrict__ p, const float* __restrict__ fb, const float* __restrict__ sb, bf16* __restrict__ next_in,
                                          int B, int M, const float* __restrict__ tgt, int To, int t, float ratio, unsigned long long seed,
                                          const unsigned long long* __restrict__ step, int* __restrict__ choice, int split) {
  pdl_wait();
  pdl_launch_dependents();
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= B * (M + 1)) return;
  bool forced = false;
  if (tgt) {
    forced = hash_uniform32(hash_seed(seed + (step ? *step : 0ull), kTfStream), (unsigned long long)t) < ratio;
    if (e == 0) choice[t] = forced ? 1 : 0;
  }
  const int m = e % (M + 1), b = e / (M + 1);
  const float v = p[b * 128 + m] + (m < M ? fb[m] : sb[0]);
  p[b * 128 + m] = v;
  if (m < M && next_in) {
    const float x = forced ? tgt[((long long)b * To + t) * M + m] : v;
    if (!split) { next_in[b * M + m] = __float2bfloat16(x); return; }
    const int Cp = (M + 63) / 64 * 64;
    const bf16 hi = __float2bfloat16(x);
    next_in[b * 2 * Cp + m] = hi; next_in[b * 2 * Cp + Cp + m] = __float2bfloat16(x - __bfloat162float(hi));
  }
}
// normalisers -> s[5] (mel terms), s[6] (stop term); out (nullable) = the four normalised loss terms
__global__ void loss_norm_kernel(float* s, float* out, float n_mel, float n_stop, float regw, const int* tlen, int B, int To, int M) {
  if (tlen) {
    float frames = 0.f;
    for (int b = 0; b < B; ++b) frames += float(tlen[b] < To ? tlen[b] : To);
    n_mel = fmaxf(frames * float(M), 1.f);      // count_nonzero of the broadcast mask (tf.losses.mean_squared_error weights)
    n_stop = fmaxf(s[4], 1.f);                  // count_nonzero of the masked stop-token losses
  }
  s[5] = n_mel; s[6] = n_stop;
  if (out) { out[0] = s[0] / n_mel; out[1] = s[1] / n_mel; out[2] = s[2] / n_stop; out[3] = s[3] * regw; }
}

struct StepCtx {
  const TL* lo; uint8_t* ws; const uint8_t* pk; const float* params; cudaStream_t st; unsigned long long seed;
  const unsigned long long* d_step; int training;
};

// one LSTM step on the swapped GEMM: gates^T = Wrec[4H perm][K] x S[B][K]^T (+ pre / bias) -> cell + zoneout
// split_bf16: Wrec rows are [W_hi | W_hi | W_lo] (pitch 3K) and the state rows S [hi | lo | hi] (pitch 3K): one segment contracts
// W_hi against [hi | lo], the next W_lo against the second hi copy. h_prev / h_state are state rows of this layout (lo at +K), h_out
// gets its lo half at +out_lo and, when out_state, the second hi copy at +2 out_lo (see EPI_LSTM); the backward stashes are skipped.
int lstm_step(const StepCtx& s, const void* wrec, int H, int K, const void* state, int B, const float* pre, int pre_stride, const float* bias,
              const float* c_prev, float* c_out, const bf16* h_prev, int ld_hp, bf16* h_state, int ld_hs, bf16* h_out, int ld_ho,
              bf16* gst, bf16* tst, const int* lens, int t, int stream_id, float zone, int out_lo = 0, int out_state = 0) {
  ActGemmCall g;
  memset(&g, 0, sizeof(g));
  const int split = s.lo->c.split_bf16;
  if (split) {
    g.a[0] = make_act(wrec, 3 * K, 4 * H, 1, 1, 3 * K); g.na = 1;
    g.seg[0] = Seg{0, 0, 0, 2 * K / kBK, 0, 1}; g.seg[1] = Seg{0, 0, 2 * K, K / kBK, 0, 1}; g.nseg = 2;
    g.w = state; g.wN = B; g.wK = 3 * K; g.wL = 1;
    gst = nullptr; tst = nullptr;
    g.epi.i[2] = out_lo; g.epi.i[10] = K; g.epi.i[11] = out_state ? 2 : 1;
  } else {
  g.a[0] = make_act(wrec, K, 4 * H, 1, 1, K); g.na = 1;
  g.seg[0] = Seg{0, 0, 0, K / kBK, 0, 1}; g.nseg = 1;
  g.w = state; g.wN = B; g.wK = K; g.wL = 1;
  }
  g.T = 4 * H; g.B = 1; g.n_tiles = (B + 31) / 32;
  g.epi.ptr[0] = const_cast<float*>(pre); g.epi.ptr[1] = const_cast<float*>(bias); g.epi.ptr[2] = const_cast<float*>(c_prev); g.epi.ptr[3] = c_out;
  g.epi.ptr[4] = const_cast<bf16*>(h_prev); g.epi.ptr[5] = h_state; g.epi.ptr[6] = h_out; g.epi.ptr[7] = gst; g.epi.ptr[8] = tst;
  g.epi.ptr[9] = const_cast<int*>(lens); g.epi.ptr[10] = const_cast<unsigned long long*>(s.d_step);
  g.epi.i[0] = H; g.epi.i[1] = B; g.epi.i[3] = pre_stride; g.epi.i[4] = ld_hp; g.epi.i[5] = ld_hs; g.epi.i[6] = ld_ho; g.epi.i[7] = t;
  g.epi.i[8] = stream_id; g.epi.i[9] = s.training; g.epi.f[0] = zone; g.epi.seed = s.seed;
  return launch_act_gemm(EPI_LSTM, 32, g, s.st);
}

int conv_block_fwd(const StepCtx& s, const ConvL& L, const void* x_in, int T, int training) {
  const TL& lo = *s.lo;
  int shifts[8];
  for (int j = 0; j < L.k; ++j) shifts[j] = conv_tap_shift(L.k, j);
  const int split = lo.c.split_bf16;
  bf16* y = reinterpret_cast<bf16*>(s.ws + L.w_y);
  float* yf = reinterpret_cast<float*>(s.ws + L.w_y);     // split mode keeps the pre-batch-norm activation in fp32
  int rc = launch_bias_act({.a = x_in, .C = L.cin, .T = T, .B = lo.B, .ntaps = L.k, .shifts = shifts, .split = split, .w = s.pk + L.k_w, .N = L.cout,
                            .wK = L.k * L.cinp, .BN = L.cout % 256 == 0 ? 256 : 128, .bias = s.params + L.p.bias, .act = L.act,
                            .out_bf16 = split ? nullptr : y, .out_f32 = split ? yf : nullptr, .ldo = L.cout, .nvalid = L.cout},
                           s.st);
  if (rc) return rc;
  float* stats = reinterpret_cast<float*>(s.ws + L.w_stats);
  const long long rows = (long long)lo.B * T;
  float* pp = const_cast<float*>(s.params);
  bf16* x = reinterpret_cast<bf16*>(s.ws + L.w_x);
  const BnDropout drop{lo.c.dropout_rate, s.seed, s.d_step, L.stream};
  if (training) T2_CHECK_CUDA(cudaMemsetAsync(stats, 0, 2 * L.cout * sizeof(float), s.st));
  if (split)
    bn_fwd(yf, L.cout, 0, x, 1, nullptr, nullptr, stats, L.cout, s.params + L.p.gamma, s.params + L.p.beta, pp + L.p.mm, pp + L.p.mv, rows, L.cout,
           training, drop, 256, s.st);
  else
    bn_fwd(y, L.cout, 0, x, 0, nullptr, nullptr, stats, L.cout, s.params + L.p.gamma, s.params + L.p.beta, pp + L.p.mm, pp + L.p.mv, rows, L.cout,
           training, drop, 256, s.st);
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}


// ======================================================================================================
// backward
// ======================================================================================================
// fixed-order list of weight-gradient GEMM launches; tiles live in the workspace (uploaded by t2_taco_init)
struct WgL { std::vector<WgradTile> tiles; };
enum { WG_PP = 0, WG_POST0 = 1 /* .. +postnet layers */ };
void build_tiles(const TL& lo, std::vector<WgL>& L) {
  L.clear();
  const int H = lo.H, D = lo.D, K1r = 2 * H + D, K2 = 2 * D, PIK = D + 2 * H;
  auto conv = [&](const ConvL& c) { WgL w; append_conv_wgrad_tiles(w.tiles, c.k, 0, c.cin, 0, c.cout, c.p.kernel); L.push_back(w); };
  { WgL w; append_wgrad_tiles(w.tiles, dense_proto(0, 1), 0, lo.PC, 0, lo.M, lo.p_ppk, lo.M); L.push_back(w); }            // 0: postnet projection
  for (int i = int(lo.post.size()) - 1; i >= 0; --i) conv(lo.post[i]);                                // 1..: postnet convs (reverse)
  { WgL w; append_wgrad_tiles(w.tiles, dense_proto(0, 1), 0, PIK, 0, lo.M, lo.p_fk, lo.M); append_wgrad_tiles(w.tiles, dense_proto(0, 1), 0, PIK, lo.M, 1, lo.p_sk, 1); L.push_back(w); }  // proj
  { WgL w;                                                                                               // decoder LSTMs + prenet-to-LSTM
    append_wgrad_tiles(w.tiles, dense_proto(0, 1), 0, K2, 0, 4 * D, lo.p_l2k, 4 * D);                                          // maps: 0 S2, 1 dg2, 2 S1, 3 dg1, 4 pn2
    append_wgrad_tiles(w.tiles, dense_proto(2, 3), 0, K1r, 0, 4 * D, lo.p_l1k + (long long)lo.P2 * 4 * D, 4 * D);
    append_wgrad_tiles(w.tiles, dense_proto(4, 3), 0, lo.P2, 0, 4 * D, lo.p_l1k, 4 * D);
    L.push_back(w); }
  { WgL w;                                                                                               // prenet + query layer
    append_wgrad_tiles(w.tiles, dense_proto(0, 1), 0, lo.P1, 0, lo.P2, lo.p_p2k, lo.P2);                                       // maps: 0 pn1, 1 dz2, 2 decin, 3 dz1, 4 PI, 5 dq_all
    append_wgrad_tiles(w.tiles, dense_proto(2, 3), 0, lo.M, 0, lo.P1, lo.p_p1k, lo.P1);
    append_wgrad_tiles(w.tiles, dense_proto(4, 5), 0, D, 0, lo.A, lo.p_qry, lo.A);
    L.push_back(w); }
  { WgL w; append_wgrad_tiles(w.tiles, dense_proto(0, 1), 0, 2 * H, 0, lo.A, lo.p_mem, lo.A); L.push_back(w); }               // memory layer: values x dkeys
  for (int d = 0; d < 2; ++d) {                                                                          // encoder LSTM d
    WgL w;  // maps: 0 h history (time-major), 1 gate grads time-major, 2 x3 (batch-major), 3 gate grads batch-major
    append_wgrad_tiles(w.tiles, dense_proto(0, 1), 0, H, 0, 4 * H, lo.p_elk[d] + (long long)lo.C * 4 * H, 4 * H);
    L.push_back(w);
    WgL w2; append_wgrad_tiles(w2.tiles, dense_proto(0, 1), 0, lo.C, 0, 4 * H, lo.p_elk[d], 4 * H); L.push_back(w2);
  }
  for (int i = int(lo.enc.size()) - 1; i >= 0; --i) conv(lo.enc[i]);
}

// loss seeds: dmel = 2 (mel - tgt) / N * [not clipped] (bf16, 128-col padded) ; ddec_direct = dmel + 2 (dec - tgt) / N
__global__ void loss_seed_kernel(const float* __restrict__ dec_f, const float* __restrict__ resid, const float* __restrict__ mel,
                                 const float* __restrict__ tgt, bf16* __restrict__ dmel, float* __restrict__ ddec, long long npos, int M,
                                 int clip, float lo, float hi, const int* __restrict__ tlen, int To, const float* __restrict__ scal,
                                 const float* __restrict__ extra) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= npos * 128) return;
  const long long pos = e / 128; const int m = int(e % 128);
  float g = 0.f;
  if (m < M) {
    const long long o = pos * M + m;
    const float n = scal[5];
    const float raw = dec_f[o] + resid[pos * 128 + m];
    const bool masked = tlen && int(pos % To) >= tlen[pos / To];             // masked frame: no mel-loss gradient
    g = masked ? 0.f : 2.f * (mel[o] - tgt[o]) / n;
    if (extra) g += extra[o];          // gradient of the post-processing net w.r.t. the clipped mel_outputs (not masked: its convs / GRU mix frames)
    if (clip && (raw < lo || raw > hi)) g = 0.f;
    ddec[o] = g + (masked ? 0.f : 2.f * (dec_f[o] - tgt[o]) / n);
  }
  dmel[e] = __float2bfloat16(g);
}
// ddec_tm[t][b][0..M) = (ddec_direct + ddec_post)[b][t][:] * [decoder clip inactive] ; col M = d BCE / d stop logit; steps [t0, t1).
// fb (teacher_forcing_ratio < 1, one step): + fb[b][:] = d(loss)/d(input frame of step t + 1) when that step consumed the frame step t
// predicted (choice[t] == 0). The fed-back frame is the raw projection output, so this term does not pass the clip mask.
__global__ void ddec_tm_kernel(const float* __restrict__ ddec, const bf16* __restrict__ dpost, const float* __restrict__ projo,
                               const float* __restrict__ stop_tgt, bf16* __restrict__ out, int B, int To, int M, int clip, float lo, float hi,
                               const int* __restrict__ tlen, float pos_w, const float* __restrict__ scal, int t0, int t1,
                               const float* __restrict__ fb, const int* __restrict__ choice) {
  const long long e = (long long)t0 * B * 128 + blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)t1 * B * 128) return;
  const int m = int(e % 128), b = int((e / 128) % B), t = int(e / (128LL * B));
  float g = 0.f;
  if (m < M) {
    const long long o = ((long long)b * To + t) * M + m;
    g = ddec[o] + __bfloat162float(dpost[o]);
    const float raw = projo[((long long)t * B + b) * 128 + m];
    if (clip && (raw < lo || raw > hi)) g = 0.f;
    if (fb && !choice[t]) g += fb[(long long)b * M + m];
  } else if (m == M) {
    const float x = projo[((long long)t * B + b) * 128 + M];
    const float z = stop_tgt[(long long)b * To + t];
    if (!tlen) g = (1.f / (1.f + __expf(-x)) - z) / scal[6];
    else if (t < tlen[b]) g = ((1.f - z) - (1.f + (pos_w - 1.f) * z) / (1.f + __expf(x))) / scal[6];     // d/dx of the weighted CE
  }
  out[e] = __float2bfloat16(g);
}
// d(pre-activation) of relu + inverted dropout given the stored post-dropout output y: dz = y > 0 ? d / keep : 0
__global__ void relu_drop_bwd_kernel(const bf16* __restrict__ d, const bf16* __restrict__ y, bf16* __restrict__ dz, long long n, float p) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e < n) dz[e] = __float2bfloat16(__bfloat162float(y[e]) > 0.f ? __bfloat162float(d[e]) / (1.f - p) : 0.f);
}

// backward of one LSTM cell + zoneout (see EPI_LSTM): produces the pre-activation gate gradients and the state grads
struct CellBwd {
  float* dh_ext; long long ld_ext;            // grad wrt the un-zoned output h_new: dh_ext[b*ld_ext + u]
  int zero_ext;                                // clear dh_ext after reading (its producer accumulates atomically, split-K)
  float* dhs; float* dcs;                      // [B][H] running grads wrt the carried (zoned) state (in/out)
  const bf16* gst; const bf16* tst; const float* c_prev;
  bf16* dg_a; long long ld_a;                  // gate grads, gate-major [4H] per batch row (row stride ld_a)
  bf16* dg_b; long long ld_b;                  // optional second copy
  const int* lens; int t, B, H, stream;
  float zone; unsigned long long seed; const unsigned long long* step;
};
__global__ void lstm_cell_bwd_kernel(CellBwd a) {
  pdl_wait();
  pdl_launch_dependents();
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)a.B * a.H) return;
  const int b = int(e / a.H), u = int(e % a.H);
  unsigned long long seed = a.seed + (a.step ? *a.step : 0ull);
  const bool live = a.lens ? (a.t < a.lens[b]) : true;
  float dzi = 0.f, dzj = 0.f, dzf = 0.f, dzo = 0.f;
  if (live) {
    const bf16* g = a.gst + (long long)b * 4 * a.H;
    const float gi = __bfloat162float(g[u]), gj = __bfloat162float(g[a.H + u]), gf = __bfloat162float(g[2 * a.H + u]),
                go = __bfloat162float(g[3 * a.H + u]);
    const float tc = __bfloat162float(a.tst[e]);
    const uint64_t idx = (uint64_t(a.t) * a.B + b) * a.H + u;
    const bool mc = a.zone <= 0.f || hash_uniform32(hash_seed(seed, uint32_t(a.stream) * 2u), idx) >= a.zone;
    const bool mh = a.zone <= 0.f || hash_uniform32(hash_seed(seed, uint32_t(a.stream) * 2u + 1u), idx) >= a.zone;
    const float dhs = a.dhs[e], dcs = a.dcs[e];
    const float dh_new = a.dh_ext[(long long)b * a.ld_ext + u] + (mh ? dhs : 0.f);
    if (a.zero_ext) a.dh_ext[(long long)b * a.ld_ext + u] = 0.f;
    const float dc_new = (mc ? dcs : 0.f) + dh_new * go * (1.f - tc * tc);
    dzo = dh_new * tc * go * (1.f - go);
    dzi = dc_new * gj * gi * (1.f - gi);
    dzj = dc_new * gi * (1.f - gj * gj);
    dzf = dc_new * a.c_prev[e] * gf * (1.f - gf);
    a.dcs[e] = dc_new * gf + (mc ? 0.f : dcs);
    a.dhs[e] = mh ? 0.f : dhs;
  }
  bf16* o = a.dg_a + (long long)b * a.ld_a;
  o[u] = __float2bfloat16(dzi); o[a.H + u] = __float2bfloat16(dzj); o[2 * a.H + u] = __float2bfloat16(dzf); o[3 * a.H + u] = __float2bfloat16(dzo);
  if (a.dg_b) {
    bf16* o2 = a.dg_b + (long long)b * a.ld_b;
    o2[u] = __float2bfloat16(dzi); o2[a.H + u] = __float2bfloat16(dzj); o2[2 * a.H + u] = __float2bfloat16(dzf); o2[3 * a.H + u] = __float2bfloat16(dzo);
  }
}

// backward step GEMM: dS^T [K rows][B] = W^T-packed [K][4H] x dgates [B][4H]^T, rows split over two fp32 destinations
int lstm_bwd_gemm(const StepCtx& s, const void* wT, int K, int H4, const void* dg, int B, float* dst0, int rows0, int ld0, int acc0, float* dst1,
                  int ld1, int acc1, int ksplit) {
  ActGemmCall g;
  memset(&g, 0, sizeof(g));
  g.a[0] = make_act(wT, H4, K, 1, 1, H4); g.na = 1;
  g.seg[0] = Seg{0, 0, 0, H4 / kBK, 0, 1}; g.nseg = 1;
  g.w = dg; g.wN = B; g.wK = H4; g.wL = 1;
  g.T = K; g.B = 1; g.n_tiles = (B + 31) / 32;
  // few output tiles (K / 128 <= 16) but a long reduction (4H): slice the reduction over `ksplit` CTAs per tile
  g.ksplit = ksplit;
  g.epi.ptr[0] = dst0; g.epi.ptr[1] = dst1;
  g.epi.i[0] = rows0; g.epi.i[1] = ld0; g.epi.i[2] = acc0; g.epi.i[3] = K; g.epi.i[4] = ld1; g.epi.i[5] = acc1; g.epi.i[6] = B;
  return launch_act_gemm(EPI_TOUT, 32, g, s.st);
}

// ---- attention backward, one CTA per batch item per step ----------------------------------------------------------
struct AttBwd {
  const bf16* h2out; int ld_h2; const bf16* WqT; const float* Wq;   // Wq fp32 [D][A]
  const float* U; const float* v;
  const float* keys; const bf16* values; const int* lens;
  const float* alpha;      // [B][Ti] of this step
  float* cumrun;           // cumulative: [B][Ti] cum_t on entry, cum_{t-1} on exit
  const float* alpha_prev; // non-cumulative: [B][Ti] alpha_{t-1} = the state the step read (nullptr at t = 0: zeros)
  float* dcum;             // [B][Ti] running grad wrt state_t (in) / state_{t-1} (out)
  const float* dPI; int ld_dPI;   // dPI_all[t]: [B][PIK] fp32
  float* dctxl;            // [B][C2] grad wrt ctx_t from LSTM-1 of step t+1 (read, then cleared for the split-K accumulation)
  float* dh2ext;           // [B][D] out: grad wrt the un-zoned LSTM-2 output of this step
  bf16* dctx_save;         // [B][C2]
  bf16* dq_save;           // [B][A]
  float* dkeys;            // [B][Ti][A] accumulated
  float* acc;              // per item: dU [(KA+1)][A] (row KA = d u0) | dv [A]
  int B, Ti, D, A, KA, C2;
  int unmasked, noncumulative;   // pick the att_bwd_kernel instantiation (host side only)
};
inline size_t att_bwd_smem(int Ti, int KA, int A, int D, int C2) {
  const int Tip = (Ti + 3) & ~3;
  return sizeof(float) * (size_t)((KA + 1) * (A + kAttPad) + att_cumlen(Ti, KA) + A + 4 * Tip + D + C2 + 2 * A +
                                  att_erows(Ti, KA) * (A + kAttPad) + 32) + 64;
}
constexpr size_t kSmemOptin = 232448;   // per-block shared-memory opt-in limit of sm_90
// Training runs att_bwd_kernel, whose [T_in + KA - 1][A + 8] fp32 dE tile lives in shared memory: refuse (before any launch) a
// T_in it cannot hold. The forward-only paths (inference, GTA) are not limited by it.
int check_att_bwd_fits(const TL& lo) {
  const int C2 = 2 * lo.H;
  const size_t need = att_bwd_smem(lo.Ti, lo.KA, lo.A, lo.D, C2);
  if (need <= kSmemOptin) return T2_OK;
  int tmax = lo.Ti;
  while (tmax > 1 && att_bwd_smem(tmax, lo.KA, lo.A, lo.D, C2) > kSmemOptin) --tmax;
  return t2_set_error(T2_ERR_UNSUPPORTED_SHAPE,
                      "training: T_in = %d needs %zu B of shared memory in the attention backward, over the %zu B per-block limit; "
                      "T_in <= %d at these attention widths",
                      lo.Ti, need, kSmemOptin, tmax);
}
// kMasked / kCumulative as in att_fwd_kernel. Un-masked, d alpha_j past lens[b] is d state_j alone (the values rows there are zero)
// and every energy gets a gradient. Non-cumulative, state_{t-1} is alpha_{t-1}, and d state_{t-1} is the location-path term only:
// alpha_t does not carry state_{t-1} forward.
template <bool kMasked, bool kCumulative>
__global__ void __launch_bounds__(kAttThreads) att_bwd_kernel(AttBwd a) {
  extern __shared__ __align__(16) float sm[];
  pdl_wait();
  pdl_launch_dependents();
  ATT_STAMP(16);
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int Ti = a.Ti, A = a.A, AP = A + kAttPad, half = a.KA / 2, NW = kAttThreads / 32;
  const int Tip = (Ti + 3) & ~3, cumlen = att_cumlen(Ti, a.KA), RE = att_erows(Ti, a.KA);
  float* Us = sm;                         // [(KA+1)][AP]
  float* cum = Us + (a.KA + 1) * AP;      // [cumlen] cum_{t-1}, zero-padded
  float* q = cum + cumlen;                // [A]
  float* al = q + A;                      // [Ti]
  float* de = al + Tip;                   // [Ti]
  float* dcs = de + Tip;                  // [Ti] incoming dcum_t
  float* dca = dcs + Tip;                 // [Ti] location-path contribution to dcum_{t-1}
  float* hs = dca + Tip;                  // [D]
  float* dctx = hs + a.D;                 // [C2]
  float* dq = dctx + a.C2;                // [A]
  float* dv = dq + A;                     // [A]
  float* dE = dv + A;                     // [RE][AP]: position j lives in row j + half; everything else stays zero
  float* red = dE + RE * AP;              // [32]
  const int len = a.lens[b];
  const int el = kMasked ? len : Ti;      // positions with an energy
  for (int i = tid; i < (a.KA + 1) * A; i += kAttThreads) Us[(i / A) * AP + (i % A)] = a.U[i];
  for (int i = tid; i < cumlen; i += kAttThreads) {
    const int j = i - half;
    float cp = 0.f;
    if (j >= 0 && j < Ti) {
      const float aj = a.alpha[(long long)b * Ti + j];
      al[j] = aj;
      if (kCumulative) {
        cp = a.cumrun[(long long)b * Ti + j] - aj;
        a.cumrun[(long long)b * Ti + j] = cp;
      } else if (a.alpha_prev) {
        cp = a.alpha_prev[(long long)b * Ti + j];
      }
      dcs[j] = a.dcum[(long long)b * Ti + j];
      dca[j] = 0.f;
    }
    cum[i] = cp;
  }
  for (int i = tid; i < a.D; i += kAttThreads) hs[split8(i, a.D)] = __bfloat162float(a.h2out[(long long)b * a.ld_h2 + i]);
  for (int c = tid; c < a.C2; c += kAttThreads) {
    const float gg = a.dPI[(long long)b * a.ld_dPI + a.D + c] + a.dctxl[(long long)b * a.C2 + c];
    a.dctxl[(long long)b * a.C2 + c] = 0.f;
    dctx[split8(c, a.C2)] = gg;            // split layout: dotted against 16-byte bf16 pieces of the values rows
    a.dctx_save[(long long)b * a.C2 + c] = __float2bfloat16(gg);
  }
  for (int i = tid; i < A; i += kAttThreads) { dq[i] = 0.f; dv[i] = 0.f; }
  for (int i = tid * 4; i < RE * AP; i += kAttThreads * 4) *reinterpret_cast<float4*>(dE + i) = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  ATT_STAMP(17);
  att_query<false>(a.WqT, hs, q, A, a.D);
  ATT_STAMP(18);
  // d alpha[j] = dctx . values[j] + dcum[j] : one warp per row, 8-wide bf16 loads, four rows in flight
  float part = 0.f;
  {
    const int nch = a.C2 >> 3;
    const uint4* vb = reinterpret_cast<const uint4*>(a.values + (long long)b * Ti * a.C2);
    for (int j = warp; j < len; j += 4 * NW) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int ch = lane; ch < nch; ch += 32) {
        uint4 u[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int jr = j + r * NW;
          u[r] = jr < len ? __ldg(vb + (long long)jr * nch + ch) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[r] += dot8s(u[r], dctx, ch, a.C2);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[r] = warp_sum(acc[r]);
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int jr = j + r * NW;
          if (jr < len) { const float da = acc[r] + dcs[jr]; de[jr] = da; part += al[jr] * da; }
        }
      }
    }
    if (kMasked) {
      for (int j = len + tid; j < Ti; j += kAttThreads) de[j] = 0.f;
    } else {
      float tail = 0.f;      // past the length dctx . values[j] = 0: d alpha[j] = dcum[j]
      for (int j = len + tid; j < Ti; j += kAttThreads) { const float da = dcs[j]; de[j] = da; tail += al[j] * da; }
      tail = warp_sum(tail);
      if (lane == 0) part += tail;
    }
  }
  if (lane == 0) red[warp] = part;
  __syncthreads();
  ATT_STAMP(19);
  float dot = 0.f;
  for (int w = 0; w < NW; ++w) dot += red[w];
  __syncthreads();
  for (int j = tid; j < Ti; j += kAttThreads) de[j] = j < el ? al[j] * (de[j] - dot) : 0.f;
  __syncthreads();
  // energies backward: units of 16 rows x 64 channels (pl recomputed on the tensor cores, see loc_tile)
  {
    const int n_nh = A >> 6, n_units = ((el + 15) >> 4) * n_nh;
    for (int u = warp; u < n_units; u += NW) {
      const int j0 = (u / n_nh) * 16, n0 = (u % n_nh) * 64;
      float acc[8][4];
      loc_tile<false>(Us, AP, cum, a.KA, j0, n0, acc);
      const int r0 = j0 + g, r1 = r0 + 8;
      const bool ok0 = r0 < el, ok1 = r1 < el;
      const long long kr0 = ((long long)b * Ti + (ok0 ? r0 : 0)) * A + n0 + 2 * t, kr1 = ((long long)b * Ti + (ok1 ? r1 : 0)) * A + n0 + 2 * t;
      float2 ky0[8], ky1[8];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        ky0[nt] = __ldg(reinterpret_cast<const float2*>(a.keys + kr0 + nt * 8));
        ky1[nt] = __ldg(reinterpret_cast<const float2*>(a.keys + kr1 + nt * 8));
      }
      const float de0 = ok0 ? de[r0] : 0.f, de1 = ok1 ? de[r1] : 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int c = n0 + nt * 8 + 2 * t;
        const float2 qq = *reinterpret_cast<const float2*>(q + c);
        const float2 vv = __ldg(reinterpret_cast<const float2*>(a.v + c));
        const float t00 = tanhf_(ky0[nt].x + qq.x + acc[nt][0]), t01 = tanhf_(ky0[nt].y + qq.y + acc[nt][1]);
        const float t10 = tanhf_(ky1[nt].x + qq.x + acc[nt][2]), t11 = tanhf_(ky1[nt].y + qq.y + acc[nt][3]);
        const float2 d0 = make_float2(de0 * vv.x * (1.f - t00 * t00), de0 * vv.y * (1.f - t01 * t01));
        const float2 d1 = make_float2(de1 * vv.x * (1.f - t10 * t10), de1 * vv.y * (1.f - t11 * t11));
        // column sums over the unit's 16 rows: this lane's two rows, then the 8 row groups (lanes with equal t)
        float sq0 = d0.x + d1.x, sq1 = d0.y + d1.y, sv0 = de0 * t00 + de1 * t10, sv1 = de0 * t01 + de1 * t11;
#pragma unroll
        for (int m = 4; m < 32; m <<= 1) {
          sq0 += __shfl_xor_sync(0xffffffffu, sq0, m); sq1 += __shfl_xor_sync(0xffffffffu, sq1, m);
          sv0 += __shfl_xor_sync(0xffffffffu, sv0, m); sv1 += __shfl_xor_sync(0xffffffffu, sv1, m);
        }
        if (g == 0) { atomicAdd(&dq[c], sq0); atomicAdd(&dq[c + 1], sq1); atomicAdd(&dv[c], sv0); atomicAdd(&dv[c + 1], sv1); }
        if (ok0) {
          atomicAdd(reinterpret_cast<float2*>(a.dkeys + kr0 + nt * 8), d0);    // accumulates over decoder steps, no read-back
          *reinterpret_cast<float2*>(dE + (r0 + half) * AP + c) = d0;
        }
        if (ok1) {
          atomicAdd(reinterpret_cast<float2*>(a.dkeys + kr1 + nt * 8), d1);
          *reinterpret_cast<float2*>(dE + (r1 + half) * AP + c) = d1;
        }
      }
    }
  }
  __syncthreads();
  ATT_STAMP(20);
  float* accp = a.acc + (long long)b * ((a.KA + 2) * A);
  for (int c = tid; c < A; c += kAttThreads) {
    a.dq_save[(long long)b * A + c] = __float2bfloat16(dq[c]);
    accp[a.KA * A + c] += dq[c];          // d u0 (also the gradient of attention_bias)
    accp[(a.KA + 1) * A + c] += dv[c];
  }
  // dU[k][c] += sum_j cum_{t-1}[j + k - half] dE[j][c] = (T^T dE)[k][c]: M = 32 taps (2 m-tiles), N = A (one n-tile per
  // warp pass), K = memory rows
  {
    const int nks = (el + 7) >> 3;
    for (int nt = warp; nt < (A >> 3); nt += NW) {
      float acc[2][4];
#pragma unroll
      for (int m = 0; m < 2; ++m) acc[m][0] = acc[m][1] = acc[m][2] = acc[m][3] = 0.f;
      for (int ks = 0; ks < nks; ++ks) {
        const int j = ks * 8 + t;
        const uint32_t b0 = f2tf32(dE[(j + half) * AP + nt * 8 + g]), b1 = f2tf32(dE[(j + 4 + half) * AP + nt * 8 + g]);
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          const int k = m * 16 + g;
          uint32_t af[4];
          af[0] = f2tf32(k < a.KA ? cum[j + k] : 0.f); af[1] = f2tf32(k + 8 < a.KA ? cum[j + k + 8] : 0.f);
          af[2] = f2tf32(k < a.KA ? cum[j + 4 + k] : 0.f); af[3] = f2tf32(k + 8 < a.KA ? cum[j + 4 + k + 8] : 0.f);
          mma_tf32(acc[m], af, b0, b1);
        }
      }
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const int k0 = m * 16 + g, k1 = k0 + 8, c = nt * 8 + 2 * t;
        if (k0 < a.KA) atomicAdd(reinterpret_cast<float2*>(accp + k0 * A + c), make_float2(acc[m][0], acc[m][1]));
        if (k1 < a.KA) atomicAdd(reinterpret_cast<float2*>(accp + k1 * A + c), make_float2(acc[m][2], acc[m][3]));
      }
    }
  }
  ATT_STAMP(21);
  // dcum_{t-1}[i] = dcum_t[i] (cumulative only) + sum_k P[i - k + 2*half][k] with P = dE U^T ([RE rows] x [32 taps], K = A): one
  // m-tile of dE rows per warp pass, the anti-diagonal sums go through shared-memory atomics
  {
    for (int mt = warp; mt < (RE >> 4); mt += NW) {
      const int r0 = mt * 16 + g, r1 = r0 + 8;
      if (mt * 16 >= el + 2 * half) continue;      // rows past the last written position are zero (warp-uniform)
      float acc[4][4];
#pragma unroll
      for (int n = 0; n < 4; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
      for (int ks = 0; ks < (A >> 3); ++ks) {
        const int c = ks * 8 + t;
        uint32_t af[4];
        af[0] = f2tf32(dE[r0 * AP + c]); af[1] = f2tf32(dE[r1 * AP + c]);
        af[2] = f2tf32(dE[r0 * AP + c + 4]); af[3] = f2tf32(dE[r1 * AP + c + 4]);
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          const int tap = n * 8 + g;
          const uint32_t b0 = tap < a.KA ? f2tf32(Us[tap * AP + c]) : 0u, b1 = tap < a.KA ? f2tf32(Us[tap * AP + c + 4]) : 0u;
          mma_tf32(acc[n], af, b0, b1);
        }
      }
#pragma unroll
      for (int n = 0; n < 4; ++n) {
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          const int tap = n * 8 + 2 * t + (x & 1), r = (x & 2) ? r1 : r0;
          const int i = r + tap - 2 * half;
          if (tap < a.KA && i >= 0 && i < Ti) atomicAdd(&dca[i], acc[n][x]);
        }
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < Ti; i += kAttThreads) a.dcum[(long long)b * Ti + i] = kCumulative ? dcs[i] + dca[i] : dca[i];
  ATT_STAMP(22);
  // dh2ext = dPI[:, 0:D] + dq . Wq^T   (bf16 [A][D] copy of the query weights: coalesced along D)
  for (int k2 = tid; k2 < (a.D >> 1); k2 += kAttThreads) {
    const float2 gg = *reinterpret_cast<const float2*>(a.dPI + (long long)b * a.ld_dPI + 2 * k2);
    float a0 = gg.x, a1 = gg.y;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a.WqT) + k2;
#pragma unroll 16
    for (int c = 0; c < A; ++c) {
      const uint32_t u = __ldg(w + (long long)c * (a.D >> 1));
      a0 += dq[c] * bf16lo(u); a1 += dq[c] * bf16hi(u);
    }
    *reinterpret_cast<float2*>(a.dh2ext + (long long)b * a.D + 2 * k2) = make_float2(a0, a1);
  }
  ATT_STAMP(23);
}
// after the loop: reduce the per-item accumulators over the batch and push dU / du0 / dv through the U = K . Wl
// factorisation: dK = dU Wl^T, dWl = K^T dU + bK (x) du0, dbK = Wl du0, d attention_bias = du0, dv
__global__ void att_finish_kernel(const float* __restrict__ acc, const float* __restrict__ K, const float* __restrict__ bK,
                                  const float* __restrict__ Wl, float* __restrict__ grads, int B, int KA, int F, int A, long long o_k,
                                  long long o_bk, long long o_wl, long long o_v, long long o_ba, float* __restrict__ scratch) {
  // phase 1 (all blocks): reduce over the batch into scratch [(KA+2)][A]
  const int n = (KA + 2) * A;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += acc[(long long)b * n + i];
    scratch[i] = s;
  }
}
__global__ void att_finish2_kernel(const float* __restrict__ dU, const float* __restrict__ K, const float* __restrict__ bK,
                                   const float* __restrict__ Wl, float* __restrict__ grads, int KA, int F, int A, long long o_k, long long o_bk,
                                   long long o_wl, long long o_v, long long o_ba) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const float* du0 = dU + KA * A;
  const float* dv = dU + (KA + 1) * A;
  if (i < KA * F) {            // dK[k][f] = sum_a dU[k][a] Wl[f][a]
    const int k = i / F, f = i % F;
    float s = 0.f;
    for (int c = 0; c < A; ++c) s += dU[k * A + c] * Wl[f * A + c];
    grads[o_k + i] += s;
  } else if (i < KA * F + F * A) {   // dWl[f][a] = sum_k K[k][f] dU[k][a] + bK[f] du0[a]
    const int j = i - KA * F, f = j / A, c = j % A;
    float s = bK[f] * du0[c];
    for (int k = 0; k < KA; ++k) s += K[k * F + f] * dU[k * A + c];
    grads[o_wl + j] += s;
  } else if (i < KA * F + F * A + F) {   // dbK[f] = sum_a Wl[f][a] du0[a]
    const int f = i - KA * F - F * A;
    float s = 0.f;
    for (int c = 0; c < A; ++c) s += Wl[f * A + c] * du0[c];
    grads[o_bk + f] += s;
  } else if (i < KA * F + F * A + F + A) {
    const int c = i - KA * F - F * A - F;
    grads[o_v + c] += dv[c];
    grads[o_ba + c] += du0[c];
  }
}
// dvalues[b][j][c] += sum_t alpha[t][b][j] * dctx[t][b][c]; then apply the memory mask in place
__global__ void dvalues_ctx_kernel(const float* __restrict__ alpha, const bf16* __restrict__ dctx, const int* __restrict__ lens,
                                   float* __restrict__ dvalues, int B, int Ti, int To, int C2) {
  const int b = blockIdx.y, j = blockIdx.x;
  const bool live = j < lens[b];
  for (int c = threadIdx.x; c < C2; c += blockDim.x) {
    float acc = dvalues[((long long)b * Ti + j) * C2 + c];
    if (live) for (int t = 0; t < To; ++t) acc += alpha[((long long)t * B + b) * Ti + j] * __bfloat162float(dctx[((long long)t * B + b) * C2 + c]);
    dvalues[((long long)b * Ti + j) * C2 + c] = live ? acc : 0.f;
  }
}
// launch helpers shared by the backward pass and t2_dbg_taco_kernel
using AttBwdFn = void (*)(AttBwd);
AttBwdFn att_bwd_fn(int unmasked, int noncumulative) {
  return unmasked ? (noncumulative ? att_bwd_kernel<false, false> : att_bwd_kernel<false, true>)
                  : (noncumulative ? att_bwd_kernel<true, false> : att_bwd_kernel<true, true>);
}
int att_bwd_setup(size_t smem, int unmasked, int noncumulative) {
  T2_CHECK_CUDA(cudaFuncSetAttribute(att_bwd_fn(unmasked, noncumulative), cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  return T2_OK;
}
int launch_att_bwd(const AttBwd& a, size_t smem, cudaStream_t st) {
  T2_CHECK_CUDA(launch_pdl(att_bwd_fn(a.unmasked, a.noncumulative), dim3(a.B), dim3(kAttThreads), smem, st, a)); t2_count_launch();
  return T2_OK;
}
int launch_cell_bwd(const CellBwd& c, cudaStream_t st) {
  T2_CHECK_CUDA(launch_pdl(lstm_cell_bwd_kernel, dim3(grid1d((long long)c.B * c.H)), dim3(256), 0, st, c)); t2_count_launch();
  return T2_OK;
}
// scratch: [(KA+2)][A] fp32 for the batch-reduced accumulators
void launch_att_finish(const float* acc, const float* K, const float* bK, const float* Wl, float* grads, int B, int KA, int F, int A, long long o_k,
                       long long o_bk, long long o_wl, long long o_v, long long o_ba, float* scratch, cudaStream_t st) {
  att_finish_kernel<<<grid1d((long long)(KA + 2) * A), 256, 0, st>>>(acc, K, bK, Wl, grads, B, KA, F, A, o_k, o_bk, o_wl, o_v, o_ba, scratch); t2_count_launch();
  att_finish2_kernel<<<grid1d(KA * F + F * A + F + A), 256, 0, st>>>(scratch, K, bK, Wl, grads, KA, F, A, o_k, o_bk, o_wl, o_v, o_ba); t2_count_launch();
}
void launch_dvalues_ctx(const float* alpha, const bf16* dctx, const int* lens, float* dvalues, int B, int Ti, int To, int C2, cudaStream_t st) {
  dvalues_ctx_kernel<<<dim3(Ti, B), 256, 0, st>>>(alpha, dctx, lens, dvalues, B, Ti, To, C2); t2_count_launch();
}

int conv_block_bwd(const StepCtx& s, const ConvL& L, const void* x_in, int T, const bf16* dout, bf16* dpre, bf16* dx, float* grads,
                   const WgradTile* tiles, int ntiles) {
  const TL& lo = *s.lo;
  const long long rows = (long long)lo.B * T;
  float* stats = reinterpret_cast<float*>(s.ws + L.w_stats);
  const bf16* y = reinterpret_cast<const bf16*>(s.ws + L.w_y);
  float* bsum = stats + 4 * L.cout;
  T2_CHECK_CUDA(cudaMemsetAsync(bsum, 0, 2 * L.cout * sizeof(float), s.st));
  bn_bwd(dout, L.cout, y, L.cout, 0, stats, L.cout, bsum, s.params + L.p.gamma, dpre, L.cout, grads + L.p.gamma, grads + L.p.beta, rows, L.cout, L.act,
         BnDropout{lo.c.dropout_rate, s.seed, s.d_step, L.stream}, 256, s.st);
  colsum(dpre, rows, L.cout, L.cout, grads + L.p.bias, 256, s.st);
  T2_CHECK_CUDA(cudaGetLastError());
  ActT maps[2] = {make_act(x_in, L.cin, T, lo.B), make_act(dpre, L.cout, T, lo.B)};
  int rc = launch_wgrad(maps, 2, tiles, ntiles, grads, T, lo.B, s.st);
  if (rc) return rc;
  if (dx) {
    int shifts[8];
    for (int j = 0; j < L.k; ++j) shifts[j] = -conv_tap_shift(L.k, j);
    rc = launch_bias_act({.a = dpre, .C = L.cout, .T = T, .B = lo.B, .ntaps = L.k, .shifts = shifts, .w = s.pk + L.k_wT, .N = L.cin, .wK = L.k * L.cout,
                          .BN = L.cin % 256 == 0 ? 256 : 128, .out_bf16 = dx, .ldo = L.cin, .nvalid = L.cin},
                         s.st);
    if (rc) return rc;
  }
  return T2_OK;
}

}  // namespace
}  // namespace t2

using namespace t2;

extern "C" int t2_taco_sizes(const t2_taco_config_t* cfg, long long* n_params, long long* packed_bytes, long long* workspace_bytes,
                             int* n_tensors) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  if (n_params) *n_params = lo.n_params;
  if (packed_bytes) *packed_bytes = lo.packed_bytes;
  if (workspace_bytes) *workspace_bytes = lo.workspace_bytes;
  if (n_tensors) *n_tensors = int(lo.params.size());
  return T2_OK;
}

extern "C" int t2_taco_param_info(const t2_taco_config_t* cfg, int i, char* name, int cap, long long* offset, int* ndim, int* shape4,
                                  int* trainable) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  return param_info(lo.params, i, name, cap, offset, ndim, shape4, trainable);
}

extern "C" int t2_taco_init(const t2_taco_config_t* cfg, void* d_packed, void* d_workspace, void* stream) {
  TL lo;
  std::vector<PackJob> jobs;
  int rc = build(cfg, lo, &jobs);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  T2_CHECK_CUDA(cudaMemsetAsync(d_packed, 0, lo.packed_bytes, st));
  T2_CHECK_CUDA(cudaMemsetAsync(d_workspace, 0, lo.workspace_bytes, st));
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_packjobs, jobs.data(), jobs.size() * sizeof(PackJob), cudaMemcpyHostToDevice, st));
  rc = upload_reg_table(lo.params, ws + lo.w_regtab, st);
  if (rc) return rc;
  std::vector<WgL> wl;
  build_tiles(lo, wl);
  std::vector<WgradTile> all;
  for (auto& w : wl) all.insert(all.end(), w.tiles.begin(), w.tiles.end());
  T2_REQUIRE(all.size() <= 16384, T2_ERR_UNSUPPORTED_SHAPE, "too many weight-gradient tiles (%d)", int(all.size()));
  T2_CHECK_CUDA(cudaMemcpyAsync(ws + lo.w_tiles, all.data(), all.size() * sizeof(WgradTile), cudaMemcpyHostToDevice, st));
  T2_CHECK_CUDA(cudaStreamSynchronize(st));
  return T2_OK;
}

extern "C" int t2_taco_pack_weights(const t2_taco_config_t* cfg, const float* d_params, void* d_packed, void* d_workspace, void* stream) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  return launch_pack(d_params, d_packed, reinterpret_cast<const PackJob*>(static_cast<uint8_t*>(d_workspace) + lo.w_packjobs), lo.n_packjobs,
                     32, 32, static_cast<cudaStream_t>(stream));
}

// ---- encoder: embedding -> conv blocks -> BiLSTM -> masked values -> attention keys (tacotron.py:113-131) ----
// The two directions of the encoder BiLSTM are independent chains of small launches (8-16 CTAs each): the backward
// direction runs on the side stream (fork / join through events; capturable).
static int encoder_fwd(const StepCtx& s, const int* d_inputs, const int* d_input_lengths, int training) {
  const TL& lo = *s.lo;
  uint8_t* ws = s.ws; const uint8_t* pk = s.pk; const float* d_params = s.params; cudaStream_t st = s.st;
  const int B = lo.B, Ti = lo.Ti, H = lo.H;
  int rc;
  bf16* emb = reinterpret_cast<bf16*>(ws + lo.w_emb);
  embed_fwd_kernel<<<grid1d((long long)B * Ti * lo.E), 256, 0, st>>>(d_inputs, d_params + lo.p_emb, emb, (long long)B * Ti, lo.E, lo.c.split_bf16); t2_count_launch();
  const void* x = emb;
  for (auto& L : lo.enc) { rc = conv_block_fwd(s, L, x, Ti, training); if (rc) return rc; x = ws + L.w_x; }
  SideStream* side = side_stream();
  if (side) {
    T2_CHECK_CUDA(cudaEventRecord(side->fork, st));
    T2_CHECK_CUDA(cudaStreamWaitEvent(side->s, side->fork, 0));
  }
  for (int d = 0; d < 2; ++d) {
    cudaStream_t sx = (d == 1 && side) ? side->s : st;
    StepCtx sc = s; sc.st = sx;
    float* pre = reinterpret_cast<float*>(ws + lo.w_encpre[d]);
    rc = launch_bias_act({.a = x, .C = lo.C, .T = Ti, .B = B, .split = lo.c.split_bf16, .w = pk + lo.k_encWx[d], .N = 4 * H,
                          .wK = lo.C, .BN = 256, .bias = d_params + lo.p_elb[d], .out_f32 = pre, .ldo = 4 * H, .nvalid = 4 * H},
                         sx);
    if (rc) return rc;
    bf16* hh = reinterpret_cast<bf16*>(ws + lo.w_ench[d]);
    float* cc = reinterpret_cast<float*>(ws + lo.w_encc[d]);
    const int hw = lo.c.split_bf16 ? 3 * H : H;     // h history rows; split: state rows [hi | lo | hi]
    T2_CHECK_CUDA(cudaMemsetAsync(hh, 0, (size_t)B * hw * 2, sx));
    T2_CHECK_CUDA(cudaMemsetAsync(cc, 0, (size_t)B * H * 4, sx));
    bf16* memory = reinterpret_cast<bf16*>(ws + lo.w_memory);
    for (int sidx = 0; sidx < Ti; ++sidx) {
      const int t = d == 0 ? sidx : Ti - 1 - sidx;
      rc = lstm_step(sc, pk + lo.k_encWr[d], H, H, hh + (long long)sidx * B * hw, B, pre + (long long)t * 4 * H, Ti * 4 * H, nullptr,
                     cc + (long long)sidx * B * H, cc + (long long)(sidx + 1) * B * H, hh + (long long)sidx * B * hw, hw,
                     hh + (long long)(sidx + 1) * B * hw, hw, memory + (long long)t * lo.ld_mem + d * H, Ti * lo.ld_mem,
                     reinterpret_cast<bf16*>(ws + lo.w_encg[d]) + (long long)sidx * B * 4 * H,
                     reinterpret_cast<bf16*>(ws + lo.w_enct[d]) + (long long)sidx * B * H, d_input_lengths, t, 52 + d, lo.c.zoneout_rate,
                     2 * H, 0);
      if (rc) return rc;
    }
  }
  if (side) {
    T2_CHECK_CUDA(cudaEventRecord(side->join, side->s));
    T2_CHECK_CUDA(cudaStreamWaitEvent(st, side->join, 0));
  }
  bf16* values = reinterpret_cast<bf16*>(ws + lo.w_values);
  mask_values_kernel<<<grid1d((long long)B * Ti * lo.ld_mem), 256, 0, st>>>(reinterpret_cast<bf16*>(ws + lo.w_memory), d_input_lengths, values, B, Ti,
                                                                        lo.ld_mem);
  t2_count_launch();
  float* keys = reinterpret_cast<float*>(ws + lo.w_keys);
  return launch_bias_act({.a = values, .C = 2 * H, .T = Ti, .B = B, .split = lo.c.split_bf16, .w = pk + lo.k_mem, .N = lo.A,
                          .wK = 2 * H, .BN = 128, .out_f32 = keys, .ldo = lo.A, .nvalid = lo.A},
                         st);
}

struct DecBufs { bf16 *S1, *S2, *PI, *values; float *c1, *c2, *cum, *attU, *keys, *pre1; size_t att_smem; int K1r, K2, PIK; };
static void decoder_bufs(const TL& lo, uint8_t* ws, DecBufs& d) {
  const int H = lo.H, D = lo.D;
  d.K1r = 2 * H + D; d.K2 = 2 * D; d.PIK = D + 2 * H;
  d.S1 = reinterpret_cast<bf16*>(ws + lo.w_S1); d.S2 = reinterpret_cast<bf16*>(ws + lo.w_S2); d.PI = reinterpret_cast<bf16*>(ws + lo.w_PI);
  d.c1 = reinterpret_cast<float*>(ws + lo.w_c1); d.c2 = reinterpret_cast<float*>(ws + lo.w_c2);
  d.cum = reinterpret_cast<float*>(ws + lo.w_cum); d.attU = reinterpret_cast<float*>(ws + lo.w_attU);
  d.keys = reinterpret_cast<float*>(ws + lo.w_keys); d.values = reinterpret_cast<bf16*>(ws + lo.w_values);
  d.pre1 = reinterpret_cast<float*>(ws + lo.w_pre1);
  d.att_smem = att_fwd_smem(lo.Ti, lo.KA, lo.A, D, 2 * H);
}
// zero initial decoder state (Architecture_wrappers.py:134-167) + the merged location filter bank
static int decoder_reset(const StepCtx& s, DecBufs& d) {
  const TL& lo = *s.lo;
  const float* d_params = s.params; cudaStream_t st = s.st;
  const int B = lo.B, Ti = lo.Ti, D = lo.D;
  decoder_bufs(lo, s.ws, d);
  T2_CHECK_CUDA(cudaMemsetAsync(d.S1, 0, (size_t)B * lo.ld_S1 * 2, st));
  T2_CHECK_CUDA(cudaMemsetAsync(d.S2, 0, (size_t)B * lo.ld_S2 * 2, st));
  T2_CHECK_CUDA(cudaMemsetAsync(d.c1, 0, (size_t)B * D * 4, st));
  T2_CHECK_CUDA(cudaMemsetAsync(d.c2, 0, (size_t)B * D * 4, st));
  T2_CHECK_CUDA(cudaMemsetAsync(d.cum, 0, (size_t)B * Ti * 4, st));
  return att_fwd_setup(d_params + lo.p_lck, d_params + lo.p_lcb, d_params + lo.p_lfl, d_params + lo.p_ba, d.attU, lo.KA, lo.F, lo.A, d.att_smem,
                       lo.c.unmasked_encoder, lo.c.noncumulative_weights, lo.c.split_bf16, st);
}
// decoder step t: LSTM-1 (prenet part of its gates precomputed in pre1[t]), LSTM-2, attention (Architecture_wrappers.py:169-213)
static int decoder_step(const StepCtx& s, const DecBufs& d, const int* d_input_lengths, int t) {
  const TL& lo = *s.lo;
  uint8_t* ws = s.ws; const uint8_t* pk = s.pk; const float* d_params = s.params; cudaStream_t st = s.st;
  const int B = lo.B, Ti = lo.Ti, H = lo.H, D = lo.D, K1r = d.K1r, K2 = d.K2, PIK = d.PIK;
  const int ld1 = lo.ld_S1, ld2 = lo.ld_S2, ldp = lo.ld_PI;   // row pitches: K1r / K2 / PIK, split 3 K1r / 3 K2 / 2 PIK
  bf16* S1t = d.S1 + (long long)t * B * ld1;
  bf16* S1n = d.S1 + (long long)(t + 1) * B * ld1;
  bf16* S2t = d.S2 + (long long)t * B * ld2;
  bf16* S2n = d.S2 + (long long)(t + 1) * B * ld2;
  bf16* PIt = d.PI + (long long)t * B * ldp;
  // LSTM 1: state operand [ctx_{t-1} | h1_{t-1}], input part precomputed in pre1[t]
  int rc = lstm_step(s, pk + lo.k_l1r, D, K1r, S1t, B, d.pre1 + (long long)t * B * 4 * D, 4 * D, nullptr, d.c1 + (long long)t * B * D,
                     d.c1 + (long long)(t + 1) * B * D, S1t + 2 * H, ld1, S1n + 2 * H, ld1, S2t, ld2,
                     reinterpret_cast<bf16*>(ws + lo.w_g1) + (long long)t * B * 4 * D, reinterpret_cast<bf16*>(ws + lo.w_t1) + (long long)t * B * D,
                     nullptr, t, 54, lo.c.zoneout_rate, K2, 1);
  if (rc) return rc;
  // LSTM 2: state operand [h1out_t | h2_{t-1}]
  rc = lstm_step(s, pk + lo.k_l2, D, K2, S2t, B, nullptr, 0, d_params + lo.p_l2b, d.c2 + (long long)t * B * D, d.c2 + (long long)(t + 1) * B * D,
                 S2t + D, ld2, S2n + D, ld2, PIt, ldp, reinterpret_cast<bf16*>(ws + lo.w_g2) + (long long)t * B * 4 * D,
                 reinterpret_cast<bf16*>(ws + lo.w_t2) + (long long)t * B * D, nullptr, t, 55, lo.c.zoneout_rate, PIK, 0);
  if (rc) return rc;
  AttArgs a;
  a.h2out = PIt; a.ld_h2 = ldp; a.WqT = reinterpret_cast<const bf16*>(pk + lo.k_qT);
  a.U = d.attU; a.v = d_params + lo.p_v;
  a.keys = d.keys; a.values = d.values; a.lens = d_input_lengths; a.cum = d.cum;
  a.alpha = reinterpret_cast<float*>(ws + lo.w_alpha) + (long long)t * B * Ti;
  a.ctx_a = S1n; a.ld_a = ld1; a.ctx_b = PIt + D; a.ld_b = ldp;
  a.B = B; a.Ti = Ti; a.D = D; a.A = lo.A; a.KA = lo.KA; a.C2 = 2 * H;
  a.unmasked = lo.c.unmasked_encoder; a.noncumulative = lo.c.noncumulative_weights;
  a.split = lo.c.split_bf16; a.lo_h2 = PIK; a.lo_a = K1r; a.lo_b = PIK;
  return launch_att_fwd(a, d.att_smem, st);
}
// prenet (two ReLU + dropout layers) and the prenet part of LSTM-1's gates (pre1) over rows [row0, row0 + nrows) of the [T_out * B]
// decoder buffers; the dropout masks are drawn under seed + *step (step nullable) at hash row offset hash_row0
static int prenet_fwd(const StepCtx& s, int row0, int nrows, unsigned long long seed, const unsigned long long* step, int hash_row0) {
  const TL& lo = *s.lo;
  const uint8_t* pk = s.pk; const float* d_params = s.params;
  const int D = lo.D, sp = lo.c.split_bf16;
  bf16* decin = reinterpret_cast<bf16*>(s.ws + lo.w_decin) + (long long)row0 * lo.ld_decin;
  bf16* pn1 = reinterpret_cast<bf16*>(s.ws + lo.w_pn1) + (long long)row0 * lo.ld_pn1;
  bf16* pn2 = reinterpret_cast<bf16*>(s.ws + lo.w_pn2) + (long long)row0 * lo.ld_pn2;
  float* pre1 = reinterpret_cast<float*>(s.ws + lo.w_pre1) + (long long)row0 * 4 * D;
  int rc = launch_bias_act({.a = decin, .C = lo.M, .T = nrows, .B = 1, .split = sp, .w = pk + lo.k_p1, .N = lo.P1, .wK = (lo.M + 63) / 64 * 64,
                            .BN = lo.P1 >= 256 ? 256 : 128, .bias = d_params + lo.p_p1b, .act = 1, .out_bf16 = pn1, .ldo = lo.P1, .nvalid = lo.P1,
                            .pdrop = lo.c.dropout_rate, .stream = 20, .seed = seed, .step = step, .hash_row0 = hash_row0},
                           s.st);
  if (rc) return rc;
  rc = launch_bias_act({.a = pn1, .C = lo.P1, .T = nrows, .B = 1, .split = sp, .w = pk + lo.k_p2, .N = lo.P2, .wK = lo.P1,
                        .BN = lo.P2 >= 256 ? 256 : 128, .bias = d_params + lo.p_p2b, .act = 1, .out_bf16 = pn2, .ldo = lo.P2, .nvalid = lo.P2,
                        .pdrop = lo.c.dropout_rate, .stream = 21, .seed = seed, .step = step, .hash_row0 = hash_row0},
                       s.st);
  if (rc) return rc;
  return launch_bias_act({.a = pn2, .C = lo.P2, .T = nrows, .B = 1, .split = sp, .w = pk + lo.k_l1x, .N = 4 * D, .wK = lo.P2, .BN = 256,
                          .bias = d_params + lo.p_l1b, .out_f32 = pre1, .ldo = 4 * D, .nvalid = 4 * D},
                         s.st);
}
// frame + stop projections of rows [row0, row0 + nrows) into projo; the bias vector [M frames | 1 stop] lives in two parameter
// tensors, so the caller's finishing kernel adds it
static int proj_fwd(const StepCtx& s, const DecBufs& d, int row0, int nrows) {
  const TL& lo = *s.lo;
  return launch_bias_act({.a = d.PI + (long long)row0 * lo.ld_PI, .C = d.PIK, .T = nrows, .B = 1, .split = lo.c.split_bf16, .w = s.pk + lo.k_proj,
                          .N = lo.M + 1, .wK = d.PIK, .BN = 128,
                          .out_f32 = reinterpret_cast<float*>(s.ws + lo.w_projo) + (long long)row0 * 128, .ldo = 128, .nvalid = lo.M + 1},
                         s.st);
}
// decoder step t of a decoder that feeds its own frames back: prenet(t), decoder_step, projection(t), then proj_bias_feedback_kernel
// adds the biases and writes step t + 1's input. With tgt (teacher-forcing ratio < 1) one draw under seed + *step picks the target frame
// instead when it falls below ratio, and choice[t] records it.
static int decoder_step_fed(const StepCtx& s, const DecBufs& d, const int* d_input_lengths, int t, const float* tgt, float ratio,
                            unsigned long long seed, const unsigned long long* step, int* choice, int hash_row0) {
  const TL& lo = *s.lo;
  const int B = lo.B;
  int rc = prenet_fwd(s, t * B, B, seed, step, hash_row0);
  if (rc) return rc;
  rc = decoder_step(s, d, d_input_lengths, t);
  if (rc) return rc;
  rc = proj_fwd(s, d, t * B, B);
  if (rc) return rc;
  bf16* decin = reinterpret_cast<bf16*>(s.ws + lo.w_decin);
  T2_CHECK_CUDA(launch_pdl(proj_bias_feedback_kernel, dim3(grid1d((long long)B * (lo.M + 1))), dim3(256), 0, s.st,
                           reinterpret_cast<float*>(s.ws + lo.w_projo) + (long long)t * B * 128, s.params + lo.p_fb, s.params + lo.p_sb,
                           t + 1 < lo.To ? decin + (long long)(t + 1) * B * lo.ld_decin : (bf16*)nullptr, B, lo.M, tgt, lo.To, t, ratio, seed, step,
                           choice, lo.c.split_bf16));
  t2_count_launch();
  return T2_OK;
}
// clip the T decoded frames of every item (dec_finish_kernel), the postnet conv blocks (batch norm in training mode when s.training)
// and the residual projection (mel_finish_kernel). With targets the losses go to the workspace scalars: tlen (nullable) masks frames,
// pos_weight weighs the stop loss.
static int postnet_fwd(const StepCtx& s, int T, const float* mel_tgt, const float* stop_tgt, const int* tlen, float pos_weight) {
  const TL& lo = *s.lo;
  uint8_t* ws = s.ws; cudaStream_t st = s.st;
  const int B = lo.B;
  float* scal = reinterpret_cast<float*>(ws + lo.w_scal);
  const float lo_c = -lo.c.max_abs_value - lo.c.lower_bound_decay, hi_c = lo.c.max_abs_value;
  bf16* dec_bm = reinterpret_cast<bf16*>(ws + lo.w_decbm);
  float* dec_f = reinterpret_cast<float*>(ws + lo.w_decf);
  dec_finish_kernel<<<grid1d((long long)B * T * (lo.M + 1)), 256, 0, st>>>(reinterpret_cast<float*>(ws + lo.w_projo), mel_tgt, stop_tgt, dec_bm, dec_f,
                                                                       reinterpret_cast<float*>(ws + lo.w_stop), scal, B, T, lo.M, lo.c.clip_outputs,
                                                                       lo_c, hi_c, lo.c.split_bf16, tlen, pos_weight); t2_count_launch();
  const void* x = dec_bm;
  for (auto& L : lo.post) { int rc = conv_block_fwd(s, L, x, T, s.training); if (rc) return rc; x = ws + L.w_x; }
  float* resid = reinterpret_cast<float*>(ws + lo.w_resid);
  int rc = launch_bias_act({.a = x, .C = lo.PC, .T = T, .B = B, .split = lo.c.split_bf16, .w = s.pk + lo.k_pp, .N = lo.M,
                            .wK = lo.PC, .BN = 128, .bias = s.params + lo.p_ppb, .out_f32 = resid, .ldo = 128, .nvalid = lo.M},
                           st);
  if (rc) return rc;
  mel_finish_kernel<<<grid1d((long long)B * T * lo.M), 256, 0, st>>>(dec_f, resid, mel_tgt, reinterpret_cast<float*>(ws + lo.w_mel), scal, (long long)B * T,
                                                                 lo.M, lo.c.clip_outputs, lo_c, hi_c, tlen, T); t2_count_launch();
  return T2_OK;
}

// forward + losses. d_inputs int32 [B][T_in]; d_input_lengths int32 [B]; d_mel_targets fp32 [B][T_out][M];
// d_stop_targets fp32 [B][T_out]. d_loss fp32[4] = {before, after, stop, regularisation} (already normalised).
extern "C" int t2_taco_forward(const t2_taco_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace, const int* d_inputs,
                               const int* d_input_lengths, const float* d_mel_targets, const float* d_stop_targets, float* d_loss,
                               int training, unsigned long long seed, const unsigned long long* d_step, void* stream) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  if (training) { rc = check_att_bwd_fits(lo); if (rc) return rc; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  StepCtx s{&lo, ws, static_cast<const uint8_t*>(d_packed), d_params, st, seed, d_step, training};
  const int B = lo.B, To = lo.To;
  float* scal = reinterpret_cast<float*>(ws + lo.w_scal);
  T2_CHECK_CUDA(cudaMemsetAsync(scal, 0, 16 * sizeof(float), st));
  const int* tlen = lo.c.mask_decoder ? reinterpret_cast<const int*>(ws + lo.w_tlen) : nullptr;     // t2_taco_set_target_lengths
  rc = encoder_fwd(s, d_inputs, d_input_lengths, training);
  if (rc) return rc;
  bf16* decin = reinterpret_cast<bf16*>(ws + lo.w_decin);
  decin_kernel<<<grid1d((long long)To * B * lo.M), 256, 0, st>>>(d_mel_targets, decin, B, To, lo.M, lo.c.split_bf16); t2_count_launch();
  const long long TB = (long long)To * B;
  DecBufs db;
  if (lo.c.teacher_forcing_ratio >= 1.f) {
    // ---- decoder: everything that does not depend on the recurrence is batched over time (teacher forcing) ----
    rc = prenet_fwd(s, 0, int(TB), seed, d_step, 0);
    if (rc) return rc;
    rc = decoder_reset(s, db);
    if (rc) return rc;
    for (int t = 0; t < To; ++t) { rc = decoder_step(s, db, d_input_lengths, t); if (rc) return rc; }
    T2_CHECK_CUDA(cudaGetLastError());
    // frame + stop projections for all steps at once, then their biases in place (tiny)
    rc = proj_fwd(s, db, 0, int(TB));
    if (rc) return rc;
    proj_bias_kernel<<<grid1d(TB * (lo.M + 1)), 256, 0, st>>>(reinterpret_cast<float*>(ws + lo.w_projo), d_params + lo.p_fb, d_params + lo.p_sb, TB, lo.M);
    t2_count_launch();
  } else {
    // ---- decoder at a teacher-forcing ratio < 1: step t + 1's input is known only once step t has drawn and projected, so the
    // prenet, the LSTM-1 input projection and the projections run per step (the steps of t2_taco_infer_steps). The prenet masks are the
    // elements the batched launches draw (hash row offset t * B), so a step that takes the target repeats the batched arithmetic. ----
    rc = decoder_reset(s, db);
    if (rc) return rc;
    int* choice = reinterpret_cast<int*>(ws + lo.w_tfsel);
    for (int t = 0; t < To; ++t) {
      rc = decoder_step_fed(s, db, d_input_lengths, t, d_mel_targets, lo.c.teacher_forcing_ratio, seed, d_step, choice, t * B);
      if (rc) return rc;
    }
    T2_CHECK_CUDA(cudaGetLastError());
  }
  rc = postnet_fwd(s, To, d_mel_targets, d_stop_targets, tlen, lo.c.cross_entropy_pos_weight);
  if (rc) return rc;
  launch_reg_loss(d_params, reinterpret_cast<const long long*>(ws + lo.w_regtab), lo.n_reg, scal + 3, st);
  T2_CHECK_CUDA(cudaGetLastError());
  loss_norm_kernel<<<1, 1, 0, st>>>(scal, d_loss, float((long long)B * To * lo.M), float((long long)B * To), lo.c.reg_weight, tlen, B, To, lo.M);
  t2_count_launch();
  return T2_OK;
}

// ======================================================================================================
// free-running synthesis (TacoTestHelper, helpers.py:6-59; tacotron.py:150-200 with is_training = False)
// ======================================================================================================
// encoder + zero decoder state + go frame. inputs int32 [B][T_in], lengths int32 [B].
extern "C" int t2_taco_infer_begin(const t2_taco_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace, const int* d_inputs,
                                   const int* d_input_lengths, void* stream) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  StepCtx s{&lo, ws, static_cast<const uint8_t*>(d_packed), d_params, st, 0ull, nullptr, 0};
  rc = encoder_fwd(s, d_inputs, d_input_lengths, 0);
  if (rc) return rc;
  DecBufs db;
  rc = decoder_reset(s, db);
  if (rc) return rc;
  T2_CHECK_CUDA(cudaMemsetAsync(ws + lo.w_decin, 0, (size_t)lo.B * lo.ld_decin * 2, st));   // go frame (helpers.py:31)
  return T2_OK;
}

// decoder steps [t_begin, t_end) of the free-running loop; t_end <= cfg->T_out (= max_iters). After the call
// workspace "stop_logits_tm" [T_out][B] (col M of the projection rows) holds the stop logits of the finished steps:
// the host applies the helper's rule (all rows round(sigmoid) == 1, helpers.py:40-54) and decides whether to continue.
extern "C" int t2_taco_infer_steps(const t2_taco_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace,
                                   const int* d_input_lengths, int t_begin, int t_end, unsigned long long seed, void* stream) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  T2_REQUIRE(t_begin >= 0 && t_begin <= t_end && t_end <= lo.To, T2_ERR_INVALID_ARG, "bad step range [%d, %d)", t_begin, t_end);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  StepCtx s{&lo, ws, static_cast<const uint8_t*>(d_packed), d_params, st, seed, nullptr, 0};
  DecBufs db;
  decoder_bufs(lo, ws, db);
  for (int t = t_begin; t < t_end; ++t) {
    const unsigned long long seed_t = seed + 0x9E3779B97F4A7C15ull * (unsigned long long)(t + 1);   // fresh prenet masks per step
    rc = decoder_step_fed(s, db, d_input_lengths, t, nullptr, 0.f, seed_t, nullptr, nullptr, 0);
    if (rc) return rc;
  }
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

// clip, postnet (inference batch-norm) and residual over the T_used decoded frames. Results (compact, batch-major):
// workspace "decoder_output" / "mel_outputs" [B][T_used][M], "stop_logits" [B][T_used]; alignments stay [T_out][B][T_in].
extern "C" int t2_taco_infer_finish(const t2_taco_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace, int T_used, void* stream) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  T2_REQUIRE(T_used >= 1 && T_used <= lo.To, T2_ERR_INVALID_ARG, "T_used %d outside [1, %d]", T_used, lo.To);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  StepCtx s{&lo, ws, static_cast<const uint8_t*>(d_packed), d_params, st, 0ull, nullptr, 0};
  rc = postnet_fwd(s, T_used, nullptr, nullptr, nullptr, 1.f);
  if (rc) return rc;
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

// tools only: device buffer of 32 int64 that receives clock64() phase stamps of the attention kernels (NULL = off)
extern "C" int t2_dbg_att_stamps(long long* d_buf) {
  T2_CHECK_CUDA(cudaMemcpyToSymbol(g_att_dbg, &d_buf, sizeof(d_buf)));
  return T2_OK;
}

extern "C" int t2_taco_workspace_tensor(const t2_taco_config_t* cfg, void* d_workspace, const char* name, void** ptr, long long* count,
                                        int* elem_bytes) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  const long long B = lo.B, Ti = lo.Ti, To = lo.To;
  struct E { const char* n; long long off, cnt; int eb; };
  const E table[] = {
      {"memory", lo.w_memory, B * Ti * lo.ld_mem, 2}, {"keys", lo.w_keys, B * Ti * lo.A, 4}, {"alignments", lo.w_alpha, To * B * Ti, 4},
      {"decoder_output", lo.w_decf, B * To * lo.M, 4}, {"mel_outputs", lo.w_mel, B * To * lo.M, 4}, {"stop_logits", lo.w_stop, B * To, 4},
      {"projection_rows", lo.w_projo, To * B * 128, 4}, {"enc_conv_out", lo.enc.back().w_x, B * Ti * lo.C, 2}, {"prenet", lo.w_pn2, To * B * lo.ld_pn2, 2}, {"proj_in", lo.w_PI, To * B * lo.ld_PI, 2},
      {"attention_filter_bank", lo.w_attU, (lo.KA + 1) * lo.A, 4},   // merged location filters U [KA][A] + offset row u0
      {"teacher_forced", lo.w_tfsel, To, 4},   // int32 per-step choices of the last forward at teacher_forcing_ratio < 1
  };
  for (const E& e : table)
    if (strcmp(e.n, name) == 0) { *ptr = ws + e.off; *count = e.cnt; *elem_bytes = e.eb; return T2_OK; }
  // per-layer conv-block tensors: "enc_conv_y<i>" / "enc_conv_x<i>" / "post_conv_y<i>" / "post_conv_x<i>" (y = conv + activation,
  // x = batch norm + dropout; bf16 [B][T][C]) and the postnet projection "postnet_residual" (fp32 [B][T_out][128])
  if (strcmp(name, "postnet_residual") == 0) { *ptr = ws + lo.w_resid; *count = B * To * 128; *elem_bytes = 4; return T2_OK; }
  for (int which = 0; which < 2; ++which) {
    const std::vector<ConvL>& v = which == 0 ? lo.enc : lo.post;
    const char* pre = which == 0 ? "enc_conv_" : "post_conv_";
    const size_t pl = strlen(pre);
    if (strncmp(name, pre, pl) == 0 && (name[pl] == 'x' || name[pl] == 'y') && name[pl + 1] >= '0' && name[pl + 1] <= '9') {
      const int i = name[pl + 1] - '0';
      if (i < int(v.size())) {
        *ptr = ws + (name[pl] == 'x' ? v[i].w_x : v[i].w_y);
        *count = B * (which == 0 ? Ti : To) * v[i].cout; *elem_bytes = 2;
        return T2_OK;
      }
    }
  }
  return t2_set_error(T2_ERR_INVALID_ARG, "unknown workspace tensor '%s'", name);
}

extern "C" int t2_taco_set_target_lengths(const t2_taco_config_t* cfg, void* d_workspace, const int* d_target_lengths, void* stream) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  T2_REQUIRE(d_target_lengths != nullptr, T2_ERR_INVALID_ARG, "null target lengths");
  T2_CHECK_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(d_workspace) + lo.w_tlen, d_target_lengths, lo.B * sizeof(int), cudaMemcpyDeviceToDevice,
                                static_cast<cudaStream_t>(stream)));
  return T2_OK;
}

// prenet backward over rows [row0, row0 + nrows) of the [T_out * B] decoder buffers: the input part of LSTM-1's gate gradient (dg1)
// through the input projection and both prenet layers (ReLU + dropout) into dz2 (w_dz) and dpn1 (in place)
static int prenet_bwd(const StepCtx& s, int row0, int nrows) {
  const TL& lo = *s.lo;
  uint8_t* ws = s.ws; cudaStream_t st = s.st;
  const int D = lo.D;
  const long long r2 = (long long)row0 * lo.P2, r1 = (long long)row0 * lo.P1;
  const bf16* dg1 = reinterpret_cast<const bf16*>(ws + lo.w_dg1) + (long long)row0 * 4 * D;
  const bf16* pn1 = reinterpret_cast<const bf16*>(ws + lo.w_pn1) + r1;
  const bf16* pn2 = reinterpret_cast<const bf16*>(ws + lo.w_pn2) + r2;
  bf16* dpn2 = reinterpret_cast<bf16*>(ws + lo.w_dpn2) + r2;
  bf16* dpn1 = reinterpret_cast<bf16*>(ws + lo.w_dpn1) + r1;
  bf16* dz2 = reinterpret_cast<bf16*>(ws + lo.w_dz) + r2;
  int rc = launch_bias_act({.a = dg1, .C = 4 * D, .T = nrows, .B = 1, .w = s.pk + lo.k_l1xT, .N = lo.P2, .wK = 4 * D, .BN = lo.P2 % 256 == 0 ? 256 : 128,
                            .out_bf16 = dpn2, .ldo = lo.P2, .nvalid = lo.P2},
                           st);
  if (rc) return rc;
  relu_drop_bwd_kernel<<<grid1d((long long)nrows * lo.P2), 256, 0, st>>>(dpn2, pn2, dz2, (long long)nrows * lo.P2, lo.c.dropout_rate); t2_count_launch();
  rc = launch_bias_act({.a = dz2, .C = lo.P2, .T = nrows, .B = 1, .w = s.pk + lo.k_p2T, .N = lo.P1, .wK = lo.P2, .BN = lo.P1 % 256 == 0 ? 256 : 128,
                        .out_bf16 = dpn1, .ldo = lo.P1, .nvalid = lo.P1},
                       st);
  if (rc) return rc;
  relu_drop_bwd_kernel<<<grid1d((long long)nrows * lo.P1), 256, 0, st>>>(dpn1, pn1, dpn1, (long long)nrows * lo.P1, lo.c.dropout_rate); t2_count_launch();
  return T2_OK;
}
// loss gradient of the projection outputs of steps [t0, t1) into ddec_tm (ddec_tm_kernel; fb / choice: the gradient of the frame a
// per-step decoder fed back, both nullable) and its product with the transposed frame / stop projections into dPI
static int proj_bwd(const StepCtx& s, const bf16* ddec_post, const float* stop_tgt, int t0, int t1, const float* fb, const int* choice) {
  const TL& lo = *s.lo;
  uint8_t* ws = s.ws; cudaStream_t st = s.st;
  const int B = lo.B, PIK = lo.D + 2 * lo.H;
  const float lo_c = -lo.c.max_abs_value - lo.c.lower_bound_decay, hi_c = lo.c.max_abs_value;
  const int* tlen = lo.c.mask_decoder ? reinterpret_cast<const int*>(ws + lo.w_tlen) : nullptr;
  bf16* ddec_tm = reinterpret_cast<bf16*>(ws + lo.w_ddec_tm);
  ddec_tm_kernel<<<grid1d((long long)(t1 - t0) * B * 128), 256, 0, st>>>(reinterpret_cast<const float*>(ws + lo.w_ddecf), ddec_post,
                                                                       reinterpret_cast<const float*>(ws + lo.w_projo), stop_tgt, ddec_tm, B, lo.To, lo.M,
                                                                       lo.c.clip_outputs, lo_c, hi_c, tlen, lo.c.cross_entropy_pos_weight,
                                                                       reinterpret_cast<const float*>(ws + lo.w_scal), t0, t1, fb, choice);
  t2_count_launch();
  return launch_bias_act({.a = ddec_tm + (long long)t0 * B * 128, .C = 128, .T = (t1 - t0) * B, .B = 1, .w = s.pk + lo.k_projT, .N = PIK, .wK = 128,
                          .BN = PIK % 256 == 0 ? 256 : 128, .out_f32 = reinterpret_cast<float*>(ws + lo.w_dPI) + (long long)t0 * B * PIK, .ldo = PIK,
                          .nvalid = PIK},
                         st);
}

// backward of the last t2_taco_forward(training=1): writes d(total loss)/d(theta) for every trainable tensor
extern "C" int t2_taco_backward(const t2_taco_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                                const int* d_inputs, const int* d_input_lengths, const float* d_mel_targets, const float* d_stop_targets,
                                float* d_grads, unsigned long long seed, const unsigned long long* d_step, void* stream) {
  return t2_taco_backward_ex(cfg, d_params, d_packed, d_workspace, d_inputs, d_input_lengths, d_mel_targets, d_stop_targets, d_grads, nullptr, seed,
                             d_step, stream);
}

extern "C" int t2_taco_backward_ex(const t2_taco_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                                   const int* d_inputs, const int* d_input_lengths, const float* d_mel_targets, const float* d_stop_targets,
                                   float* d_grads, const float* d_mel_outputs_grad, unsigned long long seed, const unsigned long long* d_step,
                                   void* stream) {
  TL lo;
  int rc = build(cfg, lo, nullptr);
  if (rc) return rc;
  T2_REQUIRE(!lo.c.split_bf16, T2_ERR_INVALID_ARG, "split_bf16 (fp32-class conv stacks) mode has no backward pass");
  rc = check_att_bwd_fits(lo);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  const uint8_t* pk = static_cast<const uint8_t*>(d_packed);
  StepCtx s{&lo, ws, pk, d_params, st, seed, d_step, 1};
  const int B = lo.B, Ti = lo.Ti, To = lo.To, H = lo.H, D = lo.D, M = lo.M, A = lo.A;
  const int K1r = 2 * H + D, K2 = 2 * D, PIK = D + 2 * H;
  const long long TB = (long long)To * B, BTo = (long long)B * To;
  std::vector<WgL> wl;
  build_tiles(lo, wl);
  std::vector<int> toff(wl.size());
  { int o = 0; for (size_t i = 0; i < wl.size(); ++i) { toff[i] = o; o += int(wl[i].tiles.size()); } }
  const WgradTile* tiles = reinterpret_cast<const WgradTile*>(ws + lo.w_tiles);
  auto TILES = [&](int i) { return tiles + toff[i]; };
  auto NT = [&](int i) { return int(wl[i].tiles.size()); };
  int li = 0;  // running wgrad-launch index (must follow build_tiles order)
  T2_CHECK_CUDA(cudaMemsetAsync(d_grads, 0, lo.n_params * sizeof(float), st));
  const float lo_c = -lo.c.max_abs_value - lo.c.lower_bound_decay, hi_c = lo.c.max_abs_value;
  bf16* dY0 = reinterpret_cast<bf16*>(ws + lo.w_dY);
  bf16* dY1 = dY0 + (long long)B * (To > Ti ? To : Ti) * (lo.PC > lo.C ? lo.PC : lo.C);
  bf16* dmel = reinterpret_cast<bf16*>(ws + lo.w_dmel);
  float* ddecf = reinterpret_cast<float*>(ws + lo.w_ddecf);
  bf16* dec_bm = reinterpret_cast<bf16*>(ws + lo.w_decbm);
  const int* tlen = lo.c.mask_decoder ? reinterpret_cast<const int*>(ws + lo.w_tlen) : nullptr;
  const float* scal = reinterpret_cast<const float*>(ws + lo.w_scal);      // [5], [6]: the loss normalisers of the forward pass
  // ---- loss seeds + postnet ----
  loss_seed_kernel<<<grid1d(BTo * 128), 256, 0, st>>>(reinterpret_cast<float*>(ws + lo.w_decf), reinterpret_cast<float*>(ws + lo.w_resid),
                                                  reinterpret_cast<float*>(ws + lo.w_mel), d_mel_targets, dmel, ddecf, BTo, M, lo.c.clip_outputs,
                                                  lo_c, hi_c, tlen, To, scal, d_mel_outputs_grad); t2_count_launch();
  rc = launch_bias_act({.a = dmel, .C = 128, .T = To, .B = B, .w = pk + lo.k_ppT, .N = lo.PC, .wK = 128, .BN = lo.PC % 256 == 0 ? 256 : 128, .out_bf16 = dY0,
                        .ldo = lo.PC, .nvalid = lo.PC},
                       st);
  if (rc) return rc;
  {
    ActT maps[2] = {make_act(ws + lo.post.back().w_x, lo.PC, To, B), make_act(dmel, 128, To, B)};
    rc = launch_wgrad(maps, 2, TILES(li), NT(li), d_grads, To, B, st); if (rc) return rc; ++li;
    colsum(dmel, BTo, M, 128, d_grads + lo.p_ppb, 256, st);
  }
  // teacher_forcing_ratio < 1: the frame projection's gradient of step t waits for step t + 1's prenet backward inside the loop below,
  // which writes the prenet gradients into w_dz step by step; the decoder-output gradient then goes to dY0 (the first postnet block's
  // output gradient is dead once its batch-norm backward has run)
  const bool per_step = lo.c.teacher_forcing_ratio < 1.f;
  T2_REQUIRE(!per_step || (To > Ti ? To : Ti) * (long long)(lo.PC > lo.C ? lo.PC : lo.C) >= (long long)To * M, T2_ERR_UNSUPPORTED_SHAPE,
             "teacher_forcing_ratio < 1 needs postnet_channels or enc_conv_channels >= num_mels");
  bf16* ddec_post = per_step ? dY0 : reinterpret_cast<bf16*>(ws + lo.w_dz);
  for (int i = int(lo.post.size()) - 1; i >= 0; --i) {
    const void* xin = i > 0 ? (const void*)(ws + lo.post[i - 1].w_x) : (const void*)dec_bm;
    rc = conv_block_bwd(s, lo.post[i], xin, To, dY0, dY1, i > 0 ? dY0 : ddec_post, d_grads, TILES(li), NT(li));
    if (rc) return rc;
    ++li;
  }
  // ---- projections ----
  bf16* ddec_tm = reinterpret_cast<bf16*>(ws + lo.w_ddec_tm);
  float* dPI = reinterpret_cast<float*>(ws + lo.w_dPI);
  bf16* PI = reinterpret_cast<bf16*>(ws + lo.w_PI);
  auto proj_wgrad = [&]() -> int {
    ActT maps[2] = {make_act(PI, PIK, int(TB), 1), make_act(ddec_tm, 128, int(TB), 1)};
    int r = launch_wgrad(maps, 2, TILES(li), NT(li), d_grads, int(TB), 1, st); if (r) return r; ++li;
    colsum(ddec_tm, TB, M, 128, d_grads + lo.p_fb, 256, st);
    colsum(ddec_tm + M, TB, 1, 128, d_grads + lo.p_sb, 256, st);
    return T2_OK;
  };
  if (!per_step) {
    rc = proj_bwd(s, ddec_post, d_stop_targets, 0, To, nullptr, nullptr);
    if (rc) return rc;
    rc = proj_wgrad();
    if (rc) return rc;
  }
  // ---- decoder: backward through time ----
  float* dh1ext = reinterpret_cast<float*>(ws + lo.w_dh1ext);
  float* dh2ext = reinterpret_cast<float*>(ws + lo.w_dh2ext);
  float* dhs1 = reinterpret_cast<float*>(ws + lo.w_dhs1);
  float* dhs2 = reinterpret_cast<float*>(ws + lo.w_dhs2);
  float* dcs1 = reinterpret_cast<float*>(ws + lo.w_dcs1);
  float* dcs2 = reinterpret_cast<float*>(ws + lo.w_dcs2);
  float* dctxl = reinterpret_cast<float*>(ws + lo.w_dctxl);
  float* dcum = reinterpret_cast<float*>(ws + lo.w_dcum);
  float* cumrun = reinterpret_cast<float*>(ws + lo.w_cumrun);
  float* dkeys = reinterpret_cast<float*>(ws + lo.w_dkeys);
  float* attacc = reinterpret_cast<float*>(ws + lo.w_attacc);
  const int nacc = (lo.KA + 2) * A;
  for (float* p : {dhs1, dhs2, dcs1, dcs2}) T2_CHECK_CUDA(cudaMemsetAsync(p, 0, (size_t)B * D * 4, st));
  T2_CHECK_CUDA(cudaMemsetAsync(dctxl, 0, (size_t)B * 2 * H * 4, st));
  T2_CHECK_CUDA(cudaMemsetAsync(dh1ext, 0, (size_t)B * D * 4, st));
  const int ks_dec = (4 * D / kBK) >= 16 ? 8 : 1, ks_enc = (4 * H / kBK) >= 16 ? 8 : 1;   // k-blocks per slice >= 2
  T2_CHECK_CUDA(cudaMemsetAsync(dcum, 0, (size_t)B * Ti * 4, st));
  T2_CHECK_CUDA(cudaMemsetAsync(dkeys, 0, (size_t)B * Ti * A * 4, st));
  T2_CHECK_CUDA(cudaMemsetAsync(attacc, 0, (size_t)B * nacc * 4, st));
  const int unmasked = lo.c.unmasked_encoder, noncum = lo.c.noncumulative_weights;
  // cumulative state: rebuilt step by step from the final cum_{T_out} (cum_{t-1} = cum_t - alpha_t); non-cumulative: read from the
  // stored alignments of the previous step
  if (!noncum) T2_CHECK_CUDA(cudaMemcpyAsync(cumrun, ws + lo.w_cum, (size_t)B * Ti * 4, cudaMemcpyDeviceToDevice, st));
  bf16* dg1 = reinterpret_cast<bf16*>(ws + lo.w_dg1);
  bf16* dg2 = reinterpret_cast<bf16*>(ws + lo.w_dg2);
  bf16* dctx_all = reinterpret_cast<bf16*>(ws + lo.w_dctx_all);
  bf16* dq_all = reinterpret_cast<bf16*>(ws + lo.w_dq_all);
  const size_t ab_smem = att_bwd_smem(Ti, lo.KA, A, D, 2 * H);
  const float* attU = reinterpret_cast<const float*>(ws + lo.w_attU);
  rc = att_bwd_setup(ab_smem, unmasked, noncum);
  if (rc) return rc;
  bf16* pn1 = reinterpret_cast<bf16*>(ws + lo.w_pn1);
  bf16* pn2 = reinterpret_cast<bf16*>(ws + lo.w_pn2);
  bf16* dpn1 = reinterpret_cast<bf16*>(ws + lo.w_dpn1);
  bf16* dz2 = reinterpret_cast<bf16*>(ws + lo.w_dz);
  float* dfb = reinterpret_cast<float*>(ws + lo.w_dfb);
  const int* choice = reinterpret_cast<const int*>(ws + lo.w_tfsel);
  for (int t = To - 1; t >= 0; --t) {
    if (per_step) {
      // loss gradient of step t's projection outputs + (when step t + 1 consumed step t's frame) the gradient of step t + 1's input,
      // left in dfb by the previous iteration; then dPI_t through the frame / stop projections
      rc = proj_bwd(s, ddec_post, d_stop_targets, t, t + 1, t + 1 < To ? dfb : nullptr, choice);
      if (rc) return rc;
    }
    AttBwd a;
    a.h2out = PI + (long long)t * B * PIK; a.ld_h2 = PIK; a.WqT = reinterpret_cast<const bf16*>(pk + lo.k_qT); a.Wq = d_params + lo.p_qry;
    a.U = attU; a.v = d_params + lo.p_v;
    a.keys = reinterpret_cast<const float*>(ws + lo.w_keys); a.values = reinterpret_cast<const bf16*>(ws + lo.w_values); a.lens = d_input_lengths;
    a.alpha = reinterpret_cast<const float*>(ws + lo.w_alpha) + (long long)t * B * Ti; a.cumrun = cumrun; a.dcum = dcum;
    a.alpha_prev = t > 0 ? a.alpha - (long long)B * Ti : nullptr;
    a.dPI = dPI + (long long)t * B * PIK; a.ld_dPI = PIK; a.dctxl = dctxl; a.dh2ext = dh2ext;
    a.dctx_save = dctx_all + (long long)t * B * 2 * H; a.dq_save = dq_all + (long long)t * B * A; a.dkeys = dkeys; a.acc = attacc;
    a.B = B; a.Ti = Ti; a.D = D; a.A = A; a.KA = lo.KA; a.C2 = 2 * H; a.unmasked = unmasked; a.noncumulative = noncum;
    rc = launch_att_bwd(a, ab_smem, st); if (rc) return rc;
    CellBwd c2;
    c2.dh_ext = dh2ext; c2.zero_ext = 0; c2.ld_ext = D; c2.dhs = dhs2; c2.dcs = dcs2;
    c2.gst = reinterpret_cast<const bf16*>(ws + lo.w_g2) + (long long)t * B * 4 * D; c2.tst = reinterpret_cast<const bf16*>(ws + lo.w_t2) + (long long)t * B * D;
    c2.c_prev = reinterpret_cast<const float*>(ws + lo.w_c2) + (long long)t * B * D;
    c2.dg_a = dg2 + (long long)t * B * 4 * D; c2.ld_a = 4 * D; c2.dg_b = nullptr; c2.ld_b = 0; c2.lens = nullptr; c2.t = t; c2.B = B; c2.H = D; c2.stream = 55;
    c2.zone = lo.c.zoneout_rate; c2.seed = seed; c2.step = d_step;
    rc = launch_cell_bwd(c2, st); if (rc) return rc;
    rc = lstm_bwd_gemm(s, pk + lo.k_l2T, K2, 4 * D, c2.dg_a, B, dh1ext, D, D, 2, dhs2, D, 2, ks_dec);   // dh1ext: zeroed by its consumer
    if (rc) return rc;
    CellBwd c1 = c2;
    c1.dh_ext = dh1ext; c1.zero_ext = 1; c1.dhs = dhs1; c1.dcs = dcs1;
    c1.gst = reinterpret_cast<const bf16*>(ws + lo.w_g1) + (long long)t * B * 4 * D; c1.tst = reinterpret_cast<const bf16*>(ws + lo.w_t1) + (long long)t * B * D;
    c1.c_prev = reinterpret_cast<const float*>(ws + lo.w_c1) + (long long)t * B * D; c1.dg_a = dg1 + (long long)t * B * 4 * D; c1.stream = 54;
    rc = launch_cell_bwd(c1, st); if (rc) return rc;
    rc = lstm_bwd_gemm(s, pk + lo.k_l1rT, K1r, 4 * D, c1.dg_a, B, dctxl, 2 * H, 2 * H, 2, dhs1, D, 2, ks_dec);  // dctxl: zeroed by att_bwd
    if (rc) return rc;
    if (per_step) {
      // the input part of LSTM-1's gate gradient back through the input projection and both prenet layers (ReLU + dropout), into the
      // [T_out * B] buffers of the batched path; for t >= 1 on to d(input frame of step t) = dfb
      rc = prenet_bwd(s, t * B, B);
      if (rc) return rc;
      if (t >= 1) {
        rc = launch_bias_act({.a = dpn1 + (long long)t * B * lo.P1, .C = lo.P1, .T = B, .B = 1, .w = pk + lo.k_p1T, .N = M, .wK = lo.P1, .BN = 128,
                              .out_f32 = dfb, .ldo = M, .nvalid = M},
                             st);
        if (rc) return rc;
      }
    }
  }
  T2_CHECK_CUDA(cudaGetLastError());
  if (per_step) { rc = proj_wgrad(); if (rc) return rc; }
  // ---- recurrent / prenet weight gradients: one wgrad GEMM over all steps ----
  {
    ActT maps[5] = {make_act(ws + lo.w_S2, K2, int(TB), 1), make_act(dg2, 4 * D, int(TB), 1), make_act(ws + lo.w_S1, K1r, int(TB), 1),
                    make_act(dg1, 4 * D, int(TB), 1), make_act(pn2, lo.P2, int(TB), 1)};
    rc = launch_wgrad(maps, 5, TILES(li), NT(li), d_grads, int(TB), 1, st); if (rc) return rc; ++li;
    colsum(dg2, TB, 4 * D, 4 * D, d_grads + lo.p_l2b, 256, st);
    colsum(dg1, TB, 4 * D, 4 * D, d_grads + lo.p_l1b, 256, st);
  }
  if (!per_step) {   // prenet data gradients over all steps (the per-step path wrote them inside the loop)
    rc = prenet_bwd(s, 0, int(TB));
    if (rc) return rc;
  }
  {
    ActT maps[6] = {make_act(pn1, lo.P1, int(TB), 1), make_act(dz2, lo.P2, int(TB), 1), make_act(ws + lo.w_decin, M, int(TB), 1),
                    make_act(dpn1, lo.P1, int(TB), 1), make_act(PI, PIK, int(TB), 1), make_act(dq_all, A, int(TB), 1)};
    rc = launch_wgrad(maps, 6, TILES(li), NT(li), d_grads, int(TB), 1, st); if (rc) return rc; ++li;
    colsum(dz2, TB, lo.P2, lo.P2, d_grads + lo.p_p2b, 256, st);
    colsum(dpn1, TB, lo.P1, lo.P1, d_grads + lo.p_p1b, 256, st);
  }
  {
    float* scratch = reinterpret_cast<float*>(ws + lo.w_attU) + (lo.KA + 1) * A;   // [(KA+2)][A] reduced accumulators
    launch_att_finish(attacc, d_params + lo.p_lck, d_params + lo.p_lcb, d_params + lo.p_lfl, d_grads, B, lo.KA, lo.F, A, lo.p_lck, lo.p_lcb, lo.p_lfl,
                      lo.p_v, lo.p_ba, scratch, st);
  }
  // ---- attention memory: keys / values ----
  bf16* dkeysb = reinterpret_cast<bf16*>(ws + lo.w_dkeysb);
  launch_f32_to_bf16(dkeys, dkeysb, (long long)B * Ti * A, st);
  float* dvalues = reinterpret_cast<float*>(ws + lo.w_dvalues);
  rc = launch_bias_act({.a = dkeysb, .C = A, .T = Ti, .B = B, .w = pk + lo.k_memT, .N = 2 * H, .wK = A, .BN = (2 * H) % 256 == 0 ? 256 : 128,
                        .out_f32 = dvalues, .ldo = 2 * H, .nvalid = 2 * H},
                       st);
  if (rc) return rc;
  {
    ActT maps[2] = {make_act(ws + lo.w_values, 2 * H, Ti, B), make_act(dkeysb, A, Ti, B)};
    rc = launch_wgrad(maps, 2, TILES(li), NT(li), d_grads, Ti, B, st); if (rc) return rc; ++li;
  }
  launch_dvalues_ctx(reinterpret_cast<float*>(ws + lo.w_alpha), dctx_all, d_input_lengths, dvalues, B, Ti, To, 2 * H, st);
  // ---- encoder BiLSTM, backward through time ----
  const void* x3 = ws + lo.enc.back().w_x;
  SideStream* side = side_stream();
  if (side) {
    T2_CHECK_CUDA(cudaEventRecord(side->fork, st));
    T2_CHECK_CUDA(cudaStreamWaitEvent(side->s, side->fork, 0));
  }
  for (int d = 0; d < 2; ++d) {
    cudaStream_t sx = (d == 1 && side) ? side->s : st;
    StepCtx sc = s; sc.st = sx;
    float* edh = reinterpret_cast<float*>(ws + lo.w_encdh[d]);
    float* edc = reinterpret_cast<float*>(ws + lo.w_encdc[d]);
    T2_CHECK_CUDA(cudaMemsetAsync(edh, 0, (size_t)B * H * 4, sx));
    T2_CHECK_CUDA(cudaMemsetAsync(edc, 0, (size_t)B * H * 4, sx));
    bf16* dgall = reinterpret_cast<bf16*>(ws + lo.w_encdgall[d]);
    bf16* dpre = reinterpret_cast<bf16*>(ws + lo.w_dencpre[d]);
    for (int sidx = Ti - 1; sidx >= 0; --sidx) {
      const int t = d == 0 ? sidx : Ti - 1 - sidx;
      CellBwd c;
      c.zero_ext = 0; c.dh_ext = dvalues + (long long)t * 2 * H + d * H; c.ld_ext = (long long)Ti * 2 * H; c.dhs = edh; c.dcs = edc;
      c.gst = reinterpret_cast<const bf16*>(ws + lo.w_encg[d]) + (long long)sidx * B * 4 * H;
      c.tst = reinterpret_cast<const bf16*>(ws + lo.w_enct[d]) + (long long)sidx * B * H;
      c.c_prev = reinterpret_cast<const float*>(ws + lo.w_encc[d]) + (long long)sidx * B * H;
      c.dg_a = dgall + (long long)sidx * B * 4 * H; c.ld_a = 4 * H; c.dg_b = dpre + (long long)t * 4 * H; c.ld_b = (long long)Ti * 4 * H;
      c.lens = d_input_lengths; c.t = t; c.B = B; c.H = H; c.stream = 52 + d; c.zone = lo.c.zoneout_rate; c.seed = seed; c.step = d_step;
      rc = launch_cell_bwd(c, sx); if (rc) return rc;
      rc = lstm_bwd_gemm(sc, pk + lo.k_encWrT[d], H, 4 * H, c.dg_a, B, edh, H, H, 2, nullptr, 0, 0, ks_enc);
      if (rc) return rc;
    }
    {
      ActT maps[2] = {make_act(ws + lo.w_ench[d], H, Ti * B, 1), make_act(dgall, 4 * H, Ti * B, 1)};
      rc = launch_wgrad(maps, 2, TILES(li), NT(li), d_grads, Ti * B, 1, sx); if (rc) return rc; ++li;
      ActT maps2[2] = {make_act(x3, lo.C, Ti, B), make_act(dpre, 4 * H, Ti, B)};
      rc = launch_wgrad(maps2, 2, TILES(li), NT(li), d_grads, Ti, B, sx); if (rc) return rc; ++li;
      colsum(dpre, (long long)B * Ti, 4 * H, 4 * H, d_grads + lo.p_elb[d], 256, sx);
    }
  }
  if (side) {
    T2_CHECK_CUDA(cudaEventRecord(side->join, side->s));
    T2_CHECK_CUDA(cudaStreamWaitEvent(st, side->join, 0));
  }
  // dx3 = dpre_fw x Wx_fw^T + dpre_bw x Wx_bw^T
  bf16* dx3 = reinterpret_cast<bf16*>(ws + lo.w_dx3);
  {
    ActGemmCall g;
    memset(&g, 0, sizeof(g));
    g.a[0] = make_act(ws + lo.w_dencpre[0], 4 * H, Ti, B); g.a[1] = make_act(ws + lo.w_dencpre[1], 4 * H, Ti, B); g.na = 2;
    g.seg[0] = Seg{0, 0, 0, 4 * H / kBK, 0, 1}; g.seg[1] = Seg{1, 0, 0, 4 * H / kBK, 0, 1}; g.nseg = 2;
    g.w = pk + lo.k_encWxT; g.wN = lo.C; g.wK = 8 * H; g.wL = 1;
    g.T = Ti; g.B = B; g.n_tiles = lo.C / (lo.C % 256 == 0 ? 256 : 128);
    g.epi.ptr[0] = dx3; g.epi.i[0] = lo.C; g.epi.i[1] = 0; g.epi.i[2] = lo.C;
    rc = launch_act_gemm(EPI_BIAS_ACT, lo.C % 256 == 0 ? 256 : 128, g, st);
    if (rc) return rc;
  }
  // ---- encoder conv blocks + embedding ----
  {
    const bf16* dout = dx3;   // a block's output gradient is dead once its BN backward has run, so dx may overwrite it
    bf16* demb = reinterpret_cast<bf16*>(ws + lo.w_demb);
    for (int i = int(lo.enc.size()) - 1; i >= 0; --i) {
      const void* xin = i > 0 ? (const void*)(ws + lo.enc[i - 1].w_x) : (const void*)(ws + lo.w_emb);
      bf16* dx = i > 0 ? dY0 : demb;
      rc = conv_block_bwd(s, lo.enc[i], xin, Ti, dout, dY1, dx, d_grads, TILES(li), NT(li));
      if (rc) return rc;
      ++li;
      dout = dx;
    }
    embed_bwd_kernel<<<grid1d((long long)B * Ti * lo.E), 256, 0, st>>>(d_inputs, demb, d_grads + lo.p_emb, (long long)B * Ti, lo.E); t2_count_launch();
  }
  // ---- L2 regulariser (tacotron.py:343-345) ----
  launch_reg_grad(d_params, d_grads, reinterpret_cast<const long long*>(ws + lo.w_regtab), lo.n_reg, lo.c.reg_weight, st);
  T2_CHECK_CUDA(cudaGetLastError());
  return T2_OK;
}

// test hook: one production kernel on caller buffers (include/t2b200.h, T2_DBG_TACO_*)
extern "C" int t2_dbg_taco_kernel(const t2_dbg_kernel_t* call, void* stream) {
  T2_REQUIRE(call != nullptr, T2_ERR_INVALID_ARG, "dbg_taco_kernel: null call");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  void* const* p = call->p;
  const long long* i = call->i;
  auto aligned16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  switch (call->kernel) {
    case T2_DBG_TACO_ATT_FWD: {
      const int B = int(i[0]), Ti = int(i[1]), D = int(i[2]), A = int(i[3]), KA = int(i[4]), F = int(i[5]), C2 = int(i[6]);
      for (int k = 0; k < 15; ++k)
        T2_REQUIRE(k == 13 || p[k] != nullptr, T2_ERR_INVALID_ARG, "dbg_taco_kernel ATT_FWD: null pointer argument %d", k);
      T2_REQUIRE(B >= 1 && B <= 256 && Ti >= 1 && Ti <= 1024 && D >= 32 && D % 32 == 0 && A % 64 == 0 && A >= 64 && A <= 128 && KA >= 1 &&
                     KA % 2 == 1 && KA <= 31 && F >= 1 && F <= 32 && C2 >= 64 && C2 % 64 == 0,
                 T2_ERR_UNSUPPORTED_SHAPE, "dbg_taco_kernel ATT_FWD: unsupported shape");
      T2_REQUIRE(i[7] >= D && i[8] >= C2 && i[9] >= C2 && aligned16(p[1]) && aligned16(p[9]) && (reinterpret_cast<uintptr_t>(p[8]) & 7) == 0 &&
                     (reinterpret_cast<uintptr_t>(p[7]) & 7) == 0,
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel ATT_FWD: bad pitch or alignment");
      T2_REQUIRE((i[10] == 0 || i[10] == 1) && (i[11] == 0 || i[11] == 1), T2_ERR_INVALID_ARG,
                 "dbg_taco_kernel ATT_FWD: unmasked / noncumulative must be 0 or 1");
      const int split = int(i[12]);
      T2_REQUIRE(split == 0 ? i[13] == 0 && i[14] == 0 && i[15] == 0
                            : split == 1 && i[13] >= D && i[7] >= i[13] + D && i[14] >= C2 && (!p[13] || i[8] >= 2 * i[14] + C2) &&
                                  i[15] >= C2 && i[9] >= i[15] + C2,
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel ATT_FWD: bad split flag or lo offsets");
      const size_t smem = att_fwd_smem(Ti, KA, A, D, C2);
      T2_REQUIRE(smem <= kSmemOptin, T2_ERR_UNSUPPORTED_SHAPE, "dbg_taco_kernel ATT_FWD: %zu B of shared memory", smem);
      AttArgs a;
      a.split = split; a.lo_h2 = int(i[13]); a.lo_a = int(i[14]); a.lo_b = int(i[15]);
      a.h2out = static_cast<const bf16*>(p[0]); a.ld_h2 = int(i[7]); a.WqT = static_cast<const bf16*>(p[1]);
      a.U = static_cast<float*>(p[6]); a.v = static_cast<const float*>(p[7]);
      a.keys = static_cast<const float*>(p[8]); a.values = static_cast<const bf16*>(p[9]); a.lens = static_cast<const int*>(p[10]);
      a.cum = static_cast<float*>(p[11]); a.alpha = static_cast<float*>(p[12]);
      a.ctx_a = static_cast<bf16*>(p[13]); a.ld_a = int(i[8]); a.ctx_b = static_cast<bf16*>(p[14]); a.ld_b = int(i[9]);
      a.B = B; a.Ti = Ti; a.D = D; a.A = A; a.KA = KA; a.C2 = C2; a.unmasked = int(i[10]); a.noncumulative = int(i[11]);
      int rc = att_fwd_setup(static_cast<const float*>(p[2]), static_cast<const float*>(p[3]), static_cast<const float*>(p[4]),
                             static_cast<const float*>(p[5]), static_cast<float*>(p[6]), KA, F, A, smem, a.unmasked, a.noncumulative, split, st);
      return rc ? rc : launch_att_fwd(a, smem, st);
    }
    case T2_DBG_TACO_CONV_GEMM: {
      const int C = int(i[0]), T = int(i[1]), Bn = int(i[2]), N = int(i[3]), wK = int(i[4]), ntaps = int(i[5]), BN = int(i[6]);
      const int act = int(i[7]), ldo = int(i[8]), nvalid = int(i[9]), sid = int(i[10]), split = int(i[11]), row0 = int(i[12]);
      const float pdrop = call->f[0];
      const int Cp = (C + kBK - 1) / kBK * kBK;
      T2_REQUIRE(p[0] && p[1] && (p[3] || p[4]) && aligned16(p[0]) && aligned16(p[1]) && (split == 0 || split == 1) &&
                     ntaps >= 1 && ntaps <= (split ? kMaxSeg / 2 : kMaxSeg),
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel CONV_GEMM: bad pointers, split flag or tap count");
      T2_REQUIRE(C >= 1 && C <= 4096 && (split || C % 8 == 0) && T >= 1 && Bn >= 1 && Bn <= 65535 && N >= 1 && wK % 8 == 0 &&
                     wK >= ntaps * Cp * (split ? 3 : 1) && (BN == 128 || BN == 256) && act >= 0 && act <= 2 && nvalid >= 1 && nvalid <= N &&
                     ldo >= nvalid && sid >= 0 && row0 >= 0 && pdrop >= 0.f && pdrop < 1.f && (ldo % 8 == 0 || !split),
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel CONV_GEMM: bad shape");
      int shifts[kMaxSeg];
      for (int j = 0; j < ntaps; ++j) shifts[j] = conv_tap_shift(ntaps, j);
      int rc = launch_bias_act({.a = p[0], .C = C, .T = T, .B = Bn, .ntaps = ntaps, .shifts = shifts, .split = split, .w = p[1], .N = N, .wK = wK, .BN = BN,
                                .bias = static_cast<const float*>(p[2]), .act = act, .out_bf16 = p[3], .out_f32 = static_cast<float*>(p[4]), .ldo = ldo,
                                .nvalid = nvalid, .pdrop = pdrop, .stream = sid, .seed = call->seed, .step = call->step, .hash_row0 = row0},
                               st);
      if (rc) return rc;
      T2_CHECK_CUDA(cudaGetLastError());
      return T2_OK;
    }
    case T2_DBG_TACO_LSTM_STEP: {
      const int H = int(i[0]), K = int(i[1]), B = int(i[2]), pre_stride = int(i[3]), ld_hp = int(i[4]), ld_hs = int(i[5]), ld_ho = int(i[6]);
      const int t = int(i[7]), sid = int(i[8]), out_lo = int(i[9]), out_state = int(i[10]), training = int(i[11]), split = int(i[12]);
      const float zone = call->f[0];
      T2_REQUIRE(p[0] && p[1] && p[4] && p[5] && p[6] && p[7] && p[8] && aligned16(p[0]) && aligned16(p[1]) && (split == 0 || split == 1) &&
                     (training == 0 || training == 1) && (out_state == 0 || out_state == 1) && zone >= 0.f && zone < 1.f && t >= 0 && sid >= 0,
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel LSTM_STEP: bad pointers or flags");
      T2_REQUIRE(H >= 32 && H % 32 == 0 && K >= 64 && K % 64 == 0 && B >= 1 && B <= 65535 && (!p[2] || pre_stride >= 4 * H) &&
                     (split ? ld_hp >= K + H && ld_hs >= 2 * K + H && out_lo >= H && ld_ho >= (out_state ? 2 : 1) * out_lo + H
                            : ld_hp >= H && ld_hs >= H && ld_ho >= H && out_lo == 0 && out_state == 0),
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel LSTM_STEP: bad shape or pitch");
      TL lo{};
      lo.c.split_bf16 = split;
      StepCtx s{&lo, nullptr, nullptr, nullptr, st, call->seed, call->step, training};
      int rc = lstm_step(s, p[0], H, K, p[1], B, static_cast<const float*>(p[2]), pre_stride, static_cast<const float*>(p[3]),
                         static_cast<const float*>(p[4]), static_cast<float*>(p[5]), static_cast<const bf16*>(p[6]), ld_hp,
                         static_cast<bf16*>(p[7]), ld_hs, static_cast<bf16*>(p[8]), ld_ho, static_cast<bf16*>(p[9]), static_cast<bf16*>(p[10]),
                         static_cast<const int*>(p[11]), t, sid, zone, out_lo, out_state);
      if (rc) return rc;
      T2_CHECK_CUDA(cudaGetLastError());
      return T2_OK;
    }
    case T2_DBG_TACO_ROWS: {
      const int which = int(i[0]), split = int(i[1]);
      T2_REQUIRE(which >= 0 && which <= 4 && (split == 0 || split == 1), T2_ERR_INVALID_ARG, "dbg_taco_kernel ROWS: bad writer or split flag");
      if (which == 0) {   // embed_fwd_kernel
        const long long npos = i[2];
        const int E = int(i[3]);
        T2_REQUIRE(p[0] && p[1] && p[2] && npos >= 1 && E >= 1, T2_ERR_INVALID_ARG, "dbg_taco_kernel ROWS embed: bad arguments");
        embed_fwd_kernel<<<grid1d(npos * E), 256, 0, st>>>(static_cast<const int*>(p[0]), static_cast<const float*>(p[1]), static_cast<bf16*>(p[2]),
                                                           npos, E, split);
      } else if (which == 1) {   // decin_kernel
        const int B = int(i[2]), To = int(i[3]), M = int(i[4]);
        T2_REQUIRE(p[0] && p[1] && B >= 1 && To >= 1 && M >= 1 && (!split || M <= 128), T2_ERR_INVALID_ARG,
                   "dbg_taco_kernel ROWS decin: bad arguments");
        decin_kernel<<<grid1d((long long)To * B * M), 256, 0, st>>>(static_cast<const float*>(p[0]), static_cast<bf16*>(p[1]), B, To, M, split);
      } else if (which == 2) {   // dec_finish_kernel
        const int B = int(i[2]), To = int(i[3]), M = int(i[4]), clip = int(i[5]);
        T2_REQUIRE(p[0] && p[3] && p[4] && p[5] && p[6] && B >= 1 && To >= 1 && M >= 1 && M + 1 <= 128 && (clip == 0 || clip == 1),
                   T2_ERR_INVALID_ARG, "dbg_taco_kernel ROWS dec_finish: bad arguments");
        dec_finish_kernel<<<grid1d((long long)B * To * (M + 1)), 256, 0, st>>>(
            static_cast<const float*>(p[0]), static_cast<const float*>(p[1]), static_cast<const float*>(p[2]), static_cast<bf16*>(p[3]),
            static_cast<float*>(p[4]), static_cast<float*>(p[5]), static_cast<float*>(p[6]), B, To, M, clip, call->f[0], call->f[1], split,
            static_cast<const int*>(p[7]), call->f[2]);
      } else if (which == 3) {   // proj_bias_feedback_kernel
        const int B = int(i[2]), M = int(i[3]), To = int(i[4]), t = int(i[5]);
        T2_REQUIRE(p[0] && p[1] && p[2] && (!p[4] || p[5]) && B >= 1 && M >= 1 && M + 1 <= 128 && To >= 1 && t >= 0 && t < To &&
                       call->f[0] >= 0.f && call->f[0] <= 1.f,
                   T2_ERR_INVALID_ARG, "dbg_taco_kernel ROWS proj_bias_feedback: bad arguments");
        T2_CHECK_CUDA(launch_pdl(proj_bias_feedback_kernel, dim3(grid1d((long long)B * (M + 1))), dim3(256), 0, st, static_cast<float*>(p[0]),
                                 static_cast<const float*>(p[1]), static_cast<const float*>(p[2]), static_cast<bf16*>(p[3]), B, M,
                                 static_cast<const float*>(p[4]), To, t, call->f[0], call->seed, call->step, static_cast<int*>(p[5]), split));
      } else {   // f32_to_bf16_kernel
        const long long rows = i[2];
        const int C = int(i[3]), Cp = int(i[4]);
        T2_REQUIRE(p[0] && p[1] && rows >= 1 && C >= 1 && (split ? Cp >= C : Cp == C), T2_ERR_INVALID_ARG,
                   "dbg_taco_kernel ROWS f32_to_bf16: bad arguments");
        if (split) launch_f32_to_bf16_split(static_cast<const float*>(p[0]), static_cast<bf16*>(p[1]), rows, C, Cp, st);
        else launch_f32_to_bf16(static_cast<const float*>(p[0]), static_cast<bf16*>(p[1]), rows * C, st);
      }
      if (which <= 3) t2_count_launch();
      T2_CHECK_CUDA(cudaGetLastError());
      return T2_OK;
    }
    case T2_DBG_TACO_ATT_BWD: {
      const int B = int(i[0]), Ti = int(i[1]), D = int(i[2]), A = int(i[3]), KA = int(i[4]), C2 = int(i[5]);
      const int unmasked = int(i[8]), noncum = int(i[9]);
      for (int k = 0; k < 16; ++k)
        T2_REQUIRE(k == 8 || p[k] != nullptr, T2_ERR_INVALID_ARG, "dbg_taco_kernel ATT_BWD: null pointer argument %d", k);
      T2_REQUIRE((i[8] == 0 || i[8] == 1) && (i[9] == 0 || i[9] == 1), T2_ERR_INVALID_ARG,
                 "dbg_taco_kernel ATT_BWD: unmasked / noncumulative must be 0 or 1");
      T2_REQUIRE(noncum || p[8] != nullptr, T2_ERR_INVALID_ARG, "dbg_taco_kernel ATT_BWD: the cumulative state needs cumrun (p[8])");
      T2_REQUIRE(B >= 1 && B <= 256 && Ti >= 1 && Ti <= 1024 && D >= 32 && D % 32 == 0 && A % 64 == 0 && A >= 64 && A <= 128 && KA >= 1 &&
                     KA % 2 == 1 && KA <= 31 && C2 >= 64 && C2 % 64 == 0,
                 T2_ERR_UNSUPPORTED_SHAPE, "dbg_taco_kernel ATT_BWD: unsupported shape");
      auto aligned8 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 7) == 0; };
      T2_REQUIRE(i[6] >= D && i[7] >= D + C2 && i[7] % 2 == 0 && aligned16(p[1]) && aligned16(p[5]) && aligned8(p[3]) && aligned8(p[4]) &&
                     aligned8(p[10]) && aligned8(p[12]) && aligned8(p[14]) && aligned8(p[15]),
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel ATT_BWD: bad pitch or alignment");
      const size_t smem = att_bwd_smem(Ti, KA, A, D, C2);
      T2_REQUIRE(smem <= kSmemOptin, T2_ERR_UNSUPPORTED_SHAPE, "dbg_taco_kernel ATT_BWD: %zu B of shared memory", smem);
      AttBwd a;
      a.h2out = static_cast<const bf16*>(p[0]); a.ld_h2 = int(i[6]); a.WqT = static_cast<const bf16*>(p[1]); a.Wq = nullptr;
      a.U = static_cast<const float*>(p[2]); a.v = static_cast<const float*>(p[3]);
      a.keys = static_cast<const float*>(p[4]); a.values = static_cast<const bf16*>(p[5]); a.lens = static_cast<const int*>(p[6]);
      a.alpha = static_cast<const float*>(p[7]);
      a.cumrun = noncum ? nullptr : static_cast<float*>(p[8]);
      a.alpha_prev = noncum ? static_cast<const float*>(p[8]) : nullptr;
      a.dcum = static_cast<float*>(p[9]); a.dPI = static_cast<const float*>(p[10]); a.ld_dPI = int(i[7]);
      a.dctxl = static_cast<float*>(p[11]); a.dh2ext = static_cast<float*>(p[12]);
      a.dctx_save = static_cast<bf16*>(p[13]); a.dq_save = static_cast<bf16*>(p[13]) + (long long)B * C2;
      a.dkeys = static_cast<float*>(p[14]); a.acc = static_cast<float*>(p[15]);
      a.B = B; a.Ti = Ti; a.D = D; a.A = A; a.KA = KA; a.C2 = C2; a.unmasked = unmasked; a.noncumulative = noncum;
      int rc = att_bwd_setup(smem, unmasked, noncum);
      return rc ? rc : launch_att_bwd(a, smem, st);
    }
    case T2_DBG_TACO_BN_FWD: {
      const long long rows = i[0];
      const int C = int(i[1]);
      T2_REQUIRE(rows >= 1 && C >= 1 && C <= 4096 && p[0] && p[1] && p[2] && p[3] && p[4] && p[5] && p[6] && (i[2] == 0 || i[2] == 1) &&
                     (i[3] == 0 || i[3] == 1) && (i[5] == 0 || i[5] == 1) && i[4] >= 0 && call->f[0] >= 0.f && call->f[0] < 1.f,
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel BN_FWD: bad arguments");
      float* stats = static_cast<float*>(p[2]);
      const BnDropout drop{call->f[0], call->seed, call->step, int(i[4])};
      if (i[2]) T2_CHECK_CUDA(cudaMemsetAsync(stats, 0, 2 * C * sizeof(float), st));
      if (i[3])
        bn_fwd(static_cast<const float*>(p[0]), C, 0, static_cast<bf16*>(p[1]), int(i[5]), nullptr, nullptr, stats, C, static_cast<const float*>(p[3]),
               static_cast<const float*>(p[4]), static_cast<float*>(p[5]), static_cast<float*>(p[6]), rows, C, int(i[2]), drop, 256, st);
      else
        bn_fwd(static_cast<const bf16*>(p[0]), C, 0, static_cast<bf16*>(p[1]), int(i[5]), nullptr, nullptr, stats, C, static_cast<const float*>(p[3]),
               static_cast<const float*>(p[4]), static_cast<float*>(p[5]), static_cast<float*>(p[6]), rows, C, int(i[2]), drop, 256, st);
      T2_CHECK_CUDA(cudaGetLastError());
      return T2_OK;
    }
    case T2_DBG_TACO_BN_BWD: {
      const long long rows = i[0];
      const int C = int(i[1]);
      T2_REQUIRE(rows >= 1 && C >= 1 && C <= 4096 && p[0] && p[1] && p[2] && p[3] && p[4] && p[5] && p[6] && i[2] >= 0 && i[2] <= 2 &&
                     i[3] >= 0 && call->f[0] >= 0.f && call->f[0] < 1.f,
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel BN_BWD: bad arguments");
      float* stats = static_cast<float*>(p[2]);
      T2_CHECK_CUDA(cudaMemsetAsync(stats + 4 * C, 0, 2 * C * sizeof(float), st));
      bn_bwd(static_cast<const bf16*>(p[0]), C, static_cast<const bf16*>(p[1]), C, 0, stats, C, stats + 4 * C, static_cast<const float*>(p[3]),
             static_cast<bf16*>(p[4]), C, static_cast<float*>(p[5]), static_cast<float*>(p[6]), rows, C, int(i[2]),
             BnDropout{call->f[0], call->seed, call->step, int(i[3])}, 256, st);
      T2_CHECK_CUDA(cudaGetLastError());
      return T2_OK;
    }
    case T2_DBG_TACO_CELL_BWD: {
      CellBwd c;
      c.dh_ext = static_cast<float*>(p[0]); c.ld_ext = i[0]; c.zero_ext = int(i[1]);
      c.dhs = static_cast<float*>(p[1]); c.dcs = static_cast<float*>(p[2]);
      c.gst = static_cast<const bf16*>(p[3]); c.tst = static_cast<const bf16*>(p[4]); c.c_prev = static_cast<const float*>(p[5]);
      c.dg_a = static_cast<bf16*>(p[6]); c.ld_a = i[2]; c.dg_b = static_cast<bf16*>(p[7]); c.ld_b = i[3];
      c.lens = static_cast<const int*>(p[8]); c.t = int(i[4]); c.B = int(i[5]); c.H = int(i[6]); c.stream = int(i[7]);
      c.zone = call->f[0]; c.seed = call->seed; c.step = call->step;
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && p[4] && p[5] && p[6] && c.B >= 1 && c.H >= 1 && c.t >= 0 && c.ld_ext >= c.H &&
                     c.ld_a >= 4 * c.H && (!c.dg_b || c.ld_b >= 4 * c.H) && (c.zero_ext == 0 || c.zero_ext == 1) && c.stream >= 0 &&
                     c.zone >= 0.f && c.zone < 1.f,
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel CELL_BWD: bad arguments");
      return launch_cell_bwd(c, st);
    }
    case T2_DBG_TACO_ATT_FINISH: {
      const int B = int(i[0]), KA = int(i[1]), F = int(i[2]), A = int(i[3]);
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && p[4] && p[5] && B >= 1 && KA >= 1 && KA <= 31 && F >= 1 && F <= 32 && A >= 1 && A <= 128 &&
                     i[4] >= 0 && i[5] >= 0 && i[6] >= 0 && i[7] >= 0 && i[8] >= 0,
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel ATT_FINISH: bad arguments");
      launch_att_finish(static_cast<const float*>(p[0]), static_cast<const float*>(p[1]), static_cast<const float*>(p[2]),
                        static_cast<const float*>(p[3]), static_cast<float*>(p[4]), B, KA, F, A, i[4], i[5], i[6], i[7], i[8],
                        static_cast<float*>(p[5]), st);
      T2_CHECK_CUDA(cudaGetLastError());
      return T2_OK;
    }
    case T2_DBG_TACO_DVALUES: {
      const int B = int(i[0]), Ti = int(i[1]), To = int(i[2]), C2 = int(i[3]);
      T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && B >= 1 && B <= 65535 && Ti >= 1 && To >= 1 && C2 >= 1, T2_ERR_INVALID_ARG,
                 "dbg_taco_kernel DVALUES: bad arguments");
      launch_dvalues_ctx(static_cast<const float*>(p[0]), static_cast<const bf16*>(p[1]), static_cast<const int*>(p[2]), static_cast<float*>(p[3]),
                         B, Ti, To, C2, st);
      T2_CHECK_CUDA(cudaGetLastError());
      return T2_OK;
    }
    case T2_DBG_TACO_LOSS: {
      const int which = int(i[0]);
      const float* f = call->f;
      T2_REQUIRE(which >= 0 && which <= 8, T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS: bad kernel selector %d", which);
      if (which <= 3) {   // the decoder-output losses: B, To, M (+ clip) as the engine passes them, rows of pitch 128
        const int B = int(i[1]), To = int(i[2]), M = int(i[3]), clip = int(i[4]);
        T2_REQUIRE(i[1] >= 1 && i[1] <= 65535 && i[2] >= 1 && i[2] <= 65535 && M >= 1 && M + 1 <= 128 && (which == 1 || clip == 0 || clip == 1),
                   T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS: bad shape or clip flag");
        const long long BTo = (long long)B * To;
        if (which == 0) {
          T2_REQUIRE(p[0] && p[1] && p[3] && p[4], T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS mel_finish: null pointer");
          mel_finish_kernel<<<grid1d(BTo * M), 256, 0, st>>>(static_cast<const float*>(p[0]), static_cast<const float*>(p[1]),
                                                             static_cast<const float*>(p[2]), static_cast<float*>(p[3]), static_cast<float*>(p[4]),
                                                             BTo, M, clip, f[0], f[1], static_cast<const int*>(p[5]), To);
        } else if (which == 1) {
          T2_REQUIRE(p[0], T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS loss_norm: null pointer");
          loss_norm_kernel<<<1, 1, 0, st>>>(static_cast<float*>(p[0]), static_cast<float*>(p[1]), float(BTo * M), float(BTo), f[0],
                                            static_cast<const int*>(p[2]), B, To, M);
        } else if (which == 2) {
          T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && p[4] && p[5] && p[7], T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS loss_seed: null pointer");
          loss_seed_kernel<<<grid1d(BTo * 128), 256, 0, st>>>(static_cast<const float*>(p[0]), static_cast<const float*>(p[1]),
                                                              static_cast<const float*>(p[2]), static_cast<const float*>(p[3]), static_cast<bf16*>(p[4]),
                                                              static_cast<float*>(p[5]), BTo, M, clip, f[0], f[1], static_cast<const int*>(p[6]), To,
                                                              static_cast<const float*>(p[7]), static_cast<const float*>(p[8]));
        } else {
          const int t0 = int(i[5]), t1 = int(i[6]);
          T2_REQUIRE(p[0] && p[1] && p[2] && p[3] && p[4] && p[6] && (!p[7] || p[8]), T2_ERR_INVALID_ARG,
                     "dbg_taco_kernel LOSS ddec_tm: null pointer (choice is required with fb)");
          T2_REQUIRE(t0 >= 0 && t0 < t1 && t1 <= To, T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS ddec_tm: bad step range [%d, %d)", t0, t1);
          ddec_tm_kernel<<<grid1d((long long)(t1 - t0) * B * 128), 256, 0, st>>>(
              static_cast<const float*>(p[0]), static_cast<const bf16*>(p[1]), static_cast<const float*>(p[2]), static_cast<const float*>(p[3]),
              static_cast<bf16*>(p[4]), B, To, M, clip, f[0], f[1], static_cast<const int*>(p[5]), f[2], static_cast<const float*>(p[6]), t0, t1,
              static_cast<const float*>(p[7]), static_cast<const int*>(p[8]));
        }
      } else if (which == 4) {   // proj_bias_kernel
        const long long rows = i[1];
        const int M = int(i[2]);
        T2_REQUIRE(p[0] && p[1] && p[2] && rows >= 1 && M >= 1 && M + 1 <= 128, T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS proj_bias: bad arguments");
        proj_bias_kernel<<<grid1d(rows * (M + 1)), 256, 0, st>>>(static_cast<float*>(p[0]), static_cast<const float*>(p[1]),
                                                                 static_cast<const float*>(p[2]), rows, M);
      } else if (which == 5) {   // relu_drop_bwd_kernel (dz may alias d, as the engine's second call does)
        const long long n = i[1];
        T2_REQUIRE(p[0] && p[1] && p[2] && n >= 1 && f[0] >= 0.f && f[0] < 1.f, T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS relu_drop_bwd: bad arguments");
        relu_drop_bwd_kernel<<<grid1d(n), 256, 0, st>>>(static_cast<const bf16*>(p[0]), static_cast<const bf16*>(p[1]), static_cast<bf16*>(p[2]), n, f[0]);
      } else if (which == 6) {   // embed_bwd_kernel
        const long long npos = i[1];
        const int E = int(i[2]);
        T2_REQUIRE(p[0] && p[1] && p[2] && npos >= 1 && E >= 1, T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS embed_bwd: bad arguments");
        embed_bwd_kernel<<<grid1d(npos * E), 256, 0, st>>>(static_cast<const int*>(p[0]), static_cast<const bf16*>(p[1]), static_cast<float*>(p[2]), npos, E);
      } else if (which == 7) {   // mask_values_kernel
        const int B = int(i[1]), Ti = int(i[2]), C2 = int(i[3]);
        T2_REQUIRE(p[0] && p[1] && p[2] && B >= 1 && Ti >= 1 && C2 >= 1, T2_ERR_INVALID_ARG, "dbg_taco_kernel LOSS mask_values: bad arguments");
        mask_values_kernel<<<grid1d((long long)B * Ti * C2), 256, 0, st>>>(static_cast<const bf16*>(p[0]), static_cast<const int*>(p[1]),
                                                                          static_cast<bf16*>(p[2]), B, Ti, C2);
      } else {   // bias_colsum_kernel<bf16> through colsum
        const long long rows = i[1];
        const int C = int(i[2]), ld = int(i[3]), threads = int(i[4]);
        T2_REQUIRE(p[0] && p[1] && rows >= 1 && C >= 1 && ld >= C && (threads == 128 || threads == 256), T2_ERR_INVALID_ARG,
                   "dbg_taco_kernel LOSS bias_colsum: bad arguments");
        colsum(static_cast<const bf16*>(p[0]), rows, C, ld, static_cast<float*>(p[1]), threads, st);
      }
      if (which <= 7) t2_count_launch();
      T2_CHECK_CUDA(cudaGetLastError());
      return T2_OK;
    }
    case T2_DBG_TACO_PARAMS: {
      const int which = int(i[0]);
      T2_REQUIRE(which >= 0 && which <= 3, T2_ERR_INVALID_ARG, "dbg_taco_kernel PARAMS: bad kernel selector %d", which);
      if (which >= 2) {   // reg_loss_kernel / reg_grad_kernel over a caller (offset, elements) table of i[1] tensors
        const long long n_reg = i[1];
        T2_REQUIRE(p[0] && p[1] && p[2] && n_reg >= 1 && n_reg <= 65535, T2_ERR_INVALID_ARG, "dbg_taco_kernel PARAMS reg: bad arguments");
        if (which == 2)
          launch_reg_loss(static_cast<const float*>(p[0]), static_cast<const long long*>(p[1]), int(n_reg), static_cast<float*>(p[2]), st);
        else
          launch_reg_grad(static_cast<const float*>(p[0]), static_cast<float*>(p[1]), static_cast<const long long*>(p[2]), int(n_reg), call->f[0], st);
        T2_CHECK_CUDA(cudaGetLastError());
        return T2_OK;
      }
      // pack_kernel: one job (add_pack) or the three jobs of a split-bf16 slot, built here and copied into the caller's job buffer
      const int split = which == 1, W = int(i[2]), grid_x = int(i[3]);
      const long long src = i[4], dst = i[7];
      const int K = int(i[5]), N = int(i[6]), ld = int(i[8]), perm = int(i[split ? 12 : 11]);
      const int transpose = split ? 1 : int(i[9]), col0 = int(i[split ? 9 : 10]), part = split ? 0 : int(i[12]);
      const int col_lo = split ? int(i[10]) : 0, slot = split ? int(i[11]) : 0;
      T2_REQUIRE(p[0] && p[1] && p[2] && (W == 32 || W == 128) && grid_x >= 1 && grid_x <= 65535 && src >= 0 && dst >= 0 && i[5] >= 1 &&
                     i[5] <= (1 << 20) && i[6] >= 1 && i[6] <= (1 << 20) && col0 >= 0 && (transpose == 0 || transpose == 1) &&
                     (part == 0 || part == 2) && col_lo >= 0 && slot >= 0,
                 T2_ERR_INVALID_ARG, "dbg_taco_kernel PARAMS pack: bad arguments");
      const int gates = W == 32 ? 4 : 2;
      T2_REQUIRE(perm == 0 || (perm > 0 && transpose && perm % W == 0 && (long long)gates * perm == N), T2_ERR_INVALID_ARG,
                 "dbg_taco_kernel PARAMS pack: gate permutation %d needs a transposing job with N = %d * perm and perm %% %d == 0", perm, gates, W);
      const int extent = transpose ? K : N;     // columns each destination row receives from col0 on
      T2_REQUIRE(ld >= col0 + extent && (!split || (ld >= col0 + slot + extent && ld >= col_lo + extent)), T2_ERR_INVALID_ARG,
                 "dbg_taco_kernel PARAMS pack: destination columns beyond the leading dimension %d", ld);
      std::vector<PackJob> jobs;
      if (split) {   // the three jobs of one split-bf16 weight slot (add_pack_fwd): W_hi at col_hi and col_hi + slot, W_lo at col_lo
        for (int col : {col0, col0 + slot, col_lo}) add_pack(jobs, src, K, N, 2 * dst, ld, 1, col, call->f[0], perm);
        jobs.back().part = 2;
      } else {
        add_pack(jobs, src, K, N, 2 * dst, ld, transpose, col0, call->f[0], perm);
        jobs.back().part = part;
      }
      T2_REQUIRE(i[1] >= (long long)(jobs.size() * sizeof(PackJob)), T2_ERR_INVALID_ARG, "dbg_taco_kernel PARAMS pack: job buffer of %lld B < %zu B",
                 i[1], jobs.size() * sizeof(PackJob));
      T2_CHECK_CUDA(cudaMemcpyAsync(p[2], jobs.data(), jobs.size() * sizeof(PackJob), cudaMemcpyHostToDevice, st));
      return launch_pack(static_cast<const float*>(p[0]), p[1], static_cast<const PackJob*>(p[2]), int(jobs.size()), W, grid_x, st);
    }
    default:
      return t2_set_error(T2_ERR_INVALID_ARG, "dbg_taco_kernel: unknown kernel id %d", call->kernel);
  }
}
