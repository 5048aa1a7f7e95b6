/* t2b200.h — C-ABI of libt2b200.so, the sm_90a compute library behind the Tacotron-2 hot paths.
 *
 * The reference (Rayhane-mamah/Tacotron-2) has NO FFI / plugin boundary: its hot paths are Python methods
 * that build TensorFlow-1 graph nodes. This header therefore DEFINES the boundary; each entry point names the
 * reference function (file:line under the reference tree) whose arithmetic it replaces.
 *
 * Conventions
 *   - every function returns 0 (T2_OK) or a negative T2_ERR_* code; t2_last_error() returns a thread-local
 *     message for the last failure on the calling thread;
 *   - all pointers named d_* / documented "device" are DEVICE pointers owned by the caller; the library
 *     never allocates persistent device memory (the *_sizes queries say how much the caller must provide);
 *   - all work is enqueued on the cudaStream_t passed as `void* stream`; no host synchronisation unless
 *     documented; entry points are re-entrant per stream;
 *   - no torch / C++ types cross this boundary.
 */
#ifndef T2B200_H_
#define T2B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define T2B200_ABI_VERSION 3

#define T2_OK 0
#define T2_ERR_INVALID_ARG (-1)
#define T2_ERR_UNSUPPORTED_SHAPE (-2)
#define T2_ERR_CUDA (-3)
#define T2_ERR_NCCL (-4)

const char* t2_last_error(void);
int t2_abi_version(void);
/* sizeof() of a POD struct of this header by name ("t2_wn_config_t", "t2_wn_sizes_t", "t2_taco_config_t", "t2_cbhg_config_t",
 * "t2_audio_config_t", "t2_dbg_act_t", "t2_dbg_gemm_t", "t2_dbg_wgrad_tile_t", "t2_dbg_kernel_t"), -1 for an unknown name: a binding asserts that its
 * mirror of the struct matches the library it loaded */
int t2_struct_size(const char* name);
/* kernels launched (or captured) by this library so far in this process */
long long t2_launch_count(void);

/* ---- engine-level test hooks (tests/test_gemm_engine.py) --------------------------------------------- */
/* bf16 dilated-conv-as-GEMM on the wgmma engine: out[b,t,n] = act(sum_s sum_k a[b,t+shift_s,k] w[n,s*Kp+k] + bias[n])
 * (Kp = C rounded up to 64). Replaces tf.layers.Conv1D as used by wavenet_vocoder/models/modules.py:206-224,320. */
int t2_dbg_conv_gemm(const void* d_a, int B, int T, int C, int ld, const int* shifts, int nshift,
                     const void* d_w, int N, int BN, const float* d_bias, int relu, void* d_out_bf16,
                     float* d_out_f32, void* stream);
/* debug: non-NULL => every GEMM CTA records 16 int64 stamps (clock64 phases, %globaltimer at entry / after the dependent-launch
 * wait / exit, SM id) at d_buf[(launch_offset + cta)*16 + slot], consecutive launches append; NULL disables */
int t2_dbg_set_timing_buffer(long long* d_buf);
/* weight-gradient GEMM: out[m,n] = scale * sum_{b,t} a[b,t+shift_a,m] * bm[b,t,n]  (fp32 [Ca,Cb]); synchronises. */
int t2_dbg_wgrad(const void* d_a, int Ca, const void* d_bm, int Cb, int B, int T, int shift_a, float scale,
                 float* d_out, void* stream);

/* The whole engine surface, for tests of every fused epilogue (tests/test_gemm_epilogues_gpu.py). One A operand: channels-last
 * bf16 [L][B][T][ld], the first C channels addressable (ld % 8 == 0, 16-byte aligned). */
typedef struct {
  const void* ptr;
  int C, T, B, L, ld;
} t2_dbg_act_t;
/* one K segment: nkb 64-wide K blocks of map `map` starting at channel k0, rows shifted by `shift`, looped over layers
 * [layer0, layer0 + nlayers) (outer); segments consume consecutive K blocks of the packed weight */
typedef struct {
  int map, shift, k0, nkb, layer0, nlayers;
} t2_dbg_seg_t;
/* act_gemm: D[b, t, n] = sum over segments s, layers l, k of A_map(s)[layer0 + l, b, t + shift, k0 + k] * W[w_layer, n, w_k0 + K offset],
 * rows outside [0, T) of item b read as zero, then epilogue `epi` (EPI_* of tacotron-2_b200/csrc/t2_gemm_types.h) with BN output columns
 * per tile and the raw epilogue arguments ptr / f / i / seed documented next to each epilogue in t2_gemm.cuh. ksplit > 1 splits
 * the reduction over that many CTAs per tile (EPI_TOUT with mode 2 only). cluster: 0 = library default, else 1, 2, 4 or 8 CTAs that
 * share each weight tile by TMA multicast; cluster_used returns the size actually launched. */
typedef struct {
  t2_dbg_act_t a[4];
  int na;
  t2_dbg_seg_t seg[16];
  int nseg;
  const void* w;             /* packed bf16 weights [wL][wN][wK], K contiguous */
  int wN, wK, wL, w_layer, w_k0;
  int T, B, n_tiles, ksplit, epi, BN;
  int cluster;               /* in */
  int cluster_used;          /* out */
  void* ptr[12];
  float f[6];
  int i[12];
  unsigned long long seed;
} t2_dbg_gemm_t;
int t2_dbg_act_gemm(t2_dbg_gemm_t* call, void* stream);
/* One tile of the weight-gradient GEMM: out[out_off + m * ldc + n] (=, +=, atomic +=: accumulate 0 / 1 / 2) scale / max(*div, 1e-20)
 * * sum over b, t of A_{a_map}[a_layer, b, t + a_shift, a_ch0 + m] * A_{b_map}[b_layer, b, t + b_shift, b_ch0 + n], for m < m_valid (<= 128),
 * n < n_valid (<= 256); div is a nullable device scalar. */
typedef struct {
  int a_map, a_ch0, a_shift, a_layer;
  int b_map, b_ch0, b_shift, b_layer;
  long long out_off;
  int ldc, m_valid, n_valid;
  float scale;
  int accumulate;
  const float* div;
} t2_dbg_wgrad_tile_t;
/* runs the host tile table `tiles` over up to 6 maps into the fp32 buffer d_out; synchronises */
int t2_dbg_wgrad_tiles(const t2_dbg_act_t* maps, int nmaps, const t2_dbg_wgrad_tile_t* tiles, int ntiles, float* d_out, int T, int B,
                       void* stream);
/* The fixed-point column sums behind the multi-block gradients: adds d_addends[r * ncols + c] (r < nrows) into column c with the same
 * atomics the GEMM epilogues use, then converts the totals as the gradient finalisation does: d_out[c] = value of the total (0 for an
 * empty total). Synchronises. */
int t2_dbg_fx_colsum(const float* d_addends, int nrows, int ncols, float* d_out, void* stream);

/* One launch of a Tacotron / CBHG engine kernel on caller buffers, with the grid, block and shared-memory size of the product path
 * (tests/test_taco_kernels_gpu.py). `kernel` selects the kernel; p / i / f carry its pointer, integer and float arguments in the order
 * documented next to each T2_DBG_* id; seed / step feed the dropout hash. Every argument is checked before any driver call; no
 * temporaries are allocated. Does not synchronise. */
typedef struct {
  int kernel;
  void* p[16];
  long long i[16];
  float f[4];
  unsigned long long seed;
  const unsigned long long* step;   /* nullable device int64 added to seed */
} t2_dbg_kernel_t;
/* t2_dbg_taco_kernel ids:
 * ATT_FWD  att_prep_kernel + att_fwd_kernel, one decoder step. p: h2out bf16 [B][ld_h2] (query source, first D used), WqT bf16 [A][D],
 *          K fp32 [KA][F], bK [F], Wl [F][A], ba [A], U fp32 [(KA+1)][A] (out: merged filter bank), v [A], keys fp32 [B][Ti][A],
 *          values bf16 [B][Ti][C2], lens int32 [B], cum fp32 [B][Ti] (in/out: the attention state), alpha fp32 [B][Ti] (out), ctx_a
 *          bf16 (nullable), ctx_b bf16. i: B, Ti, D, A, KA, F, C2, ld_h2, ld_a, ld_b, unmasked, noncumulative (the two
 *          t2_taco_config_t flags; 0 = masked scores and cum + alpha as the new state, 1 = all T_in scores and alpha as the new state),
 *          split (t2_taco_config_t.split_bf16: WqT rows are [hi(D) | lo(D)], values rows [hi(C2) | lo(C2)]), then lo_h2, lo_a, lo_b (0
 *          unless split): the lo half of the query source sits at +lo_h2, ctx_a is written [hi | lo at +lo_a | hi again at +2 lo_a],
 *          ctx_b [hi | lo at +lo_b].
 * BN_FWD   bn_stats_kernel (training) + bn_apply_kernel (conv-block batch norm). p: y (bf16, or fp32 when i[3]), x bf16 [rows][C] (split: [rows][2C]),
 *          stats fp32 [4C], gamma, beta, moving mean, moving variance. i: rows, C, training, y_fp32, stream, split. f: dropout p.
 * BN_BWD   bn_bwd_stats_kernel + bn_bwd_apply_kernel. p: dout bf16, y bf16, stats fp32 [6C] (mean / rstd at [2C, 4C); [4C, 6C) receives
 *          the backward sums), gamma, dpre bf16 (out), dgamma, dbeta (accumulated). i: rows, C, act, stream. f: dropout p. */
#define T2_DBG_TACO_ATT_FWD 1
#define T2_DBG_TACO_BN_FWD 2
#define T2_DBG_TACO_BN_BWD 3
/* CELL_BWD    lstm_cell_bwd_kernel, one step t. p: dh_ext fp32 [B][ld_ext] (cleared when zero_ext), dhs, dcs fp32 [B][H] (in/out), gst bf16
 *             [B][4H] gate stash (i | j | f | o), tst bf16 [B][H] tanh(c) stash, c_prev fp32 [B][H], dg_a bf16 [B][ld_a] (out), dg_b
 *             (nullable), lens int32 [B] (nullable). i: ld_ext, zero_ext, ld_a, ld_b, t, B, H, stream. f: zoneout rate.
 * ATT_FINISH  att_finish_kernel + att_finish2_kernel. p: acc fp32 [B][(KA+2)][A], K [KA][F], bK [F], Wl [F][A], grads fp32 (accumulated
 *             at the offsets), scratch fp32 [(KA+2)][A]. i: B, KA, F, A, o_k, o_bk, o_wl, o_v, o_ba.
 * DVALUES     dvalues_ctx_kernel. p: alpha fp32 [To][B][Ti], dctx bf16 [To][B][C2], lens int32 [B], dvalues fp32 [B][Ti][C2] (in/out).
 *             i: B, Ti, To, C2.
 * ATT_BWD     att_bwd_kernel, one decoder step (the training backward's grid, block and shared memory). p: h2out bf16 [B][ld_h2] (query
 *             source, first D used), WqT bf16 [A][D], U fp32 [(KA+1)][A] (merged filter bank, row KA = u0, as ATT_FWD leaves it), v [A],
 *             keys fp32 [B][Ti][A], values bf16 [B][Ti][C2], lens int32 [B], alpha fp32 [B][Ti] (this step), state: cumulative = cum_t
 *             fp32 [B][Ti] (in; out: cum_{t-1} = cum_t - alpha), non-cumulative = alpha_{t-1} fp32 [B][Ti] (read; nullable = zeros, step
 *             0), dstate fp32 [B][Ti] (in: d loss / d state_t; out: d loss / d state_{t-1}), dPI fp32 [B][ld_dPI] (cols [0, D): d h2out,
 *             [D, D + C2): d context), dctxl fp32 [B][C2] (added to the context gradient, then cleared), dh2ext fp32 [B][D] (out),
 *             dsave bf16 [B][C2] dctx followed by [B][A] dq (out), dkeys fp32 [B][Ti][A] (accumulated), acc fp32 [B][(KA+2)][A]
 *             (accumulated: dU rows 0..KA-1, du0, dv). i: B, Ti, D, A, KA, C2, ld_h2, ld_dPI, unmasked, noncumulative. */
#define T2_DBG_TACO_CELL_BWD 4
#define T2_DBG_TACO_ATT_FINISH 5
#define T2_DBG_TACO_DVALUES 6
#define T2_DBG_TACO_ATT_BWD 7
/* CONV_GEMM   launch_bias_act: a k-tap 'same' convolution / projection through the GEMM engine and EPI_BIAS_ACT, tap j reading row
 *             t + conv_tap_shift(ntaps, j) of the same item. p: a bf16 [Bn][T][C] (split: [Bn][T][hi(Cp) | lo(Cp)], Cp = C rounded up
 *             to 64), packed weight bf16 [N][wK] (split: [W_hi | W_hi | W_lo] per tap, wK >= 3 ntaps Cp), bias fp32 [N] (nullable),
 *             out bf16 [Bn T][ldo] (split: [hi(ldo) | lo(ldo)], pitch 2 ldo; nullable), out fp32 [Bn T][ldo] (nullable; one of the two
 *             outputs is required). i: C, T, Bn, N, wK, ntaps (<= 16; split <= 8), BN (128 / 256), act (0 none, 1 relu, 2 tanh), ldo,
 *             nvalid, dropout stream, split, hash_row0 (position offset of the dropout mask). f: dropout rate. seed / step: dropout seed.
 * LSTM_STEP   lstm_step: one recurrent step on the swapped GEMM (EPI_LSTM). p: wrec bf16 [4H][K] (split: [4H][W_hi | W_hi | W_lo]),
 *             state bf16 [B][K] (split: [B][hi | lo | hi]), pre fp32 (row b at + b pre_stride, nullable), bias fp32 [4H] (nullable),
 *             c_prev fp32 [B][H], c_out fp32 [B][H], h_prev bf16 (+ b ld_hp; split: lo at +K), h_state bf16 (+ b ld_hs; split: written
 *             [hi | lo at +K | hi at +2K]), h_out bf16 (+ b ld_ho; split: lo at +out_lo, and the second hi copy at +2 out_lo when
 *             out_state), gate stash bf16 [B][4H] (nullable), tanh(c) stash bf16 [B][H] (nullable; neither stash is written in split
 *             mode), lens int32 [B] (nullable). i: H, K, B, pre_stride, ld_hp, ld_hs, ld_ho, t, zoneout stream, out_lo, out_state,
 *             training, split. f: zoneout rate. seed / step: zoneout seed.
 * ROWS        one of the small row writers, i[0] selecting it and i[1] = split (0: bf16 rows, 1: split-bf16 [hi | lo] rows):
 *             0 embed_fwd_kernel    p: idx int32 [npos], table fp32 [NS][E], out bf16 ([npos][E]; split [npos][hi(E) | lo(E)]).
 *                                   i: -, -, npos, E.
 *             1 decin_kernel        p: target fp32 [B][To][M], out bf16 ([To][B][M]; split: rows [hi(M) | pad | lo(M) | pad] of pitch
 *                                   256, the padding is not written). i: -, -, B, To, M.
 *             2 dec_finish_kernel   p: projo fp32 [To][B][128], target fp32 [B][To][M] (nullable), stop target (nullable), dec bf16
 *                                   ([B][To][M]; split: rows [hi(M) | pad | lo(M) | pad] of pitch 256), dec fp32 [B][To][M], stop fp32
 *                                   [B][To], loss sums fp32 [5] (accumulated), target lengths int32 [B] (nullable). i: -, -, B, To, M,
 *                                   clip. f: clip low, clip high, stop positive weight.
 *             3 proj_bias_feedback_kernel  p: projection fp32 [B][128] (in / out), frame bias [M], stop bias [1], next input bf16
 *                                   (nullable; [B][M], split: decin rows of pitch 256), target fp32 [B][To][M] (nullable), choice int32
 *                                   [To] (required with a target). i: -, -, B, M, To, t. f: teacher-forcing ratio. seed / step: its draw.
 *             4 f32_to_bf16_kernel  p: in fp32 [rows][C], out bf16 ([rows][C]; split [rows][hi(Cp) | lo(Cp)], channels C..Cp-1
 *                                   zero). i: -, -, rows, C, Cp (= C unless split). */
#define T2_DBG_TACO_CONV_GEMM 8
#define T2_DBG_TACO_LSTM_STEP 9
#define T2_DBG_TACO_ROWS 10
/* LOSS        one of the loss / gradient-seed kernels, i[0] selecting it. The decoder-output kernels (0-3) take i: -, B, To, M (M + 1
 *             <= 128), clip, and f: clip low, clip high, stop positive weight; frames are batch-major [B][To][M], projection rows
 *             time-major [To][B][128] (col M: stop logit), the loss scalars fp32 [16] as the engine keeps them ([0] before, [1] after,
 *             [2] stop, [3] regulariser, [4] masked stop count: accumulated; [5] / [6] mel / stop normalisers).
 *             0 mel_finish_kernel   p: dec fp32, residual fp32 [B To][128], target (nullable), mel fp32 (out), scal, target lengths
 *                                   int32 [B] (nullable).
 *             1 loss_norm_kernel    p: scal, out fp32 [4] (nullable: the four normalised loss terms), target lengths (nullable).
 *                                   f[0]: regulariser weight (clip unused).
 *             2 loss_seed_kernel    p: dec fp32, residual, mel, target, dmel bf16 [B To][128] (out), ddec fp32 [B][To][M] (out),
 *                                   target lengths (nullable), scal (reads [5]), extra fp32 [B][To][M] (nullable; d loss / d mel
 *                                   outputs from a later head).
 *             3 ddec_tm_kernel      p: ddec fp32 [B][To][M], dpost bf16 [B][To][M], projection rows, stop target fp32 [B][To], out bf16
 *                                   [To][B][128] (rows of steps [t0, t1) written), target lengths (nullable), scal (reads [6]), fb fp32
 *                                   [B][M] (nullable), choice int32 [To] (required with fb). i[5], i[6]: t0, t1.
 *             4 proj_bias_kernel    p: projection rows fp32 [rows][128] (in / out), frame bias [M], stop bias [1]. i: -, rows, M.
 *             5 relu_drop_bwd_kernel  p: d bf16 [n], y bf16 [n], dz bf16 [n] (may be d). i: -, n. f[0]: dropout rate.
 *             6 embed_bwd_kernel    p: idx int32 [npos], dx bf16 [npos][E], dtable fp32 (accumulated). i: -, npos, E.
 *             7 mask_values_kernel  p: memory bf16 [B][Ti][C2], lengths int32 [B], values bf16 [B][Ti][C2]. i: -, B, Ti, C2.
 *             8 bias_colsum_kernel<bf16> (colsum)  p: src bf16 [rows][ld], dst fp32 [C] (accumulated). i: -, rows, C, ld, threads
 *                                   (128 / 256).
 * PARAMS      the parameter-table kernels, i[0] selecting one.
 *             0 pack_kernel, one job (add_pack)  p: params fp32, packed bf16, job buffer (device, >= sizeof(PackJob) B; filled
 *                                   stream-ordered). i: -, job buffer bytes, W (32: four LSTM gates, 128: two WaveNet gate halves),
 *                                   grid_x, src_off, K, N, dst_off (bf16 elements), dst_ld, transpose, col0, perm, part (0 / 2).
 *                                   f[0]: scale.
 *             1 pack_kernel, the three jobs of a split-bf16 slot in one launch p: as 0 (>= 3 sizeof(PackJob) B). i: -, bytes, W,
 *                                   grid_x, src_off, K, N, dst_off, dst_ld, col_hi, col_lo, slot, perm. f[0]: scale.
 *                                   A job with perm > 0 must transpose, with N = gates * perm (gates = 4 for W = 32, 2 for W = 128)
 *                                   and perm % W == 0.
 *             2 reg_loss_kernel     p: params fp32, table int64 [n_reg][2] (offset, elements), dst fp32 (accumulated: 0.5 sum w^2).
 *                                   i: -, n_reg.
 *             3 reg_grad_kernel     p: params, grads fp32 (accumulated: weight w), table. i: -, n_reg. f[0]: weight. */
#define T2_DBG_TACO_LOSS 11
#define T2_DBG_TACO_PARAMS 12
int t2_dbg_taco_kernel(const t2_dbg_kernel_t* call, void* stream);
/* t2_dbg_cbhg_kernel ids (the batch-norm pair works on the column slice [c0, c0 + C) of pitch-ld matrices; statistics / sums are
 * [4 Ct] / [2 Ct] indexed by absolute column, and the caller zeroes the sum sections first, as the engine does):
 * BN_FWD       bn_stats_kernel (training) + bn_apply_kernel. p: y, xb bf16 (nullable), xf fp32 [rows][C] (nullable), add fp32 [rows][C] (nullable),
 *              stats, gamma, beta, mm, mv. i: rows, C, ld, c0, Ct, training, y_fp32, stat_threads (128 or 256), split (0 / 1: xb rows are
 *              [hi(ld) | lo(ld)] at pitch 2 ld).
 * BN_BWD       bn_bwd_stats_kernel + bn_bwd_apply_kernel. p: g, y (both bf16, or both fp32 when i[9]), stats, bsum, gamma, dpre bf16, dgamma, dbeta.
 *              i: rows, C, ldg, ld, c0, Ct, ldd, act, stat_threads, fp32.
 * POOL_FWD     maxpool_fwd_k. p: x bf16 [N][C], out. i: N (= B T rows), T, C, split (0 / 1: x and out are [N][hi(C) | lo(C)] rows, the
 *              pair with the larger hi + lo wins).
 * POOL_BWD     maxpool_bwd_k. p: x, dout, dx. i: N, T, C.
 * HIGHWAY_FWD  highway_fwd_k. p: pre fp32 [N][2HU], bh, bt, h fp32 [N][HU], hf fp32, hb bf16, HT bf16 [N][2HU] (nullable). i: N, HU,
 *              split (0 / 1: hb is [N][hi(HU) | lo(HU)]).
 * HIGHWAY_BWD  highway_bwd_k. p: dh fp32, HT bf16, h fp32, dHT bf16 [N][2HU], dcarry fp32. i: N, HU.
 * GRU_FWD      gru_fwd_kernel, both directions over the whole padded sequence (rows b T + t, N = B T). p: params fp32 (flat; the kernel
 *              reads the recurrent rows [HU, HU + RU) of the two kernels and the biases), XP fp32 [N][6RU] ([fw gates | fw cand | bw gates
 *              | bw cand], no biases), out bf16 [N][2RU], then the stashes bf16 [N][RU] r, u, c, rh of fw, then of bw (all eight present,
 *              or all null as in inference). i: B, T, HU, RU (= 128), then p_gk, p_ck, p_gb, p_cb of fw, then of bw (offsets into params),
 *              then i[12] split (0 / 1: the recurrent weights are used as hi + lo pairs, out is [N][hi(2RU) | lo(2RU)] and the eight stashes
 *              must be null).
 * GRU_BWD      gru_bwd_kernel (BPTT of both directions). p: params, dout fp32 [N][2RU], out bf16 [N][2RU] (h_prev, as GRU_FWD writes it),
 *              the stashes r, u, c of fw, then of bw, dXP bf16 [N][6RU] (out: [dr_pre | du_pre | dc_pre] per direction).
 *              i: B, T, HU, RU (= 128), then p_gk, p_ck of fw, then of bw.
 * LINEAR       lin_norm_k, lin_finish_k, then loss_out_k (the linear-spectrogram clip, L1 loss and gradient seed; rows r = b T + t,
 *              N = B T). p: lin fp32 [N][NFP] (in / out: columns [0, NF) clipped), target fp32 [N][NF] (nullable: inference), dlin bf16
 *              [N][NFP] (nullable; written only with a target, as the engine does), scal fp32 [10] ([0] / [1] accumulated L1 sums, [2]
 *              regulariser sum, [8] / [9] normalisers), out fp32 [2] (nullable: loss_out_k skipped), target lengths int32 [B] (nullable).
 *              i: B, T, NF, NFP, n_prio, clip. f: clip low, clip high, regulariser weight.
 * ADD          i[0] selecting: 0 add_k  p: acc fp32 [n] (in / out: acc + a), a fp32 [n], out bf16 [n] (nullable). i: -, n.
 *                              1 dmel_k p: a, b, c fp32 [N][128], dhin fp32 [N][M], out fp32 [N][M]. i: -, N, M (<= 128). */
#define T2_DBG_CBHG_BN_FWD 1
#define T2_DBG_CBHG_BN_BWD 2
#define T2_DBG_CBHG_POOL_FWD 3
#define T2_DBG_CBHG_POOL_BWD 4
#define T2_DBG_CBHG_HIGHWAY_FWD 5
#define T2_DBG_CBHG_HIGHWAY_BWD 6
#define T2_DBG_CBHG_GRU_FWD 7
#define T2_DBG_CBHG_GRU_BWD 8
#define T2_DBG_CBHG_LINEAR 9
#define T2_DBG_CBHG_ADD 10
int t2_dbg_cbhg_kernel(const t2_dbg_kernel_t* call, void* stream);


/* ---- WaveNet vocoder: teacher-forced training path ---------------------------------------------------------
 * Replaces wavenet_vocoder/models/wavenet.py:650-721 (WaveNet.step), :476-519 (add_loss), the layers of
 * wavenet_vocoder/models/modules.py:184-521,539-654,736-817 and wavenet_vocoder/models/mixture.py:18-74.
 * Field names follow the reference's hparams.py:187-228. */
typedef struct {
  int layers, stacks, residual_channels, gate_channels, skip_out_channels;
  int kernel_size;           /* taps of the dilated causal convolution: 2, 3 or 4 (tap j reads x(t - (kernel_size-1-j) d)) */
  int cin_channels;          /* 80 (num_mels) or 0 = no local conditioning */
  int out_channels;          /* 256 (mu-law softmax), 3*nr_mix (MoL) or 2 (single Gaussian: mean, log-scale) */
  int quantize_channels;     /* 256 or 65536 */
  int input_type;            /* 0 'raw', 1 'mulaw', 2 'mulaw-quantize' */
  int legacy, residual_legacy;
  int upsample_type;         /* 0 'SubPixel', 1 '2D' (ConvTranspose2D), 2 '1D' (ConvTranspose1D: kernel = stride = s over time, mixes the
                              * cin channels; kernel [1][s][C][C] = [kh][kw][out][in], bias [C]; freq_axis_kernel_size is not read) */
  int n_upsample;
  int upsample_scales[4];
  int freq_axis_kernel_size;
  float dropout;             /* wavenet_dropout */
  float log_scale_min;
  int B, T, Tc;              /* per-GPU batch, samples per item, conditioning frames per item */
  int c_pre_upsampled;       /* 1: conditioning is given at sample rate [B, T, cin] fp32 (skip upsample net) */
  float log_scale_min_gauss; /* single-Gaussian head (out_channels == 2): clamp of the predicted log-scale (hparams.py:196) */
  int cdf_loss;              /* Gaussian head: 1 = log(CDF+ - CDF-) loss, 0 = log-density (gaussian.py:18-33) */
  int split_bf16;            /* 1 = "fp32-class" forward: activations and weights travel as bf16 hi + lo pairs (3 tensor-core products per
                              * contraction, fp32 accumulate; ~2^-17 relative operand error instead of 2^-9). Forward / loss and AR synthesis
                              * only, dropout 0: the parity mode that shows the bf16-mode deviation from the reference's fp32 graph is storage
                              * rounding. In AR synthesis (t2_wn_ar_*) it stores the synthesis weights as plain fp32 and reads the conditioning
                              * in fp32 (CUDA-core FMA: exact products without a hi + lo pair). */
  int gin_channels;          /* global (speaker) conditioning: width of the speaker embedding (wavenet.py:151-158), 0 = off */
  int n_speakers;            /* rows of gc_embedding (>= 1 when gin_channels > 0) */
  int upsample_activation;   /* after each learnable upsampling layer (wavenet.py:197-203): 0 ReLU, 1 LeakyReLU max(alpha x, x), 2 none */
  float leaky_alpha;         /* LeakyReLU slope, in [0, 1] (checked whatever the activation; 0 in a zeroed struct) */
} t2_wn_config_t;

typedef struct {
  long long n_params;        /* fp32 master parameters (TF variable layouts, concatenated) */
  long long packed_bytes;    /* bf16 GEMM-operand copies + derived fp32 biases */
  long long workspace_bytes; /* activations saved for backward, gradients of activations, tables */
  int n_tensors;
} t2_wn_sizes_t;

int t2_wn_sizes(const t2_wn_config_t* cfg, t2_wn_sizes_t* out);
/* i-th parameter tensor: TF-style name (SURVEY.md Appendix B), offset into the flat buffer, shape */
int t2_wn_param_info(const t2_wn_config_t* cfg, int i, char* name, int name_cap, long long* offset, int* ndim,
                     int* shape4);
/* one-time: zero the packed buffer / workspace and upload the static job tables (synchronises the stream) */
int t2_wn_init(const t2_wn_config_t* cfg, void* d_packed, void* d_workspace, void* stream);
/* fp32 masters -> bf16 operand layouts (run after every optimizer step) */
int t2_wn_pack_weights(const t2_wn_config_t* cfg, const float* d_params, void* d_packed, void* d_workspace,
                       void* stream);
/* forward + loss. d_x: int32 [B,T] mu-law indices (input_type 2) or fp32 [B,T] samples; d_c: fp32 [B,cin,Tc]
 * (or [B,T,cin] when c_pre_upsampled); d_targets: int32 / fp32 [B,T]; d_lengths int32 [B].
 * d_loss: fp32[2] = {sum of masked losses, normaliser} (loss = [0]/[1]); d_logits: optional fp32 [B,T,ldo]
 * (ldo = 256, or 32 for MoL). save_for_backward=0 skips the backward stashes. Dropout masks are a pure function of
 * (seed + *d_step, layer, position, channel); d_step (device u64, nullable) lets a replayed CUDA graph advance. */
int t2_wn_forward(const t2_wn_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                  const void* d_x, const float* d_c, const void* d_targets, const int* d_lengths, float* d_loss,
                  float* d_logits, int save_for_backward, unsigned long long seed,
                  const unsigned long long* d_step, void* stream);
/* backward of the last t2_wn_forward(save_for_backward=1): writes all parameter gradients (d loss / d theta) */
int t2_wn_backward(const t2_wn_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                   const void* d_x, const float* d_c, float* d_grads, unsigned long long seed,
                   const unsigned long long* d_step, void* stream);
/* Phased backward for data-parallel training (wavenet.py:561-593: tower gradients are averaged after backward). The weight
 * gradients of the residual stack come from `n_groups` launches over layer groups whose parameters are CONTIGUOUS ranges of the
 * flat gradient buffer, so the caller can all-reduce group g while group g+1 computes. phase -1: everything (== t2_wn_backward);
 * 0: data-gradient chain, head, conditioning tails; 1 + g: weight gradients of layers [g*L/n, (g+1)*L/n); 100: join of the
 * library's side stream (call after the last group, before reading gradients of the head / upsampling / first-conv tensors). */
int t2_wn_backward_phased(const t2_wn_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                          const void* d_x, const float* d_c, float* d_grads, unsigned long long seed,
                          const unsigned long long* d_step, int phase, int n_groups, void* stream);
/* measurement hook for bench.py's roofline leg: average device time (CUDA events on `stream`) of `reps` launches of
 * one per-layer GEMM over the state left in the workspace by the last forward/backward. which: 0 gate GEMM, 1 out
 * GEMM, 2 dz + gate-backward GEMM, 3 dx GEMM. Re-running 1 / 3 rewrites x[l+1] / dx[l] with identical values.
 * Synchronises. */
int t2_wn_time_kernel(const t2_wn_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                      int which, int layer, int reps, float* ms_per_launch, void* stream);
/* The forward gate / out GEMMs of every residual layer can run as ONE persistent launch, and so can the backward dz / dx GEMMs:
 * tiles wait for the neighbour tiles they read instead of for whole launches. By default (mode 0) they do where a layer's gate
 * GEMM is at most two waves of CTAs; mode 1 makes the following calls launch them per layer (the reference the chains are compared
 * with bit for bit), mode 2 always uses the chains. */
int t2_dbg_wn_per_layer(int mode);
/* The work tickets of a persistent chain (dir 0 forward, 1 backward), in the order CTAs take them: 8 ints per ticket
 * {kind (0 gate / dz, 1 out / dx), layer, M tile over all items, N tile, first and last counter waited for, count awaited,
 * counter completed}, counter of (kind, layer, M tile m) = (kind * layers + layer) * M tiles + m. out == NULL: count only.
 * Host only. Returns the ticket count. */
int t2_dbg_wn_chain(const t2_wn_config_t* cfg, int dir, int* out, int cap);
/* debug / test access to workspace tensors by name ("x", "z", "c_up", "h1", "dg", ...): returns device pointer,
 * element count and element size */
int t2_wn_workspace_tensor(const t2_wn_config_t* cfg, void* d_workspace, const char* name, void** ptr,
                           long long* count, int* elem_bytes);
/* gin_channels > 0: the speaker ids (device int32 [B]) of the next forwards, copied into the workspace, so a replayed CUDA graph
 * uses the ids set last. NULL = no speaker term (the reference skips it when g is None, modules.py:504); t2_wn_init starts there.
 * Every layer then adds b_gin + W_gin^T gc_embedding[id_b] to item b's gate pre-activations. An id outside [0, n_speakers) reads
 * nothing: it makes that item's gate biases, and so its gate activations, NaN. */
int t2_wn_set_speakers(const t2_wn_config_t* cfg, void* d_workspace, const int* d_speaker_ids, void* stream);
/* One launch of a conditioning-upsampler kernel or of a small kernel of the WaveNet engine on caller buffers (t2_dbg_kernel_t above), with
 * the product's grid, block and shared memory. Every argument is checked before any driver call; no temporaries are allocated. Upsampler
 * layouts: in fp32 [B][C][W], layer output fp32 [B][C][W*s];
 * K / bias as the layer's parameters (upsample_type 0: [3][3][1][s] / [s]; 1: [3][s][1][1] / [1]; 2: [1][s][C][C] / [C]). Common i:
 * B, C (1..128), W, s, type (0 SubPixel, 1 2D, 2 1D), act (0 ReLU, 1 LeakyReLU, 2 none); f[0]: LeakyReLU alpha in [0, 1].
 * UP_FWD        p: in, K, bias, out fp32 [B][C][W*s] (post-activation), c_up bf16 (nullable: channels-last [B][W*s][C], or the split
 *               rows [B][W*s][256] = hi | lo when i[6] = 1). i[6]: split.
 * UP_BWD_PARAM  p: in, out (post-activation), dout fp32 [B][C][W*s] (d loss / d out), dK fp32, dbias fp32 (both out), acc int64 [nK + nb]
 *               (scratch: the fixed-point totals, nK / nb = elements of K / bias). dK and dbias are overwritten with the totals converted
 *               as the engine's gradient finalisation does. Synchronises nothing.
 * UP_BWD_INPUT  p: out, dout, K, din fp32 [B][C][W] (out). */
#define T2_DBG_WN_UP_FWD 1
#define T2_DBG_WN_UP_BWD_PARAM 2
#define T2_DBG_WN_UP_BWD_INPUT 3
/* The small kernels of the WaveNet engine, one launch each with the engine's launcher (tests/test_wavenet_kernels_gpu.py); their ids
 * start at 10, ids 4 to 9 are not assigned. p / i / f:
 * FIRST_CONV      first_conv_kernel. p: xin (int32 [npos] one-hot indices in [0, Q): not checked, or fp32 [npos] samples), W fp32 ([Q][R],
 *                 or [1][R] for scalar input), bias fp32 [R], x bf16 [npos][R] (out; split: [npos][2R] = hi | lo), xd bf16 [npos][R]
 *                 (nullable: the dropout copy, kept with probability 1 - f[0], hash seed = seed + *step). i: npos, R (multiple of 8, <= 1024),
 *                 scalar_in, split (no xd). f[0]: dropout p in [0, 1).
 * FIRST_CONV_BWD  first_conv_bwd_kernel + the gradient finalisation. p: xin (as FIRST_CONV), dx0 bf16 [npos][R], acc int64 [Q][R] (scratch:
 *                 cleared, then the fixed-point totals), dW fp32 [Q][R] (in/out: each non-zero total is added). i: npos, R (<= 1024),
 *                 scalar_in, Q (1 for scalar input).
 * COLSUM          colsum_kernel + the gradient finalisation. p: ws (base of the src_off byte offsets), acc int64 [n_acc] (scratch, as above),
 *                 grads fp32 [n_acc] (in/out, as above), scalars fp32 [n_scalars] (nullable when n_scalars = 0), table (device scratch,
 *                 64 bytes per job), jobs HOST int64 [njobs][7] {src_off (bytes, bf16 [rows][ld] source), rows, C, ld (both even),
 *                 dst_off, dst2_off (-1: none), div_scalar (-1: none)}, scales HOST fp32 [njobs]. i: njobs, n_acc, ws bytes, n_scalars.
 *                 Column c of a job adds scale / max(scalars[div_scalar], 1e-20) * sum_r src[r][c] to acc[dst_off + c] (and dst2_off + c).
 * DERIVED_BIAS    derived_bias_kernel. p: params, bias_g fp32 [L][G] (out), bias_skip fp32 [S] (out), offs int64 [3L] device (per layer the
 *                 offsets of b_dil, b_cin (-1: none), b_skip), scales fp32 [L] device. i: L, G, S.
 * SKIP_BIAS       skip_bias_kernel. p: skipsum int64 [S] (fixed-point), grads fp32 (out: scales[l] * skipsum at offs[3l + 2]), offs, scales.
 *                 i: L, S.
 * FX_FINALIZE     fx_finalize_kernel. p: acc int64 [n], grads fp32 [n] (in/out: + the value of every non-zero total). i: n.
 * CL_TO_CHW       cl_to_chw_kernel. p: in fp32 [B][T][C], out fp32 [B][C][T]. i: B, T, C.
 * GIN_BIAS        gin_bias_kernel. p: params, bias fp32 (layer l at + l bias_ld), on int32 (nullable = on), ids int32 [B] (nullable = no
 *                 speaker term), out fp32 (out: [l][b][g] at + l out_l + b out_b + g). i: L, B, G, Gi, NS, bias_ld, out_l, out_b, p_k, p_b,
 *                 p_stride, p_emb (W_gin / b_gin of layer l at params + p_k / p_b + l p_stride, the embedding [NS][Gi] at p_emb).
 * SET_SPEAKERS    set_speakers_kernel. p: spk int32 [1 + B] (out: on flag, then the ids), ids int32 [B] (nullable). i: B.
 * GIN_WGRAD       gin_wgrad_kernel. p: params, spk int32 [1 + B], S int64 [L][B][G] (fixed-point per-item sums), gfx int64 (out: the
 *                 integer totals at offs[3l], offs[3l + 1] and, with spk[0], p_b + l p_stride), grads fp32 (out with spk[0]: dW_gin), offs
 *                 int64 [3L]. i: L, B, G, Gi, NS, p_k, p_b, p_stride, p_emb.
 * GIN_DEMB        gin_demb_kernel. p, i: as GIN_WGRAD; writes the embedding gradient rows of the speakers some item uses (with spk[0]). */
#define T2_DBG_WN_FIRST_CONV 10
#define T2_DBG_WN_FIRST_CONV_BWD 11
#define T2_DBG_WN_COLSUM 12
#define T2_DBG_WN_DERIVED_BIAS 13
#define T2_DBG_WN_SKIP_BIAS 14
#define T2_DBG_WN_FX_FINALIZE 15
#define T2_DBG_WN_CL_TO_CHW 16
#define T2_DBG_WN_GIN_BIAS 17
#define T2_DBG_WN_SET_SPEAKERS 18
#define T2_DBG_WN_GIN_WGRAD 19
#define T2_DBG_WN_GIN_DEMB 20
int t2_dbg_wn_kernel(const t2_dbg_kernel_t* call, void* stream);


/* ---- WaveNet vocoder: Fast-WaveNet autoregressive synthesis ---------------------------------------------------
 * Replaces WaveNet.incremental (wavenet_vocoder/models/wavenet.py:724-911), CausalConv1D incremental path
 * (modules.py:273-303) and sample_from_discretized_mix_logistic (mixture.py:76-107). cfg->B = synthesis batch,
 * cfg->T = samples to generate. cluster_size in {1,2,4,8,16}: CTAs per thread-block cluster sharing one batch group. */
int t2_wn_ar_sizes(const t2_wn_config_t* cfg, int cluster_size, long long* packed_bytes, long long* workspace_bytes);
/* fp32 masters -> slice-major synthesis weights (bf16, or fp32 when cfg->split_bf16 = 1: packed_bytes then holds 4 bytes per weight)
 * + ring tables; run once per checkpoint; synchronises */
int t2_wn_ar_pack(const t2_wn_config_t* cfg, int cluster_size, const float* d_params, void* d_packed_ar,
                  void* d_workspace, void* stream);
/* d_c: fp32 [B,cin,Tc] (feeder-normalised mels); d_initial: int32[B] (mu-law index, 127 = silence) or fp32[B];
 * conditioning: cfg->split_bf16 = 0 rounds the upsampled conditioning to a bf16 [B,T,cin] workspace copy; = 1 reads it in fp32 where it
 * lies - d_c [B,T,cin] itself when c_pre_upsampled, else the last upsampling layer's fp32 output [B,cin,T] in the workspace;
 * d_test_inputs: NULL or int32/fp32 [B,T] teacher-forcing inputs (the reference's wavenet_synth_debug path);
 * d_u_a / d_u_b: NULL (on-device counter RNG from `seed`) or injected uniforms in (0,1): MoL d_u_a [B,T,nr_mix] mixture
 * selection and d_u_b [B,T] logistic draw; mu-law d_u_a [B,T]. d_out_samples: int32 / fp32 [B,T];
 * d_out_raw: NULL or fp32 [B,T,out_channels] network outputs (what the reference collects in tower_y_hat_eval). */
int t2_wn_ar_generate(const t2_wn_config_t* cfg, int cluster_size, const float* d_params, const void* d_packed_ar,
                      void* d_workspace, const float* d_c, const void* d_initial, const void* d_test_inputs,
                      const float* d_u_a, const float* d_u_b, unsigned long long seed, void* d_out_samples,
                      float* d_out_raw, void* stream);
/* gin_channels > 0: per-item gate biases of the following t2_wn_ar_generate calls from the speaker ids (device int32 [B]; NULL = no
 * speaker term) and the masters. Call after t2_wn_ar_pack, which resets them to no speaker term. Items of one cluster may differ. */
int t2_wn_ar_set_speakers(const t2_wn_config_t* cfg, int cluster_size, const float* d_params, const void* d_packed_ar,
                          void* d_workspace, const int* d_speaker_ids, void* stream);


/* ---- Tacotron-2 mel predictor: training graph (teacher forcing, outputs_per_step = 1, predict_linear = False) ----
 * Replaces tacotron/models/tacotron.py:104-200,315-354, tacotron/models/modules.py:81-455,
 * tacotron/models/attention.py:38-226 and Architecture_wrappers.py:169-213. Names follow hparams.py:121-176,238-283. */
typedef struct {
  int B, T_in, T_out;
  int n_symbols, num_mels, embedding_dim;
  int enc_conv_layers, enc_conv_kernel, enc_conv_channels, encoder_lstm_units;
  int attention_dim, attention_filters, attention_kernel;
  int prenet1, prenet2, decoder_lstm_units;
  int postnet_layers, postnet_kernel, postnet_channels;
  int clip_outputs;
  float dropout_rate;        /* tacotron_dropout_rate (conv blocks in training; prenet always) */
  float zoneout_rate;        /* tacotron_zoneout_rate */
  float reg_weight;          /* tacotron_reg_weight */
  float max_abs_value, lower_bound_decay;
  int split_bf16;            /* 1 = "fp32-class" forward: every contraction of the training / GTA forward and of free-running synthesis
                              * (embedding, encoder conv blocks, encoder BiLSTM, memory layer, prenet, decoder LSTMs, attention query and
                              * context, frame / stop projection, postnet; the CBHG head has its own t2_cbhg_config_t.split_bf16) runs on bf16 hi + lo operand pairs (hi.hi + lo.hi + hi.lo, fp32
                              * accumulate) and every stored activation / recurrent state is a hi + lo pair; pre-batch-norm activations and
                              * cell states are fp32. Forward / losses / synthesis only (no backward); the LSTM sizes must be multiples of 64. */
  int mask_decoder;          /* 1 = masked losses (tacotron/models/modules.py:412-455): MSE terms over the frames t < targets_lengths[b]
                              * (sum / count_nonzero of the mask), stop-token loss = weighted sigmoid CE over the same frames divided by the
                              * number of NON-ZERO masked terms; the lengths come from t2_taco_set_target_lengths */
  float cross_entropy_pos_weight;  /* pos_weight of tf.nn.weighted_cross_entropy_with_logits (masked stop-token loss only) */
  int unmasked_encoder;      /* 1 = mask_encoder False (tacotron/models/attention.py:140-151, tacotron.py:135): the attention energies and
                              * the softmax cover all T_in positions of every row, not only the first input_lengths[b]. The encoder outputs
                              * (values, keys) past a length are zero either way (dynamic BiLSTM, modules.py:207-217), but their energies
                              * are not, so the results depend on the padded T_in. 0 = masked (the reference default). Other values are
                              * T2_ERR_INVALID_ARG. Applies to training, evaluation, GTA and synthesis. */
  int noncumulative_weights; /* 1 = cumulative_weights False (attention.py:220-224): the attention state after a step is that step's
                              * alignments, not their running sum. 0 = cumulative (the reference default); other values are
                              * T2_ERR_INVALID_ARG. Applies everywhere the attention runs. */
  float teacher_forcing_ratio;     /* tacotron_teacher_forcing_ratio in [0, 1] ('constant' mode, helpers.py:115-128) of t2_taco_forward /
                              * t2_taco_backward; anything else is T2_ERR_INVALID_ARG. 1 = full teacher forcing: the prenet, the LSTM-1 input
                              * projection and the frame / stop projections run batched over all T_out steps. < 1: at the end of decoder step t
                              * ONE draw u_t (hash stream 40, element t) decides for the whole batch: u_t < ratio feeds step t + 1 the target
                              * frame t, otherwise the raw (bias added, un-clipped) frame it just predicted, and the backward pass
                              * differentiates through the fed-back frames. That path runs the prenet, the input projection and the
                              * projections once per step. Workspace "teacher_forced" int32 [T_out] holds the choices of the last forward
                              * (element t = 1: step t + 1 consumed the target). Free-running synthesis ignores the field. */
} t2_taco_config_t;

int t2_taco_sizes(const t2_taco_config_t* cfg, long long* n_params, long long* packed_bytes, long long* workspace_bytes,
                  int* n_tensors);
int t2_taco_param_info(const t2_taco_config_t* cfg, int i, char* name, int name_cap, long long* offset, int* ndim,
                       int* shape4, int* trainable);
int t2_taco_init(const t2_taco_config_t* cfg, void* d_packed, void* d_workspace, void* stream);
int t2_taco_pack_weights(const t2_taco_config_t* cfg, const float* d_params, void* d_packed, void* d_workspace, void* stream);
/* forward + losses. d_inputs int32 [B,T_in] (0-padded character ids), d_input_lengths int32 [B], d_mel_targets fp32
 * [B,T_out,num_mels] (padded with -max_abs_value), d_stop_targets fp32 [B,T_out]. d_loss fp32[4] = {before MSE, after
 * MSE, stop-token CE, L2 regularisation}; total = sum. training=1: batch-norm batch statistics (moving stats in
 * d_params are updated), conv dropout, stochastic zoneout. */
int t2_taco_forward(const t2_taco_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace,
                    const int* d_inputs, const int* d_input_lengths, const float* d_mel_targets,
                    const float* d_stop_targets, float* d_loss, int training, unsigned long long seed,
                    const unsigned long long* d_step, void* stream);
/* mask_decoder = 1: copies the B target lengths (device int32) into the workspace; call before t2_taco_forward (stream-ordered,
 * capturable). Replaces the `targets_lengths` placeholder of tacotron/models/tacotron.py:28 / tacotron/feeder.py:207. */
int t2_taco_set_target_lengths(const t2_taco_config_t* cfg, void* d_workspace, const int* d_target_lengths, void* stream);
/* backward of the last t2_taco_forward(training=1): d(total loss)/d(theta) into the flat gradient buffer (non-trainable
 * batch-norm moving statistics get 0) */
int t2_taco_backward(const t2_taco_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                     const int* d_inputs, const int* d_input_lengths, const float* d_mel_targets,
                     const float* d_stop_targets, float* d_grads, unsigned long long seed,
                     const unsigned long long* d_step, void* stream);
/* same, plus an extra upstream gradient on the clipped mel_outputs (fp32 [B][T_out][num_mels], NULL = none): the CBHG head's
 * t2_cbhg_backward output (tacotron.py:203-219 hangs the post-processing net on mel_outputs) */
int t2_taco_backward_ex(const t2_taco_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace,
                     const int* d_inputs, const int* d_input_lengths, const float* d_mel_targets,
                     const float* d_stop_targets, float* d_grads, const float* d_mel_outputs_grad, unsigned long long seed,
                     const unsigned long long* d_step, void* stream);
/* Free-running synthesis (TacoTestHelper, tacotron/models/helpers.py:6-59; tacotron.py:150-200 with is_training = False:
 * inference batch-norm, deterministic zoneout blend, prenet dropout still on). cfg->T_out is max_iters (hparams.py:138).
 *   t2_taco_infer_begin   encoder, zero decoder state, go frame
 *   t2_taco_infer_steps   decoder steps [t_begin, t_end): each feeds back its own raw frame (helpers.py:56). The stop logit
 *                         of step t is workspace "projection_rows"[t][b][num_mels]; the CALLER applies the stop rule
 *                         (every row round(sigmoid) == 1, helpers.py:40-54; r = 1) between chunks - no host sync inside.
 *   t2_taco_infer_finish  clip, postnet, residual over the first T_used frames; workspace "decoder_output" /
 *                         "mel_outputs" are then COMPACT [B][T_used][num_mels], "stop_logits" [B][T_used]. */
int t2_taco_infer_begin(const t2_taco_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace,
                        const int* d_inputs, const int* d_input_lengths, void* stream);
int t2_taco_infer_steps(const t2_taco_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace,
                        const int* d_input_lengths, int t_begin, int t_end, unsigned long long seed, void* stream);
int t2_taco_infer_finish(const t2_taco_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace, int T_used,
                         void* stream);
/* tools only: clock64() phase stamps of the attention kernels into a device buffer of 32 int64 (NULL turns them off) */
/* Counter-hash RNG behind the in-kernel dropout / zoneout masks (SURVEY.md §7 "stochastic ops in parity"):
 * d_out[i] = U[0,1) drawn for element (first_index + i) of hash stream `stream_id` under `seed` (= the seed passed to
 * t2_taco_forward / t2_wn_forward plus the device step counter). Element kept / updated iff d_out[i] >= rate.
 * Tacotron stream ids: encoder conv dropout 10+i, prenet 20 / 21, postnet conv dropout 30+i (element = linear index of
 * the layer output), zoneout (c, h) = 2*s, 2*s+1 with s = 52 / 53 (encoder fw / bw), 54 / 55 (decoder LSTM 1 / 2) and
 * element = (t*B + b)*H + unit; the teacher-forcing draw (teacher_forcing_ratio < 1) is stream 40, element = decoder step t.
 * Replaces tf.layers.dropout / tf.nn.dropout draws of tacotron/models/modules.py:133-134,249,389 and the tf.random_uniform([])
 * of tacotron/models/helpers.py:121. */
int t2_rng_uniform_f32(unsigned long long seed, unsigned int stream_id, long long first_index, long long n, float* d_out,
                       void* stream);
int t2_dbg_att_stamps(long long* d_buf);
int t2_dbg_ar_stamps(long long* d_buf);    /* same for one layer pass of the AR synthesis kernel (16 int64) */
/* debug / test access to workspace tensors by name. With split_bf16 = 1 the bf16 activation tensors double their rows: "memory"
 * [B][T_in][hi(2H) | lo(2H)], "prenet" [T_out][B][hi(P2) | lo(P2)] and "proj_in" [T_out][B][hi(D + 2H) | lo(D + 2H)] (count is
 * twice the bf16-mode count); the fp32 value of a channel is float(hi) + float(lo). "keys" stays fp32 [B][T_in][attention_dim]. */
int t2_taco_workspace_tensor(const t2_taco_config_t* cfg, void* d_workspace, const char* name, void** ptr,
                             long long* count, int* elem_bytes);

/* ---- Tacotron: CBHG post-processing net + linear-spectrogram head (predict_linear = True, the reference default) ----
 * Replaces tacotron/models/tacotron.py:203-219 (CBHG_postnet, cbhg_linear_specs_projection, clip), :323-330 / the
 * MaskedLinearLoss of tacotron/models/modules.py:457-485, and modules.py:4-78 (HighwayNet, CBHG: conv bank, max-pool, projections,
 * highway layers, bidirectional GRU over the whole padded sequence). Field names follow hparams.py:64,162-169.
 * It is a separate engine chained behind t2_taco_forward: its input is the Tacotron workspace tensor "mel_outputs", its backward
 * returns d(linear loss + its regulariser)/d(mel_outputs), which t2_taco_backward_ex adds to the mel loss seed. Parameters, gradients
 * and Adam moments are sub-ranges of the caller's flat buffers (one optimizer step / one global-norm clip over both engines). */
typedef struct {
  int B, T;                  /* batch items, decoder steps (= mel frames, >= 2) */
  int num_mels;              /* 80 */
  int kernels;               /* cbhg_kernels: convolution bank sizes 1..kernels (<= 8) */
  int conv_channels;         /* cbhg_conv_channels (128) */
  int pool_size;             /* cbhg_pool_size (2) */
  int projection;            /* cbhg_projection (256); the second projection maps back to num_mels */
  int projection_kernel_size;/* cbhg_projection_kernel_size (3) */
  int highwaynet_layers;     /* cbhg_highwaynet_layers (4) */
  int highway_units;         /* cbhg_highway_units (128) */
  int rnn_units;             /* cbhg_rnn_units (128): GRU units per direction */
  int num_freq;              /* n_fft/2 + 1: 1025 at n_fft = 2048 */
  int n_priority_freq;       /* int(2000 / (sample_rate / 2) * num_freq): bins carrying the second half of the L1 weight */
  int clip_outputs, mask_decoder;
  float max_abs_value, lower_bound_decay, reg_weight;
  int split_bf16;            /* 1 = "fp32-class" forward (t2_taco_config_t.split_bf16): every contraction - conv bank, projections,
                              * dense, highway layers, GRU input projections and recurrence, linear projection - runs on bf16 hi + lo
                              * operand pairs (hi.hi + lo.hi + hi.lo, fp32 accumulate; the recurrence h.W_hi + h.W_lo with the fp32 state)
                              * and every stored bf16 activation is a hi + lo pair; pre-batch-norm activations are fp32. Forward / losses
                              * only: t2_cbhg_backward returns T2_ERR_INVALID_ARG. 0 = bf16 operands; other values are T2_ERR_INVALID_ARG. */
} t2_cbhg_config_t;
int t2_cbhg_sizes(const t2_cbhg_config_t* cfg, long long* n_params, long long* packed_bytes, long long* workspace_bytes, int* n_tensors);
int t2_cbhg_param_info(const t2_cbhg_config_t* cfg, int i, char* name, int name_cap, long long* offset, int* ndim, int* shape4,
                       int* trainable);
int t2_cbhg_init(const t2_cbhg_config_t* cfg, void* d_packed, void* d_workspace, void* stream);          /* synchronises */
int t2_cbhg_pack_weights(const t2_cbhg_config_t* cfg, const float* d_params, void* d_packed, void* d_workspace, void* stream);
/* mask_decoder = 1: the B target lengths (device int32), as t2_taco_set_target_lengths */
int t2_cbhg_set_target_lengths(const t2_cbhg_config_t* cfg, void* d_workspace, const int* d_target_lengths, void* stream);
/* d_mel: fp32 [B][T][num_mels] (the clipped mel_outputs); d_linear_targets fp32 [B][T][num_freq] or NULL (inference);
 * d_loss[0] = linear loss, d_loss[1] = reg_weight * sum l2_loss(CBHG kernels) (NULL allowed). training = 1: batch statistics
 * (+ moving-average update), stashes for the backward pass. Linear outputs: workspace tensor "linear_outputs", fp32 rows of
 * pitch (num_freq rounded up to a multiple of 8), the first num_freq columns valid. */
int t2_cbhg_forward(const t2_cbhg_config_t* cfg, float* d_params, const void* d_packed, void* d_workspace, const float* d_mel,
                    const float* d_linear_targets, float* d_loss, int training, void* stream);
/* backward of the last t2_cbhg_forward(training = 1 with targets): gradients into d_grads (this engine's range of the flat
 * buffer; overwritten), d(loss)/d(mel_outputs) into d_mel_grad fp32 [B][T][num_mels] */
int t2_cbhg_backward(const t2_cbhg_config_t* cfg, const float* d_params, const void* d_packed, void* d_workspace, const float* d_mel,
                     float* d_grads, float* d_mel_grad, void* stream);
/* debug / test access to workspace tensors by name: "linear_outputs" fp32 (as above), bf16 "rnn_outputs" [B][T][2 RU], "highway_input"
 * [B][T][num_mels], "bank_outputs" / "pooled_outputs" [B][T][kernels * conv_channels] (after the batch norm / the max-pool), "gru_input"
 * [B][T][highway_units], fp32 "gru_xp" [B][T][6 RU], and the training stashes. With split_bf16 = 1 the bf16 activation tensors double
 * their rows: "rnn_outputs" [B][T][hi(2 RU) | lo(2 RU)], "bank_outputs" / "pooled_outputs" [B][T][hi(K CC) | lo(K CC)], "gru_input"
 * [B][T][hi(HU) | lo(HU)] and "highway_input" [B][T][hi(Ms) | lo(Ms)] with num_mels zero-padded to Ms, the next multiple of 64 (count is the
 * element count of those rows); the fp32 value of a channel is float(hi) + float(lo). "linear_outputs" and "gru_xp" stay fp32. */
int t2_cbhg_workspace_tensor(const t2_cbhg_config_t* cfg, void* d_workspace, const char* name, void** ptr, long long* count);

/* ---- optimizer: tf.train.AdamOptimizer + per-tensor clip_by_norm/clip_by_value + EMA ------------------------
 * Replaces wavenet.py:586-613 (and tacotron.py:429-437 with global_norm_clip > 0).
 * d_offsets: int64 [n_tensors + 1] element offsets of the tensors inside the flat buffers.
 * grad_scale multiplies every gradient first (1/world_size after an NCCL sum all-reduce).
 * max_norm <= 0 disables per-tensor norm clipping; max_value <= 0 disables value clipping;
 * global_norm_clip > 0 applies tf.clip_by_global_norm instead. d_ema may be NULL.
 * d_scratch: fp32 [2 n_tensors + ceil(n_total / 4096)]: the norms are summed in a fixed order without float
 * atomics, so the same call on the same state gives bit-identical results (data-parallel replicas stay identical).
 * Non-finite gradients: the clips propagate NaN, as tf.clip_by_norm / clip_by_global_norm / clip_by_value do. A NaN or Inf anywhere
 * in a tensor (per-tensor clip) or in any tensor (global clip) makes the norm non-finite: NaN turns every clipped gradient of that
 * tensor (of every tensor) into NaN, Inf scales every finite gradient to 0 and the Inf ones to NaN. Without a norm clip only the
 * non-finite elements themselves go non-finite; the value clip keeps NaN as NaN and clamps +-Inf to +-max_value. */
int t2_adam_step(float* d_params, const float* d_grads, float* d_m, float* d_v, float* d_ema,
                 const long long* d_offsets, int n_tensors, long long n_total, float lr, float beta1, float beta2,
                 float eps, int step, float grad_scale, float max_norm, float max_value, float global_norm_clip,
                 float ema_decay, float* d_scratch, void* stream);

/* ---- audio front-end ----------------------------------------------------------------------------------------
 * Replaces datasets/audio.py:22-25,61-77,178-182,225-270 and wavenet_vocoder/util.py:30-129. Field names follow
 * hparams.py:63-111. */
typedef struct {
  int sample_rate, n_fft, hop_size, win_size, num_mels;
  float fmin, fmax;
  float magnitude_power;
  float min_level_db, ref_level_db, max_abs_value;
  int symmetric_mels, allow_clipping_in_normalization, signal_normalization;
} t2_audio_config_t;

/* n_fft: 512, 1024, 2048 or 4096 (else T2_ERR_UNSUPPORTED_SHAPE); 2 <= win_size <= n_fft; num_mels <= 128; fmax <= sample_rate / 2.
 * Spectra have bins = n_fft/2 + 1 rows (257, 513, 1025 or 2049). */
int t2_stft_mel_plan_bytes(const t2_audio_config_t* cfg, long long* bytes);
/* builds twiddles, the periodic Hann window and the sparse Slaney mel filterbank (librosa.filters.mel restated in
 * fp64 on the host) into d_plan; synchronises the stream */
int t2_stft_mel_plan_init(const t2_audio_config_t* cfg, void* d_plan, void* stream);
int t2_stft_mel_frames(const t2_audio_config_t* cfg, int n_samples);
/* melspectrogram (and optionally linearspectrogram) of B clips of n_samples fp32 samples.
 * sample fed to the STFT = gain * (x[n] - preemphasis * x[n-1]); preemphasis = 0, gain = 1 is the plain
 * datasets/audio.py:melspectrogram. d_mel: fp32 [B][frames][num_mels] (time_major=1, the layout the preprocessor
 * saves, datasets/preprocessor.py:158) or [B][num_mels][frames] (time_major=0, what audio.melspectrogram returns);
 * d_linear: NULL or fp32 [B][frames][n_fft/2+1] / [B][n_fft/2+1][frames]. */
int t2_stft_mel_f32(const t2_audio_config_t* cfg, const void* d_plan, const float* d_wav, int B, int n_samples,
                    float preemphasis, float gain, float* d_mel, float* d_linear, int time_major, void* stream);
/* dense Slaney mel filterbank the fused kernel uses (librosa.filters.mel as called by datasets/audio.py:243-246): HOST double
 * [num_mels][n_fft/2 + 1]; its pseudo-inverse is the reference's _mel_to_linear (audio.py:231-241) */
int t2_mel_basis_f64(const t2_audio_config_t* cfg, double* h_basis);
/* Griffin-Lim phase reconstruction on the GPU: replaces datasets/audio.py:151-161 (_griffin_lim: librosa istft / stft iterations)
 * and :163-176 (the TF-graph variant). d_mag: fp32 [B][frames][n_fft/2+1] magnitudes (already raised to hparams.power);
 * d_phase_io: optional float2 [B][frames][n_fft/2+1] unit phases (in: initial phases, out: final) - NULL draws exp(2 pi i u) from the
 * counter hash under `seed` (the reference draws np.random.rand); iters = hparams.griffin_lim_iters re-estimation rounds (iters + 1
 * inverse transforms); d_wav: fp32 [B][hop * (frames - 1)] (librosa.istft length, centre-trimmed). Workspace: t2_griffin_lim_bytes. */
int t2_griffin_lim_bytes(const t2_audio_config_t* cfg, int B, int frames, long long* bytes);
int t2_griffin_lim_f32(const t2_audio_config_t* cfg, const void* d_plan, const float* d_mag, float* d_phase_io, int B, int frames,
                       int iters, unsigned long long seed, void* d_workspace, float* d_wav, void* stream);
/* One launch of an audio front-end kernel on caller buffers (t2_dbg_kernel_t above), through the launcher t2_stft_mel_f32 /
 * t2_griffin_lim_f32 use, so grid, block and shared memory are the product's (tests/test_audio_kernels_gpu.py). cfg must pass the
 * plan checks of t2_stft_mel_plan_bytes; plan is a device plan built for cfg by t2_stft_mel_plan_init; bins = n_fft/2 + 1. Every
 * argument is checked before any driver call; no temporaries are allocated. Does not synchronise.
 * STFT_MEL       stft_mel_kernel_v2. p: plan, wav fp32 [B][n_samples], mel fp32, lin fp32 (nullable), laid out as t2_stft_mel_f32's.
 *                i: B (1..65535), n_samples (1..2^30), time_major (0 / 1). f: preemphasis, gain (finite).
 * GL_INIT_PHASE  gl_init_phase_kernel. p: phase float2 [n] (out: exp(2 pi i u), u the counter hash of the element index under seed).
 *                i: n (1..2^36). seed.
 * GL_ISTFT       gl_istft_kernel. p: plan, mag fp32 [B][frames][bins], phase float2 [B][frames][bins], frames fp32 [B][frames][win_size]
 *                (out: the windowed inverse transforms). i: B (1..65535), frames (2..2^24, hop (frames - 1) < 2^31).
 * GL_OLA         gl_ola_kernel. p: plan, frames fp32 [B][frames][win_size], y fp32 [B][hop (frames - 1)] (out). i: as GL_ISTFT.
 * GL_STFT        gl_stft_kernel. p: plan, y fp32 [B][hop (frames - 1)], phase float2 [B][frames][bins] (out: unit phases). i: as GL_ISTFT. */
#define T2_DBG_AUDIO_STFT_MEL 1
#define T2_DBG_AUDIO_GL_INIT_PHASE 2
#define T2_DBG_AUDIO_GL_ISTFT 3
#define T2_DBG_AUDIO_GL_OLA 4
#define T2_DBG_AUDIO_GL_STFT 5
int t2_dbg_audio_kernel(const t2_audio_config_t* cfg, const t2_dbg_kernel_t* call, void* stream);
int t2_preemphasis_f32(const float* d_x, float* d_y, int B, int n_samples, float k, void* stream);
/* mu-law (mu forced to 255 like util.py:48,67,99,127); quantise truncates toward zero */
int t2_mulaw_quantize_f32_i32(const float* d_in, int* d_out, long long n, void* stream);
int t2_inv_mulaw_quantize_i32_f32(const int* d_in, float* d_out, long long n, void* stream);
int t2_mulaw_f32(const float* d_in, float* d_out, long long n, void* stream);
int t2_inv_mulaw_f32(const float* d_in, float* d_out, long long n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* T2B200_H_ */
