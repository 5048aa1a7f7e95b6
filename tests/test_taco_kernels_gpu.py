"""Tacotron / CBHG engine kernels (tacotron-2_b200/csrc/t2_tacotron.cu, t2_cbhg.cu), one launch at a time through t2_dbg_taco_kernel /
t2_dbg_cbhg_kernel, against float64 references computed from the exact inputs the kernels read (bf16 inputs stay bf16, the TF32
operands of the location filter are rounded with cvt.rna semantics, dropout masks come from the host copy of the hash in
mask_hash.py). The attention is also re-derived step by step inside whole training forwards from the engine's own tensors.

Per-element bounds (u = 2^-24, fp32 unit roundoff):
  attention energies      arg = keys + q + pl; |d arg| <= 2(KA+1)u P + 2(D/32 + 8)u |h|.|Wq| + 2u |arg|, P = sum_k |tf32(cum)| |tf32(U)|
                          + |tf32(u0)| (the TF32 products are exact in fp32, only the accumulation rounds; each lane of att_query adds D/32
                          products, then 5 shuffle levels); |d e_j| <= sum_a |v_a| (4e-7 + (1 - t^2) |d arg|) + 2(18 + A/64)u sum_a |v_a t|
                          (16 products per lane, 2 shuffles, one atomic per 64-channel unit; tanhf_ = ex2.approx + rcp.approx: <= 4e-7)
  alignments              |d alpha_j| <= alpha_j (2 max_j |d e_j| + 2^-20 (1 + range e) + 2 Ti u + 4u)   (softmax of perturbed energies,
                          __expf relative error 2^-21 (1 + |x|))
  context (bf16)          1.01 (sum_j |d alpha_j| |v_j| + 2 Ti u sum_j alpha_j |v_j|) + 2^-8 |ctx|
  cum (fp32)              exactly cum + alpha (one fp32 add, the same in the test); exactly unchanged past len, alpha exactly 0 there
  batch-norm statistics   G = rows / 64 + 67 sequential fp32 adds per channel (64 blocks, then 64 atomics). A two-pass fp32 variance
                          is off by <= G u var; the kernels sum (y - y0) with y0 the channel's first row, so the bound is that of the
                          two-pass form with the margin 2 (1 + (mean - y0)^2 / var):  |d var| <= 2 G u (var + (mean - y0)^2),
                          |d mean| <= 2 G u mean|y - y0| + 2u |mean|, rstd relative 0.5 |d var| / (var + 1e-3) + 4u
  batch-norm outputs      first-order propagation of the statistics' bounds + 8u per operation chain, + 2^-8 |ref| for bf16 stores
  max-pool                exact (bf16 max; the backward adds at most two bf16 values, then one bf16 rounding: 2^-8 |ref|)
  highway                 sigmoid through __expf: |d T| <= 2^-20 (1 + |x|) T + 2u; outputs first-order + 4u |ref|, + 2^-8 |ref| for bf16
  LSTM cell backward      float64 autograd of the zoneout cell on the kernel's bf16 gate / tanh(c) stashes (tanh' = 1 - tc^2 from the
                          stash, as the kernel reads it); 8u per operation chain, + 2^-8 |ref| for the bf16 gate grads
  att_finish / dvalues    float64 autograd of U = K Wl, u0 = bK Wl + ba; fp32 sums of n terms: 2 n u times the same contraction on |.|
Every check records its worst err / bound through parity_util.record. Measured on an H100: <= 0.996 for every bf16 output; the
batch-norm gamma / beta sums sit near 1e-4 because their bounds take every one of the rows / 64 + 67 fp32 roundings at full size and
with one sign, while the real errors are random walks. Outputs start as NaN; padding columns and rows past a length must
still be NaN (or exactly 0 where the kernel promises it), and NaN in the unread channels / rows of the inputs shows they are not read.

COVERAGE maps every __global__ kernel of the two files and of the kernels they share (t2_params.cu, t2_batchnorm.cu) to the test here that
launches it (the shared batch-norm kernels are launched by both the Tacotron and the CBHG batch-norm tests);
a COVERAGE value is either the name of a test here or `file::test` for a per-kernel test in another module (att_bwd_kernel:
tests/test_attention_state_gpu.py; the two GRU kernels: tests/test_cbhg_gru_gpu.py; the split row writers:
tests/test_split_operands_gpu.py; the loss, gradient-seed, parameter-packing, regulariser and column-sum kernels:
tests/test_taco_loss_kernels_gpu.py). EXEMPT, which would name an end-to-end test covering a kernel without a per-launch test, is
empty.
test_every_engine_and_shared_kernel_is_covered (CPU) fails for a kernel added without an entry."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import mask_hash as mh
from parity_util import record
from t2_import import t2

GPU = pytest.mark.gpu
L = t2.lib
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
F64 = torch.float64
NAN = float("nan")
U = 2.0 ** -24
BF = 2.0 ** -8
TAN_ERR = 4e-7
TACO = dict(ATT_FWD=1, BN_FWD=2, BN_BWD=3, CELL_BWD=4, ATT_FINISH=5, DVALUES=6)
CBHG = dict(BN_FWD=1, BN_BWD=2, POOL_FWD=3, POOL_BWD=4, HIGHWAY_FWD=5, HIGHWAY_BWD=6)

COVERAGE = {
    "att_prep_kernel": "test_att_fwd", "att_fwd_kernel": "test_att_fwd",
    "bn_stats_kernel": "test_taco_bn_fwd", "bn_apply_kernel": "test_taco_bn_fwd",
    "bn_bwd_stats_kernel": "test_taco_bn_bwd", "bn_bwd_apply_kernel": "test_taco_bn_bwd",
    "maxpool_fwd_k": "test_maxpool", "maxpool_bwd_k": "test_maxpool", "highway_fwd_k": "test_highway", "highway_bwd_k": "test_highway",
    "lstm_cell_bwd_kernel": "test_lstm_cell_bwd", "att_finish_kernel": "test_att_finish", "att_finish2_kernel": "test_att_finish",
    "dvalues_ctx_kernel": "test_dvalues_ctx", "att_bwd_kernel": "test_attention_state_gpu.py::test_att_bwd",
    "gru_fwd_kernel": "test_cbhg_gru_gpu.py::test_gru_fwd", "gru_bwd_kernel": "test_cbhg_gru_gpu.py::test_gru_bwd",
    "embed_fwd_kernel": "test_split_operands_gpu.py::test_embed_fwd_split", "decin_kernel": "test_split_operands_gpu.py::test_decin_split",
    "proj_bias_feedback_kernel": "test_split_operands_gpu.py::test_proj_bias_feedback_split",
    "f32_to_bf16_kernel": "test_split_operands_gpu.py::test_f32_to_bf16_split",
}
_LK = "test_taco_loss_kernels_gpu.py::"
COVERAGE.update({
    "dec_finish_kernel": _LK + "test_decoder_loss_chain", "mel_finish_kernel": _LK + "test_decoder_loss_chain",
    "loss_norm_kernel": _LK + "test_decoder_loss_chain", "loss_seed_kernel": _LK + "test_decoder_loss_chain",
    "ddec_tm_kernel": _LK + "test_decoder_loss_chain", "proj_bias_kernel": _LK + "test_proj_bias",
    "relu_drop_bwd_kernel": _LK + "test_relu_drop_bwd", "embed_bwd_kernel": _LK + "test_embed_bwd", "mask_values_kernel": _LK + "test_mask_values",
    "lin_norm_k": _LK + "test_linear_loss", "lin_finish_k": _LK + "test_linear_loss", "loss_out_k": _LK + "test_linear_loss",
    "add_k": _LK + "test_add_k", "dmel_k": _LK + "test_dmel_k", "pack_kernel": _LK + "test_pack",
    "reg_loss_kernel": _LK + "test_reg_loss_and_grad", "reg_grad_kernel": _LK + "test_reg_loss_and_grad",
    "bias_colsum_kernel": _LK + "test_bias_colsum",
})
EXEMPT = {}


def test_every_engine_and_shared_kernel_is_covered():
    """CPU: every __global__ kernel of t2_tacotron.cu / t2_cbhg.cu / t2_params.cu / t2_batchnorm.cu is launched by a per-kernel test"""
    names = set()
    for f in ("t2_tacotron.cu", "t2_cbhg.cu", "t2_params.cu", "t2_batchnorm.cu"):
        src = open(os.path.join(ROOT, "tacotron-2_b200", "csrc", f)).read()
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src))
    assert len(names) >= 39
    missing = sorted(n for n in names if n not in COVERAGE and n not in EXEMPT)
    assert not missing, "kernels without a test: %s" % missing
    assert not set(COVERAGE) & set(EXEMPT) and not EXEMPT
    for k, t in list(COVERAGE.items()) + list(EXEMPT.items()):
        f, name = t.split("::") if "::" in t else (os.path.basename(__file__), t)
        assert re.search(r"^def %s\(" % name, open(os.path.join(ROOT, "tests", f)).read(), re.M), (k, t)


# ------------------------------------------------------------------------------------------------------------------------------
# plumbing
# ------------------------------------------------------------------------------------------------------------------------------
def _lib():
    lib = L.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    return lib


def launch(which, kernel, p=(), i=(), f=(), seed=0, step=None):
    lib = _lib()
    c = L.DbgKernel()
    c.kernel = (TACO if which == "taco" else CBHG)[kernel]
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate(i):
        c.i[k] = int(v)
    for k, v in enumerate(f):
        c.f[k] = float(v)
    c.seed = seed
    c.step = None if step is None else step.data_ptr()
    fn = lib.t2_dbg_taco_kernel if which == "taco" else lib.t2_dbg_cbhg_kernel
    L.check(fn(ctypes.byref(c), L.stream_ptr()))
    torch.cuda.synchronize()


def check(name, got, ref, bound, **info):
    err = (got.to(F64) - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=float("inf")).max().item() if err.numel() else 0.0
    record(name, worst_err_over_bound=ratio, **info)
    assert ratio <= 1.0, "%s: worst err / bound %.3g" % (name, ratio)


def all_nan(name, t):
    assert t.numel() == 0 or torch.isnan(t.float()).all().item(), "%s: written outside its bounds" % name


def nan_buf(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


def tf32(x):
    """cvt.rna.tf32.f32: round an fp32 tensor to 10 mantissa bits, ties away from zero"""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def lens_for(B, Ti):
    opts = [1, 16 * (Ti // 32) + 1, max(Ti - 1, 1), Ti]
    return [min(opts[b % 4], Ti) for b in range(B)]


# ------------------------------------------------------------------------------------------------------------------------------
# location-sensitive attention
# ------------------------------------------------------------------------------------------------------------------------------
def att_reference(h, WqT, U_bank, KA, v, keys, values, lens, cum):
    """float64 alignments / context of one decoder step for N rows (h [N, D] bf16, WqT [A, D] bf16, U_bank [(KA+1), A] the kernel's
    fp32 filter bank, v [A], keys [N, Ti, A] fp32, values [N, Ti, C2] bf16, lens [N], cum [N, Ti] fp32) with their bounds"""
    N, Ti, A = keys.shape
    D = WqT.shape[1]
    half = KA // 2
    valid = torch.arange(Ti, device=DEV)[None, :] < lens[:, None]
    hq, W = h.to(F64), WqT.to(F64)
    q, qabs = hq @ W.t(), hq.abs() @ W.abs().t()
    Ut = tf32(U_bank).to(F64)
    win = Fn.pad(tf32(cum).to(F64), (half, half)).unfold(1, KA, 1)            # [N, Ti, KA]: cum[j + k - half], zero outside
    pl = win @ Ut[:KA] + Ut[KA]
    P = win.abs() @ Ut[:KA].abs() + Ut[KA].abs()
    ky = torch.where(valid[..., None], keys.to(F64), torch.zeros((), dtype=F64, device=DEV))
    arg = ky + q[:, None, :] + pl
    d_arg = 2 * (KA + 1) * U * P + 2 * (D / 32 + 8) * U * qabs[:, None, :] + 2 * U * arg.abs()
    t = torch.tanh(arg)
    v64 = v.to(F64)
    e = t @ v64
    d_e = ((1 - t * t) * d_arg) @ v64.abs() + TAN_ERR * v64.abs().sum() + 2 * (18 + A / 64) * U * (t.abs() @ v64.abs())
    e = torch.where(valid, e, torch.full_like(e, -math.inf))
    alpha = torch.softmax(e, dim=1)
    emax = torch.where(valid, d_e, torch.zeros_like(d_e)).amax(1, keepdim=True)
    rng = e.amax(1, keepdim=True) - torch.where(valid, e, torch.full_like(e, math.inf)).amin(1, keepdim=True)
    d_alpha = alpha * (2 * emax + 2.0 ** -20 * (1 + rng) + 2 * Ti * U + 4 * U)
    vals = torch.where(valid[..., None], values.to(F64), torch.zeros((), dtype=F64, device=DEV))
    ctx = torch.einsum("nj,njc->nc", alpha, vals)
    d_ctx = 1.01 * (torch.einsum("nj,njc->nc", d_alpha, vals.abs()) + 2 * Ti * U * torch.einsum("nj,njc->nc", alpha, vals.abs())) + BF * ctx.abs()
    return alpha, d_alpha, ctx, d_ctx, valid


ATT_CASES = [  # B, Ti, A, KA, F, D, C2
    (3, 1, 128, 31, 32, 1024, 512), (4, 15, 128, 31, 32, 1024, 512), (4, 16, 128, 31, 32, 1024, 512), (4, 17, 128, 31, 32, 1024, 512),
    (32, 160, 128, 31, 32, 1024, 512), (3, 336, 128, 31, 32, 1024, 512), (1, 160, 64, 1, 1, 256, 256), (3, 17, 64, 31, 32, 256, 256),
    (4, 160, 128, 31, 32, 1024, 768), (4, 160, 128, 31, 32, 1024, 1024), (3, 336, 64, 31, 1, 1024, 1024), (32, 160, 128, 1, 32, 256, 768),
]


@GPU
@pytest.mark.parametrize("B,Ti,A,KA,F,D,C2", ATT_CASES)
def test_att_fwd(B, Ti, A, KA, F, D, C2):
    g = torch.Generator().manual_seed(B * 1000 + Ti + C2 + KA)
    lens = torch.tensor(lens_for(B, Ti), dtype=torch.int32)
    ld_h2, ld_a, ld_b = D + 8, C2 + 16, C2 + 8
    h2 = torch.randn(B, ld_h2, generator=g).bfloat16()
    h2[:, D:] = NAN
    WqT = (torch.randn(A, D, generator=g) / math.sqrt(D)).bfloat16()
    K = torch.randn(KA, F, generator=g) * 0.5
    bK = torch.randn(F, generator=g) * 0.1
    Wl = torch.randn(F, A, generator=g) / math.sqrt(F)
    ba = torch.randn(A, generator=g) * 0.1
    v = torch.randn(A, generator=g) / math.sqrt(A) * 2
    keys = torch.randn(B, Ti, A, generator=g) * 0.5
    values = torch.randn(B, Ti, C2, generator=g).bfloat16()
    cum = 0.05 + torch.rand(B, Ti, generator=g) * 1.5        # non-zero and different at every position
    for b in range(B):
        keys[b, lens[b]:] = NAN
        values[b, lens[b]:] = NAN
    dv = [x.to(DEV) for x in (h2, WqT, K, bK, Wl, ba, v, keys, values, lens, cum)]
    h2d, WqTd, Kd, bKd, Wld, bad, vd, keysd, valuesd, lensd, cumd = dv
    Ub = nan_buf(((KA + 1) * A,), torch.float32)
    cum_in = cumd.clone()
    alpha = nan_buf((B, Ti), torch.float32)
    ctx_a, ctx_b = nan_buf((B, ld_a), torch.bfloat16), nan_buf((B, ld_b), torch.bfloat16)
    launch("taco", "ATT_FWD", [h2d, WqTd, Kd, bKd, Wld, bad, Ub, vd, keysd, valuesd, lensd, cumd, alpha, ctx_a, ctx_b],
           [B, Ti, D, A, KA, F, C2, ld_h2, ld_a, ld_b])
    tag = "att_fwd_B%d_Ti%d_A%d_KA%d_F%d_D%d_C2%d" % (B, Ti, A, KA, F, D, C2)
    U_ref = torch.cat([Kd.to(F64) @ Wld.to(F64), (bad.to(F64) + bKd.to(F64) @ Wld.to(F64))[None]])
    U_abs = torch.cat([Kd.abs().to(F64) @ Wld.abs().to(F64), (bad.abs().to(F64) + bKd.abs().to(F64) @ Wld.abs().to(F64))[None]])
    check(tag + "_U", Ub.view(KA + 1, A), U_ref, 2 * (F + 1) * U * U_abs + 1e-30)
    ref_a, d_a, ref_c, d_c, valid = att_reference(h2d[:, :D], WqTd, Ub.view(KA + 1, A), KA, vd, keysd, valuesd, lensd, cum_in)
    check(tag + "_alpha", torch.where(valid, alpha, torch.zeros_like(alpha)), ref_a, d_a + 1e-30)
    assert (alpha[~valid] == 0).all(), "alpha past len must be exactly 0"
    assert torch.equal(cumd, cum_in + alpha), "cum must come back as cum + alpha (exactly unchanged past len)"
    check(tag + "_ctx", ctx_b[:, :C2], ref_c, d_c + 1e-30)
    assert torch.equal(ctx_a[:, :C2], ctx_b[:, :C2])
    all_nan(tag + " ctx_a pad", ctx_a[:, C2:])
    all_nan(tag + " ctx_b pad", ctx_b[:, C2:])


@GPU
@pytest.mark.parametrize("T_in,units", [(160, 256), (336, 256), (160, 384)])
def test_attention_in_training_forward(T_in, units):
    """Teacher-forced training forward at the Cfg-3 widths (B = 32, T_out = 200): every step's alignments and context re-derived in
    float64 from the engine's own query rows, keys, memory and the fp32 running sum of its earlier alignments"""
    from hparams import hparams
    hp = hparams.copy()
    hp.parse("predict_linear=False")
    hp.set_hparam("encoder_lstm_units", units)
    B, To = 32, 200
    g = torch.Generator().manual_seed(T_in + units)
    inputs = torch.randint(2, 66, (B, T_in), generator=g)
    lens = torch.tensor(lens_for(B, T_in))
    for b in range(B):
        inputs[b, lens[b]:] = 0
    mel = (torch.randn(B, To, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    stop = torch.zeros(B, To)
    stop[:, -3:] = 1
    model = t2.tacotron.Tacotron(hp, B, T_in, To)
    model.init_variables(seed=5)
    # random attention biases and a non-trivial location branch so that every term of the energies matters
    params = model.export_params()
    for name in ("attention/attention_bias", "attention/location_features_convolution/bias"):
        params[name] = torch.randn(params[name].shape, generator=g) * 0.3
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=True)
    torch.cuda.synchronize()
    H, D, A, KA = units, hp.decoder_lstm_units, hp.attention_dim, hp.attention_kernel[0]
    C2 = 2 * H
    PI = model.workspace_tensor("proj_in", (To, B, D + C2))
    keys = model.workspace_tensor("keys", (B, T_in, A))
    memory = model.workspace_tensor("memory", (B, T_in, C2))
    al = model.workspace_tensor("alignments", (To, B, T_in))
    U_bank = model.workspace_tensor("attention_filter_bank", (KA + 1, A))
    p = model.params
    off = {n: (o, s) for n, o, s, _ in model.tensors}
    o, s = off["attention/query_layer/kernel"]
    WqT = p[o:o + s[0] * s[1]].view(s).t().contiguous().bfloat16()
    o, s = off["attention/attention_variable_projection"]
    v = p[o:o + s[0]]
    lens_d = lens.int().cuda()
    cum = torch.zeros(B, T_in, dtype=torch.float32, device=DEV)
    worst_a = worst_c = 0.0
    chunk = 20
    for t0 in range(0, To, chunk):
        ts = list(range(t0, min(To, t0 + chunk)))
        cums = []
        for t in ts:
            cums.append(cum.clone())
            cum = cum + al[t]                      # the kernel's fp32 running sum, in step order
        n = len(ts)
        rows = PI[ts[0]:ts[-1] + 1].reshape(n * B, D + C2)
        ref_a, d_a, ref_c, d_c, valid = att_reference(rows[:, :D], WqT, U_bank, KA, v, keys.repeat(n, 1, 1), memory.repeat(n, 1, 1),
                                                      lens_d.repeat(n), torch.cat(cums))
        got_a = al[ts[0]:ts[-1] + 1].reshape(n * B, T_in)
        assert (got_a[~valid] == 0).all()
        ra = ((torch.where(valid, got_a, torch.zeros_like(got_a)).to(F64) - ref_a).abs() / (d_a + 1e-30)).max().item()
        rc = ((rows[:, D:].to(F64) - ref_c).abs() / (d_c + 1e-30)).max().item()
        worst_a, worst_c = max(worst_a, ra), max(worst_c, rc)
    record("att_in_situ_Tin%d_H%d" % (T_in, units), alpha_worst_err_over_bound=worst_a, ctx_worst_err_over_bound=worst_c)
    assert worst_a <= 1.0 and worst_c <= 1.0, (worst_a, worst_c)


# ------------------------------------------------------------------------------------------------------------------------------
# batch norm (two copies)
# ------------------------------------------------------------------------------------------------------------------------------
def offset_input(rows, C, ratio, g):
    """per channel: mean = ratio * std (std in [0.5, 2]), so that mean / std = ratio"""
    std = 0.5 + 1.5 * torch.rand(C, generator=g)
    return torch.randn(rows, C, generator=g) * std + ratio * std * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0)


def bn_stats_reference(y, rows):
    """two-pass float64 mean / biased variance of y [rows][C] (the values the kernel reads) and the bounds of the kernels' shifted fp32
    sums (module docstring)"""
    y64 = y.to(F64)
    mean = y64.mean(0)
    var = ((y64 - mean) ** 2).mean(0)
    y0 = y64[0]
    G = rows / 64 + 67
    d_var = 2 * G * U * (var + (mean - y0) ** 2)
    d_mean = 2 * G * U * (y64 - y0).abs().mean(0) + 2 * U * mean.abs()
    rstd = 1 / torch.sqrt(var + 1e-3)
    d_rstd = rstd * (0.5 * d_var / (var + 1e-3) + 4 * U)
    return mean, var, rstd, d_mean, d_var, d_rstd


def bn_out_reference(y, mean, rstd, d_mean, d_rstd, gamma, beta):
    y64, gm, bt = y.to(F64), gamma.to(F64), beta.to(F64)
    xh = (y64 - mean) * rstd
    x = xh * gm + bt
    d_x = gm.abs() * (rstd * d_mean + (y64 - mean).abs() * d_rstd + 8 * U * (y64.abs() + mean.abs()) * rstd) + 8 * U * (xh.abs() * gm.abs() + bt.abs())
    return x, d_x


BN_TACO_CASES = [  # rows, C, y_fp32, training, p, split, ratio
    (1, 80, 0, 1, 0.0, 0, 1), (7, 128, 0, 1, 0.5, 0, 1), (25600, 512, 0, 1, 0.5, 0, 1), (25600, 80, 1, 1, 0.0, 1, 30),
    (25600, 128, 0, 1, 0.0, 0, 30), (25600, 128, 1, 1, 0.0, 0, 300), (25600, 80, 0, 1, 0.0, 0, 300), (7, 512, 0, 0, 0.0, 0, 1),
    (25600, 128, 1, 0, 0.0, 1, 30),
]


@GPU
@pytest.mark.parametrize("rows,C,y_f32,training,p,split,ratio", BN_TACO_CASES)
def test_taco_bn_fwd(rows, C, y_f32, training, p, split, ratio):
    g = torch.Generator().manual_seed(rows + C + ratio)
    y = offset_input(rows, C, ratio, g)
    y = (y if y_f32 else y.bfloat16()).to(DEV)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV)
    beta = (0.3 * torch.randn(C, generator=g)).to(DEV)
    mm0 = (ratio * torch.randn(C, generator=g)).to(DEV)
    mv0 = (0.5 + torch.rand(C, generator=g) * 2).to(DEV)
    mm, mv = mm0.clone(), mv0.clone()
    stats = nan_buf((4 * C,), torch.float32)
    x = nan_buf((rows, 2 * C if split else C), torch.bfloat16)
    step = torch.tensor([3], dtype=torch.int64, device=DEV)
    seed, stream = 1234, 11
    launch("taco", "BN_FWD", [y, x, stats, gamma, beta, mm, mv], [rows, C, training, y_f32, stream, split], [p], seed=seed, step=step)
    tag = "taco_bn_fwd_r%d_C%d_f%d_t%d_p%g_s%d_ratio%d" % (rows, C, y_f32, training, p, split, ratio)
    if training:
        mean, var, rstd, d_mean, d_var, d_rstd = bn_stats_reference(y, rows)
        check(tag + "_mean", stats[2 * C:3 * C], mean, d_mean + 1e-30)
        check(tag + "_rstd", stats[3 * C:4 * C], rstd, d_rstd)
        check(tag + "_moving_mean", mm, 0.99 * mm0.to(F64) + 0.01 * mean, 0.01 * d_mean + 4 * U * (mm0.abs().to(F64) + mean.abs()))
        check(tag + "_moving_var", mv, 0.99 * mv0.to(F64) + 0.01 * var, 0.01 * d_var + 4 * U * (mv0.to(F64) + var))
    else:
        mean, rstd = mm0.to(F64), 1 / torch.sqrt(mv0.to(F64) + 1e-3)
        d_mean, d_rstd = torch.zeros_like(mean), rstd * 4 * U
        assert torch.equal(mm, mm0) and torch.equal(mv, mv0)
        all_nan(tag + " stats (inference)", stats)
    ref, d_ref = bn_out_reference(y, mean, rstd, d_mean, d_rstd, gamma, beta)
    if training and p > 0:
        hs = mh.hash_seed(seed + 3, stream)
        keep = torch.from_numpy(mh.hash_uniform32(hs, np.arange(rows * C, dtype=np.uint64)) >= np.float32(p)).view(rows, C).to(DEV)
        ref = torch.where(keep, ref / (1 - p), torch.zeros_like(ref))
        d_ref = torch.where(keep, d_ref / (1 - p) * (1 + 4 * U), torch.zeros_like(d_ref))
    got = x[:, :C].to(F64)
    if split:
        got = got + x[:, C:].to(F64)               # [hi | lo]: the pair carries ~16 mantissa bits
        check(tag + "_x", got, ref, d_ref + 2 ** -16 * ref.abs() + 1e-30)
    else:
        check(tag + "_x", got, ref, d_ref * (1 + BF) + BF * ref.abs() + 1e-30)


@GPU
@pytest.mark.parametrize("rows,C,act,p", [(1, 128, 0, 0.0), (7, 80, 1, 0.0), (25600, 512, 2, 0.5), (3000, 128, 1, 0.5)])
def test_taco_bn_bwd(rows, C, act, p):
    g = torch.Generator().manual_seed(rows * 7 + C + act)
    y = torch.randn(rows, C, generator=g)
    if act == 2:
        y = torch.tanh(y)
    elif act == 1:
        y = torch.relu(y)
    y = y.bfloat16().to(DEV)
    dout = torch.randn(rows, C, generator=g).bfloat16().to(DEV)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV)
    y64 = y.to(F64)
    mean32 = y64.mean(0).float()
    rstd32 = (1 / torch.sqrt(y64.var(0, unbiased=False) + 1e-3)).float()
    stats = torch.cat([torch.full((2 * C,), NAN), torch.zeros(2 * C), torch.full((2 * C,), NAN)]).to(DEV)
    stats[2 * C:3 * C], stats[3 * C:4 * C] = mean32, rstd32
    dg0, db0 = torch.randn(C, generator=g).to(DEV), torch.randn(C, generator=g).to(DEV)
    dgamma, dbeta = dg0.clone(), db0.clone()
    dpre = nan_buf((rows, C), torch.bfloat16)
    step = torch.tensor([9], dtype=torch.int64, device=DEV)
    seed, stream = 77, 31
    launch("taco", "BN_BWD", [dout, y, stats, gamma, dpre, dgamma, dbeta], [rows, C, act, stream], [p], seed=seed, step=step)
    gg = dout.to(F64)
    if p > 0:
        hs = mh.hash_seed(seed + 9, stream)
        keep = torch.from_numpy(mh.hash_uniform32(hs, np.arange(rows * C, dtype=np.uint64)) >= np.float32(p)).view(rows, C).to(DEV)
        gg = torch.where(keep, gg / (1 - p), torch.zeros_like(gg))
    mean, rstd = mean32.to(F64), rstd32.to(F64)
    xh = (y64 - mean) * rstd
    sg, sgx = gg.sum(0), (gg * xh).sum(0)
    G = rows / 64 + 67
    d_sg = 2 * G * U * gg.abs().sum(0)
    d_sgx = 2 * G * U * (gg * xh).abs().sum(0) + 4 * U * (gg.abs() * (y64.abs() + mean.abs()) * rstd).sum(0)
    gm = gamma.to(F64)
    dy = gm * rstd * (gg - sg / rows - xh * sgx / rows)
    d_dy = gm.abs() * rstd * (d_sg / rows + xh.abs() * d_sgx / rows + 4 * U * (y64.abs() + mean.abs()) * rstd * sgx.abs() / rows
                               + 8 * U * (gg.abs() + sg.abs() / rows + xh.abs() * sgx.abs() / rows))
    if act == 1:
        dy, d_dy = torch.where(y64 > 0, dy, torch.zeros_like(dy)), torch.where(y64 > 0, d_dy, torch.zeros_like(d_dy))
    elif act == 2:
        dy, d_dy = dy * (1 - y64 * y64), d_dy * (1 - y64 * y64) + 4 * U * dy.abs()
    tag = "taco_bn_bwd_r%d_C%d_act%d_p%g" % (rows, C, act, p)
    check(tag + "_dpre", dpre, dy, d_dy * (1 + BF) + BF * dy.abs() + 1e-30)
    check(tag + "_dgamma", dgamma, dg0.to(F64) + sgx, d_sgx + 2 * U * (dg0.abs().to(F64) + sgx.abs()) + 1e-30)
    check(tag + "_dbeta", dbeta, db0.to(F64) + sg, d_sg + 2 * U * (db0.abs().to(F64) + sg.abs()) + 1e-30)


BN_CBHG_CASES = [  # rows, C, ld, c0, y_fp32, training, ratio, stat_threads, outputs
    (1, 128, 1024, 0, 0, 1, 1, 128, "b"), (7, 128, 1024, 384, 0, 1, 1, 128, "b"), (25600, 128, 2048, 1920, 0, 1, 30, 128, "b"),
    (25600, 80, 80, 0, 1, 1, 300, 128, "fa"), (25600, 512, 512, 0, 0, 1, 30, 256, "b"), (7, 80, 80, 0, 1, 0, 1, 128, "fa"),
    (25600, 128, 1024, 256, 0, 0, 1, 128, "bf"),
]


@GPU
@pytest.mark.parametrize("rows,C,ld,c0,y_f32,training,ratio,thr,outs", BN_CBHG_CASES)
def test_cbhg_bn_fwd(rows, C, ld, c0, y_f32, training, ratio, thr, outs):
    g = torch.Generator().manual_seed(rows + C + c0 + ratio)
    Ct = ld
    yfull = torch.full((rows, ld), NAN)
    yfull[:, c0:c0 + C] = offset_input(rows, C, ratio, g)
    y = (yfull if y_f32 else yfull.bfloat16()).to(DEV)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV)
    beta = (0.3 * torch.randn(C, generator=g)).to(DEV)
    mm0, mv0 = (ratio * torch.randn(C, generator=g)).to(DEV), (0.5 + 2 * torch.rand(C, generator=g)).to(DEV)
    mm, mv = mm0.clone(), mv0.clone()
    stats = nan_buf((4 * Ct,), torch.float32)
    stats[c0:c0 + C] = 0
    stats[Ct + c0:Ct + c0 + C] = 0
    xb = nan_buf((rows, ld), torch.bfloat16) if "b" in outs else None
    xf = nan_buf((rows, C), torch.float32) if "f" in outs else None
    add = torch.randn(rows, C, generator=g).to(DEV) if "a" in outs else None
    launch("cbhg", "BN_FWD", [y, xb, xf, add, stats, gamma, beta, mm, mv], [rows, C, ld, c0, Ct, training, y_f32, thr])
    tag = "cbhg_bn_fwd_r%d_C%d_c0%d_f%d_t%d_ratio%d_%s" % (rows, C, c0, y_f32, training, ratio, outs)
    ys = y[:, c0:c0 + C]
    if training:
        mean, var, rstd, d_mean, d_var, d_rstd = bn_stats_reference(ys, rows)
        check(tag + "_mean", stats[2 * Ct + c0:2 * Ct + c0 + C], mean, d_mean + 1e-30)
        check(tag + "_rstd", stats[3 * Ct + c0:3 * Ct + c0 + C], rstd, d_rstd)
        check(tag + "_moving_mean", mm, 0.99 * mm0.to(F64) + 0.01 * mean, 0.01 * d_mean + 4 * U * (mm0.abs().to(F64) + mean.abs()))
        check(tag + "_moving_var", mv, 0.99 * mv0.to(F64) + 0.01 * var, 0.01 * d_var + 4 * U * (mv0.to(F64) + var))
        for sec in range(4):
            all_nan(tag + " stats outside the slice", torch.cat([stats[sec * Ct:sec * Ct + c0], stats[sec * Ct + c0 + C:(sec + 1) * Ct]]))
    else:
        mean, rstd = mm0.to(F64), 1 / torch.sqrt(mv0.to(F64) + 1e-3)
        d_mean, d_rstd = torch.zeros_like(mean), rstd * 4 * U
        assert torch.equal(mm, mm0) and torch.equal(mv, mv0)
    ref, d_ref = bn_out_reference(ys, mean, rstd, d_mean, d_rstd, gamma, beta)
    if add is not None:
        ref, d_ref = ref + add.to(F64), d_ref + 2 * U * (ref.abs() + add.abs().to(F64))
    if xb is not None:
        check(tag + "_xb", xb[:, c0:c0 + C], ref, d_ref * (1 + BF) + BF * ref.abs() + 1e-30)
        all_nan(tag + " xb outside the slice", torch.cat([xb[:, :c0], xb[:, c0 + C:]], 1))
    if xf is not None:
        check(tag + "_xf", xf, ref, d_ref + 1e-30)


@GPU
@pytest.mark.parametrize("rows,C,ld,c0,act,fp32,thr", [(7, 128, 1024, 384, 1, 0, 128), (25600, 128, 1024, 896, 1, 0, 128),
                                                        (3000, 80, 80, 0, 0, 1, 128), (1, 256, 256, 0, 1, 0, 256)])
def test_cbhg_bn_bwd(rows, C, ld, c0, act, fp32, thr):
    g = torch.Generator().manual_seed(rows + C + c0 + act)
    Ct, ldg, ldd = ld, ld, ld if not fp32 else 128
    yfull = torch.full((rows, ld), NAN)
    yfull[:, c0:c0 + C] = torch.relu(torch.randn(rows, C, generator=g)) if act else torch.randn(rows, C, generator=g)
    gfull = torch.full((rows, ldg), NAN)
    gfull[:, c0:c0 + C] = torch.randn(rows, C, generator=g)
    dt = torch.float32 if fp32 else torch.bfloat16
    y, gd = yfull.to(dt).to(DEV), gfull.to(dt).to(DEV)
    ys, gs = y[:, c0:c0 + C].to(F64), gd[:, c0:c0 + C].to(F64)
    mean32, rstd32 = ys.mean(0).float(), (1 / torch.sqrt(ys.var(0, unbiased=False) + 1e-3)).float()
    stats = nan_buf((4 * Ct,), torch.float32)
    stats[2 * Ct + c0:2 * Ct + c0 + C], stats[3 * Ct + c0:3 * Ct + c0 + C] = mean32, rstd32
    bsum = nan_buf((2 * Ct,), torch.float32)
    bsum[c0:c0 + C] = 0
    bsum[Ct + c0:Ct + c0 + C] = 0
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV)
    dg0, db0 = torch.randn(C, generator=g).to(DEV), torch.randn(C, generator=g).to(DEV)
    dgamma, dbeta = dg0.clone(), db0.clone()
    dpre = nan_buf((rows, ldd), torch.bfloat16)
    launch("cbhg", "BN_BWD", [gd, y, stats, bsum, gamma, dpre, dgamma, dbeta], [rows, C, ldg, ld, c0, Ct, ldd, act, thr, fp32])
    mean, rstd = mean32.to(F64), rstd32.to(F64)
    xh = (ys - mean) * rstd
    sg, sgx = gs.sum(0), (gs * xh).sum(0)
    G = rows / 64 + 67
    d_sg = 2 * G * U * gs.abs().sum(0)
    d_sgx = 2 * G * U * (gs * xh).abs().sum(0) + 4 * U * (gs.abs() * (ys.abs() + mean.abs()) * rstd).sum(0)
    gm = gamma.to(F64)
    dy = gm * rstd * (gs - sg / rows - xh * sgx / rows)
    d_dy = gm.abs() * rstd * (d_sg / rows + xh.abs() * d_sgx / rows + 4 * U * (ys.abs() + mean.abs()) * rstd * sgx.abs() / rows
                               + 8 * U * (gs.abs() + sg.abs() / rows + xh.abs() * sgx.abs() / rows))
    if act == 1:
        dy, d_dy = torch.where(ys > 0, dy, torch.zeros_like(dy)), torch.where(ys > 0, d_dy, torch.zeros_like(d_dy))
    tag = "cbhg_bn_bwd_r%d_C%d_c0%d_act%d_fp32%d" % (rows, C, c0, act, fp32)
    check(tag + "_dpre", dpre[:, c0:c0 + C], dy, d_dy * (1 + BF) + BF * dy.abs() + 1e-30)
    all_nan(tag + " dpre outside the slice", torch.cat([dpre[:, :c0], dpre[:, c0 + C:]], 1))
    check(tag + "_dgamma", dgamma, dg0.to(F64) + sgx, d_sgx + 2 * U * (dg0.abs().to(F64) + sgx.abs()) + 1e-30)
    check(tag + "_dbeta", dbeta, db0.to(F64) + sg, d_sg + 2 * U * (db0.abs().to(F64) + sg.abs()) + 1e-30)
    all_nan(tag + " bsum outside the slice", torch.cat([bsum[:c0], bsum[c0 + C:Ct + c0], bsum[Ct + c0 + C:]]))


# ------------------------------------------------------------------------------------------------------------------------------
# max-pool and highway (CBHG)
# ------------------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize("B,T,C", [(3, 2, 128), (5, 3, 80), (4, 37, 256), (1, 37, 128)])
def test_maxpool(B, T, C):
    """tf.layers.max_pooling1d(2, 1, 'same') per item (rows never pool across an item boundary); values from a 4-value set so that ties
    are common; the gradient of each window goes to its FIRST maximum (TF's rule)"""
    g = torch.Generator().manual_seed(B * T + C)
    N = B * T
    vals = torch.tensor([-1.0, 0.0, 0.5, 2.0])
    x = vals[torch.randint(0, 4, (N, C), generator=g)].bfloat16().to(DEV)
    dout = torch.randn(N, C, generator=g).bfloat16().to(DEV)
    out, dx = nan_buf((N, C), torch.bfloat16), nan_buf((N, C), torch.bfloat16)
    launch("cbhg", "POOL_FWD", [x, out], [N, T, C])
    launch("cbhg", "POOL_BWD", [x, dout, dx], [N, T, C])
    x3, d3 = x.view(B, T, C).to(F64), dout.view(B, T, C).to(F64)
    nxt = torch.cat([x3[:, 1:], torch.full_like(x3[:, :1], -math.inf)], 1)
    ref = torch.maximum(x3, nxt)
    assert torch.equal(out.view(B, T, C).to(F64), ref)
    ref_dx = torch.zeros_like(x3)
    first_wins = x3 >= nxt                                   # window t = (x[t], x[t+1]); the last window holds x[T-1] alone
    ref_dx += torch.where(first_wins, d3, torch.zeros_like(d3))
    ref_dx[:, 1:] += torch.where(first_wins[:, :-1], torch.zeros_like(d3[:, :-1]), d3[:, :-1])
    check("maxpool_bwd_B%d_T%d_C%d" % (B, T, C), dx.view(B, T, C), ref_dx, BF * ref_dx.abs() + 1e-30)
    assert (x3[:, :-1] == x3[:, 1:]).any(), "the case must contain ties"


@GPU
@pytest.mark.parametrize("N,HU", [(7, 128), (3000, 128), (64, 80)])
def test_highway(N, HU):
    g = torch.Generator().manual_seed(N + HU)
    sel = torch.tensor([0.0, 1e-3, -1e-3, 0.5, -0.5, 2.0, -2.0])
    pre = torch.randn(N, 2 * HU, generator=g) * 2
    pre[:, :HU] = sel[torch.randint(0, 7, (N, HU), generator=g)]          # H pre-activations exactly 0 and on both sides of it
    bh = torch.zeros(HU)
    bt = torch.randn(HU, generator=g) * 0.5
    h = torch.randn(N, HU, generator=g)
    pre, bh, bt, h = pre.to(DEV), bh.to(DEV), bt.to(DEV), h.to(DEV)
    hf, hb, HT = nan_buf((N, HU), torch.float32), nan_buf((N, HU), torch.bfloat16), nan_buf((N, 2 * HU), torch.bfloat16)
    launch("cbhg", "HIGHWAY_FWD", [pre, bh, bt, h, hf, hb, HT], [N, HU])
    p64 = pre.to(F64)
    Hh = torch.relu(p64[:, :HU] + bh.to(F64))
    tx = p64[:, HU:] + bt.to(F64)
    T = torch.sigmoid(tx)
    d_T = 2.0 ** -20 * (1 + tx.abs()) * T + 2 * U
    h64 = h.to(F64)
    ref = Hh * T + h64 * (1 - T)
    d_ref = (Hh - h64).abs() * d_T + 4 * U * (Hh * T + (h64 * (1 - T)).abs())
    tag = "highway_N%d_HU%d" % (N, HU)
    check(tag + "_hf", hf, ref, d_ref + 1e-30)
    check(tag + "_hb", hb, ref, d_ref * (1 + BF) + BF * ref.abs() + 1e-30)
    assert torch.equal(HT[:, :HU].to(F64), Hh.to(torch.bfloat16).to(F64))         # relu of exact fp32 sums, rounded once
    check(tag + "_HT_T", HT[:, HU:], T, d_T * (1 + BF) + BF * T + 1e-30)
    # backward from the stash
    dh = torch.randn(N, HU, generator=g).to(DEV)
    dHT, dcar = nan_buf((N, 2 * HU), torch.bfloat16), nan_buf((N, HU), torch.float32)
    launch("cbhg", "HIGHWAY_BWD", [dh, HT, h, dHT, dcar], [N, HU])
    Hs, Ts, d64 = HT[:, :HU].to(F64), HT[:, HU:].to(F64), dh.to(F64)
    rH = torch.where(Hs > 0, d64 * Ts, torch.zeros_like(Ts))
    rT = d64 * (Hs - h64) * Ts * (1 - Ts)
    rc = d64 * (1 - Ts)
    assert (dHT[:, :HU][Hs == 0] == 0).all(), "relu gradient at H = 0 must be exactly 0"
    check(tag + "_dH", dHT[:, :HU], rH, (BF + 2 * U) * rH.abs() + 1e-30)
    check(tag + "_dT", dHT[:, HU:], rT, (BF + 8 * U) * rT.abs() + 8 * U * (d64 * h64 * Ts * (1 - Ts)).abs() + 1e-30)
    check(tag + "_dcarry", dcar, rc, 2 * U * rc.abs() + 1e-30)


# ------------------------------------------------------------------------------------------------------------------------------
# LSTM cell backward (zoneout), attention finish, d values
# ------------------------------------------------------------------------------------------------------------------------------
CELL_CASES = [  # B, H, zone, zero_ext, with lens, with dg_b, t
    (1, 128, 0.0, 0, False, False, 0), (3, 256, 0.1, 1, True, True, 7), (32, 1024, 0.1, 0, True, False, 40), (32, 128, 0.0, 1, True, True, 3),
    (3, 1024, 0.1, 1, False, False, 2),
]


@GPU
@pytest.mark.parametrize("B,H,zone,zero_ext,with_lens,with_dgb,t", CELL_CASES)
def test_lstm_cell_bwd(B, H, zone, zero_ext, with_lens, with_dgb, t):
    g = torch.Generator().manual_seed(B * H + t + zero_ext)
    lens = torch.tensor([t + 1 if b % 2 == 0 else t for b in range(B)], dtype=torch.int32) if with_lens else None    # odd items are dead
    live = torch.ones(B, dtype=torch.bool) if lens is None else (t < lens)
    gates = torch.cat([torch.sigmoid(torch.randn(B, H, generator=g) * 2), torch.tanh(torch.randn(B, H, generator=g) * 2),
                       torch.sigmoid(torch.randn(B, H, generator=g) * 2), torch.sigmoid(torch.randn(B, H, generator=g) * 2)], 1).bfloat16()
    c_prev = torch.randn(B, H, generator=g) * 1.5
    g64 = gates.double()
    c_new = g64[:, 2 * H:3 * H] * c_prev.double() + g64[:, :H] * g64[:, H:2 * H]
    tst = torch.tanh(c_new).bfloat16()
    ld_ext, ld_a, ld_b = H + 4, 4 * H + 8, 4 * H + 16
    dh_ext = torch.randn(B, ld_ext, generator=g)
    dh_ext[:, H:] = NAN
    dhs, dcs = torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
    gst_in, tst_in, cp_in = gates.clone(), tst.clone(), c_prev.clone()
    gst_in[~live], tst_in[~live], cp_in[~live] = NAN, NAN, NAN            # dead items must not be read
    dv = [x.to(DEV) for x in (dh_ext, dhs, dcs, gst_in, tst_in, cp_in)]
    dh_d, dhs_d, dcs_d, gst_d, tst_d, cp_d = dv
    dg_a = nan_buf((B, ld_a), torch.bfloat16)
    dg_b = nan_buf((B, ld_b), torch.bfloat16) if with_dgb else None
    lens_d = lens.to(DEV) if lens is not None else None
    step = torch.tensor([5], dtype=torch.int64, device=DEV)
    seed, stream = 4321, 55
    launch("taco", "CELL_BWD", [dh_d, dhs_d, dcs_d, gst_d, tst_d, cp_d, dg_a, dg_b, lens_d], [ld_ext, zero_ext, ld_a, ld_b, t, B, H, stream],
           [zone], seed=seed, step=step)
    # masks: element (t, b, u) of streams 2 * stream (c) and 2 * stream + 1 (h); kept (the state updates) iff u >= zone
    idx = ((t * B + np.arange(B, dtype=np.uint64)[:, None]) * H + np.arange(H, dtype=np.uint64)[None, :]).astype(np.uint64)
    mc = torch.from_numpy(mh.hash_uniform32(mh.hash_seed(seed + 5, 2 * stream), idx) >= np.float32(zone)).double()
    mhm = torch.from_numpy(mh.hash_uniform32(mh.hash_seed(seed + 5, 2 * stream + 1), idx) >= np.float32(zone)).double()
    if zone <= 0:
        mc, mhm = torch.ones_like(mc), torch.ones_like(mhm)
    # float64 autograd of the cell on the stashed values (gate pre-activations are the exact inverses of the stashed gates)
    z = [torch.logit(g64[:, :H]), torch.atanh(g64[:, H:2 * H]), torch.logit(g64[:, 2 * H:3 * H]), torch.logit(g64[:, 3 * H:])]
    z = [x.clone().requires_grad_(True) for x in z]
    cp = c_prev.double().clone().requires_grad_(True)
    hp = torch.zeros(B, H, dtype=F64, requires_grad=True)
    gi, gj, gf, go = torch.sigmoid(z[0]), torch.tanh(z[1]), torch.sigmoid(z[2]), torch.sigmoid(z[3])
    cn = gf * cp + gi * gj
    tc = tst.double()
    T = tc + (1 - tc * tc) * (cn - cn.detach())                           # value and derivative from the bf16 stash, as the kernel reads it
    hn = go * T
    c_out, h_out = mc * cn + (1 - mc) * cp, mhm * hn + (1 - mhm) * hp
    dh64, dhs64, dcs64 = dh_ext[:, :H].double(), dhs.double(), dcs.double()
    (dh64 * hn + dhs64 * h_out + dcs64 * c_out).sum().backward()
    ref_g = torch.cat([x.grad for x in z], 1)
    ref_dcs, ref_dhs = cp.grad, hp.grad
    # fp32 error of dc_new (8u per chain), carried into the gate and state gradients
    dh_new = dh64 + mhm * dhs64
    e_c = 8 * U * ((dh_new * go.detach() * (1 - tc * tc)).abs() + dcs64.abs())
    dc_new = mc * dcs64 + dh_new * go.detach() * (1 - tc * tc)
    gd = g64
    fac = torch.cat([(gd[:, H:2 * H] * gd[:, :H] * (1 - gd[:, :H])).abs(), (gd[:, :H] * (1 - gd[:, H:2 * H] ** 2)).abs(),
                     (c_prev.double() * gd[:, 2 * H:3 * H] * (1 - gd[:, 2 * H:3 * H])).abs(), torch.zeros(B, H, dtype=F64)], 1)
    d_g = e_c.repeat(1, 4) * fac + 8 * U * ref_g.abs() + 8 * U * (dh_new.abs() * tc.abs()).repeat(1, 4) * torch.cat([torch.zeros(B, 3 * H, dtype=F64), torch.ones(B, H, dtype=F64)], 1)
    d_dcs = e_c * gd[:, 2 * H:3 * H] + 4 * U * ((dc_new * gd[:, 2 * H:3 * H]).abs() + dcs64.abs())
    livem = live[:, None].to(DEV)
    ref_g, d_g = torch.where(live[:, None], ref_g, torch.zeros_like(ref_g)).to(DEV), d_g.to(DEV)
    tag = "cell_bwd_B%d_H%d_z%g_ze%d_l%d" % (B, H, zone, zero_ext, int(with_lens))
    check(tag + "_dg", dg_a[:, :4 * H], ref_g, d_g * (1 + BF) + BF * ref_g.abs() + 1e-30)
    assert (dg_a[:, :4 * H][~livem.expand(B, 4 * H)] == 0).all(), "dead items: gate gradients must be exactly 0"
    all_nan(tag + " dg_a pad", dg_a[:, 4 * H:])
    if dg_b is not None:
        assert torch.equal(dg_b[:, :4 * H], dg_a[:, :4 * H])
        all_nan(tag + " dg_b pad", dg_b[:, 4 * H:])
    l2 = live.to(DEV)
    check(tag + "_dcs", dcs_d[l2], ref_dcs.to(DEV)[l2], d_dcs.to(DEV)[l2] + 1e-30)
    assert torch.equal(dhs_d[l2], ref_dhs.to(DEV)[l2].float()), "dhs: exactly dhs or 0 by the h mask"
    assert torch.equal(dcs_d[~l2], dcs.to(DEV)[~l2]) and torch.equal(dhs_d[~l2], dhs.to(DEV)[~l2]), "dead items: carried grads unchanged"
    dh_out = dh_d[:, :H]
    if zero_ext:
        assert (dh_out[l2] == 0).all()
    else:
        assert torch.equal(dh_out[l2], dh_ext[:, :H].to(DEV)[l2])
    assert torch.equal(dh_out[~l2], dh_ext[:, :H].to(DEV)[~l2])
    all_nan(tag + " dh_ext pad", dh_d[:, H:])


@GPU
@pytest.mark.parametrize("B,KA,F,A", [(1, 31, 32, 128), (3, 31, 32, 128), (32, 1, 1, 64), (5, 31, 7, 64)])
def test_att_finish(B, KA, F, A):
    g = torch.Generator().manual_seed(B + KA + F + A)
    acc = torch.randn(B, KA + 2, A, generator=g)
    K, bK, Wl = torch.randn(KA, F, generator=g) * 0.5, torch.randn(F, generator=g) * 0.3, torch.randn(F, A, generator=g) / math.sqrt(F)
    o_k, o_bk = 3, 3 + KA * F + 1
    o_wl = o_bk + F + 2
    o_v, o_ba = o_wl + F * A + 5, o_wl + F * A + 5 + A + 3
    n = o_ba + A + 4
    start = torch.randn(n, generator=g)
    dv = [x.to(DEV) for x in (acc, K, bK, Wl, start)]
    acc_d, K_d, bK_d, Wl_d, grads = dv
    grads = grads.clone()
    scratch = nan_buf(((KA + 2) * A,), torch.float32)
    launch("taco", "ATT_FINISH", [acc_d, K_d, bK_d, Wl_d, grads, scratch], [B, KA, F, A, o_k, o_bk, o_wl, o_v, o_ba])
    a64 = acc_d.double().sum(0)
    aabs = acc_d.double().abs().sum(0)
    Kx, bKx, Wlx = (x.double().clone().requires_grad_(True) for x in (K_d, bK_d, Wl_d))
    bax, vx = torch.zeros(A, dtype=F64, device=DEV, requires_grad=True), torch.zeros(A, dtype=F64, device=DEV, requires_grad=True)
    Ux, u0x = Kx @ Wlx, bKx @ Wlx + bax
    ((a64[:KA] * Ux).sum() + (a64[KA] * u0x).sum() + (a64[KA + 1] * vx).sum()).backward()
    Ka, bKa, Wla = K_d.double().abs(), bK_d.double().abs(), Wl_d.double().abs()
    nn_ = B + A + KA + 2
    ab = {"dK": aabs[:KA] @ Wla.t(), "dWl": Ka.t() @ aabs[:KA] + bKa[:, None] * aabs[KA][None, :], "dbK": Wla @ aabs[KA],
          "dv": aabs[KA + 1], "dba": aabs[KA]}
    ref = {"dK": Kx.grad, "dWl": Wlx.grad, "dbK": bKx.grad, "dv": vx.grad, "dba": bax.grad}
    offs = {"dK": (o_k, KA * F), "dWl": (o_wl, F * A), "dbK": (o_bk, F), "dv": (o_v, A), "dba": (o_ba, A)}
    s64 = start.to(DEV).double()
    touched = torch.zeros(n, dtype=torch.bool, device=DEV)
    for k, (o, m) in offs.items():
        r = s64[o:o + m] + ref[k].reshape(-1)
        check("att_finish_B%d_KA%d_F%d_A%d_%s" % (B, KA, F, A, k), grads[o:o + m], r,
              2 * nn_ * U * ab[k].reshape(-1) + 2 * U * r.abs() + 1e-30)
        touched[o:o + m] = True
    assert torch.equal(grads[~touched], start.to(DEV)[~touched]), "att_finish wrote outside its tensors"
    check("att_finish_B%d_KA%d_F%d_A%d_scratch" % (B, KA, F, A), scratch.view(KA + 2, A), a64, 2 * B * U * aabs + 1e-30)


@GPU
@pytest.mark.parametrize("B,Ti,To,C2", [(3, 17, 50, 512), (2, 160, 200, 768), (1, 1, 3, 256)])
def test_dvalues_ctx(B, Ti, To, C2):
    g = torch.Generator().manual_seed(B + Ti + To + C2)
    lens = torch.tensor(lens_for(B, Ti), dtype=torch.int32)
    alpha = torch.softmax(torch.randn(To, B, Ti, generator=g) * 2, -1)
    dctx = torch.randn(To, B, C2, generator=g).bfloat16()
    start = torch.randn(B, Ti, C2, generator=g)
    al_d, dc_d, ln_d, dv_d = alpha.to(DEV), dctx.to(DEV), lens.to(DEV), start.to(DEV).clone()
    launch("taco", "DVALUES", [al_d, dc_d, ln_d, dv_d], [B, Ti, To, C2])
    ref = start.to(DEV).double() + torch.einsum("tbj,tbc->bjc", al_d.double(), dc_d.double())
    ab = start.to(DEV).double().abs() + torch.einsum("tbj,tbc->bjc", al_d.double(), dc_d.double().abs())
    valid = (torch.arange(Ti, device=DEV)[None, :] < ln_d[:, None].long())
    tag = "dvalues_B%d_Ti%d_To%d_C2%d" % (B, Ti, To, C2)
    check(tag, dv_d[valid], ref[valid], 2 * (To + 1) * U * ab[valid] + 1e-30)
    assert (dv_d[~valid] == 0).all(), "rows past len must be exactly 0"
