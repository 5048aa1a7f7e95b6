"""Tacotron / CBHG loss, gradient-seed and parameter-packing kernels (t2_tacotron.cu, t2_cbhg.cu, t2_params.cu, t2_batchnorm.cu), one launch
at a time through t2_dbg_taco_kernel (LOSS, PARAMS, ROWS 2) / t2_dbg_cbhg_kernel (LINEAR, ADD), against float64 references computed from
the exact fp32 / bf16 values the kernels read. Outputs start as NaN: padding columns, rows outside [t0, t1) and destination elements
outside a pack job's block must still be NaN, and the elements the kernels promise as zeros must be exactly 0.

Per-element bounds (u = 2^-24, fp32 unit roundoff; BF = 2^-8 bounds one bf16 rounding relative to the value):
  exact kernels          mask_values, proj_bias (one fp32 add), add_k (one fp32 add, then bf16 RNE), dmel_k (fp32 ((a + b) + c) + d in
                         that order), relu_drop_bwd at dropout rates 0 and 0.5 (d / (1 - p) is exact, so the stored value is one bf16
                         rounding of the float64 value; at other rates one fp32 division precedes it: BF + u) and pack (bf16 RNE of
                         the fp32 product w * scale; part 2 the bf16 RNE of that product minus its bf16 high half) are compared bit for bit.
  loss sums              every sum is a per-warp shuffle tree (5 levels) whose results go to one fp32 atomic per warp, in any order: a
                         sum of n terms with nw = ceil(n / 32) warps is off by <= (8 + nw) u sum |term| (+ 3u per squared difference).
                         The normalised terms add u for the division; the regulariser (8 blocks x 256 threads, ceil(len / 2048)
                         sequential adds per thread, then at most 64 atomics per tensor) is off by <= (len / 2048 + 8 + 64 n_reg) u sum w^2.
  stop loss              each term (1 - z) v + c (log1p(exp(-|v|)) + max(-v, 0)), c = 1 + (pos_weight - 1) z, goes through __expf
                         (relative error 2^-21 (1 + |v|)) and a cancellation of size |v|: |d term| <= 4u (|v| + c sp) + c 2^-20 (1 + |v|)
                         exp(-|v|). Its normaliser is the count of masked terms that are NON-ZERO IN FP32 (tf.count_nonzero of the fp32
                         losses, as TensorFlow evaluates MaskedSigmoidCrossEntropy): for z = 0 and v below about -15 the fp32 sum
                         v + (log1p(e^v) - v) is exactly 0 and the frame leaves the count, although its float64 loss is not 0. The test
                         takes the count from an fp32 evaluation of the formula and keeps its logits away from the band where that zero
                         depends on the exp rounding (every count is checked to be the same with exp perturbed by 2^-20). With no
                         non-zero term (every live frame saturated, or no live frame) the kernel's normaliser is fmaxf(0, 1) = 1 and the
                         stop loss 0, where TensorFlow's fp32 evaluation divides 0 by 0 (NaN): test_stop_loss_with_no_counted_frame.
  gradient seeds         float64 autograd of loss_fn's formulas (masked_mse, masked_sigmoid_cross_entropy, F.mse_loss, BCE) through both
                         clamps (the clip passes the gradient at equality, raw == lo or hi), with the residual sum dec + resid taken from
                         its fp32 value (the clip tests compare that value): dmel <= 4u A, ddec <= 6u (A + |2 (dec - tgt) / n|) with
                         A = |2 (mel - tgt) / n| + |extra|; ddec_tm adds 2u (|ddec| + |dpost| + |fb|); the stop column
                         (1 - z - c sigmoid(-v)) / n (plain: (sigmoid(v) - z) / n) is off by c s (2^-21 (1 + |v|) + 3u) + 2u (|1 - z| + c s)
                         over n; bf16 outputs add BF |ref| and scale the fp32 bound by 1 + BF.
  linear L1              lin_finish_k: sums of |lin - tgt| as the loss sums above; the seed sign(d) (0.5 / n_all + [f < n_prio] 0.5 / n_low)
                         is off by 3u, then one bf16 rounding. The masked normalisers are sum(mask) NF for BOTH terms (MaskedLinearLoss),
                         the plain ones N NF and N n_prio.
  embed_bwd / colsum     fp32 sums in any order: embed_bwd adds the count of each index plus the start value (2 (count + 1) u sum |.|);
                         bias_colsum runs 64 blocks of ceil(rows / 64) sequential adds, then 64 atomics: (rows / 64 + 66) u sum |.|.
  reg_grad               grads + w params, one fp32 FMA or a multiply and an add: u |w p| + u |ref|.
Every check records its worst err / bound through parity_util.record. Measured on an H100 80GB HBM3 at its 700 W power limit: <= 0.996 for
the bf16 seeds (dmel, ddec_tm, whose bound is mostly the one bf16 rounding), 0.999 for reg_grad, <= 0.38 for ddec, <= 0.75 for dlin and
<= 0.05 for every loss sum; the exact kernels are bit-identical."""
import ctypes
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from oracle import tacotron as ot
from parity_util import record
from t2_import import t2
from test_taco_kernels_gpu import all_nan, check, nan_buf

GPU = pytest.mark.gpu
L = t2.lib
DEV = "cuda"
F64 = torch.float64
NAN = float("nan")
U = 2.0 ** -24
BF = 2.0 ** -8
EXP_ERR = 2.0 ** -21
TACO_ROWS, TACO_LOSS, TACO_PARAMS = 10, 11, 12
CBHG_LINEAR, CBHG_ADD = 9, 10
LO = float(np.float32(-4.1))        # -max_abs_value - lower_bound_decay of the default hparams, as the engines pass it (fp32)
HI = 4.0


def hook(which, kernel, p=(), i=(), f=()):
    lib = L.load()
    c = L.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate(i):
        c.i[k] = int(v)
    for k, v in enumerate(f):
        c.f[k] = float(v)
    fn = lib.t2_dbg_taco_kernel if which == "taco" else lib.t2_dbg_cbhg_kernel
    L.check(fn(ctypes.byref(c), L.stream_ptr()))
    torch.cuda.synchronize()


def bits(t):
    return t.contiguous().view(torch.int16) if t.dtype == torch.bfloat16 else t.contiguous().view(torch.int32)


def assert_bits(name, got, ref):
    assert torch.equal(bits(got), bits(ref)), "%s: not bit-identical (%d elements differ)" % (name, int((bits(got) != bits(ref)).sum()))
    record(name, worst_err_over_bound=0.0)


def f32(x):
    return torch.tensor(x, dtype=torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# decoder loss chain: dec_finish, mel_finish, reg_loss, loss_norm, then loss_seed and ddec_tm
# ------------------------------------------------------------------------------------------------------------------------------
def stop_terms32(v, z, pw, masked, exp_scale=1.0):
    """the per-frame stop loss as the kernel evaluates it, in fp32 (exp optionally scaled to probe the rounding band)"""
    v, z = v.float(), z.float()
    e = (torch.exp(-v.abs()).double() * exp_scale).float()
    sp = torch.log1p(e)
    if not masked:
        return torch.clamp(v, min=0) - v * z + sp
    c = 1 + (f32(pw) - 1) * z
    return (1 - z) * v + c * (sp + torch.clamp(-v, min=0))


def stop_terms64(v, z, pw, masked):
    v, z = v.double(), z.double()
    sp = torch.log1p(torch.exp(-v.abs()))
    if not masked:
        return torch.clamp(v, min=0) - v * z + sp
    return (1 - z) * v + (1 + (pw - 1) * z) * (sp + torch.clamp(-v, min=0))


def stop_logits(B, To, z, g):
    """z = 0 frames: saturated logits in [-40, -20] or ordinary ones in [-12, 12]; z = 1 frames: ordinary or large positive [15, 40]"""
    sat = torch.rand(B, To, generator=g) < 0.35
    ordinary = (torch.rand(B, To, generator=g) * 2 - 1) * 12
    neg = -20 - torch.rand(B, To, generator=g) * 20
    pos = 15 + torch.rand(B, To, generator=g) * 25
    return torch.where(sat, torch.where(z > 0, pos, neg), ordinary)


CHAIN_CASES = [  # B, To, M, mask_decoder, clip, pos_weight, extra, (t0, t1) of ddec_tm (None: all steps), fb
    (5, 23, 80, 1, 1, 5.5, 0, None, 0), (5, 23, 80, 1, 1, 1.0, 1, (3, 17), 1), (5, 17, 8, 0, 1, 1.0, 0, None, 0),
    (6, 31, 120, 1, 0, 3.0, 1, None, 1), (3, 9, 120, 0, 0, 1.0, 1, (2, 9), 0), (5, 40, 8, 1, 1, 2.0, 0, (0, 1), 1),
    (7, 50, 80, 0, 1, 1.0, 0, None, 1),
]


@GPU
@pytest.mark.parametrize("B,To,M,mask,clip,pw,with_extra,rng,with_fb", CHAIN_CASES)
def test_decoder_loss_chain(B, To, M, mask, clip, pw, with_extra, rng, with_fb):
    g = torch.Generator().manual_seed(B * 100 + To + M + mask * 7 + clip * 3 + with_fb)
    tag = "loss_chain_B%d_To%d_M%d_mask%d_clip%d_pw%g_x%d_fb%d" % (B, To, M, mask, clip, pw, with_extra, with_fb)
    tl = [0, 1, To - 1, To, To + 5] + [int(x) for x in torch.randint(0, To + 1, (B - 5,), generator=g)] if mask else None
    full = 3 if mask else 0                                      # an item every frame of which is live
    x = torch.randn(To, B, M, generator=g) * 2.2                 # raw frame projections
    resid = torch.randn(B * To, M, generator=g) * 0.5
    x[0, full, :4] = torch.tensor([LO, HI, 5.0, -6.0])           # decoder clip: at both bounds and beyond them
    x[1, full, 4:8] = torch.tensor([3.5, -4.0, 3.5, -4.0])       # postnet clip: raw = dec + resid at HI, at LO, then beyond
    resid[full * To + 1, 4:8] = torch.tensor([0.5, float(f32(LO) + 4.0), 1.0, -1.0])
    z = (torch.rand(B, To, generator=g) < 0.3).float()
    v = stop_logits(B, To, z, g)
    tgt = torch.randn(B, To, M, generator=g) * 2
    projo = torch.full((To, B, 128), NAN)
    projo[..., :M], projo[..., M] = x, v.t()
    resid_p = torch.full((B * To, 128), NAN)
    resid_p[:, :M] = resid
    # regulariser table: two tensors at 16-byte aligned offsets, NaN between them (not read)
    params = torch.full((304 + 80,), NAN)
    params[:300], params[304:381] = torch.randn(300, generator=g) * 0.1, torch.randn(77, generator=g) * 0.1
    tab = torch.tensor([0, 300, 304, 77], dtype=torch.int64)
    regw = 1e-3
    d = {k: t.to(DEV) for k, t in dict(projo=projo, resid=resid_p, tgt=tgt, z=z, params=params, tab=tab).items()}
    tlen = torch.tensor(tl, dtype=torch.int32, device=DEV) if mask else None
    dec_bm, dec_f, stop = nan_buf((B, To, M), torch.bfloat16), nan_buf((B, To, M), torch.float32), nan_buf((B, To), torch.float32)
    mel, out = nan_buf((B, To, M), torch.float32), nan_buf((4,), torch.float32)
    scal = torch.zeros(16, device=DEV)
    hook("taco", TACO_ROWS, [d["projo"], d["tgt"], d["z"], dec_bm, dec_f, stop, scal, tlen], [2, 0, B, To, M, clip], [LO, HI, pw])
    hook("taco", TACO_LOSS, [dec_f, d["resid"], d["tgt"], mel, scal, tlen], [0, B, To, M, clip], [LO, HI])
    hook("taco", TACO_PARAMS, [d["params"], d["tab"], scal[3:]], [2, 2])
    hook("taco", TACO_LOSS, [scal, out, tlen], [1, B, To, M, 0], [regw])

    # ---- forward values ----
    xb = d["projo"][..., :M].permute(1, 0, 2)
    dec32 = xb.clamp(LO, HI) if clip else xb
    assert torch.equal(dec_f, dec32) and torch.equal(stop, d["projo"][..., M].t())
    raw32 = dec_f + d["resid"][:, :M].view(B, To, M)             # one fp32 add, as mel_finish / loss_seed form it
    assert torch.equal(mel, raw32.clamp(LO, HI) if clip else raw32)
    live = torch.ones(B, To, dtype=torch.bool, device=DEV) if not mask else \
        torch.arange(To, device=DEV)[None, :] < tlen.long()[:, None]
    n_mel = max(int(live.sum()) * M, 1) if mask else B * To * M
    t32 = stop_terms32(stop.cpu(), z, pw, mask)
    for s in (1 - 2.0 ** -20, 1 + 2.0 ** -20):                  # the test's logits keep the fp32 zeros away from the exp rounding band
        assert torch.equal(stop_terms32(stop.cpu(), z, pw, mask, s) != 0, t32 != 0), "stop logits inside the rounding band"
    counted = (t32 != 0) & live.cpu()
    n_stop = max(int(counted.sum()), 1) if mask else B * To
    if mask:
        assert ((t32 == 0) & live.cpu() & (z == 0)).any(), "the case must contain saturated live frames that leave the count"
        assert scal[4].item() == int(counted.sum())
    assert scal[5].item() == n_mel and scal[6].item() == n_stop, (scal[5].item(), n_mel, scal[6].item(), n_stop)

    lm = live[..., None].to(F64)
    t64, m64, dec64 = d["tgt"].to(F64), mel.to(F64), dec_f.to(F64)
    nw1, nw2 = math.ceil(B * To * (M + 1) / 32), math.ceil(B * To * M / 32)
    sq_b, sq_a = (dec64 - t64) ** 2 * lm, (m64 - t64) ** 2 * lm
    ref_b, ref_a = sq_b.sum() / n_mel, sq_a.sum() / n_mel
    s64 = stop_terms64(stop, d["z"], pw, mask) * live
    ref_s = s64.sum() / n_stop
    vv = stop.to(F64).abs()
    c = (1 + (pw - 1) * d["z"].to(F64)) if mask else torch.ones_like(vv)
    sp = torch.log1p(torch.exp(-vv)) + (torch.clamp(-stop.to(F64), min=0) if mask else 0)
    e_terms = ((4 * U * (vv + c * sp) + c * 2 * EXP_ERR * (1 + vv) * torch.exp(-vv)) * live).sum()
    w = d["params"][:381].double()
    reg = 0.5 * (w[:300] ** 2).sum() + 0.5 * (w[304:] ** 2).sum()
    if mask:                                                     # the oracle's formulas give the same float64 values
        tl_c, n64 = tlen.cpu().long(), int(torch.count_nonzero(stop_terms64(stop.cpu(), z, pw, True) * live.cpu()))
        assert abs(ot.masked_mse(t64.cpu(), dec64.cpu(), tl_c).item() - ref_b.item()) <= 1e-12 * ref_b.item()
        assert abs(ot.masked_mse(t64.cpu(), m64.cpu(), tl_c).item() - ref_a.item()) <= 1e-12 * ref_a.item()
        s_or = ot.masked_sigmoid_cross_entropy(z.double(), stop.cpu().double(), tl_c, pw).item()
        assert n64 > n_stop and abs(s_or * n64 / n_stop - ref_s.item()) <= 1e-12 * abs(ref_s.item()), "float64 counts the saturated frames"
    else:
        assert abs(Fn.mse_loss(dec64, t64).item() - ref_b.item()) <= 1e-12 * ref_b.item()
        assert abs(Fn.mse_loss(m64, t64).item() - ref_a.item()) <= 1e-12 * ref_a.item()
        assert abs(Fn.binary_cross_entropy_with_logits(stop.to(F64), d["z"].to(F64)).item() - ref_s.item()) <= 1e-12 * ref_s.item()
    check(tag + "_before", out[0], ref_b, (11 + nw1) * U * sq_b.sum() / n_mel + U * ref_b)
    check(tag + "_after", out[1], ref_a, (11 + nw2) * U * sq_a.sum() / n_mel + U * ref_a)
    check(tag + "_stop", out[2], ref_s, ((8 + nw1) * U * s64.abs().sum() + e_terms) / n_stop + U * ref_s.abs())
    check(tag + "_reg", out[3], reg * regw, (300 / 2048 + 8 + 128 + 1) * U * reg * regw)

    # ---- gradient seeds: loss_seed, then ddec_tm on the kernel's ddec ----
    extra = (torch.randn(B, To, M, generator=g) * 1e-3).to(DEV) if with_extra else None
    dmel, ddec = nan_buf((B * To, 128), torch.bfloat16), nan_buf((B, To, M), torch.float32)
    hook("taco", TACO_LOSS, [dec_f, d["resid"], mel, d["tgt"], dmel, ddec, tlen, scal, extra], [2, B, To, M, clip], [LO, HI])
    t0, t1 = rng or (0, To)
    dpost = (torch.randn(B, To, M, generator=g) * 1e-3).bfloat16().to(DEV)
    fb = (torch.randn(B, M, generator=g) * 1e-3).to(DEV) if with_fb else None
    choice = torch.tensor([t % 2 for t in range(To)], dtype=torch.int32, device=DEV) if with_fb else None
    dtm = nan_buf((To, B, 128), torch.bfloat16)
    hook("taco", TACO_LOSS, [ddec, dpost, d["projo"], d["z"], dtm, tlen, scal, fb, choice], [3, B, To, M, clip, t0, t1], [LO, HI, pw])

    xs = d["projo"][..., :M].to(F64).requires_grad_(True)
    vs = d["projo"][..., M].to(F64).requires_grad_(True)
    xbs = xs.permute(1, 0, 2)
    dec = xbs.clamp(LO, HI) if clip else xbs
    r64 = d["resid"][:, :M].view(B, To, M).to(F64)
    raw = dec + r64 + (raw32.to(F64) - (dec + r64)).detach()      # value of the fp32 sum, derivative 1
    melg = raw.clamp(LO, HI) if clip else raw
    before = ((dec - t64) ** 2 * lm).sum() / n_mel
    after = ((melg - t64) ** 2 * lm).sum() / n_mel
    if extra is not None:
        after = after + (melg * extra.to(F64)).sum()
    stop_loss = (stop_terms64(vs.t(), d["z"], pw, mask) * live).sum() / n_stop
    dmel_ref, ddec_ref = torch.autograd.grad(after, raw, retain_graph=True)[0], torch.autograd.grad(before + after, dec, retain_graph=True)[0]
    total = before + after + stop_loss + (dec * dpost.to(F64)).sum()
    if fb is not None:
        total = total + sum((xbs[:, t] * fb.to(F64)).sum() for t in range(t0, t1) if choice[t].item() == 0)
    dx_ref, dv_ref = torch.autograd.grad(total, [xs, vs])
    A = 2 * (m64 - t64).abs() * lm / n_mel + (extra.abs().to(F64) if extra is not None else 0)
    check(tag + "_dmel", dmel[:, :M].view(B, To, M), dmel_ref, 4 * U * A * (1 + BF) + BF * dmel_ref.abs() + 1e-30)
    assert (dmel[:, M:] == 0).all(), "dmel padding columns must be exactly 0"
    e_ddec = 6 * U * (A + 2 * (dec64 - t64).abs() * lm / n_mel)
    check(tag + "_ddec", ddec, ddec_ref, e_ddec + 1e-30)
    if extra is None and mask:
        assert (ddec[~live] == 0).all() and (dmel[:, :M].view(B, To, M)[~live] == 0).all(), "masked frames: exact zero seeds"
    ts = slice(t0, t1)
    e_tm = (e_ddec + 2 * U * (ddec_ref.abs() + dpost.abs().to(F64) + (fb.abs().to(F64)[:, None] if fb is not None else 0))).permute(1, 0, 2)
    check(tag + "_ddec_tm", dtm[ts, :, :M], dx_ref[ts], e_tm[ts] * (1 + BF) + BF * dx_ref[ts].abs() + 1e-30)
    xv = vs.detach()
    zt = d["z"].t().to(F64)
    if mask:
        ct, s = (1 + (pw - 1) * zt), torch.sigmoid(-xv)
        e_st = (ct * s * (EXP_ERR * (1 + xv.abs()) + 3 * U) + 2 * U * ((1 - zt).abs() + ct * s)) / n_stop
    else:
        s = torch.sigmoid(xv)
        e_st = (s * (EXP_ERR * (1 + xv.abs()) + 3 * U) + 2 * U * (s + zt)) / n_stop
    check(tag + "_dstop", dtm[ts, :, M], dv_ref[ts], e_st[ts] * (1 + BF) + BF * dv_ref[ts].abs() + 1e-30)
    if mask:
        assert (dtm[ts, :, M][~live.t()[ts]] == 0).all(), "masked frames: the stop gradient must be exactly 0"
    assert (dtm[ts, :, M + 1:] == 0).all(), "ddec_tm padding columns must be exactly 0"
    all_nan(tag + " ddec_tm outside [t0, t1)", torch.cat([dtm[:t0].flatten(), dtm[t1:].flatten()]))


@GPU
def test_stop_loss_with_no_counted_frame():
    """every live frame saturated at z = 0 (its fp32 loss is exactly 0) and one item without live frames: the masked count is 0, the
    kernel's normaliser fmaxf(0, 1) = 1 and the stop loss exactly 0, where TensorFlow's fp32 evaluation gives 0 / 0 = NaN"""
    B, To, M = 2, 5, 8
    projo = torch.full((To, B, 128), NAN)
    projo[..., :M] = 0.5
    projo[..., M] = -30.0
    tgt, z = torch.zeros(B, To, M), torch.zeros(B, To)
    d = [t.to(DEV) for t in (projo, tgt, z)]
    tlen = torch.tensor([3, 0], dtype=torch.int32, device=DEV)
    dec_bm, dec_f, stop = nan_buf((B, To, M), torch.bfloat16), nan_buf((B, To, M), torch.float32), nan_buf((B, To), torch.float32)
    scal, out = torch.zeros(16, device=DEV), nan_buf((4,), torch.float32)
    hook("taco", TACO_ROWS, [d[0], d[1], d[2], dec_bm, dec_f, stop, scal, tlen], [2, 0, B, To, M, 1], [LO, HI, 2.0])
    hook("taco", TACO_LOSS, [scal, out, tlen], [1, B, To, M, 0], [0.0])
    assert scal[4].item() == 0 and scal[6].item() == 1 and out[2].item() == 0
    assert scal[5].item() == 3 * M and out[0].item() == 0.25
    live = torch.arange(To)[None, :] < tlen.cpu()[:, None]
    t32 = stop_terms32(stop.cpu(), z, 2.0, True) * live
    assert (t32 == 0).all() and math.isnan((t32.sum() / torch.count_nonzero(t32)).item()), "TensorFlow's fp32 evaluation: 0 / 0"
    record("stop_loss_no_counted_frame", worst_err_over_bound=0.0)


# ------------------------------------------------------------------------------------------------------------------------------
# linear-spectrogram loss (CBHG head)
# ------------------------------------------------------------------------------------------------------------------------------
LIN_CASES = [  # B, T, NF, NFP, sample_rate, mask_decoder, clip, with_target
    (3, 17, 1025, 1032, 22050, 1, 1, 1), (3, 17, 1025, 1032, 22050, 0, 1, 1), (2, 9, 65, 72, 80000, 0, 0, 1),
    (5, 7, 65, 72, 80000, 1, 1, 1), (3, 17, 1025, 1032, 22050, 0, 1, 0),
]


@GPU
@pytest.mark.parametrize("B,T,NF,NFP,sr,mask,clip,with_tgt", LIN_CASES)
def test_linear_loss(B, T, NF, NFP, sr, mask, clip, with_tgt):
    """n_prio from the hparams formula (185 at 22.05 kHz / 1025 bins) or a small value (3 of 65 bins at 80 kHz)"""
    g = torch.Generator().manual_seed(B * T + NF + mask + 2 * clip + 4 * with_tgt)
    hp = types.SimpleNamespace(sample_rate=sr, num_freq=NF, mask_decoder=bool(mask))
    n_prio = int(2000 / (sr * 0.5) * NF)
    N = B * T
    tag = "linear_B%d_T%d_NF%d_prio%d_mask%d_clip%d_tgt%d" % (B, T, NF, n_prio, mask, clip, with_tgt)
    tl = ([0, 1, T - 1, T, T + 2] if B >= 5 else [5, T, T + 3][:B]) if mask else None
    raw = torch.full((N, NFP), NAN)
    raw[:, :NF] = torch.randn(N, NF, generator=g) * 2.5
    r_live = (3 if B >= 5 else 1) * T + 1                        # frame 1 of an item that is live in every case
    raw[r_live, :4] = torch.tensor([LO, HI, 4.5, -5.0])
    tgt = torch.randn(N, NF, generator=g) * 2
    tgt[r_live, 4:8] = raw[r_live, 4:8].clamp(LO, HI) if clip else raw[r_live, 4:8]     # d = 0 exactly: a zero gradient (sign 0)
    lin = raw.to(DEV)
    tgt_d = tgt.to(DEV) if with_tgt else None
    dlin = nan_buf((N, NFP), torch.bfloat16)
    scal = nan_buf((10,), torch.float32)
    if with_tgt:
        scal[:2] = 0
    scal[2] = 3.25
    out = nan_buf((2,), torch.float32) if with_tgt else None
    tlen = torch.tensor(tl, dtype=torch.int32, device=DEV) if mask else None
    regw = 1e-6
    hook("cbhg", CBHG_LINEAR, [lin, tgt_d, dlin, scal, out, tlen], [B, T, NF, NFP, n_prio, clip], [LO, HI, regw])
    raw_d = raw.to(DEV)
    assert torch.equal(lin[:, :NF], raw_d[:, :NF].clamp(LO, HI) if clip else raw_d[:, :NF])
    all_nan(tag + " lin padding", lin[:, NF:])
    if not with_tgt:
        all_nan(tag + " dlin (inference)", dlin)
        all_nan(tag + " scal sums (inference)", torch.cat([scal[:2], scal[3:8]]))
        return
    tl_t = torch.tensor(tl) if mask else None
    live = (torch.arange(T)[None, :] < tl_t[:, None]).reshape(N) if mask else torch.ones(N, dtype=torch.bool)
    n_live = int(live.sum())
    n_all, n_low = (max(n_live * NF, 1), max(n_live * NF, 1)) if mask else (N * NF, N * n_prio)
    assert scal[8].item() == n_all and scal[9].item() == n_low
    x = raw[:, :NF].to(F64).requires_grad_(True)                 # the oracle runs on the host
    y = x.clamp(LO, HI) if clip else x
    loss = ot.linear_loss(tgt.to(F64).view(B, T, NF), y.view(B, T, NF), hp, tl_t)
    gx, = torch.autograd.grad(loss, x)
    loss, gx, t64 = loss.detach().to(DEV), gx.to(DEV), tgt_d.to(F64)
    l1 = (lin[:, :NF].to(F64) - t64).abs() * live.to(DEV)[:, None]
    nw = math.ceil(N * NFP / 32)
    check(tag + "_loss", out[0], loss.detach(),
          0.5 * (6 + nw) * U * (l1.sum() / n_all + l1[:, :n_prio].sum() / n_low) + 4 * U * loss.abs())
    check(tag + "_reg", out[1], torch.tensor(3.25 * regw, dtype=F64, device=DEV), U * 3.25 * regw)
    check(tag + "_dlin", dlin[:, :NF], gx, 3 * U * gx.abs() * (1 + BF) + BF * gx.abs() + 1e-30)
    assert (dlin[:, NF:] == 0).all(), "dlin padding columns must be exactly 0"
    assert (dlin[:, 4:8][r_live] == 0).all() and (dlin[~live.to(DEV)] == 0).all(), "exact zeros: d = 0 and masked rows"
    if clip:
        assert dlin[r_live, 0].item() != 0 and dlin[r_live, 1].item() != 0, "the clip passes the gradient at equality"
        assert dlin[r_live, 2].item() == 0 and dlin[r_live, 3].item() == 0


# ------------------------------------------------------------------------------------------------------------------------------
# embedding gradient, column sums, regulariser
# ------------------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize("npos,E,NS", [(37, 8, 5), (320, 512, 66), (3000, 512, 1), (1000, 7, 3)])
def test_embed_bwd(npos, E, NS):
    """NS = 1: every position on one index (the longest chain of atomics)"""
    g = torch.Generator().manual_seed(npos + E + NS)
    rows = NS + 2                                                # rows NS, NS + 1 are never indexed
    idx = torch.randint(0, NS, (npos,), generator=g, dtype=torch.int32)
    dx = torch.randn(npos, E, generator=g).bfloat16()
    start = torch.randn(rows, E, generator=g)
    idx_d, dx_d, tab = idx.to(DEV), dx.to(DEV), start.to(DEV).clone()
    hook("taco", TACO_LOSS, [idx_d, dx_d, tab], [6, npos, E])
    ref = start.to(DEV).to(F64).index_add(0, idx_d.long(), dx_d.to(F64))
    absum = start.to(DEV).to(F64).abs().index_add(0, idx_d.long(), dx_d.to(F64).abs())
    cnt = torch.bincount(idx.long(), minlength=rows).to(DEV).to(F64)[:, None]
    check("embed_bwd_n%d_E%d_NS%d" % (npos, E, NS), tab, ref, 2 * (cnt + 1) * U * absum + 1e-30)
    assert torch.equal(tab[NS:], start.to(DEV)[NS:]), "rows no position points at must not change"


@GPU
@pytest.mark.parametrize("rows,C,ld,thr", [(1, 80, 80, 256), (37, 300, 304, 128), (1000, 300, 320, 256), (6401, 128, 130, 128),
                                           (25600, 80, 128, 256), (63, 1, 1, 128)])
def test_bias_colsum(rows, C, ld, thr):
    """64 blocks of ceil(rows / 64) rows: rows < 64 leaves blocks empty, rows % 64 != 0 gives a partial last block"""
    g = torch.Generator().manual_seed(rows + C + thr)
    src = torch.full((rows, ld), NAN)
    src[:, :C] = torch.randn(rows, C, generator=g)
    src = src.bfloat16().to(DEV)
    d0 = torch.randn(C, generator=g).to(DEV)
    dst = nan_buf((C + 5,), torch.float32)
    dst[:C] = d0
    hook("taco", TACO_LOSS, [src, dst], [8, rows, C, ld, thr])
    s = src[:, :C].to(F64)
    ref = d0.to(F64) + s.sum(0)
    check("bias_colsum_r%d_C%d_ld%d_t%d" % (rows, C, ld, thr), dst[:C], ref, (rows / 64 + 66) * U * (d0.abs().to(F64) + s.abs().sum(0)) + 1e-30)
    all_nan("bias_colsum past C", dst[C:])


def reg_layout(lengths, gap):
    """offsets as add_param lays tensors out (16-byte aligned), with a non-regularised tensor of `gap` elements after each"""
    offs, n = [], 0
    for ln in lengths:
        offs.append(n)
        n += (ln + 3) // 4 * 4
        n += (gap + 3) // 4 * 4
    return offs, n


@GPU
def test_reg_loss_and_grad():
    lengths = [1, 255, 2049, 100003]
    offs, n = reg_layout(lengths, 7)
    g = torch.Generator().manual_seed(17)
    params = torch.full((n,), NAN)
    inside = torch.zeros(n, dtype=torch.bool)
    for o, ln in zip(offs, lengths):
        params[o:o + ln] = torch.randn(ln, generator=g) * 0.3
        inside[o:o + ln] = True
    tab = torch.tensor([x for o, ln in zip(offs, lengths) for x in (o, ln)], dtype=torch.int64).to(DEV)
    p_d, inside = params.to(DEV), inside.to(DEV)
    dst = torch.tensor([0.75, NAN], device=DEV)
    hook("taco", TACO_PARAMS, [p_d, tab, dst], [2, len(lengths)])
    w = torch.where(inside, p_d, torch.zeros_like(p_d)).to(F64)
    ref = 0.75 + 0.5 * (w * w).sum()
    check("reg_loss", dst[0], ref, (max(lengths) / 2048 + 8 + 64 * len(lengths)) * U * ref)
    assert math.isnan(dst[1].item())
    g0 = torch.randn(n, generator=g).to(DEV)
    grads = g0.clone()
    weight = 1e-6 * 3.7
    hook("taco", TACO_PARAMS, [p_d, grads, tab], [3, len(lengths)], [weight])
    wp = w * f32(weight).item()
    r = g0.to(F64) + wp
    check("reg_grad", grads[inside], r[inside], (U * wp.abs()[inside] + U * r.abs()[inside]) * (1 + 4 * U) + 1e-30)
    assert torch.equal(grads[~inside], g0[~inside]), "elements outside the table must not change"


# ------------------------------------------------------------------------------------------------------------------------------
# pack_kernel
# ------------------------------------------------------------------------------------------------------------------------------
JOB_BYTES = 4096


def pack_rows(N, perm, W):
    """destination row of source column n (launch_pack's permutation)"""
    n = torch.arange(N)
    if perm <= 0:
        return n
    gates = 4 if W == 32 else 2
    gi, u = n // perm, n % perm
    return (u // W) * (gates * W) + gi * W + u % W


def pack_expect(dst, src, K, N, dst_off, ld, transpose, col0, perm, W, part, scale):
    """writes the job's bf16 block into the flat bf16 tensor dst and returns the mask of the elements it covers"""
    a = src * f32(scale)                                          # fp32 product, as the kernel forms it
    if part == 2:
        a = a - a.bfloat16().float()
    v = a.bfloat16()
    cover = torch.zeros(dst.numel(), dtype=torch.bool)
    if transpose:
        rows = pack_rows(N, perm, W)
        ix = dst_off + rows[:, None] * ld + col0 + torch.arange(K)[None, :]
        dst[ix.flatten()] = v.t().flatten()
    else:
        ix = dst_off + torch.arange(K)[:, None] * ld + col0 + torch.arange(N)[None, :]
        dst[ix.flatten()] = v.flatten()
    cover[ix.flatten()] = True
    return cover


def run_pack(which, K, N, src_off, dst_off, ld, cols, transpose, perm, W, part, scale, grid_x, seed):
    g = torch.Generator().manual_seed(seed)
    params = torch.full((src_off + K * N + 9,), NAN)
    params[src_off:src_off + K * N] = torch.randn(K * N, generator=g) * 0.2
    nrows = N if transpose else K
    size = dst_off + nrows * ld + 11
    packed = nan_buf((size,), torch.bfloat16)
    jobs = torch.zeros(JOB_BYTES, dtype=torch.uint8, device=DEV)
    p_d = params.to(DEV)
    if which == 0:
        hook("taco", TACO_PARAMS, [p_d, packed, jobs], [0, JOB_BYTES, W, grid_x, src_off, K, N, dst_off, ld, transpose, cols[0], perm, part], [scale])
    else:
        hook("taco", TACO_PARAMS, [p_d, packed, jobs], [1, JOB_BYTES, W, grid_x, src_off, K, N, dst_off, ld, cols[0], cols[1], cols[2], perm], [scale])
    src = params[src_off:src_off + K * N].view(K, N)
    ref = torch.full((size,), NAN, dtype=torch.bfloat16)
    if which == 0:
        cover = pack_expect(ref, src, K, N, dst_off, ld, transpose, cols[0], perm, W, part, scale)
    else:                                                          # split slot: hi at col_hi and col_hi + slot, lo at col_lo
        cover = pack_expect(ref, src, K, N, dst_off, ld, 1, cols[0], perm, W, 0, scale)
        cover |= pack_expect(ref, src, K, N, dst_off, ld, 1, cols[0] + cols[2], perm, W, 0, scale)
        cover |= pack_expect(ref, src, K, N, dst_off, ld, 1, cols[1], perm, W, 2, scale)
    got = packed.cpu()
    tag = "pack%s_K%d_N%d_src%d_dst%d_ld%d_c%s_t%d_perm%d_W%d_part%d_s%g_g%d" % (
        "_split" if which else "", K, N, src_off, dst_off, ld, "-".join(map(str, cols)), transpose, perm, W, part, scale, grid_x)
    assert_bits(tag, got[cover], ref[cover])
    all_nan(tag + " outside the job's block", got[~cover])


PACK_CASES = [  # K, N, src_off, dst_off, dst_ld, col0, transpose, perm, W, part, scale, grid_x
    (1, 1, 0, 0, 2, 0, 0, 0, 32, 0, 1.0, 32), (63, 65, 3, 1, 67, 1, 0, 0, 32, 0, 1.0, 32), (64, 80, 4, 0, 80, 0, 0, 0, 32, 0, 1.0, 16),
    (65, 63, 5, 7, 97, 3, 1, 0, 32, 0, 0.5, 3), (80, 64, 2, 8, 160, 80, 1, 0, 128, 0, 1.0, 32), (257, 257, 1, 0, 258, 1, 1, 0, 32, 2, 1.0, 32),
    (257, 1, 9, 3, 3, 1, 0, 0, 32, 0, 1.0, 1), (1, 257, 0, 0, 257, 0, 0, 0, 32, 0, 1.0, 32), (257, 80, 6, 2, 259, 2, 1, 0, 128, 0, 0.25, 16),
    (64, 128, 0, 0, 64, 0, 1, 32, 32, 0, 1.0, 32), (65, 256, 4, 0, 96, 31, 1, 64, 32, 0, 1.0, 32), (80, 256, 0, 0, 80, 0, 1, 128, 128, 0, 1.0, 16),
    (63, 512, 2, 2, 70, 6, 1, 256, 128, 2, 0.75, 16), (257, 128, 3, 1, 257, 0, 1, 32, 32, 2, 1.0, 5),
]


@GPU
@pytest.mark.parametrize("K,N,src_off,dst_off,ld,col0,transpose,perm,W,part,scale,grid_x", PACK_CASES)
def test_pack(K, N, src_off, dst_off, ld, col0, transpose, perm, W, part, scale, grid_x):
    """odd src_off / N take the scalar loads, odd dst_ld / col0 / dst_off the scalar stores; even ones the vector paths"""
    run_pack(0, K, N, src_off, dst_off, ld, (col0,), transpose, perm, W, part, scale, grid_x, K * 1000 + N + col0)


PACK_SPLIT_CASES = [  # K, N, src_off, dst_off, dst_ld, col_hi, col_lo, slot, perm, W, scale, grid_x
    (80, 128, 0, 0, 240, 0, 160, 80, 32, 32, 1.0, 32), (63, 64, 1, 0, 193, 1, 129, 64, 0, 128, 0.7071, 16),
    (257, 256, 4, 64, 771, 0, 514, 257, 128, 128, 1.5, 16), (64, 256, 2, 0, 192, 0, 128, 64, 64, 32, 0.5, 32),
]


@GPU
@pytest.mark.parametrize("K,N,src_off,dst_off,ld,col_hi,col_lo,slot,perm,W,scale,grid_x", PACK_SPLIT_CASES)
def test_pack_split(K, N, src_off, dst_off, ld, col_hi, col_lo, slot, perm, W, scale, grid_x):
    """the three jobs of one split-bf16 weight slot in one launch (grid.y = 3): [W_hi | W_hi | W_lo] of the scaled weights"""
    run_pack(1, K, N, src_off, dst_off, ld, (col_hi, col_lo, slot), 1, perm, W, 0, scale, grid_x, K + N + slot)


# ------------------------------------------------------------------------------------------------------------------------------
# exact element-wise kernels
# ------------------------------------------------------------------------------------------------------------------------------
@GPU
@pytest.mark.parametrize("B,Ti,C2", [(1, 1, 64), (5, 37, 512), (3, 160, 768)])
def test_mask_values(B, Ti, C2):
    g = torch.Generator().manual_seed(B + Ti + C2)
    lens = [min(x, Ti + 3) for x in ([0, 1, Ti, Ti + 3, max(Ti // 2, 1)] * B)[:B]]
    mem = torch.randn(B, Ti, C2, generator=g).bfloat16()
    for b, ln in enumerate(lens):
        mem[b, ln:] = NAN                                          # rows past the length are not read
    vals = nan_buf((B * Ti * C2 + 33,), torch.bfloat16)
    hook("taco", TACO_LOSS, [mem.to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV), vals], [7, B, Ti, C2])
    valid = (torch.arange(Ti)[None, :] < torch.tensor(lens)[:, None])[..., None].expand(B, Ti, C2)
    ref = torch.where(valid, mem, torch.zeros((), dtype=torch.bfloat16))
    assert_bits("mask_values_B%d_Ti%d_C2%d" % (B, Ti, C2), vals[:B * Ti * C2].cpu(), ref.flatten())
    all_nan("mask_values tail", vals[B * Ti * C2:])


@GPU
@pytest.mark.parametrize("rows,M", [(1, 8), (37, 80), (4000, 120)])
def test_proj_bias(rows, M):
    g = torch.Generator().manual_seed(rows + M)
    p0 = torch.full((rows, 128), NAN)
    p0[:, :M + 1] = torch.randn(rows, M + 1, generator=g) * 3
    fb, sb = torch.randn(M, generator=g), torch.randn(1, generator=g)
    p = p0.to(DEV)
    hook("taco", TACO_LOSS, [p, fb.to(DEV), sb.to(DEV)], [4, rows, M])
    assert_bits("proj_bias_r%d_M%d" % (rows, M), p[:, :M + 1], (p0[:, :M + 1] + torch.cat([fb, sb])[None]).to(DEV))
    all_nan("proj_bias padding", p[:, M + 1:])


@GPU
@pytest.mark.parametrize("n,p,inplace", [(1, 0.5, 0), (1000, 0.5, 1), (65537, 0.0, 0), (4099, 0.1, 1)])
def test_relu_drop_bwd(n, p, inplace):
    g = torch.Generator().manual_seed(n)
    d = torch.randn(n, generator=g).bfloat16()
    y = torch.relu(torch.randn(n, generator=g)).bfloat16()
    y[::7] = 0.0
    y[1::11] = -0.0
    y[2::13] = -1.0
    d_d, y_d = d.to(DEV), y.to(DEV)
    dz = d_d if inplace else nan_buf((n,), torch.bfloat16)
    hook("taco", TACO_LOSS, [d_d, y_d, dz], [5, n], [p])
    keep = float(np.float32(1) - np.float32(p))
    ref64 = torch.where(y.to(F64) > 0, d.to(F64) / keep, torch.zeros((), dtype=F64))
    tag = "relu_drop_bwd_n%d_p%g_inplace%d" % (n, p, inplace)
    if p in (0.0, 0.5):
        assert_bits(tag, dz.cpu(), ref64.bfloat16())
    else:
        check(tag, dz.cpu(), ref64, (BF + U) * ref64.abs() + 1e-30)
    assert (dz.cpu()[y.to(F64) <= 0] == 0).all()


@GPU
@pytest.mark.parametrize("n,with_b", [(1, 1), (5000, 0), (65541, 1)])
def test_add_k(n, with_b):
    g = torch.Generator().manual_seed(n)
    acc0, a = torch.randn(n, generator=g), torch.randn(n, generator=g) * 1e-3
    acc = acc0.to(DEV)
    outb = nan_buf((n + 3,), torch.bfloat16) if with_b else None
    hook("cbhg", CBHG_ADD, [acc, a.to(DEV), outb], [0, n])
    ref = acc0 + a
    assert_bits("add_k_n%d" % n, acc.cpu(), ref)
    if with_b:
        assert_bits("add_k_bf16_n%d" % n, outb[:n].cpu(), ref.bfloat16())
        all_nan("add_k tail", outb[n:])


@GPU
@pytest.mark.parametrize("N,M", [(1, 8), (37, 80), (2000, 120)])
def test_dmel_k(N, M):
    g = torch.Generator().manual_seed(N + M)
    abc = []
    for k in range(3):
        t = torch.full((N, 128), NAN)
        t[:, :M] = torch.randn(N, M, generator=g) * 10.0 ** (k - 1)
        abc.append(t)
    dh = torch.randn(N, M, generator=g)
    out = nan_buf((N * M + 7,), torch.float32)
    hook("cbhg", CBHG_ADD, [abc[0].to(DEV), abc[1].to(DEV), abc[2].to(DEV), dh.to(DEV), out], [1, N, M])
    ref = ((abc[0][:, :M] + abc[1][:, :M]) + abc[2][:, :M]) + dh
    assert_bits("dmel_k_N%d_M%d" % (N, M), out[:N * M].cpu(), ref.flatten())
    all_nan("dmel_k tail", out[N * M:])
