"""The CBHG bidirectional GRU kernels (gru_fwd_kernel / gru_bwd_kernel, t2_cbhg.cu) one launch at a time through t2_dbg_cbhg_kernel
(T2_DBG_CBHG_GRU_FWD / GRU_BWD), and inside a CBHG training step, against the float64 references and bounds of tests/gru_reference.py.

The forward is checked step by step: each step is re-derived from the kernel's own bf16 output of the previous step, so every bound
spans one step of the recurrence. The BPTT is checked the same way: a float64 BPTT of the kernel's own inputs, re-anchored every step on
the kernel's g recovered from its own dXP of the previously processed step. The in-engine test re-derives the GRU outputs, stashes, dXP and the eight weight row blocks and four biases of the GRU from
the engine's own operands, which pins the parameter offsets, stash pointers, the XP column layout d 3RU + {0, RU, 2RU} and the +-1
shifts of the recurrent weight-gradient tiles at item boundaries. Every check records its worst err / bound through parity_util.record."""
import ctypes

import pytest
import torch

import gru_reference as gr
from hparams import hparams
from oracle import tacotron as ot
from parity_util import record
from t2_import import t2

pytestmark = pytest.mark.gpu
L = t2.lib
DEV = "cuda"
F64 = torch.float64
NAN = float("nan")
HU, RU = 128, 128
GUARD = 3                                       # rows past N that must stay untouched
DIRS = ("forward", "backward")
CASES = [(1, 1), (1, 2), (3, 37), (4, 64), (5, 37), (9, 200), (32, 800)]
GRU_FWD, GRU_BWD = 7, 8


def launch(kernel, p, i):
    lib = L.load()
    c = L.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate(i):
        c.i[k] = int(v)
    L.check(lib.t2_dbg_cbhg_kernel(ctypes.byref(c), L.stream_ptr()))
    torch.cuda.synchronize()


def check(name, got, ref, bound, **info):
    err = (got.to(F64) - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=float("inf")).max().item() if err.numel() else 0.0
    record(name, worst_err_over_bound=ratio, **info)
    assert ratio <= 1.0, "%s: worst err / bound %.3g" % (name, ratio)
    return ratio


def nan_buf(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


def _hp():
    hp = hparams.copy()
    hp.parse("predict_linear=True")
    return hp


def _params(regime, seed):
    """flat fp32 parameter buffer with the two directions' GRU tensors at odd offsets; the input rows (< HU) of both kernels are NaN
    (the recurrent kernels never read them). Returns (flat, offsets [fw, bw] of (gk, ck, gb, cb), Ws for the reference)."""
    g = torch.Generator().manual_seed(seed)
    p = ot.init_params(_hp(), seed=seed, random_bias=regime == "random_bias")
    parts, offs, Ws, o = [torch.full((3,), NAN)], [], [], 3
    for n in DIRS:
        q = "CBHG_postnet/%s_RNN/" % n
        gk, ck, gb, cb = p[q + "gates/kernel"].clone(), p[q + "candidate/kernel"].clone(), p[q + "gates/bias"].clone(), p[q + "candidate/bias"].clone()
        if regime == "random_bias":
            gb, cb = torch.randn(2 * RU, generator=g) * 0.5, torch.randn(RU, generator=g) * 0.5
        Ws.append(dict(gk=gk.to(DEV), gb=gb.to(DEV), ck=ck.to(DEV), cb=cb.to(DEV)))
        gk[:HU], ck[:HU] = NAN, NAN
        d = {}
        for k, t in (("gk", gk), ("ck", ck), ("gb", gb), ("cb", cb)):
            d[k] = o
            parts.append(t.reshape(-1))
            o += t.numel()
            parts.append(torch.full((5,), NAN))
            o += 5
        offs.append(d)
    return torch.cat(parts).to(DEV), offs, Ws


def _xp(B, T, regime, seed):
    g = torch.Generator().manual_seed(seed + 1)
    return (torch.randn(B, T, 6 * RU, generator=g) * (8.0 if regime == "saturating" else 1.0)).to(DEV)


def run_fwd(flat, offs, XP, B, T, stashes=True):
    N = B * T
    out = nan_buf((N + GUARD, 2 * RU), torch.bfloat16)
    st = [nan_buf((N + GUARD, RU), torch.bfloat16) if stashes else None for _ in range(8)]
    ints = [B, T, HU, RU]
    for d in range(2):
        ints += [offs[d]["gk"], offs[d]["ck"], offs[d]["gb"], offs[d]["cb"]]
    launch(GRU_FWD, [flat, XP, out] + st, ints)
    return out, st


def check_fwd(tag, ref, out, st, B, T):
    """out / stashes (views [N + GUARD, .]) against the re-anchored reference; worst ratio"""
    N = B * T
    worst = check(tag + "_out", out[:N].view(B, T, 2 * RU), ref["out"], ref["out_b"])
    for d in range(2):
        for j, k in enumerate(("r", "u", "c", "rh")):
            worst = max(worst, check("%s_%s_%s" % (tag, k, "fb"[d] + "w"), st[4 * d + j][:N].view(B, T, RU), ref[k][d], ref[k + "_b"][d]))
    return worst


@pytest.mark.parametrize("regime", ["normal", "saturating", "gate_bias_1", "random_bias"])
@pytest.mark.parametrize("B,T", CASES)
def test_gru_fwd(B, T, regime):
    seed = B * 1000 + T + len(regime)
    flat, offs, Ws = _params("random_bias" if regime == "random_bias" else "init", seed)
    if regime == "normal":          # small random gate biases instead of the initialiser's 1.0
        for W in Ws:
            W["gb"] = torch.randn(2 * RU, generator=torch.Generator().manual_seed(seed), device="cpu").to(DEV) * 0.1
        for d in range(2):
            flat[offs[d]["gb"]:offs[d]["gb"] + 2 * RU] = Ws[d]["gb"]
    XP = _xp(B, T, regime, seed)
    out, st = run_fwd(flat, offs, XP, B, T)
    N = B * T
    tag = "gru_fwd_B%d_T%d_%s" % (B, T, regime)
    ref = gr.forward(XP, Ws, HU, anchor=out[:N].view(B, T, 2 * RU))
    check_fwd(tag, ref, out, st, B, T)
    assert torch.isnan(out[N:].float()).all() and all(torch.isnan(s[N:].float()).all() for s in st), "written past row N"
    out_inf, _ = run_fwd(flat, offs, XP, B, T, stashes=False)
    assert torch.equal(out_inf[:N], out[:N]), "inference (no stashes) must store the same outputs"


@pytest.mark.parametrize("B,T", CASES)
def test_gru_bwd(B, T):
    seed = B * 7 + T
    flat, offs, Ws = _params("init", seed)
    XP = _xp(B, T, "normal", seed)
    out, st = run_fwd(flat, offs, XP, B, T)
    N = B * T
    g = torch.Generator().manual_seed(seed + 2)
    dout = (torch.randn(N, 2 * RU, generator=g) * 0.1).to(DEV)
    stb = [st[0], st[1], st[2], st[4], st[5], st[6]]                       # r, u, c of fw, then of bw
    ints = [B, T, HU, RU, offs[0]["gk"], offs[0]["ck"], offs[1]["gk"], offs[1]["ck"]]
    dXP = nan_buf((N + GUARD, 6 * RU), torch.bfloat16)
    launch(GRU_BWD, [flat, dout, out] + stb + [dXP], ints)
    dXP2 = nan_buf((N + GUARD, 6 * RU), torch.bfloat16)
    launch(GRU_BWD, [flat, dout, out] + stb + [dXP2], ints)
    assert torch.equal(dXP[:N], dXP2[:N]), "two launches must be bit-identical"
    assert torch.isnan(dXP[N:].float()).all(), "written past row N"
    v = lambda t: t[:N].view(B, T, -1)
    got = v(dXP).to(F64)
    ref, bnd = gr.bptt(dout.view(B, T, 2 * RU), v(out), [v(st[0]), v(st[4])], [v(st[1]), v(st[5])], [v(st[2]), v(st[6])], Ws, HU, anchor=got)
    tag = "gru_bwd_B%d_T%d" % (B, T)
    # the precision the design gives up: dXP against a float64 BPTT on the exact float64 forward (fp32 state, unrounded stashes)
    ex = gr.forward(XP, Ws, HU)
    ref_x, _ = gr.bptt(dout.view(B, T, 2 * RU), ex["out"], ex["r"], ex["u"], ex["c"], Ws, HU)
    rel_x = ((got - ref_x).norm() / ref_x.norm()).item()
    check_dxp(tag + "_dXP", got, ref, bnd, rel_l2_vs_exact_forward=rel_x)


def check_dxp(tag, got, ref, bnd, **info):
    """dXP within its re-anchored bound, and that bound as tight at the last step as at the first: the median bound / |dXP| of every
    time step stays below 2^-3 (tests/test_cbhg_gru_cpu.py::test_bptt_anchored_bound_does_not_decay_with_the_step)"""
    T = ref.shape[1]
    per_step = (bnd / (ref.abs() + 1e-30)).transpose(0, 1).reshape(T, -1).median(1).values
    worst_step = per_step.max().item()
    ratio = check(tag, got, ref, bnd, worst_step_median_bound_rel=worst_step, **info)
    assert worst_step < 2 ** -3, "%s: the bound of some step is loose (median bound / |dXP| %.3g)" % (tag, worst_step)
    return ratio


def _ws(model, name, dtype, shape):
    lib = model.lib
    p, cnt = ctypes.c_void_p(), ctypes.c_longlong()
    L.check(lib.t2_cbhg_workspace_tensor(ctypes.byref(model.cbhg), L.ptr(model.cb_workspace), name.encode(), ctypes.byref(p), ctypes.byref(cnt)))
    off = p.value - model.cb_workspace.data_ptr()
    es = 2 if dtype == torch.bfloat16 else 4
    n = 1
    for s in shape:
        n *= s
    assert cnt.value == n, (name, cnt.value, n)
    return model.cb_workspace[off:off + n * es].view(dtype).reshape(shape)


@pytest.mark.parametrize("B,T", [(5, 37), (32, 800)])
def test_gru_in_engine(B, T):
    hp = hparams.copy()         # the CBHG widths of the defaults, a smaller Tacotron around them (tests/test_cbhg_gpu.py)
    hp.parse("predict_linear=True,tacotron_dropout_rate=0.0,tacotron_zoneout_rate=0.0,enc_conv_channels=256,embedding_dim=256,"
             "encoder_lstm_units=128,decoder_lstm_units=256,postnet_channels=256,prenet_layers=[128,128],attention_dim=128,num_freq=513")
    params = ot.init_params(hp, seed=11, random_bias=True)
    g = torch.Generator().manual_seed(B + T)
    mel = (torch.randn(B, T, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    lin_t = (torch.randn(B, T, hp.num_freq, generator=g) * 1.5 - 1).clamp(-4, 4)
    model = t2.tacotron.Tacotron(hp, B, 16, T)
    model.load_params(params)
    model.pack()
    lib, cfg = model.lib, ctypes.byref(model.cbhg)
    prm = model.params[model.n_taco:]
    mel_d, lin_d = mel.cuda().contiguous(), lin_t.cuda().contiguous()
    L.check(lib.t2_cbhg_forward(cfg, L.ptr(prm), L.ptr(model.cb_packed), L.ptr(model.cb_workspace), L.ptr(mel_d), L.ptr(lin_d), L.ptr(model.cb_loss), 1,
                                L.stream_ptr()))
    torch.cuda.synchronize()
    Ws = []
    for n in DIRS:
        q = "CBHG_postnet/%s_RNN/" % n
        Ws.append({k: params[q + s].to(DEV) for k, s in (("gk", "gates/kernel"), ("gb", "gates/bias"), ("ck", "candidate/kernel"), ("cb", "candidate/bias"))})
    XP = _ws(model, "gru_xp", torch.float32, (B, T, 6 * RU)).clone()          # the highway backward reuses this buffer
    out = _ws(model, "rnn_outputs", torch.bfloat16, (B, T, 2 * RU))
    st = {k: [_ws(model, "gru_%s_%s" % (k, dn), torch.bfloat16, (B, T, RU)) for dn in ("fw", "bw")] for k in ("r", "u", "c", "rh")}
    h_last = _ws(model, "gru_input", torch.bfloat16, (B, T, HU))
    tag = "gru_engine_B%d_T%d" % (B, T)
    ref = gr.forward(XP, Ws, HU, anchor=out)
    ratios = {"out": check(tag + "_out", out, ref["out"], ref["out_b"])}
    for k in ("r", "u", "c", "rh"):
        ratios[k] = max(check("%s_%s_%sw" % (tag, k, "fb"[d]), st[k][d], ref[k][d], ref[k + "_b"][d]) for d in range(2))
    # the input projections themselves: h_last times the input rows of both kernels, fp32 accumulation of HU bf16 products
    Win = torch.cat([torch.cat([gr.bf16(W["gk"][:HU]), gr.bf16(W["ck"][:HU])], 1) for W in Ws], 1)
    xr, xa = h_last.to(F64) @ Win, h_last.to(F64).abs() @ Win.abs()
    ratios["xp"] = check(tag + "_xp", XP, xr, 2 * (HU / 16 + 16) * gr.U * xa + 1e-30)
    model.grads = torch.zeros_like(model.params)
    L.check(lib.t2_cbhg_backward(cfg, L.ptr(prm), L.ptr(model.cb_packed), L.ptr(model.cb_workspace), L.ptr(mel_d), L.ptr(model.grads[model.n_taco:]),
                                 L.ptr(model.cb_dmel), L.stream_ptr()))
    torch.cuda.synchronize()
    dout = _ws(model, "gru_dout", torch.float32, (B, T, 2 * RU))
    dXP = _ws(model, "gru_dxp", torch.bfloat16, (B, T, 6 * RU))
    ref_d, bnd = gr.bptt(dout, out, st["r"], st["u"], st["c"], Ws, HU, anchor=dXP)
    ratios["dxp"] = check_dxp(tag + "_dXP", dXP, ref_d, bnd)
    grads = model.export_grads()
    wg = gr.weight_grads(h_last, dXP, out, st["rh"], HU)
    for d, n in enumerate(DIRS):
        q = "CBHG_postnet/%s_RNN/" % n
        gk, ck = grads[q + "gates/kernel"].to(DEV), grads[q + "candidate/kernel"].to(DEV)
        got = {"gk_in": gk[:HU], "gk_rec": gk[HU:], "ck_in": ck[:HU], "ck_rec": ck[HU:], "gb": grads[q + "gates/bias"].to(DEV),
               "cb": grads[q + "candidate/bias"].to(DEV)}
        for k, v in got.items():
            r, b = wg[(d, k)]
            ratios["%s_%s" % (k, n)] = check("%s_%s_%s" % (tag, k, n), v, r, b)
    record(tag + "_summary", **{"worst_" + k: v for k, v in ratios.items()})
