"""The float64 GRU references of tests/gru_reference.py without a GPU: pinned to oracle.tacotron.gru_cell and to float64 autograd, shown to
be tight enough that each of a list of plausible kernel faults leaves the bound, and the GRU test hooks' argument checks (they run before
any driver call, so the pointers passed here are never dereferenced)."""
import ctypes

import pytest
import torch

import gru_reference as gr
from hparams import hparams
from oracle import tacotron as ot
from t2_import import t2

F64 = torch.float64
HU, RU = 128, 128
DIRS = ("forward", "backward")


def _weights(seed, gate_bias=None, scale=1.0):
    hp = hparams.copy()
    hp.parse("predict_linear=True")
    p = ot.init_params(hp, seed=seed, random_bias=gate_bias is None)
    Ws = []
    for n in DIRS:
        q = "CBHG_postnet/%s_RNN/" % n
        W = dict(gk=p[q + "gates/kernel"] * scale, gb=p[q + "gates/bias"], ck=p[q + "candidate/kernel"] * scale, cb=p[q + "candidate/bias"])
        if gate_bias is not None:
            W["gb"] = torch.full_like(W["gb"], gate_bias)
        Ws.append(W)
    return Ws


def _rounded_weights(Ws):
    """the kernels' view: recurrent rows in bf16, input rows and biases as given"""
    out = []
    for W in Ws:
        gk, ck = W["gk"].clone().double(), W["ck"].clone().double()
        gk[HU:], ck[HU:] = gr.bf16(W["gk"][HU:]), gr.bf16(W["ck"][HU:])
        out.append(dict(gk=gk, gb=W["gb"].double(), ck=ck, cb=W["cb"].double()))
    return out


def _exact_bigru(x, Ws):
    """float64 bidirectional GRU through oracle.tacotron.gru_cell (autograd-capable): x [B, T, HU] -> [B, T, 2RU]"""
    B, T, _ = x.shape
    outs = []
    for d in range(2):
        W = Ws[d]
        st = torch.zeros(B, RU, dtype=F64)
        seq = [None] * T
        for t in (range(T) if d == 0 else range(T - 1, -1, -1)):
            st = ot.gru_cell(x[:, t], st, W["gk"], W["gb"], W["ck"], W["cb"])
            seq[t] = st
        outs.append(torch.stack(seq, 1))
    return torch.cat(outs, -1)


def _xp(x, Ws):
    """the input projections [B, T, 6RU] (no biases) of x [B, T, HU]"""
    return torch.cat([torch.cat([x @ W["gk"][:HU], x @ W["ck"][:HU]], -1) for W in Ws], -1)


def test_forward_reference_is_the_oracle_gru_cell():
    g = torch.Generator().manual_seed(1)
    Ws = _rounded_weights(_weights(3))
    x = torch.randn(3, 11, HU, generator=g, dtype=F64)
    ref = _exact_bigru(x, Ws)
    res = gr.forward(_xp(x, Ws), Ws, HU)
    assert (res["out"] - ref).abs().max().item() < 1e-12
    # re-anchored on the exact states, every step reproduces them
    res_a = gr.forward(_xp(x, Ws), Ws, HU, anchor=ref)
    assert (res_a["out"] - ref).abs().max().item() < 1e-12


def _autograd_case(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    Ws = [{k: v.clone().requires_grad_(True) for k, v in W.items()} for W in _rounded_weights(_weights(seed))]
    x = torch.randn(B, T, HU, generator=g, dtype=F64).requires_grad_(True)
    dout = torch.randn(B, T, 2 * RU, generator=g, dtype=F64)
    return Ws, x, dout


def test_bptt_reference_is_float64_autograd():
    """dXP of the BPTT formulas, fed the float64 forward's unrounded states and stashes, equals autograd's d loss / d pre-activations"""
    Ws, x, dout = _autograd_case(3, 9, 4)
    XP = _xp(x.detach(), Ws).detach().requires_grad_(True)
    Wd = [{k: v.detach() for k, v in W.items()} for W in Ws]
    # the same recurrence, written on the pre-activations so that autograd yields their gradients
    B, T, _ = x.shape
    outs = []
    for d in range(2):
        W = Wd[d]
        h = torch.zeros(B, RU, dtype=F64)
        seq = [None] * T
        for t in (range(T) if d == 0 else range(T - 1, -1, -1)):
            o = d * 3 * RU
            ru = torch.sigmoid(XP[:, t, o:o + 2 * RU] + W["gb"] + h @ W["gk"][HU:])
            r, u = ru[:, :RU], ru[:, RU:]
            c = torch.tanh(XP[:, t, o + 2 * RU:o + 3 * RU] + W["cb"] + (r * h) @ W["ck"][HU:])
            h = u * h + (1 - u) * c
            seq[t] = h
        outs.append(torch.stack(seq, 1))
    out = torch.cat(outs, -1)
    (out * dout).sum().backward()
    res = gr.forward(XP.detach(), Wd, HU)
    assert (res["out"] - out.detach()).abs().max().item() < 1e-12
    dXP, bnd = gr.bptt(dout, res["out"], res["r"], res["u"], res["c"], Wd, HU)
    assert (dXP - XP.grad).abs().max().item() < 1e-12 * max(1.0, XP.grad.abs().max().item())
    assert torch.isfinite(bnd).all()


def test_weight_gradient_reference_is_float64_autograd():
    """input / recurrent row blocks of both kernels and both biases from h_last, dXP, out and r h equal autograd through the oracle cell"""
    Ws, x, dout = _autograd_case(4, 7, 5)
    out = _exact_bigru(x, Ws)
    (out * dout).sum().backward()
    Wd = [{k: v.detach() for k, v in W.items()} for W in Ws]
    res = gr.forward(_xp(x.detach(), Wd), Wd, HU)
    dXP, _ = gr.bptt(dout, res["out"], res["r"], res["u"], res["c"], Wd, HU)
    wg = gr.weight_grads(x.detach(), dXP, res["out"], res["rh"], HU)
    for d in range(2):
        got = {"gk_in": Ws[d]["gk"].grad[:HU], "gk_rec": Ws[d]["gk"].grad[HU:], "ck_in": Ws[d]["ck"].grad[:HU],
               "ck_rec": Ws[d]["ck"].grad[HU:], "gb": Ws[d]["gb"].grad, "cb": Ws[d]["cb"].grad}
        for k, v in got.items():
            ref, _ = wg[(d, k)]
            assert (ref - v).abs().max().item() < 1e-11 * max(1.0, v.abs().max().item()), (d, k)


# ---- sensitivity: each fault leaves the bound ----------------------------------------------------------------------------------
_CASES = {}


def _case(B, T):
    """clean reference of one (B, T) case: forward re-anchored on its own bf16 out, the kernel's bf16 stashes, BPTT and gradients"""
    if (B, T) not in _CASES:
        g = torch.Generator().manual_seed(B * 1000 + T)
        Ws = _weights(7, gate_bias=1.0)
        XP = torch.randn(B, T, 6 * RU, generator=g)
        exact = gr.forward(XP, Ws, HU)
        out = gr.bf16(exact["out"])
        st = {k: [gr.bf16(exact[k][d]) for d in range(2)] for k in ("r", "u", "c", "rh")}
        dout = torch.randn(B, T, 2 * RU, generator=g) * 0.01
        dXP, dXP_b = gr.bptt(dout, out, st["r"], st["u"], st["c"], Ws, HU)
        h_last = gr.bf16(torch.randn(B, T, HU, generator=g))
        wg = gr.weight_grads(h_last, gr.bf16(dXP), out, st["rh"], HU)
        _CASES[(B, T)] = dict(Ws=Ws, XP=XP, out=out, st=st, dout=dout, dXP=dXP, dXP_b=dXP_b, h_last=h_last, wg=wg)
    return _CASES[(B, T)]


def _leaves(got, ref, bound):
    return ((got.double() - ref).abs() / bound).max().item()


@pytest.mark.parametrize("B,T", [(5, 37), (32, 800)])
@pytest.mark.parametrize("fault", ["swap_ru", "no_gate_bias", "carry_items"])
def test_forward_faults_leave_the_bound(B, T, fault):
    c = _case(B, T)
    bad_out = gr.bf16(gr.forward(c["XP"], c["Ws"], HU, fault=fault)["out"])     # what a faulty kernel would store
    ref = gr.forward(c["XP"], c["Ws"], HU, anchor=bad_out)                           # the check: each step from the kernel's own out
    assert _leaves(bad_out, ref["out"], ref["out_b"]) > 1
    good = gr.forward(c["XP"], c["Ws"], HU, anchor=c["out"])
    assert _leaves(c["out"], good["out"], good["out_b"]) <= 1                         # and the fault-free kernel stays inside


def _late_step_fault(dXP, T):
    """the dXP of the step each direction processes halfway through (fw t = T/2, bw t = T - 1 - T/2) scaled by 1.5"""
    bad = dXP.clone()
    s = T // 2
    bad[:, s, :3 * RU] *= 1.5
    bad[:, T - 1 - s, 3 * RU:] *= 1.5
    return bad


@pytest.mark.parametrize("B,T", [(5, 37), (32, 800)])
@pytest.mark.parametrize("fault", ["bw_off", "no_drh_r", "late_step"])
def test_bptt_faults_leave_the_bound(B, T, fault):
    """the check of the GPU tests: a float64 BPTT re-anchored on the (here: faulty) kernel's own dXP"""
    c = _case(B, T)
    st = c["st"]
    args = (c["dout"], c["out"], st["r"], st["u"], st["c"], c["Ws"], HU)
    if fault == "late_step":
        bad = gr.bf16(_late_step_fault(c["dXP"], T))
    else:
        bad = gr.bf16(gr.bptt(*args, fault=fault)[0])
    ref, bnd = gr.bptt(*args, anchor=bad)
    assert _leaves(bad, ref, bnd) > 1
    good = gr.bf16(c["dXP"])
    ref, bnd = gr.bptt(*args, anchor=good)
    assert _leaves(good, ref, bnd) <= 1


@pytest.mark.parametrize("B,T", [(5, 37), (32, 800)])
def test_bptt_anchored_bound_does_not_decay_with_the_step(B, T):
    """re-anchored on the kernel's dXP, the bound does not grow with the step index: the median bound / |dXP| of each time step (over
    items, units and both directions) is below 2^-3 at every step (0.011 to 0.065 here at both shapes; carried without anchoring
    through all steps the median is 1.5e4 at T = 37 and 3e32 at T = 800)"""
    c = _case(B, T)
    st = c["st"]
    ref, bnd = gr.bptt(c["dout"], c["out"], st["r"], st["u"], st["c"], c["Ws"], HU, anchor=gr.bf16(c["dXP"]))
    rel = (bnd / (ref.abs() + 1e-30)).transpose(0, 1).reshape(T, -1)
    per_step = rel.median(1).values
    assert per_step.max().item() < 2 ** -3, per_step.max().item()


@pytest.mark.parametrize("B,T", [(5, 37), (32, 800)])
@pytest.mark.parametrize("fault", ["shift_flip", "boundary"])
def test_weight_gradient_faults_leave_the_bound(B, T, fault):
    c = _case(B, T)
    bad = gr.weight_grads(c["h_last"], gr.bf16(c["dXP"]), c["out"], c["st"]["rh"], HU, fault=fault)
    worst = max(_leaves(bad[(d, "gk_rec")][0], *c["wg"][(d, "gk_rec")]) for d in range(2))
    assert worst > 1


# ---- hook argument checks --------------------------------------------------------------------------------------------------------
def _hook(kernel, p, i):
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    c = t2.lib.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = v
    for k, v in enumerate(i):
        c.i[k] = v
    return lib.t2_dbg_cbhg_kernel(ctypes.byref(c), None), lib.t2_last_error()


FWD_I = [5, 37, HU, RU, 0, 1000, 2000, 3000, 4000, 5000, 6000, 7000]
BWD_I = [5, 37, HU, RU, 0, 1000, 4000, 5000]


@pytest.mark.parametrize("kernel,n_p,ints", [(7, 11, FWD_I), (8, 10, BWD_I)])
def test_gru_hooks_check_their_arguments_before_any_launch(kernel, n_p, ints):
    ptrs = [16 * (k + 1) for k in range(n_p)]                  # never dereferenced: the checks come first
    rng = b"must be in [1, 2^20]"
    for k, v, msg in ((3, 64, b"RU must be 128"), (0, 0, rng), (1, 0, rng), (2, 0, rng), (0, -(2 ** 32) + 5, rng), (1, 2 ** 32 + 37, rng)):
        bad = list(ints)
        bad[k] = v
        rc, err = _hook(kernel, ptrs, bad)
        assert rc != 0 and msg in err, (k, v, rc, err)
    for k in range(n_p):
        p = list(ptrs)
        p[k] = None
        rc, err = _hook(kernel, p, ints)
        if kernel == 7 and k >= 3:
            assert rc != 0 and b"all present or all null" in err, (k, err)        # one missing stash: a partial group
        else:
            assert rc != 0 and b"null" in err, (k, err)
    if kernel == 7:
        rc, err = _hook(kernel, ptrs[:3] + [None] * 4 + ptrs[7:], ints)            # fw stashes absent, bw present
        assert rc != 0 and b"all present or all null" in err
