"""The Tacotron attention without encoder masking (mask_encoder=False: energies and softmax over every T_in position of the padded
batch) and without cumulative state (cumulative_weights=False: the location features read the previous step's alignments) on the
CUDA path, against the oracle (oracle/tacotron.py implements both; tests/test_attention_state_cpu.py pins it to the executed
reference).

End to end: training forward / backward, the per-step teacher-forcing path, Cfg-3 widths with the device's dropout / zoneout masks,
evaluation, GTA and free-running synthesis through the drop-in model, and a CUDA-graph replay, at the tolerances of
tests/test_tacotron_gpu.py and tests/test_teacher_forcing_gpu.py. One launch at a time: att_fwd_kernel (T2_DBG_TACO_ATT_FWD with the two
flags) and att_bwd_kernel (T2_DBG_TACO_ATT_BWD) for all four flag combinations against float64 references computed from the kernels'
exact inputs, with bounds of the form of tests/test_taco_kernels_gpu.py::test_att_fwd (TF32 on the location products)."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as Fn

from hparams import hparams
from oracle import tacotron as ot
from parity_util import record
from t2_import import t2

from test_tacotron_gpu import _trained_like_stats
from test_teacher_forcing_gpu import FWD_TOL, _batch, _check_draws, _compare, _hp, _oracle_step, _outputs, _run, _seed_where
from test_taco_kernels_gpu import BF, DEV, F64, NAN, TAN_ERR, U, att_reference, check, lens_for, nan_buf, tf32

pytestmark = pytest.mark.gpu

COMBOS = {"nomask": dict(mask_encoder=False), "nocum": dict(cumulative_weights=False),
          "both": dict(mask_encoder=False, cumulative_weights=False)}
ATT_FWD, ATT_BWD = 1, 7


def _pad_mask(lens, T_in):
    return torch.arange(T_in)[None, :] >= lens[:, None]


# ------------------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("combo", list(COMBOS))
def test_training_matches_oracle(combo):
    """forward, losses and every gradient, B = 3 with two rows shorter than T_in"""
    hp = _hp(**COMBOS[combo])
    B, T_in, T_out, M = 3, 40, 24, hp.num_mels
    params = ot.init_params(hp, seed=71, random_bias=True)
    batch = _batch(hp, B, T_in, T_out, 71)
    assert (batch[1] < T_in).sum() == 2
    model = _run(hp, params, batch, 1.0, 5)
    grads_ref, ref, parts = _oracle_step(params, *batch, hp, 1.0, None)
    _compare("tacotron_att_%s_B%d_Tin%d_Tout%d" % (combo, B, T_in, T_out), model, ref, parts, grads_ref, B, T_in, T_out, M, FWD_TOL)


def test_the_flags_change_the_results():
    """un-masked: alignment mass on the padded positions (exactly 0 when masked); non-cumulative: alignments differ by > 1e-3"""
    B, T_in, T_out, M = 3, 40, 24, 80
    params = ot.init_params(_hp(), seed=72, random_bias=True)
    batch = _batch(_hp(), B, T_in, T_out, 72)
    pad = _pad_mask(batch[1], T_in)
    al = {}
    for combo, flags in [("default", {})] + list(COMBOS.items()):
        model = _run(_hp(**flags), params, batch, 1.0, 5, backward=False)
        al[combo] = _outputs(model, B, T_in, T_out, M)["alignments"]          # [B, T_out, T_in]
        del model
    leak = {k: min(float(a[b][:, pad[b]].sum(-1).min()) for b in range(B) if pad[b].any()) for k, a in al.items()}
    on_pad = {k: max(float(a[b][:, pad[b]].abs().max()) for b in range(B) if pad[b].any()) for k, a in al.items()}
    nocum_diff = (al["nocum"] - al["default"]).abs().max().item()
    print("smallest padded mass per step:", leak, "non-cumulative vs cumulative max |d alpha|:", nocum_diff)
    record("tacotron_att_flags_effect", nomask_pad_mass=leak["nomask"], both_pad_mass=leak["both"], nocum_diff=nocum_diff)
    assert leak["nomask"] > 0 and leak["both"] > 0
    assert on_pad["default"] == 0 and on_pad["nocum"] == 0
    assert nocum_diff > 1e-3


def test_cfg3_stochastic_paths_with_both_flags():
    """Cfg-3 widths (B = 32, T_in = 160, T_out = 200), conv and prenet dropout 0.5, zoneout 0.1: the masks the kernels drew are
    rebuilt from the hash and injected into the oracle"""
    from test_parity_full_gpu import taco_batch, taco_masks
    hp = hparams.copy()
    hp.parse("predict_linear=False")
    hp.set_hparam("mask_encoder", False)
    hp.set_hparam("cumulative_weights", False)
    B, T_in, T_out, M = 32, 160, 200, hp.num_mels
    params = ot.init_params(hp, seed=73, random_bias=True)
    batch = taco_batch(hp, B, T_in, T_out, 73)
    assert (batch[1] < T_in).any()
    model = _run(hp, params, batch, 1.0, 99)
    masks = taco_masks(model, hp, B, T_in, T_out)
    grads_ref, ref, parts = _oracle_step(params, *batch, hp, 1.0, None, masks=masks)
    _compare("tacotron_att_both_cfg3_B32_Tin160_Tout200_stochastic", model, ref, parts, grads_ref, B, T_in, T_out, M, FWD_TOL)


@pytest.mark.parametrize("combo", ["nomask", "nocum"])
def test_teacher_forcing_ratio_half(combo):
    """the per-step decoder path (ratio < 1) with each flag, against oracle.forward(tf_ratio=, tf_draws=) with the device's draws"""
    hp = _hp(**COMBOS[combo])
    B, T_in, T_out, M = 3, 40, 24, hp.num_mels
    ratio = 0.5
    params = ot.init_params(hp, seed=74, random_bias=True)
    batch = _batch(hp, B, T_in, T_out, 74)
    seed = _seed_where(lambda c: 6 <= c.sum() <= len(c) - 6, T_out, ratio, start=4000)
    model = _run(hp, params, batch, ratio, seed)
    draws, choices = _check_draws(model, ratio, seed, T_out)
    assert 0 < int(choices[:-1].sum()) < T_out - 1
    grads_ref, ref, parts = _oracle_step(params, *batch, hp, ratio, draws)
    _compare("tacotron_att_%s_tf0.5" % combo, model, ref, parts, grads_ref, B, T_in, T_out, M, FWD_TOL)


@pytest.mark.parametrize("combo", list(COMBOS))
def test_synthesis_gta_and_evaluation_through_the_dropin_model(combo):
    """free running (TacoTestHelper), GTA and evaluation (inference batch norm, zoneout blend) through tacotron.models: the engines
    pick the flags up from the hparams"""
    from tacotron.models import create_model
    hp = _hp(tacotron_zoneout_rate=0.1, max_iters=24, **COMBOS[combo])
    B, T_in, T_out, M = 3, 40, 24, hp.num_mels
    params = _trained_like_stats(ot.init_params(hp, seed=75, random_bias=True), 75)
    params["stop_token_projection/bias"] = torch.full((1,), -6.0)        # never stops: runs to max_iters
    inputs, lens, mel, stop = _batch(hp, B, T_in, T_out, 75)
    m = create_model("Tacotron", hp)
    m.load_variables(params)
    m.initialize(inputs.cuda(), lens.cuda())
    eng = m._eng
    assert (eng.cfg.unmasked_encoder, eng.cfg.noncumulative_weights) == (int(not hp.mask_encoder), int(not hp.cumulative_weights))
    ref = ot.synthesize(params, inputs, lens, hp, max_iters=T_out)
    assert m.tower_mel_outputs[0].shape[1] == ref["mel_outputs"].shape[1] == T_out
    e_al = (m.tower_alignments[0].transpose(1, 2).cpu() - ref["alignments"]).abs().max().item()
    e_dec = (m.tower_decoder_output[0].cpu() - ref["decoder_output"]).abs().mean().item()
    e_mel = (m.tower_mel_outputs[0].cpu() - ref["mel_outputs"]).abs().mean().item()
    e_stop = (m.tower_stop_token_prediction[0].cpu() - ref["stop_token_prediction"]).abs().max().item()
    res = dict(synth_align=e_al, synth_dec_l1=e_dec, synth_mel_l1=e_mel, synth_stop=e_stop)
    assert e_al < 1e-4 and e_dec < 1e-3 and e_mel < 4e-3 and e_stop < 1e-4, res      # test_free_running_synthesis_matches_oracle
    with torch.no_grad():
        ref_tf = ot.forward(params, inputs, lens, mel, hp, training=False)
    for mode in ("gta", "eval"):
        if mode == "gta":
            m.initialize(inputs.cuda(), lens.cuda(), mel.cuda(), gta=True)
        else:
            m.initialize(inputs.cuda(), lens.cuda(), mel.cuda(), stop.cuda(), is_evaluating=True)
        torch.cuda.synchronize()
        e_al = (m.tower_alignments[0].transpose(1, 2).cpu() - ref_tf["alignments"]).abs().max().item()
        e_dec = (m.tower_decoder_output[0].cpu() - ref_tf["decoder_output"]).abs().mean().item()
        e_mel = (m.tower_mel_outputs[0].cpu() - ref_tf["mel_outputs"]).abs().mean().item()
        res.update({mode + "_align": e_al, mode + "_dec_l1": e_dec, mode + "_mel_l1": e_mel})
        assert e_al < FWD_TOL["align"] and e_dec < FWD_TOL["dec_l1"] and e_mel < FWD_TOL["mel_l1"], (mode, res)
    print(combo, res)
    record("tacotron_att_%s_synth_gta_eval" % combo, **res)


def test_cuda_graph_replay_equals_the_eager_step():
    """both flags, dropout 0.5 / zoneout 0.1: a replay of the captured pack + forward + backward against an eager step at the same
    device step counter. Losses within the fp32-reordering tolerance of test_tacotron_gpu.py, gradients within the batched path's
    run-to-run spread (test_teacher_forcing_gpu.py: the batch-norm statistics are fp32 atomic sums)"""
    hp = _hp(tacotron_dropout_rate=0.5, tacotron_zoneout_rate=0.1, mask_encoder=False, cumulative_weights=False)
    B, T_in, T_out = 3, 40, 24
    params = ot.init_params(hp, seed=76, random_bias=True)
    inputs, lens, mel, stop = [x.cuda() for x in _batch(hp, B, T_in, T_out, 76)]
    g = t2.tacotron.Tacotron(hp, B, T_in, T_out)
    g.load_params(params)
    graph = g.capture(inputs.int(), lens.int(), mel, stop)
    graph.replay()
    torch.cuda.synchronize()
    e = t2.tacotron.Tacotron(hp, B, T_in, T_out)
    e.load_params(params)
    e.step_dev.copy_(g.step_dev - 1)
    e.step_dev.add_(1)
    e.forward(inputs.int(), lens.int(), mel, stop)
    e.backward()
    torch.cuda.synchronize()
    assert torch.equal(e.step_dev, g.step_dev)
    lg, le = g.losses(), e.losses()
    ga, gb = g.export_grads(), e.export_grads()
    al_err = (g.workspace_tensor("alignments") - e.workspace_tensor("alignments")).abs().max().item()
    rel = lambda x, y: ((x - y).norm() / y.norm().clamp_min(1e-12)).item()
    cos = lambda x, y: ((x * y).sum() / (x.norm() * y.norm()).clamp_min(1e-20)).item()
    keys = [k for k in gb if gb[k].norm() > 1e-6 and not (k.endswith("/bias") and "conv_layer" in k)]
    worst = max(keys, key=lambda k: rel(ga[k], gb[k]))
    print("graph vs eager: losses", lg, le, "align", al_err, "worst", worst, rel(ga[worst], gb[worst]))
    record("tacotron_att_both_graph_vs_eager", align_max_err=al_err, worst_rel=rel(ga[worst], gb[worst]),
           worst_cos=min(cos(ga[k], gb[k]) for k in keys))
    for k in ("before", "after", "stop", "reg"):
        assert abs(lg[k] - le[k]) < 2e-3 + 1e-3 * abs(le[k]), (k, lg, le)
    assert al_err < FWD_TOL["align"]
    bad = [k for k in keys if rel(ga[k], gb[k]) > 0.15 or cos(ga[k], gb[k]) < 0.995]
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------------------------
# one launch at a time
# ------------------------------------------------------------------------------------------------------------------------------
def _launch(kernel, p, i):
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    c = t2.lib.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate(i):
        c.i[k] = int(v)
    t2.lib.check(lib.t2_dbg_taco_kernel(ctypes.byref(c), t2.lib.stream_ptr()))
    torch.cuda.synchronize()


FLAG_CASES = [(um, nc) for um in (0, 1) for nc in (0, 1)]
SHAPES = [(4, 17, 128, 31, 32, 1024, 512), (3, 160, 128, 31, 32, 1024, 512), (3, 336, 128, 31, 32, 1024, 512), (3, 40, 64, 1, 4, 256, 256)]


def _att_inputs(B, Ti, A, KA, F, D, C2, unmasked, seed):
    """random inputs in the engine's layouts; values rows past a length are zero (the encoder's outputs there are), keys past it are
    zero too when masked is off (memory_layer has no bias) and NaN when it is on (never read)"""
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor(lens_for(B, Ti), dtype=torch.int32)
    h2 = torch.randn(B, D + 8, generator=g).bfloat16()
    h2[:, D:] = NAN
    WqT = (torch.randn(A, D, generator=g) / math.sqrt(D)).bfloat16()
    K = torch.randn(KA, F, generator=g) * 0.5
    bK = torch.randn(F, generator=g) * 0.1
    Wl = torch.randn(F, A, generator=g) / math.sqrt(F)
    ba = torch.randn(A, generator=g) * 0.1
    v = torch.randn(A, generator=g) / math.sqrt(A) * 2
    keys = torch.randn(B, Ti, A, generator=g) * 0.5
    values = torch.randn(B, Ti, C2, generator=g).bfloat16()
    state = 0.05 + torch.rand(B, Ti, generator=g) * 1.5
    for b in range(B):
        keys[b, lens[b]:] = 0 if unmasked else NAN
        values[b, lens[b]:] = 0 if unmasked else NAN
    return [x.to(DEV) for x in (h2, WqT, K, bK, Wl, ba, v, keys, values, lens, state)]


@pytest.mark.parametrize("unmasked,noncum", FLAG_CASES)
@pytest.mark.parametrize("B,Ti,A,KA,F,D,C2", SHAPES)
def test_att_fwd_flags(B, Ti, A, KA, F, D, C2, unmasked, noncum):
    h2, WqT, K, bK, Wl, ba, v, keys, values, lens, state = _att_inputs(B, Ti, A, KA, F, D, C2, unmasked, B * 1000 + Ti + 7 * unmasked + noncum)
    Ub = nan_buf(((KA + 1) * A,), torch.float32)
    st_in = state.clone()
    alpha = nan_buf((B, Ti), torch.float32)
    ctx_a, ctx_b = nan_buf((B, C2 + 16), torch.bfloat16), nan_buf((B, C2 + 8), torch.bfloat16)
    _launch(ATT_FWD, [h2, WqT, K, bK, Wl, ba, Ub, v, keys, values, lens, state, alpha, ctx_a, ctx_b],
            [B, Ti, D, A, KA, F, C2, D + 8, C2 + 16, C2 + 8, unmasked, noncum])
    tag = "att_fwd_um%d_nc%d_B%d_Ti%d_A%d_KA%d" % (unmasked, noncum, B, Ti, A, KA)
    # un-masked: every score counts (reference lengths = T_in); the zero values rows past a length add nothing to the context
    ref_lens = torch.full_like(lens, Ti) if unmasked else lens
    ref_a, d_a, ref_c, d_c, valid = att_reference(h2[:, :D], WqT, Ub.view(KA + 1, A), KA, v, keys, values, ref_lens, st_in)
    check(tag + "_alpha", torch.where(valid, alpha, torch.zeros_like(alpha)), ref_a, d_a + 1e-30)
    pad = ~(torch.arange(Ti, device=DEV)[None, :] < lens[:, None])
    if unmasked:
        assert bool((alpha[pad] > 0).all()), "un-masked: every padded position gets weight"
    else:
        assert bool((alpha[pad] == 0).all()), "masked: alpha past len must be exactly 0"
    want_state = alpha if noncum else st_in + alpha
    assert torch.equal(state, want_state), "state must come back as alpha (non-cumulative) or cum + alpha"
    check(tag + "_ctx", ctx_b[:, :C2], ref_c, d_c + 1e-30)
    assert torch.equal(ctx_a[:, :C2], ctx_b[:, :C2])


def _att_bwd_reference(h, WqT, Ub, KA, v, keys, values, lens, alpha, prev, dstate, dPI, dctxl, unmasked, cumulative):
    """float64 gradients of one attention step on the kernel's inputs (prev = the state the step read, alpha = its alignments) and
    first-order bounds. dE = d loss / d (keys + q + pl), with pl through the TF32 location products as the kernel computes them."""
    B, Ti, A = keys.shape
    D, C2 = WqT.shape[1], values.shape[2]
    half = KA // 2
    live = torch.arange(Ti, device=DEV)[None, :] < lens[:, None]
    ev = torch.ones_like(live) if unmasked else live                      # positions with an energy
    q = h.to(F64) @ WqT.to(F64).t()
    qabs = h.to(F64).abs() @ WqT.to(F64).abs().t()
    Ut = tf32(Ub).to(F64)
    win = Fn.pad(tf32(prev).to(F64), (half, half)).unfold(1, KA, 1)
    pl = win @ Ut[:KA] + Ut[KA]
    P = win.abs() @ Ut[:KA].abs() + Ut[KA].abs()
    ky = torch.where(ev[..., None], keys.to(F64), torch.zeros((), dtype=F64, device=DEV))
    arg = ky + q[:, None, :] + pl
    d_arg = 2 * (KA + 1) * U * P + 2 * (D / 32 + 8) * U * qabs[:, None, :] + 2 * U * arg.abs()
    t = torch.tanh(arg)
    d_t = (1 - t * t) * d_arg + TAN_ERR
    v64, al = v.to(F64), alpha.to(F64)
    vals = torch.where(live[..., None], values.to(F64), torch.zeros((), dtype=F64, device=DEV))
    dctx32 = dPI[:, D:D + C2] + dctxl                                    # fp32, as the kernel adds them
    dctx = dctx32.to(F64)
    ds = dstate.to(F64)
    da = torch.einsum("bjc,bc->bj", vals, dctx) + ds
    da_abs = torch.einsum("bjc,bc->bj", vals.abs(), dctx.abs()) + ds.abs()
    d_da = 2 * (C2 / 8 + 16) * U * da_abs
    al_e = torch.where(ev, al, torch.zeros_like(al))
    dot = (al_e * da).sum(1, keepdim=True)
    de = al_e * (da - dot)
    de_abs = al_e * (da_abs + (al_e * da_abs).sum(1, keepdim=True))
    d_de = al_e * (d_da + (al_e * d_da).sum(1, keepdim=True)) + 2 * (Ti + 16) * U * de_abs
    s = 1 - t * t
    dE = de[..., None] * v64 * s
    dE_abs = de_abs[..., None] * v64.abs() * s
    d_dE = d_de[..., None] * v64.abs() * s + de.abs()[..., None] * v64.abs() * 2 * t.abs() * d_t + 4 * U * dE_abs
    n_sum = 2 * (Ti + 40) * U
    out, bnd = {}, {}
    out["dq"] = dE.sum(1)
    bnd["dq"] = d_dE.sum(1) + n_sum * dE_abs.sum(1)
    out["dv"] = (de[..., None] * t).sum(1)
    bnd["dv"] = (d_de[..., None] * t.abs() + de.abs()[..., None] * d_t).sum(1) + n_sum * (de_abs[..., None] * t.abs()).sum(1)
    out["dkeys"] = dE
    bnd["dkeys"] = d_dE
    # TF32 products: operands rounded with rna (relative 2^-11 each); the state operand is rounded exactly as here, dE may round
    # differently when it is perturbed, hence the 2^-10 margin on top of its own error
    tE, tE_abs = dE, dE_abs
    d_tE = d_dE + 2.0 ** -10 * dE_abs
    winT = win                                                          # [B, Ti, KA] tf32(prev)[j + k - half]
    out["dU"] = torch.einsum("bjk,bjc->bkc", winT, tE)
    bnd["dU"] = torch.einsum("bjk,bjc->bkc", winT.abs(), d_tE) + n_sum * torch.einsum("bjk,bjc->bkc", winT.abs(), tE_abs)
    # d prev[i] = sum_k sum_c dE[i - k + half][c] U[k][c]
    Pm = tE @ Ut[:KA].t()                                               # [B, Ti, KA]
    Pm_b = d_tE @ Ut[:KA].abs().t() + 2 * (A + 16) * U * (tE_abs @ Ut[:KA].abs().t()) + 2.0 ** -10 * (tE_abs @ Ut[:KA].abs().t())
    dprev = torch.zeros(B, Ti, dtype=F64, device=DEV)
    dprev_b = torch.zeros_like(dprev)
    for k in range(KA):
        # position j, tap k feeds prev[j + k - half]
        lo, hi = max(0, half - k), min(Ti, Ti + half - k)
        dprev[:, lo + k - half:hi + k - half] += Pm[:, lo:hi, k]
        dprev_b[:, lo + k - half:hi + k - half] += Pm_b[:, lo:hi, k]
    if cumulative:
        dprev = dprev + ds
        dprev_b = dprev_b + ds.abs() * 2 * U
    out["dprev"], bnd["dprev"] = dprev, dprev_b + 2 * KA * U * dprev.abs()
    Wt = WqT.to(F64)
    out["dh2ext"] = dPI[:, :D].to(F64) + out["dq"] @ Wt
    bnd["dh2ext"] = bnd["dq"] @ Wt.abs() + 2 * (A + 4) * U * (out["dq"].abs() @ Wt.abs() + dPI[:, :D].abs().to(F64))
    out["dctx"], bnd["dctx"] = dctx, BF * dctx.abs() + 1e-30
    return out, bnd, live, ev


@pytest.mark.parametrize("unmasked,noncum", FLAG_CASES)
@pytest.mark.parametrize("B,Ti,A,KA,F,D,C2", SHAPES)
def test_att_bwd(B, Ti, A, KA, F, D, C2, unmasked, noncum):
    h2, WqT, K, bK, Wl, ba, v, keys, values, lens, state = _att_inputs(B, Ti, A, KA, F, D, C2, unmasked, B * 2000 + Ti + 7 * unmasked + noncum)
    g = torch.Generator().manual_seed(Ti * 3 + KA + unmasked * 2 + noncum)
    # the forward of the step gives the alignments the backward reads, and the merged filter bank
    Ub = nan_buf(((KA + 1) * A,), torch.float32)
    prev = state.clone()
    st = state.clone()
    alpha = nan_buf((B, Ti), torch.float32)
    ctx = nan_buf((B, C2), torch.bfloat16)
    _launch(ATT_FWD, [h2, WqT, K, bK, Wl, ba, Ub, v, keys, values, lens, st, alpha, None, ctx],
            [B, Ti, D, A, KA, F, C2, D + 8, C2, C2, unmasked, noncum])
    ld_dPI = D + C2 + 4
    dPI = torch.randn(B, ld_dPI, generator=g).to(DEV)
    dPI[:, D + C2:] = NAN
    dctxl = (torch.randn(B, C2, generator=g) * 0.5).to(DEV)
    dctxl_in = dctxl.clone()
    dstate = (torch.randn(B, Ti, generator=g) * 0.3).to(DEV)
    dstate_in = dstate.clone()
    dh2ext = nan_buf((B, D), torch.float32)
    dsave = nan_buf((B * C2 + B * A,), torch.bfloat16)
    dkeys0 = (torch.randn(B, Ti, A, generator=g) * 0.01).to(DEV)
    dkeys = dkeys0.clone()
    acc0 = (torch.randn(B, KA + 2, A, generator=g) * 0.01).to(DEV)
    acc = acc0.clone()
    state_arg = prev if noncum else st.clone()         # non-cumulative: alpha_{t-1}; cumulative: cum_t (in), cum_{t-1} (out)
    cum_t = state_arg.clone()
    _launch(ATT_BWD, [h2, WqT, Ub, v, keys, values, lens, alpha, state_arg, dstate, dPI, dctxl, dh2ext, dsave, dkeys, acc],
            [B, Ti, D, A, KA, C2, D + 8, ld_dPI, unmasked, noncum])
    tag = "att_bwd_um%d_nc%d_B%d_Ti%d_A%d_KA%d" % (unmasked, noncum, B, Ti, A, KA)
    if noncum:
        assert torch.equal(state_arg, prev), "the non-cumulative state is read only"
    else:
        assert torch.equal(state_arg, cum_t - alpha), "cum_{t-1} = cum_t - alpha_t"
    assert bool((dctxl == 0).all()), "dctxl is cleared for the next step's split-K accumulation"
    ref, bnd, live, ev = _att_bwd_reference(h2[:, :D], WqT, Ub.view(KA + 1, A), KA, v, keys, values, lens, alpha,
                                            state_arg if not noncum else prev, dstate_in, dPI, dctxl_in, unmasked, not noncum)
    check(tag + "_dh2ext", dh2ext, ref["dh2ext"], bnd["dh2ext"] + 1e-30)
    check(tag + "_dctx", dsave[:B * C2].view(B, C2), ref["dctx"], bnd["dctx"])
    check(tag + "_dq", dsave[B * C2:].view(B, A), ref["dq"], bnd["dq"] + BF * ref["dq"].abs() + 1e-30)
    dk = torch.where(ev[..., None], dkeys - dkeys0, torch.zeros_like(dkeys))
    check(tag + "_dkeys", dk, ref["dkeys"], bnd["dkeys"] + 2 * U * dkeys.abs().to(F64) + 1e-30)
    assert torch.equal(dkeys[~ev], dkeys0[~ev]), "dkeys past the energies must be untouched"
    accd = (acc - acc0).to(F64)
    sl = 2 * U * acc.abs().to(F64)
    check(tag + "_dU", accd[:, :KA], ref["dU"], bnd["dU"] + sl[:, :KA] + 1e-30)
    check(tag + "_du0", accd[:, KA], ref["dq"], bnd["dq"] + sl[:, KA] + 1e-30)
    check(tag + "_dv", accd[:, KA + 1], ref["dv"], bnd["dv"] + sl[:, KA + 1] + 1e-30)
    check(tag + "_dstate", dstate, ref["dprev"], bnd["dprev"] + 1e-30)
    if unmasked:
        assert bool((dk[~live.unsqueeze(-1).expand_as(dk)] != 0).any()), "un-masked: the padded keys get gradient"


def test_att_bwd_reference_is_float64_autograd():
    """the explicit float64 formulas of _att_bwd_reference equal torch.autograd through one attention step (softmax alignments,
    location features from the previous state, the next state) for every flag combination, on small random inputs"""
    B, Ti, A, KA, D, C2 = 2, 11, 64, 5, 32, 64
    g = torch.Generator().manual_seed(3)
    for unmasked in (0, 1):
        for cumulative in (0, 1):
            lens = torch.tensor([Ti, 6], dtype=torch.int32, device=DEV)
            h = torch.randn(B, D, generator=g).bfloat16().to(DEV)
            WqT = torch.randn(A, D, generator=g).bfloat16().to(DEV) * 0.2
            Ub = tf32(torch.randn(KA + 1, A, generator=g) * 0.3).to(DEV)
            v = torch.randn(A, generator=g).to(DEV)
            keys = torch.randn(B, Ti, A, generator=g).to(DEV)
            values = torch.randn(B, Ti, C2, generator=g).bfloat16().to(DEV)
            values[1, 6:] = 0
            keys[1, 6:] = 0
            prev = tf32(torch.rand(B, Ti, generator=g)).to(DEV)
            dstate = torch.randn(B, Ti, generator=g).to(DEV)
            dPI = torch.randn(B, D + C2, generator=g).to(DEV)
            dctxl = torch.zeros(B, C2, device=DEV)
            live = torch.arange(Ti, device=DEV)[None, :] < lens[:, None]
            hq = h.to(F64).requires_grad_(True)
            ky = keys.to(F64).requires_grad_(True)
            U64 = Ub.to(F64).requires_grad_(True)
            v64 = v.to(F64).requires_grad_(True)
            pv = prev.to(F64).requires_grad_(True)
            q = hq @ WqT.to(F64).t()
            win = Fn.pad(pv, (KA // 2, KA // 2)).unfold(1, KA, 1)
            e = torch.tanh(ky + q[:, None, :] + win @ U64[:KA] + U64[KA]) @ v64
            if not unmasked:
                e = torch.where(live, e, torch.full_like(e, -math.inf))
            a = torch.softmax(e, 1)
            ctx = torch.einsum("bj,bjc->bc", a, values.to(F64))
            new_state = pv + a if cumulative else a
            loss = (ctx * dPI[:, D:].to(F64)).sum() + (new_state * dstate.to(F64)).sum()
            gq, gk, gU, gv, gp = torch.autograd.grad(loss, [hq, ky, U64, v64, pv])
            out, _, _, ev = _att_bwd_reference(h, WqT, Ub, KA, v, keys, values, lens, a.detach().float(), prev, dstate, dPI, dctxl,
                                               unmasked, cumulative)
            # the step's alignments enter the explicit formulas rounded to fp32, as the kernel reads them
            tol = lambda x: 1e-5 * (1 + x.abs().max().item())
            assert (out["dkeys"] - torch.where(ev[..., None], gk, torch.zeros_like(gk))).abs().max() <= tol(gk)
            assert (out["dU"].sum(0) - gU[:KA]).abs().max() <= tol(gU) and (out["dq"].sum(0) - gU[KA]).abs().max() <= tol(gU)
            assert (out["dv"].sum(0) - gv).abs().max() <= tol(gv)
            assert (out["dprev"] - gp).abs().max() <= tol(gp)
            assert (out["dh2ext"] - dPI[:, :D].to(F64) - gq).abs().max() <= tol(gq)
