"""Training at a teacher-forcing ratio below 1 ('constant' mode, helpers.py:115-128): at the end of every decoder step ONE uniform draw
(hash stream 40, element t) decides whether step t + 1 consumes the target frame or the raw frame step t just predicted, and the loss
back-propagates through the fed-back frames. The CUDA engine runs that path step by step; oracle.tacotron.forward(tf_ratio=, tf_draws=)
runs it on the CPU with the draws the device made, and autograd gives the reference gradients.

Tolerances are those of tests/test_tacotron_gpu.py (forward: test_forward_matches_oracle; gradients: test_backward_matches_oracle,
cos >= 0.97 and rel <= 0.25, 0.9 / 0.5 for conv biases in front of a batch norm) and, at Cfg-3 widths, of
tests/test_parity_full_gpu.py."""
import math

import numpy as np
import pytest
import torch

from hparams import hparams
from oracle import tacotron as ot
from t2_import import t2
from parity_util import record

import mask_hash as mh

pytestmark = pytest.mark.gpu

TF_STREAM = 40
FWD_TOL = dict(align=6e-4, dec_l1=1.6e-3, mel_l1=4e-2, stop=5e-3, loss=2e-3)


def _hp(**kw):
    hp = hparams.copy()
    hp.parse("predict_linear=False,tacotron_dropout_rate=0.0,tacotron_zoneout_rate=0.0,enc_conv_channels=256,embedding_dim=256,"
             "encoder_lstm_units=128,decoder_lstm_units=256,postnet_channels=256,prenet_layers=[128,128],attention_dim=128")
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


def _batch(hp, B, T_in, T_out, seed):
    g = torch.Generator().manual_seed(seed)
    inputs = torch.randint(2, 66, (B, T_in), generator=g)
    lens = torch.tensor([T_in] + [max(T_in - 7 * (i + 1), 3) for i in range(B - 1)])
    for b in range(B):
        inputs[b, lens[b]:] = 0
    mel = (torch.randn(B, T_out, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    stop = torch.zeros(B, T_out)
    stop[:, -3:] = 1
    return inputs, lens, mel, stop


def _host_choices(seed, T_out, ratio):
    """the choices a forward under `seed` (+ device step 0) makes, from the host copy of the hash"""
    u = mh.hash_uniform32(mh.hash_seed(seed, TF_STREAM), np.arange(T_out, dtype=np.uint64))
    return u < np.float32(ratio)


def _seed_where(pred, T_out, ratio, start=1000):
    for s in range(start, start + 100000):
        c = _host_choices(s, T_out, ratio)[:T_out - 1]       # the last draw feeds no step
        if pred(c):
            return s
    raise AssertionError("no seed found")


def _oracle_step(params, inputs, lens, mel, stop, hp, ratio, draws, masks=None):
    ps = {k: (v.clone().requires_grad_(True) if ot.is_trainable(k) else v.clone()) for k, v in params.items()}
    out = ot.forward(ps, inputs, lens, mel, hp, True, masks, tf_ratio=ratio, tf_draws=draws)
    loss, parts = ot.loss_fn(out, mel, stop, ps, hp)
    names = [k for k in ps if ot.is_trainable(k)]
    gr = torch.autograd.grad(loss, [ps[k] for k in names], allow_unused=True)
    grads = {k: (g if g is not None else torch.zeros_like(ps[k])) for k, g in zip(names, gr)}
    return grads, {k: v.detach() for k, v in out.items()}, {k: v.detach() for k, v in parts.items()}


def _run(hp, params, batch, ratio, seed, backward=True):
    inputs, lens, mel, stop = batch
    B, T_in = inputs.shape
    T_out = mel.shape[1]
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out, teacher_forcing_ratio=ratio)
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=True, seed=seed)
    if backward:
        model.backward()
    torch.cuda.synchronize()
    return model


def _outputs(model, B, T_in, T_out, M):
    return dict(alignments=model.workspace_tensor("alignments", (T_out, B, T_in)).float().cpu().transpose(0, 1).clone(),
                decoder_output=model.workspace_tensor("decoder_output", (B, T_out, M)).cpu().clone(),
                mel_outputs=model.workspace_tensor("mel_outputs", (B, T_out, M)).cpu().clone(),
                stop_logits=model.workspace_tensor("stop_logits", (B, T_out)).cpu().clone())


def _check_draws(model, ratio, seed, T_out):
    draws = model.rng_uniform(TF_STREAM, T_out).cpu()
    choices = model.teacher_forcing_choices().cpu()
    assert torch.equal(choices, draws < ratio), (choices, draws)
    assert np.array_equal(choices.numpy(), _host_choices(seed, T_out, ratio))
    return draws, choices


def _compare(tag, model, ref, parts, grads_ref, B, T_in, T_out, M, tol, grad_tol=(0.25, 0.97)):
    out = _outputs(model, B, T_in, T_out, M)
    los = model.losses()
    m = dict(align_max_err=(out["alignments"] - ref["alignments"]).abs().max().item(),
             dec_l1=(out["decoder_output"] - ref["decoder_output"]).abs().mean().item(),
             mel_l1=(out["mel_outputs"] - ref["mel_outputs"]).abs().mean().item(),
             stop_max=(out["stop_logits"] - ref["stop_logits"]).abs().max().item())
    for k in ("before", "after", "stop", "reg"):
        m["loss_%s_err" % k] = abs(los[k] - parts[k].item())
    grads = model.export_grads()
    bad, rels, coss = [], [], []
    for name, g_ref in grads_ref.items():
        g = grads[name]
        den = g_ref.norm().item()
        rel = (g - g_ref).norm().item() / max(den, 1e-12)
        cos = (g * g_ref).sum().item() / max(den * g.norm().item(), 1e-20)
        noise_floor = name.endswith("/bias") and "conv_layer" in name
        rel_tol, cos_tol = (0.5, 0.9) if noise_floor else grad_tol
        if den >= 1e-6 and not noise_floor:
            rels.append(rel); coss.append(cos)
        if den >= 1e-6 and (rel >= rel_tol or cos < cos_tol):
            bad.append("%-60s rel %.4g cos %.4f |ref| %.3g |cuda| %.3g" % (name, rel, cos, den, g.norm().item()))
    m["grad_worst_rel"], m["grad_worst_cos"] = max(rels), min(coss)
    print(tag, m)
    record(tag, **m)
    assert m["align_max_err"] < tol["align"] and m["dec_l1"] < tol["dec_l1"] and m["mel_l1"] < tol["mel_l1"], m
    assert m["stop_max"] < tol["stop"], m
    for k in ("before", "after", "stop", "reg"):
        assert m["loss_%s_err" % k] < tol["loss"] + 1e-3 * abs(parts[k].item()), (k, m)
    assert not bad, "gradient mismatch:\n" + "\n".join(bad)
    return grads


@pytest.mark.parametrize("ratio", [0.5, 0.0])
def test_feedback_training_matches_oracle(ratio):
    """forward, losses and every gradient at ratio 0.5 (draws that mix both inputs) and 0 (every step after the first consumes the
    previous prediction). The prenet, its LSTM-1 input projection and the embedding get gradient through the fed-back frames too."""
    hp = _hp()
    B, T_in, T_out, M = 3, 40, 24, hp.num_mels
    params = ot.init_params(hp, seed=61, random_bias=True)
    batch = _batch(hp, B, T_in, T_out, 61)
    seed = _seed_where(lambda c: 6 <= c.sum() <= len(c) - 6, T_out, ratio) if ratio > 0 else 7
    model = _run(hp, params, batch, ratio, seed)
    draws, choices = _check_draws(model, ratio, seed, T_out)
    if ratio == 0.0:
        assert not choices.any()
    else:
        assert 0 < int(choices[:-1].sum()) < T_out - 1
    grads_ref, ref, parts = _oracle_step(params, *batch, hp, ratio, draws)
    _compare("tacotron_tf%g_B%d_Tin%d_Tout%d" % (ratio, B, T_in, T_out), model, ref, parts, grads_ref, B, T_in, T_out, M, FWD_TOL)


def test_draws_that_change_the_input_change_the_gradients():
    """the feedback term is real: at a seed whose draws mix both choices the prenet, LSTM-1 and projection gradients differ from the
    teacher-forced ones by more than 10 % (the bf16 difference to the oracle is 2-15 %, test_feedback_training_matches_oracle)"""
    hp = _hp()
    B, T_in, T_out = 3, 40, 24
    ratio = 0.5
    params = ot.init_params(hp, seed=62, random_bias=True)
    batch = _batch(hp, B, T_in, T_out, 62)
    seed = _seed_where(lambda c: 6 <= c.sum() <= len(c) - 6, T_out, ratio, start=2000)
    g_mix = _run(hp, params, batch, ratio, seed).export_grads()
    g_tf = _run(hp, params, batch, 1.0, seed).export_grads()
    rel = lambda a, b: ((a - b).norm() / b.norm().clamp_min(1e-12)).item()
    diffs = {k: rel(g_mix[k], g_tf[k]) for k in ("decoder_prenet/dense_1/kernel", "decoder_prenet/dense_2/kernel", "decoder_LSTM/cell_1/kernel",
                                                 "linear_transform_projection/kernel", "linear_transform_projection/bias")}
    print("relative gradient change vs teacher forcing:", diffs)
    record("tacotron_tf_mix_vs_forced", **{k.replace("/", "_"): v for k, v in diffs.items()})
    assert all(v > 0.1 for v in diffs.values()), diffs


def _nonzero_grad_tensors(grads):
    """conv biases in front of a batch norm are left out: the normalisation cancels them, so their gradients are rounding noise
    (the last postnet layer has no activation, so its bias gradient is exactly zero in exact arithmetic)"""
    return [k for k in grads if not (k.endswith("/bias") and "conv_layer" in k)]


def test_per_step_forward_is_bitwise_the_batched_forward_when_every_draw_teacher_forces():
    """ratio just below 1 at a seed whose draws all take the target, prenet dropout 0.5 and zoneout 0.1 on. In an evaluation forward
    (batch norm on the moving statistics) nothing is summed with atomics, so the per-step decoder (per-step prenet GEMMs drawing the
    masks of the batched launch through the hash row offset, per-step input projection and projections, the feedback kernel writing the
    targets) must give the batched ratio-1 path's results bit for bit."""
    hp = _hp(tacotron_dropout_rate=0.5, tacotron_zoneout_rate=0.1)
    B, T_in, T_out, M = 3, 40, 24, hp.num_mels
    ratio = 0.9999
    params = ot.init_params(hp, seed=63, random_bias=True)
    inputs, lens, mel, stop = _batch(hp, B, T_in, T_out, 63)
    seed = _seed_where(lambda c: c.all(), T_out, ratio, start=3000)
    res = {}
    for r in (ratio, 1.0):
        model = t2.tacotron.Tacotron(hp, B, T_in, T_out, teacher_forcing_ratio=r)
        model.load_params(params)
        model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=False, seed=seed)
        torch.cuda.synchronize()
        if r < 1:
            assert model.teacher_forcing_choices()[:-1].all()
        res[r] = dict(_outputs(model, B, T_in, T_out, M), prenet=model.workspace_tensor("prenet").cpu().clone(),
                      projection_rows=model.workspace_tensor("projection_rows").cpu().clone())
        del model
    same = {k: torch.equal(res[ratio][k], res[1.0][k]) for k in res[1.0]}
    err = {k: (res[ratio][k].float() - res[1.0][k].float()).abs().max().item() for k in res[1.0]}
    print("per-step vs batched evaluation forward: bitwise", same, "max abs", err)
    record("tacotron_tf_per_step_vs_batched_eval_fwd", bitwise=all(same.values()), **{k + "_max": v for k, v in err.items()})
    assert all(same.values()), err


def test_per_step_training_step_matches_the_batched_step_when_every_draw_teacher_forces():
    """the same in a training step, backward included. The prenet outputs (targets, weights and hash masks only) must agree bit for
    bit. Everything else is not bit-reproducible even between two runs of the SAME path: the batch-norm statistics are fp32 atomic sums,
    whose order changes the encoder's bf16 activations now and then, and that change reaches every output and gradient of this tiny
    batch. Two runs of the batched path differ by up to 5 % (cos 0.9992) in a gradient tensor and 4.5e-4 in a loss here on an H100;
    the bounds below are the losses' fp32-reordering tolerance of test_tacotron_gpu.py and 3x that gradient spread. A per-step
    backward that added the feedback term for a forced step, or misplaced a prenet row, moves these gradients by 30-80 %."""
    hp = _hp(tacotron_dropout_rate=0.5, tacotron_zoneout_rate=0.1)
    B, T_in, T_out, M = 3, 40, 24, hp.num_mels
    ratio = 0.9999
    params = ot.init_params(hp, seed=63, random_bias=True)
    batch = _batch(hp, B, T_in, T_out, 63)
    seed = _seed_where(lambda c: c.all(), T_out, ratio, start=3000)
    runs = []
    for r in (ratio, 1.0, 1.0):
        m = _run(hp, params, batch, r, seed)
        runs.append((m.workspace_tensor("prenet").cpu().clone(), m.losses(), m.export_grads()))
        del m
    (pa, la, ga), (pb, lb, gb), (_, lc, gc) = runs
    assert torch.equal(pa, pb)
    rel = lambda x, y: ((x - y).norm() / y.norm().clamp_min(1e-12)).item()
    cos = lambda x, y: ((x * y).sum() / (x.norm() * y.norm()).clamp_min(1e-20)).item()
    keys = [k for k in _nonzero_grad_tensors(gb) if gb[k].norm() > 1e-6]
    d = {k: (rel(ga[k], gb[k]), cos(ga[k], gb[k])) for k in keys}
    spread = max(rel(gc[k], gb[k]) for k in keys)
    worst = max(d, key=lambda k: d[k][0])
    l_err = {k: abs(la[k] - lb[k]) for k in ("before", "after", "stop", "reg")}
    print("per-step vs batched training step: worst %s rel %.3g cos %.5f | batched run-to-run worst rel %.3g | losses %s" % (
        worst, d[worst][0], d[worst][1], spread, l_err))
    record("tacotron_tf_per_step_vs_batched_train", worst_rel=d[worst][0], worst_cos=min(c for _, c in d.values()),
           batched_run_to_run_worst_rel=spread, loss_max_err=max(l_err.values()))
    for k in l_err:
        assert l_err[k] < 2e-3 + 1e-3 * abs(lb[k]), (k, l_err)
    bad = ["%-60s rel %.4g cos %.5f" % (k, r_, c_) for k, (r_, c_) in d.items() if r_ > 0.15 or c_ < 0.995]
    assert not bad, "per-step step differs from the batched step:\n" + "\n".join(bad)


def test_cfg3_stochastic_paths_at_ratio_half():
    """Cfg-3 widths (B = 32, T_in = 160, T_out = 200), conv and prenet dropout 0.5 and zoneout 0.1 on: the masks the kernels drew are
    rebuilt from the hash and injected into the oracle together with the teacher-forcing draws"""
    from test_parity_full_gpu import taco_batch, taco_masks
    hp = hparams.copy()
    hp.parse("predict_linear=False")
    B, T_in, T_out, M = 32, 160, 200, hp.num_mels
    ratio = 0.5
    params = ot.init_params(hp, seed=64, random_bias=True)
    batch = taco_batch(hp, B, T_in, T_out, 64)
    seed = 99
    model = _run(hp, params, batch, ratio, seed)
    draws, choices = _check_draws(model, ratio, seed, T_out)
    assert 0 < int(choices.sum()) < T_out
    masks = taco_masks(model, hp, B, T_in, T_out)
    grads_ref, ref, parts = _oracle_step(params, *batch, hp, ratio, draws, masks=masks)
    _compare("tacotron_tf0.5_cfg3_B32_Tin160_Tout200_stochastic", model, ref, parts, grads_ref, B, T_in, T_out, M, FWD_TOL)


def test_cuda_graph_replays_draw_fresh_choices():
    hp = _hp(tacotron_dropout_rate=0.5, tacotron_zoneout_rate=0.1)
    B, T_in, T_out = 3, 40, 24
    ratio = 0.5
    params = ot.init_params(hp, seed=65, random_bias=True)
    inputs, lens, mel, stop = [x.cuda() for x in _batch(hp, B, T_in, T_out, 65)]
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out, teacher_forcing_ratio=ratio)
    model.load_params(params)
    graph = model.capture(inputs.int(), lens.int(), mel, stop)
    seen = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        draws = model.rng_uniform(TF_STREAM, T_out).cpu()          # seed + the device step counter the replay advanced
        choices = model.teacher_forcing_choices().cpu()
        assert torch.equal(choices, draws < ratio)
        assert all(math.isfinite(v) for v in model.losses().values()) and torch.isfinite(model.grads).all()
        seen.append((draws, choices))
    assert not torch.equal(seen[0][0], seen[1][0]) and not torch.equal(seen[0][1], seen[1][1])


def test_gta_feeds_the_targets_and_evaluation_draws():
    from tacotron.models import create_model
    hp = _hp(tacotron_teacher_forcing_ratio=0.5, tacotron_zoneout_rate=0.1)
    B, T_in, T_out, M = 3, 40, 24, hp.num_mels
    params = ot.init_params(hp, seed=66, random_bias=True)
    inputs, lens, mel, stop = [x.cuda() for x in _batch(hp, B, T_in, T_out, 66)]
    m = create_model("Tacotron", hp)
    m.load_variables(params)
    m.initialize(inputs, lens, mel, gta=True)
    assert m._eng.cfg.teacher_forcing_ratio == 1.0
    gta_mel = m.tower_mel_outputs[0].clone()
    ref = t2.tacotron.Tacotron(hp, B, T_in, T_out, teacher_forcing_ratio=1.0)
    ref.load_params(params)
    ref.forward(inputs.int(), lens.int(), mel, stop, training=False)
    torch.cuda.synchronize()
    assert torch.equal(gta_mel, ref.workspace_tensor("mel_outputs", (B, T_out, M)))
    m.initialize(inputs, lens, mel, stop, is_evaluating=True)
    eng = m._eng
    assert eng.cfg.teacher_forcing_ratio == pytest.approx(0.5)
    torch.cuda.synchronize()
    draws = eng.rng_uniform(TF_STREAM, T_out).cpu()
    assert torch.equal(eng.teacher_forcing_choices().cpu(), draws < 0.5)
    assert math.isfinite(float(m.add_loss()))


def test_dropin_training_loop_at_ratio_half():
    from tacotron.models import create_model
    hp = _hp(tacotron_teacher_forcing_ratio=0.5, tacotron_dropout_rate=0.5, tacotron_zoneout_rate=0.1)
    B, T_in, T_out = 3, 40, 24
    inputs, lens, mel, stop = [x.cuda() for x in _batch(hp, B, T_in, T_out, 67)]
    m = create_model("Tacotron", hp)
    losses = []
    for step in range(4):
        m.initialize(inputs, lens, mel, stop, global_step=step, is_training=True)
        losses.append(float(m.add_loss()))
        m.add_optimizer(step)
    torch.cuda.synchronize()
    print("drop-in losses at ratio 0.5:", losses)
    assert all(math.isfinite(l) for l in losses) and torch.isfinite(m.gradients).all()


@pytest.mark.parametrize("precision", ["bf16", "fp32-class"])
def test_synthesis_is_bitwise_the_ratio_zero_evaluation_forward(precision):
    """free-running synthesis (t2_taco_infer_*) and an evaluation forward at teacher-forcing ratio 0 run the same decoder step: each
    feeds the frame it just predicted to the next step. With prenet dropout off nothing random is left, so over the T_used steps
    synthesis ran both give the same decoder outputs, alignments and stop logits bit for bit. The postnet's 'same' convolutions read
    past T_used, so mel_outputs agree only when synthesis ran all T_out steps."""
    hp = _hp(tacotron_zoneout_rate=0.1)
    B, T_in, T_out, M = 3, 40, 24, hp.num_mels
    params = ot.init_params(hp, seed=68, random_bias=True)
    inputs, lens, mel, stop = [x.cuda() for x in _batch(hp, B, T_in, T_out, 68)]
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out, precision=precision, teacher_forcing_ratio=0.0)
    model.load_params(params)
    model.forward(inputs.int(), lens.int(), mel, stop, training=False, seed=5)
    torch.cuda.synchronize()
    fwd = _outputs(model, B, T_in, T_out, M)
    syn = model.synthesize(inputs.int(), lens.int(), max_iters=T_out, seed=5)
    T = syn["T"]
    syn_stop = model.workspace_tensor("stop_logits", (B, T)).cpu()
    same = dict(decoder_output=torch.equal(syn["decoder_output"].cpu(), fwd["decoder_output"][:, :T]),
                alignments=torch.equal(syn["alignments"].cpu(), fwd["alignments"][:, :T]),
                stop_logits=torch.equal(syn_stop, fwd["stop_logits"][:, :T]))
    if T == T_out:
        same["mel_outputs"] = torch.equal(syn["mel_outputs"].cpu(), fwd["mel_outputs"])
    print("synthesis (T_used %d of %d) vs ratio-0 evaluation forward, %s: bitwise" % (T, T_out, precision), same)
    record("tacotron_synthesis_vs_ratio0_fwd_%s" % precision, T_used=T, bitwise=all(same.values()))
    assert all(same.values()), same
