"""CUDA Tacotron (through the C-ABI) vs the fp32 CPU oracle, dropout / zoneout off (rates are hparams), same seeded
inputs. Tolerances (bf16 GEMM operands, fp32 accumulate / state; <= 2x the values measured on an H100):
losses <= 2e-3 absolute + 1e-3 relative, alignments max abs err <= 6e-4, decoder-output L1 <= 1.6e-3, stop logits <= 5e-3, mel outputs
mean abs err <= 4e-2 (measured 2.5e-2: five batch-normalised postnet layers each add ~0.2 % of a unit-variance activation in bf16 storage
- tools/taco_layer_diag.py; 6e-4 in the fp32-class mode, tests/test_precision_modes_gpu.py).
Gradients vs the fp32 oracle: per tensor cosine >= 0.97 and relative error <= 0.25 (conv biases in front of a batch norm: 0.9 / 0.5) (measured: 2-4 % for the large
tensors; 10-18 % for the small encoder-conv / location-attention tensors of the tiny B=3 problem, shrinking as the batch
grows — the bf16 sign-flip noise floor discussed in tests/test_wavenet_gpu.py, amplified by batch-norm over ~100 rows)."""
import pytest
import torch

from hparams import hparams
from oracle import tacotron as ot
from t2_import import t2
from parity_util import record

pytestmark = pytest.mark.gpu


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


def _run_forward(hp, B, T_in, T_out, seed):
    params = ot.init_params(hp, seed=seed, random_bias=True)
    inputs, lens, mel, stop = _batch(hp, B, T_in, T_out, seed)
    ref = ot.forward(params, inputs, lens, mel, hp, training=True)
    _, parts = ot.loss_fn(ref, mel, stop, params, hp)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out)
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda())
    torch.cuda.synchronize()
    return model, params, ref, parts, (inputs, lens, mel, stop)


@pytest.mark.parametrize("B,T_in,T_out", [(3, 40, 24), (2, 150, 33)])
def test_forward_matches_oracle(B, T_in, T_out):
    hp = _hp()
    model, params, ref, parts, _ = _run_forward(hp, B, T_in, T_out, 31)
    mem_ref = None
    al = model.workspace_tensor("alignments", (T_out, B, T_in)).float().cpu().transpose(0, 1)
    err_al = (al - ref["alignments"]).abs().max().item()
    dec = model.workspace_tensor("decoder_output", (B, T_out, hp.num_mels)).cpu()
    melo = model.workspace_tensor("mel_outputs", (B, T_out, hp.num_mels)).cpu()
    stop = model.workspace_tensor("stop_logits", (B, T_out)).cpu()
    e_dec = (dec - ref["decoder_output"]).abs()
    e_mel = (melo - ref["mel_outputs"]).abs()
    e_stop = (stop - ref["stop_logits"]).abs()
    los = model.losses()
    print("align err %.3g | dec max %.3g mean %.3g | mel max %.3g mean %.3g | stop max %.3g | losses cuda %s oracle %s" % (
        err_al, e_dec.max(), e_dec.mean(), e_mel.max(), e_mel.mean(), e_stop.max(), los, {k: round(v.item(), 6) for k, v in parts.items()}))
    record("tacotron_small_fwd_B%d_Tin%d_Tout%d" % (B, T_in, T_out), align_max_err=err_al, dec_l1=e_dec.mean().item(), dec_max=e_dec.max().item(),
           mel_l1=e_mel.mean().item(), mel_max=e_mel.max().item(), stop_max=e_stop.max().item(),
           **{"loss_%s_err" % k: abs(los[k] - parts[k].item()) for k in ("before", "after", "stop", "reg")})
    assert err_al < 6e-4                                            # measured 6e-5 .. 3e-4
    assert e_dec.mean().item() < 1.6e-3 and e_mel.mean().item() < 4e-2 and e_stop.max().item() < 5e-3     # measured 7e-4 / 2.5e-2 / 1.5e-3
    for k in ("before", "after", "stop", "reg"):
        # 2e-3 absolute + 1e-3 relative: the losses here are O(3-5) at random init and the batch-norm statistics / loss sums
        # are fp32 atomics (run-to-run reordering moves the 4th digit)
        assert abs(los[k] - parts[k].item()) < 2e-3 + 1e-3 * abs(parts[k].item()), k


def test_forward_matches_oracle_at_384_encoder_units():
    """2 * encoder_lstm_units = 768 > 512: the attention context needs more work items than the attention CTA has threads"""
    B, T_in, T_out = 3, 40, 24
    hp = _hp(encoder_lstm_units=384)
    model, params, ref, parts, _ = _run_forward(hp, B, T_in, T_out, 37)
    al = model.workspace_tensor("alignments", (T_out, B, T_in)).float().cpu().transpose(0, 1)
    err_al = (al - ref["alignments"]).abs().max().item()
    dec = model.workspace_tensor("decoder_output", (B, T_out, hp.num_mels)).cpu()
    e_dec = (dec - ref["decoder_output"]).abs()
    los = model.losses()
    record("tacotron_fwd_H384_B%d_Tin%d_Tout%d" % (B, T_in, T_out), align_max_err=err_al, dec_l1=e_dec.mean().item())
    assert err_al < 6e-4 and e_dec.mean().item() < 1.6e-3                 # the same tolerances as test_forward_matches_oracle
    for k in ("before", "after", "stop", "reg"):
        assert abs(los[k] - parts[k].item()) < 2e-3 + 1e-3 * abs(parts[k].item()), k


@pytest.mark.parametrize("B,T_in,T_out", [(3, 40, 24), (8, 60, 64)])
def test_backward_matches_oracle(B, T_in, T_out):
    hp = _hp()
    model, params, ref, parts, (inputs, lens, mel, stop) = _run_forward(hp, B, T_in, T_out, 32)
    model.backward()
    torch.cuda.synchronize()
    _, grads_ref, _, _ = ot.train_step(params, inputs, lens, mel, stop, hp)
    grads = model.export_grads()
    report, bad, rels, coss = [], [], [], []
    for name, g_ref in grads_ref.items():
        g = grads[name]
        den = g_ref.norm().item()
        rel = (g - g_ref).norm().item() / max(den, 1e-12)
        cos = (g * g_ref).sum().item() / max(den * g.norm().item(), 1e-20)
        if den >= 1e-6 and not (name.endswith("/bias") and "conv_layer" in name):
            rels.append(rel); coss.append(cos)
        report.append("%-60s rel %.4g cos %.4f |ref| %.3g |cuda| %.3g" % (name, rel, cos, den, g.norm().item()))
        # conv biases in front of a batch norm: the normalisation cancels the bias except through the activation's
        # curvature, so these gradients are ~50x smaller than their kernels' and sit in the bf16 noise of the tiny batch
        noise_floor = name.endswith("/bias") and "conv_layer" in name
        rel_tol, cos_tol = (0.5, 0.9) if noise_floor else (0.25, 0.97)
        if den >= 1e-6 and (rel >= rel_tol or cos < cos_tol):
            bad.append(report[-1])
    print("\n".join(report))
    record("tacotron_small_bwd_B%d_Tin%d_Tout%d" % (B, T_in, T_out), worst_rel=max(r for r in rels), worst_cos=min(coss))
    assert not bad, "gradient mismatch:\n" + "\n".join(bad)


def test_adam_global_norm_clip_matches_oracle():
    hp = _hp()
    B, T_in, T_out = 2, 24, 12
    model, params, ref, parts, (inputs, lens, mel, stop) = _run_forward(hp, B, T_in, T_out, 33)
    model.backward()
    grads = model.export_grads()
    state = {}
    p_ref = {k: v.clone() for k, v in params.items() if ot.is_trainable(k)}
    ot.adam_step(p_ref, {k: grads[k] for k in p_ref}, state, hp, 0)
    model.optimizer_step()
    torch.cuda.synchronize()
    p_new = model.export_params()
    for k in p_ref:
        assert (p_new[k] - p_ref[k]).abs().max().item() < 2e-6, k


def test_fine_tuning_freezes_embedding_and_encoder():
    """tacotron_fine_tuning (tacotron.py:401): only variables without 'inputs_embedding' / 'encoder_' in their names are optimised, and
    only their gradients enter the global-norm clip"""
    hp = _hp(tacotron_fine_tuning=True)
    B, T_in, T_out = 2, 24, 12
    model, params, ref, parts, _ = _run_forward(hp, B, T_in, T_out, 35)
    model.backward()
    grads = model.export_grads()
    frozen = lambda k: "inputs_embedding" in k or "encoder_" in k
    p_ref = {k: v.clone() for k, v in params.items() if ot.is_trainable(k) and not frozen(k)}
    ot.adam_step(p_ref, {k: grads[k] for k in p_ref}, {}, hp, 0)
    model.optimizer_step()
    torch.cuda.synchronize()
    p_new = model.export_params()
    for k, v in params.items():
        if not ot.is_trainable(k):
            continue
        if frozen(k):
            assert torch.equal(p_new[k], v), k
        else:
            assert (p_new[k] - p_ref[k]).abs().max().item() < 2e-6, k


def _trained_like_stats(params, seed):
    """non-trivial batch-norm moving statistics so that the inference path is really exercised"""
    g = torch.Generator().manual_seed(seed)
    for k in params:
        if k.endswith("moving_mean"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.1
        elif k.endswith("moving_variance"):
            params[k] = torch.rand(params[k].shape, generator=g) * 0.5 + 0.75
    return params


def test_free_running_synthesis_matches_oracle():
    """TacoTestHelper path: own predictions fed back, inference batch-norm / zoneout blend, stop rule on the host.
    Tolerances as in the teacher-forced test, a little wider on the frames since bf16 errors are fed back 24 times."""
    hp = _hp(tacotron_zoneout_rate=0.1)
    B, T_in, steps = 3, 40, 24
    params = _trained_like_stats(ot.init_params(hp, seed=41, random_bias=True), 41)
    params["stop_token_projection/bias"] = torch.full((1,), -6.0)        # never stops: runs to max_iters
    inputs, lens, _, _ = _batch(hp, B, T_in, steps, 41)
    ref = ot.synthesize(params, inputs, lens, hp, max_iters=steps)
    model = t2.tacotron.Tacotron(hp, B, T_in, steps)
    model.load_params(params)
    out = model.synthesize(inputs.int().cuda(), lens.int().cuda(), chunk=10)
    assert out["T"] == steps == ref["mel_outputs"].shape[1]
    e_al = (out["alignments"].cpu() - ref["alignments"]).abs().max().item()
    e_dec = (out["decoder_output"].cpu() - ref["decoder_output"]).abs()
    e_mel = (out["mel_outputs"].cpu() - ref["mel_outputs"]).abs()
    e_stop = (out["stop_token_prediction"].cpu() - ref["stop_token_prediction"]).abs().max().item()
    print("synthesis: align %.3g | dec max %.3g mean %.3g | mel max %.3g mean %.3g | stop %.3g" % (
        e_al, e_dec.max(), e_dec.mean(), e_mel.max(), e_mel.mean(), e_stop))
    record("tacotron_synthesis_24steps", align_max_err=e_al, dec_l1=e_dec.mean().item(), mel_l1=e_mel.mean().item(), stop_max=e_stop)
    assert e_al < 1e-4 and e_dec.mean().item() < 1e-3 and e_mel.mean().item() < 4e-3 and e_stop < 1e-4       # measured 3e-5 / 4e-4 / 1.6e-3 / 2e-6


def test_synthesis_stop_rule():
    """finished <=> every row's stop probability rounds to 1 (helpers.py:40-54): the frame of that step is kept."""
    hp = _hp()
    B, T_in, max_iters = 2, 20, 40
    params = ot.init_params(hp, seed=42, random_bias=True)
    inputs, lens, _, _ = _batch(hp, B, T_in, max_iters, 42)
    model = t2.tacotron.Tacotron(hp, B, T_in, max_iters)
    params["stop_token_projection/bias"] = torch.full((1,), 6.0)          # stops at the very first step
    model.load_params(params)
    out = model.synthesize(inputs.int().cuda(), lens.int().cuda(), chunk=16)
    ref = ot.synthesize(params, inputs, lens, hp, max_iters=max_iters)
    assert out["T"] == 1 == ref["mel_outputs"].shape[1]
    assert (out["mel_outputs"].cpu() - ref["mel_outputs"]).abs().mean().item() < 4e-2
    # a stop vector that crosses zero mid-sequence: the stop logit follows the decoder state, so make the projection
    # read a time ramp out of the cumulative-free part: use the oracle's own decision as the expectation
    params["stop_token_projection/bias"] = torch.full((1,), 0.0)
    params["stop_token_projection/kernel"] = params["stop_token_projection/kernel"] * 8
    model.load_params(params)
    ref = ot.synthesize(params, inputs, lens, hp, max_iters=max_iters)
    out = model.synthesize(inputs.int().cuda(), lens.int().cuda(), chunk=7)
    margin = (torch.logit(ref["stop_token_prediction"].clamp(1e-6, 1 - 1e-6))).abs().min().item()
    print("oracle stops after %d steps (min |logit| %.3g), cuda after %d" % (ref["mel_outputs"].shape[1], margin, out["T"]))
    if margin > 0.05:        # no marginal decisions: the two must agree exactly
        assert out["T"] == ref["mel_outputs"].shape[1]


def test_gta_mode_uses_inference_statistics():
    """GTA / eval graph: teacher forcing with is_training = False (tacotron.py:157-160): moving-average batch norm,
    no conv dropout, deterministic zoneout blend."""
    hp = _hp(tacotron_zoneout_rate=0.1)
    B, T_in, T_out = 3, 40, 24
    params = _trained_like_stats(ot.init_params(hp, seed=43, random_bias=True), 43)
    inputs, lens, mel, stop = _batch(hp, B, T_in, T_out, 43)
    ref = ot.forward(params, inputs, lens, mel, hp, training=False)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out)
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=False)
    torch.cuda.synchronize()
    melo = model.workspace_tensor("mel_outputs", (B, T_out, hp.num_mels)).cpu()
    al = model.workspace_tensor("alignments", (T_out, B, T_in)).float().cpu().transpose(0, 1)
    assert (al - ref["alignments"]).abs().max().item() < 1e-3
    assert (melo - ref["mel_outputs"]).abs().mean().item() < 4e-2
    p_after = model.export_params()
    for k in params:
        if "moving_" in k:
            assert torch.equal(p_after[k], params[k]), k          # inference must not touch the moving statistics


def test_masked_decoder_losses_match_oracle():
    """mask_decoder=True (modules.py:412-455): MSE terms over the frames inside each target length, weighted sigmoid CE (pos_weight 3)
    divided by the number of non-zero masked terms; forward losses and the gradients they seed"""
    hp = _hp(mask_decoder=True, cross_entropy_pos_weight=3.0)
    B, T_in, T_out = 4, 40, 32
    params = ot.init_params(hp, seed=45, random_bias=True)
    inputs, lens, mel, stop = _batch(hp, B, T_in, T_out, 45)
    tl = torch.tensor([32, 27, 20, 9])
    stop = (torch.arange(T_out)[None, :] >= (tl[:, None] - 1)).float()
    _, grads_ref, ref, parts = ot.train_step(params, inputs, lens, mel, stop, hp, targets_lengths=tl)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out)
    model.load_params(params)
    with pytest.raises(t2.lib.T2Error):
        model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda())             # lengths are mandatory, as in the reference
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), targets_lengths=tl.int().cuda())
    model.backward()
    torch.cuda.synchronize()
    los = model.losses()
    for k in ("before", "after", "stop", "reg"):
        assert abs(los[k] - parts[k].item()) < 2e-3 + 1e-3 * abs(parts[k].item()), (k, los[k], parts[k].item())
    grads = model.export_grads()
    for name in ("linear_transform_projection/kernel", "stop_token_projection/kernel", "postnet_projection/kernel", "decoder_LSTM/cell_2/kernel"):
        g, gr = grads[name], grads_ref[name]
        cos = (g * gr).sum().item() / (g.norm().item() * gr.norm().item())
        assert cos > 0.97 and abs(g.norm().item() / gr.norm().item() - 1) < 0.1, (name, cos)
    # the unmasked model gives different losses on the same batch: the mask is really applied
    hp0 = _hp()
    _, parts0 = ot.loss_fn(ot.forward(params, inputs, lens, mel, hp0, training=True), mel, stop, params, hp0)
    assert abs(parts0["before"].item() - parts["before"].item()) > 1e-2
