"""The Tacotron fp32-class mode (precision='fp32-class', t2_taco_config_t.split_bf16 = 1) end to end against the fp32 oracle at the
Cfg-3 widths (512 / 1024 / 512). Every contraction of the forward and of free-running synthesis - the convolution stacks, the encoder
BiLSTM, the prenet, both decoder LSTMs, the attention query / context and the frame / stop projection - runs on bf16 hi + lo operand pairs
(hi.hi + lo.hi + hi.lo, fp32 accumulation) with every stored activation a hi / lo pair, so the north-star mel-L1 <= 1e-3 is asserted.
The other bounds are twice the values measured on an H100 SXM (80 GB, 700 W power limit)."""
import pytest
import torch

from hparams import hparams
from oracle import tacotron as ot
from t2_import import t2
from parity_util import record
from test_parity_full_gpu import taco_batch, taco_compare
from test_tacotron_gpu import _trained_like_stats

pytestmark = pytest.mark.gpu

MEL_L1 = 1e-3          # BASELINE.json north star: mel-L1 against the fp32 reference


def _hp(stochastic=False, **kw):
    hp = hparams.copy()
    hp.parse("predict_linear=False" + ("" if stochastic else ",tacotron_dropout_rate=0.0,tacotron_zoneout_rate=0.0"))
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


def _split_rows(t, n):
    """recombine a split-mode workspace tensor whose rows are [hi(n) | lo(n)] into fp32 [..., n]"""
    t = t.reshape(-1, 2 * n).float()
    return t[:, :n] + t[:, n:]


def _tol(align, dec_l1, stop, loss):
    return dict(align=align, dec_l1=dec_l1, mel_l1=MEL_L1, stop=stop, loss=loss, grad_rel=1.0, grad_cos=0.0)


@pytest.mark.parametrize("stochastic,num_mels", [(False, 80), (True, 80), (False, 40)], ids=["False", "True", "num_mels40"])
def test_teacher_forced_cfg3(stochastic, num_mels):
    """B = 32, T_in 160, T_out 200; stochastic: conv / prenet dropout 0.5 and zoneout 0.1 with the device's masks injected. 40 mels fill
    one 64-wide K block per half of the split mel rows (decoder input, postnet input) instead of two."""
    hp = _hp(stochastic, num_mels=num_mels)
    tag = "tacotron_fp32_class_cfg3_%s%s" % ("stochastic" if stochastic else "deterministic", "" if num_mels == 80 else "_mels%d" % num_mels)
    m = taco_compare(tag, hp, 32, 160, 200, 61, _tol(2.7e-5, 5.5e-6, 3e-5, 5e-5), backward=False, precision="fp32-class").measured
    assert m["mel_l1"] <= MEL_L1, m


def test_stages_cfg3():
    """memory, keys, alignments and decoder_output of one deterministic training forward against the oracle, stage by stage"""
    hp = _hp()
    B, T_in, T_out = 32, 160, 200
    params = ot.init_params(hp, seed=62, random_bias=True)
    inputs, lens, mel, stop = taco_batch(hp, B, T_in, T_out, 62)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out, precision="fp32-class")
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=True)
    torch.cuda.synchronize()
    H = hp.encoder_lstm_units
    with torch.no_grad():
        x = params["inputs_embedding"][inputs]
        for i in range(hp.enc_conv_num_layers):
            x = ot.conv_block(x, params, "encoder_convolutions/conv_layer_%d/" % (i + 1), "relu", True, 0.0)
        memory = ot.encoder_rnn(x, lens, params, hp, True)
        keys = (memory * (torch.arange(T_in)[None, :] < lens[:, None]).float().unsqueeze(-1)) @ params["attention/memory_layer/kernel"]
        ref = ot.forward(params, inputs, lens, mel, hp, training=True)
    mem = _split_rows(model.workspace_tensor("memory").cpu(), 2 * H).reshape(B, T_in, 2 * H)
    live = (torch.arange(T_in)[None, :] < lens[:, None]).unsqueeze(-1)
    k = model.workspace_tensor("keys", (B, T_in, hp.attention_dim)).cpu()
    al = model.workspace_tensor("alignments", (T_out, B, T_in)).cpu().transpose(0, 1)
    dec = model.workspace_tensor("decoder_output", (B, T_out, hp.num_mels)).cpu()
    vals = dict(memory_max=((mem - memory) * live).abs().max().item(), keys_max=(k - keys).abs().max().item(),
                align_max=(al - ref["alignments"]).abs().max().item(), dec_l1=(dec - ref["decoder_output"]).abs().mean().item(),
                dec_max=(dec - ref["decoder_output"]).abs().max().item())
    m = record("tacotron_fp32_class_cfg3_stages", **vals)
    assert m["memory_max"] < 1.2e-4 and m["keys_max"] < 7e-5, m
    assert m["align_max"] < 1.4e-5 and m["dec_l1"] < 6e-6 and m["dec_max"] < 4e-5, m


@pytest.mark.parametrize("variant", ["mask_encoder=False", "cumulative_weights=False"])
def test_attention_variants_cfg3(variant):
    hp = _hp()
    hp.parse(variant)
    tag = "tacotron_fp32_class_cfg3_" + variant.split("=")[0]
    m = taco_compare(tag, hp, 32, 160, 200, 63, _tol(4e-6, 5.5e-6, 1e-5, 4e-5), backward=False, precision="fp32-class").measured
    assert m["mel_l1"] <= MEL_L1, m


def test_teacher_forcing_ratio_half_cfg3():
    """ratio 0.5: the oracle replays the device's per-step choices between the target frame and the fed-back prediction"""
    hp = _hp()
    B, T_in, T_out = 32, 160, 200
    params = ot.init_params(hp, seed=64, random_bias=True)
    inputs, lens, mel, stop = taco_batch(hp, B, T_in, T_out, 64)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out, precision="fp32-class", teacher_forcing_ratio=0.5)
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=True, seed=1234)
    torch.cuda.synchronize()
    choices = model.teacher_forcing_choices().cpu()
    assert 0 < int(choices[:T_out - 1].sum()) < T_out - 1
    draws = [0.0 if bool(c) else 1.0 for c in choices]
    with torch.no_grad():
        ref = ot.forward(params, inputs, lens, mel, hp, training=True, tf_ratio=0.5, tf_draws=draws)
    al = model.workspace_tensor("alignments", (T_out, B, T_in)).cpu().transpose(0, 1)
    dec = model.workspace_tensor("decoder_output", (B, T_out, hp.num_mels)).cpu()
    melo = model.workspace_tensor("mel_outputs", (B, T_out, hp.num_mels)).cpu()
    m = record("tacotron_fp32_class_cfg3_tf_half", align_max=(al - ref["alignments"]).abs().max().item(),
               dec_l1=(dec - ref["decoder_output"]).abs().mean().item(), mel_l1=(melo - ref["mel_outputs"]).abs().mean().item())
    assert m["mel_l1"] <= MEL_L1 and m["align_max"] < 2.1e-5 and m["dec_l1"] < 5e-6, m


def test_gta_eval_cfg3():
    """training=False (GTA / eval): inference batch norm on non-trivial moving statistics, zoneout's deterministic blend"""
    hp = _hp(tacotron_zoneout_rate=0.1)
    B, T_in, T_out = 32, 160, 200
    params = _trained_like_stats(ot.init_params(hp, seed=65, random_bias=True), 65)
    inputs, lens, mel, stop = taco_batch(hp, B, T_in, T_out, 65)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out, precision="fp32-class")
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=False)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = ot.forward(params, inputs, lens, mel, hp, training=False)
    al = model.workspace_tensor("alignments", (T_out, B, T_in)).cpu().transpose(0, 1)
    dec = model.workspace_tensor("decoder_output", (B, T_out, hp.num_mels)).cpu()
    melo = model.workspace_tensor("mel_outputs", (B, T_out, hp.num_mels)).cpu()
    m = record("tacotron_fp32_class_cfg3_gta_eval", align_max=(al - ref["alignments"]).abs().max().item(),
               dec_l1=(dec - ref["decoder_output"]).abs().mean().item(), mel_l1=(melo - ref["mel_outputs"]).abs().mean().item())
    assert m["mel_l1"] <= MEL_L1 and m["align_max"] < 8e-6 and m["dec_l1"] < 5.5e-6, m


def _synth(hp, params, inputs, lens, steps):
    model = t2.tacotron.Tacotron(hp, inputs.shape[0], inputs.shape[1], steps, precision="fp32-class")
    model.load_params(params)
    return model.synthesize(inputs.int().cuda(), lens.int().cuda(), chunk=32)


def test_free_running_synthesis_cfg3():
    """120 free-running steps (stop bias held low), each feeding back its own frame: mel_outputs against ot.synthesize"""
    hp = _hp(tacotron_zoneout_rate=0.1)
    B, T_in, steps = 8, 120, 120
    params = _trained_like_stats(ot.init_params(hp, seed=66, random_bias=True), 66)
    params["stop_token_projection/bias"] = torch.full((1,), -20.0)
    inputs, lens, _, _ = taco_batch(hp, B, T_in, steps, 66)
    with torch.no_grad():
        ref = ot.synthesize(params, inputs, lens, hp, max_iters=steps)
    out = _synth(hp, params, inputs, lens, steps)
    assert out["T"] == steps == ref["mel_outputs"].shape[1]
    m = record("tacotron_fp32_class_cfg3_synthesis_120", mel_l1=(out["mel_outputs"].cpu() - ref["mel_outputs"]).abs().mean().item(),
               dec_l1=(out["decoder_output"].cpu() - ref["decoder_output"]).abs().mean().item(),
               align_max=(out["alignments"].cpu() - ref["alignments"]).abs().max().item())
    assert m["mel_l1"] <= MEL_L1 and m["align_max"] < 7e-6 and m["dec_l1"] < 5e-6, m


def test_synthesis_stop_step_cfg3():
    """a stop projection set to a scaled (possibly negated) frame channel, with a bias that puts the stop rule's smallest |logit| margin
    over the run at 0.1 or more: the device stops at exactly the oracle's step. The stop logits do not feed back, so the trajectory is
    the one of a run that never stops, and the channel / step pair is picked from that run's frames."""
    hp = _hp(tacotron_zoneout_rate=0.1)
    B, T_in, steps = 4, 100, 140
    params = _trained_like_stats(ot.init_params(hp, seed=67, random_bias=True), 67)
    params["stop_token_projection/bias"] = torch.full((1,), -30.0)
    inputs, lens, _, _ = taco_batch(hp, B, T_in, steps, 67)
    with torch.no_grad():
        free = ot.synthesize(params, inputs, lens, hp, max_iters=steps)
    frames = free["decoder_output"].double()                   # [B, steps, M]
    assert free["mel_outputs"].shape[1] == steps and frames.abs().max().item() < hp.max_abs_value
    best = None
    for m in range(hp.num_mels):
        for sign in (1.0, -1.0):
            rule = (sign * frames[:, :, m]).min(dim=0).values   # a step ends the run when every row's logit + bias > 0
            for T in range(10, steps - 1):
                gap = rule[T].item() - rule[:T].max().item()
                if best is None or gap > best[0]:
                    best = (gap, T, m, sign, rule[T].item() + rule[:T].max().item())
    gap, T_stop, m, sign, mid = best
    assert gap > 0, "no frame channel reaches a new maximum of the stop rule"
    mag = max(1.0, 0.2 / gap)                                  # margin = mag * gap / 2 >= 0.1 on both sides of the stop step
    wf, bf = params["linear_transform_projection/kernel"], params["linear_transform_projection/bias"]
    params["stop_token_projection/kernel"] = wf[:, m:m + 1] * (sign * mag)
    params["stop_token_projection/bias"] = (bf[m:m + 1] * (sign * mag) - mag * mid / 2).float()
    with torch.no_grad():
        ref = ot.synthesize(params, inputs, lens, hp, max_iters=steps)
    out = _synth(hp, params, inputs, lens, steps)
    record("tacotron_fp32_class_cfg3_stop_step", T_ref=ref["mel_outputs"].shape[1], T_dev=out["T"], margin=mag * gap / 2, scale=sign * mag,
           channel=m)
    assert ref["mel_outputs"].shape[1] == T_stop + 1
    assert out["T"] == T_stop + 1
    assert (out["mel_outputs"].cpu() - ref["mel_outputs"]).abs().mean().item() <= MEL_L1
