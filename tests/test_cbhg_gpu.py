"""CBHG post-processing net + linear head (predict_linear = True, the reference default: tacotron.py:203-219, modules.py:4-78,457-485)
through the C-ABI vs the fp32 CPU oracle.

1. the CBHG engine alone on a GIVEN mel tensor (both sides see identical inputs): linear outputs, linear loss, regulariser, every
   weight gradient and the gradient handed back to the Tacotron graph (d loss / d mel_outputs);
2. the whole Tacotron training step with the head attached: the extra gradient path through mel_outputs into postnet / decoder.
Tolerances follow the bf16-operand figures of tests/test_tacotron_gpu.py (<= 2x the values measured on an H100)."""
import ctypes

import pytest
import torch

from hparams import hparams
from oracle import tacotron as ot
from t2_import import t2
from parity_util import record, grad_report

pytestmark = pytest.mark.gpu
L = t2.lib


def _hp(**kw):
    hp = hparams.copy()
    hp.parse("predict_linear=True,tacotron_dropout_rate=0.0,tacotron_zoneout_rate=0.0,enc_conv_channels=256,embedding_dim=256,"
             "encoder_lstm_units=128,decoder_lstm_units=256,postnet_channels=256,prenet_layers=[128,128],attention_dim=128,num_freq=513")
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


def _batch(hp, B, T_in, T_out, seed):
    g = torch.Generator().manual_seed(seed)
    inputs = torch.randint(2, 66, (B, T_in), generator=g)
    lens = torch.tensor([T_in] + [max(T_in - 5 * (i + 1), 3) for i in range(B - 1)])
    for b in range(B):
        inputs[b, lens[b]:] = 0
    mel = (torch.randn(B, T_out, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    lin = (torch.randn(B, T_out, hp.num_freq, generator=g) * 1.5 - 1).clamp(-4, 4)
    stop = torch.zeros(B, T_out)
    stop[:, -3:] = 1
    return inputs, lens, mel, stop, lin


def _is_cbhg(name):
    return name.startswith(("CBHG_postnet", "cbhg_"))


@pytest.mark.parametrize("B,T,mask", [(5, 37, False), (8, 64, True)])
def test_cbhg_engine_matches_oracle(B, T, mask):
    hp = _hp(mask_decoder=mask)
    params = ot.init_params(hp, seed=11, random_bias=True)
    g = torch.Generator().manual_seed(5)
    mel = (torch.randn(B, T, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    lin_t = (torch.randn(B, T, hp.num_freq, generator=g) * 1.5 - 1).clamp(-4, 4)
    tl = torch.tensor([T] + [max(T - 6 * (i + 1), 4) for i in range(B - 1)])
    # oracle
    ps = {k: (v.clone().requires_grad_(True) if (_is_cbhg(k) and ot.is_trainable(k)) else v.clone()) for k, v in params.items()}
    mel_r = mel.clone().requires_grad_(True)
    lin_ref = ot.linear_head(mel_r, ps, hp, True)
    loss_lin = ot.linear_loss(lin_t, lin_ref, hp, tl if mask else None)
    reg = sum((v * v).sum() / 2 for k, v in ps.items() if _is_cbhg(k) and ot.is_regularized(k)) * hp.tacotron_reg_weight
    names = [k for k in ps if _is_cbhg(k) and ot.is_trainable(k)]
    gr = torch.autograd.grad(loss_lin + reg, [ps[k] for k in names] + [mel_r])
    grads_ref = dict(zip(names, gr[:-1]))
    dmel_ref = gr[-1]
    # CUDA: the CBHG engine of a Tacotron model, driven directly on `mel`
    model = t2.tacotron.Tacotron(hp, B, 16, T)
    model.load_params(params)
    model.pack()
    lib, cfg = model.lib, ctypes.byref(model.cbhg)
    prm = model.params[model.n_taco:]
    mel_d, lin_d = mel.cuda().contiguous(), lin_t.cuda().contiguous()
    if mask:
        L.check(lib.t2_cbhg_set_target_lengths(cfg, L.ptr(model.cb_workspace), L.ptr(tl.int().cuda()), L.stream_ptr()))
    L.check(lib.t2_cbhg_forward(cfg, L.ptr(prm), L.ptr(model.cb_packed), L.ptr(model.cb_workspace), L.ptr(mel_d), L.ptr(lin_d), L.ptr(model.cb_loss), 1,
                                L.stream_ptr()))
    model.grads = torch.zeros_like(model.params)
    L.check(lib.t2_cbhg_backward(cfg, L.ptr(prm), L.ptr(model.cb_packed), L.ptr(model.cb_workspace), L.ptr(mel_d), L.ptr(model.grads[model.n_taco:]),
                                 L.ptr(model.cb_dmel), L.stream_ptr()))
    torch.cuda.synchronize()
    lin = model.linear_outputs().cpu()
    e = (lin - lin_ref.detach()).abs()
    l_lin, l_reg = model.cb_loss.tolist()
    grads = {k: v for k, v in model.export_grads().items() if _is_cbhg(k)}
    rows, worst_rel, worst_cos = grad_report(grads, grads_ref)
    for name, rel, cos, den in rows:
        print("%-60s rel %.4f cos %.5f |g| %.3g" % (name, rel, cos, den))
    dmel = model.cb_dmel.view(B, T, hp.num_mels).cpu()
    dm_rel = (dmel - dmel_ref).norm().item() / dmel_ref.norm().item()
    dm_cos = (dmel * dmel_ref).sum().item() / (dmel.norm().item() * dmel_ref.norm().item())
    m = record("cbhg_engine_B%d_T%d_mask%d" % (B, T, int(mask)), lin_mean_err=e.mean().item(), lin_max_err=e.max().item(),
               loss_lin_err=abs(l_lin - loss_lin.item()), loss_lin_ref=loss_lin.item(), loss_reg_err=abs(l_reg - reg.item()), loss_reg_ref=reg.item(),
               grad_worst_rel=worst_rel, grad_worst_cos=worst_cos, dmel_rel=dm_rel, dmel_cos=dm_cos)
    assert m["lin_mean_err"] < 3e-2 and m["loss_lin_err"] < 5e-3 and m["loss_reg_err"] < 1e-6 + 1e-3 * reg.item()
    assert worst_cos > 0.95 and worst_rel < 0.35 and dm_cos > 0.97 and dm_rel < 0.25


def test_cbhg_inference_mode_and_batch_padding():
    """synthesis path: moving-average batch norm, B not a multiple of 4, arbitrary T (linear_from_mel)"""
    hp = _hp()
    params = ot.init_params(hp, seed=12, random_bias=True)
    for k in params:                                    # non-trivial moving statistics
        if k.endswith("moving_mean"):
            params[k] = torch.randn_like(params[k]) * 0.1
        if k.endswith("moving_variance"):
            params[k] = torch.rand_like(params[k]) + 0.5
    g = torch.Generator().manual_seed(6)
    mel = (torch.randn(3, 29, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    ref = ot.linear_head(mel, params, hp, False)
    model = t2.tacotron.Tacotron(hp, 4, 16, 32)
    model.load_params(params)
    lin = model.linear_from_mel(mel.cuda()).cpu()
    e = (lin - ref).abs()
    m = record("cbhg_inference_B3_T29", lin_mean_err=e.mean().item(), lin_max_err=e.max().item())
    assert lin.shape == ref.shape and m["lin_mean_err"] < 3e-2


def test_tacotron_train_step_with_linear_head():
    hp = _hp()
    B, T_in, T_out = 4, 30, 28
    params = ot.init_params(hp, seed=21, random_bias=True)
    inputs, lens, mel, stop, lin_t = _batch(hp, B, T_in, T_out, 21)
    loss_ref, grads_ref, out_ref, parts = ot.train_step(params, inputs, lens, mel, stop, hp, linear_targets=lin_t)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out)
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), linear_targets=lin_t.cuda())
    model.backward()
    torch.cuda.synchronize()
    los = model.losses()
    e = (model.linear_outputs().cpu() - out_ref["linear_outputs"]).abs()
    grads = model.export_grads()
    rows, worst_rel, worst_cos = grad_report(grads, grads_ref)
    for name, rel, cos, den in rows:
        print("%-70s rel %.4f cos %.5f |g| %.3g" % (name, rel, cos, den))
    # tensors upstream of mel_outputs receive the head's gradient through t2_taco_backward_ex (conv biases in front of a batch norm
    # have a true gradient of zero: excluded by their norm)
    post = [r for r in rows if r[0].startswith(("postnet", "decoder_LSTM", "linear_transform")) and r[3] >= 1e-6]
    m = record("tacotron_linear_head_B4_Tin30_Tout28", lin_mean_err=e.mean().item(), loss_linear_err=abs(los["linear"] - parts["linear"].item()),
               loss_linear_ref=parts["linear"].item(), loss_total_err=abs(los["total"] - loss_ref.item()), loss_total_ref=loss_ref.item(),
               loss_reg_err=abs(los["reg"] - parts["reg"].item()), grad_worst_rel=worst_rel, grad_worst_cos=worst_cos,
               upstream_worst_rel=max(r[1] for r in post), upstream_worst_cos=min(r[2] for r in post))
    assert m["lin_mean_err"] < 6e-2 and m["loss_linear_err"] < 1e-2 and m["loss_total_err"] < 2e-2
    assert m["upstream_worst_cos"] > 0.95 and worst_cos > 0.9
