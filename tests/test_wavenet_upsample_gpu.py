"""The conditioning upsampler kernels on the H100: ConvTranspose1D (upsample_type '1D') and the LeakyReLU / linear activations of all
three learnable upsamplers, one launch at a time through t2_dbg_wn_kernel and end to end through the engine.

Bounds:
  executed reference   tests/golden/reference_wavenet_graph.npz, scenario ce_1d (cin 6, scales [2, 3]): the forward of both layers
                       reproduces the reference's upsampled conditioning within 2e-6 (the oracle's own bound); fed the oracle's
                       d loss / d c_up, the backward launches reproduce the reference's upsampler gradients within 2e-4 x max (ditto).
  kernel sweeps        float64 torch references on the exact fp32 inputs and outputs the kernels read (the activation derivative is
                       taken from the kernel's own stored output, as the kernels do). Every element within 1e-5 of the same contraction
                       over absolute values (+1e-9 for the 2^-40 fixed-point quantum of the weight-gradient sums): fp32-sized.
                       The bf16 conditioning copies are exactly the bf16 rounding of the kernel's fp32 output (hi, and lo = the rest).
  end to end           against the fp32 oracle with the bounds of tests/test_wavenet_gpu.py: loss 1e-4 (CE) / 6e-4 (MoL), logits max 8e-3
                       and mean 1.5e-3, every gradient tensor within 1e-1 relative (L2) (SubPixel / 2D under the new activations:
                       the upsampler tensors within 2e-3 of float64 on the engine's own d loss / d c_up, see that test); the
                       fp32-class forward within 1e-4; two
                       backward runs bit-identical; Adam within 2e-6. AR: the bounds of tests/test_wavenet_ar_gpu.py.
MEASURED lines are printed for the record."""
import ctypes
import math
import os
import types

import numpy as np
import pytest
import torch

import t2_tf_bundle as tb
from hparams import hparams
from oracle import wavenet as ow
from t2_import import t2

pytestmark = pytest.mark.gpu
L = t2.lib
DEV = "cuda"
F64 = torch.float64
NAN = float("nan")
UP_FWD, UP_BWD_PARAM, UP_BWD_INPUT = 1, 2, 3
TYPES = {"SubPixel": 0, "2D": 1, "1D": 2}
ACTS = {"Relu": 0, "LeakyRelu": 1, None: 2}
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_wavenet_graph.npz")


# ------------------------------------------------------------------------------------------------------------------------------
# one launch at a time
# ------------------------------------------------------------------------------------------------------------------------------
def launch(kernel, p, B, C, W, s, utype, act, alpha=0.0, split=0):
    c = L.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate((B, C, W, s, TYPES[utype], ACTS[act], split)):
        c.i[k] = int(v)
    c.f[0] = float(alpha)
    L.check(L.load().t2_dbg_wn_kernel(ctypes.byref(c), L.stream_ptr()))
    torch.cuda.synchronize()


def _layer_hp(utype, s, act, alpha):
    return types.SimpleNamespace(upsample_type=utype, upsample_scales=[s], upsample_activation=act, leaky_alpha=alpha)


def _pre(x, K, b, utype, s):
    """pre-activation of one layer (the oracle's layer code, activation off)"""
    return ow.upsample(x, {"local_conditioning_upsampling_1/kernel": K, "local_conditioning_upsampling_1/bias": b},
                       _layer_hp(utype, s, "none", 0.0))


def _dact(out, act, alpha):
    if act == "Relu":
        return (out > 0).to(F64)
    if act == "LeakyRelu":
        return torch.where(out > 0, torch.ones_like(out), torch.full_like(out, alpha))
    return torch.ones_like(out)


def _shapes(utype, s, C):
    return {"SubPixel": ((3, 3, 1, s), (s,)), "2D": ((3, s, 1, 1), (1,)), "1D": ((1, s, C, C), (C,))}[utype]


def check(name, got, ref, bound):
    err = (got.to(F64) - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=float("inf")).max().item()
    assert ratio <= 1.0, "%s: worst err / bound %.3g" % (name, ratio)
    return ratio


def _sweep_case(utype, act, s, B, C, W, seed, split=0):
    alpha = 0.4 if act == "LeakyRelu" else 0.0
    g = torch.Generator().manual_seed(seed)
    ks, bs = _shapes(utype, s, C)
    x = torch.randn(B, C, W, generator=g)
    K = torch.randn(ks, generator=g) * (0.5 / math.sqrt(C if utype == "1D" else 3))
    b = torch.randn(bs, generator=g) * 0.1
    dout = torch.randn(B, C, W * s, generator=g)
    xd, Kd, bd, doutd = (t.to(DEV) for t in (x, K, b, dout))
    out = torch.full((B, C, W * s), NAN, device=DEV)
    cup = torch.full((B, W * s, 256 if split else C), NAN, device=DEV).to(torch.bfloat16)
    launch(UP_FWD, [xd, Kd, bd, out, cup], B, C, W, s, utype, act, alpha, split)
    # forward: float64 on the same inputs
    x64, K64, b64 = x.to(F64), K.to(F64), b.to(F64)
    pre = _pre(x64, K64, b64, utype, s)
    ref = pre if act is None else (torch.relu(pre) if act == "Relu" else torch.nn.functional.leaky_relu(pre, alpha))
    pre_abs = _pre(x64.abs(), K64.abs(), b64.abs(), utype, s)
    o = out.cpu()
    r_fwd = check("fwd %s %s s%d" % (utype, act, s), o, ref, 1e-5 * pre_abs + 1e-30)
    v = o.transpose(1, 2)
    hi = v.to(torch.bfloat16)
    if split:
        cc = cup.cpu()
        assert torch.equal(cc[:, :, :C], hi) and torch.equal(cc[:, :, 128:128 + C], (v - hi.float()).to(torch.bfloat16))
    else:
        assert torch.equal(cup.cpu(), hi)
    # weight gradients: dpre from the kernel's own output, autograd of the pre-activation in float64
    dpre = doutd.cpu().to(F64) * _dact(o.to(F64), act, alpha)
    Kr, br, xr = K64.clone().requires_grad_(), b64.clone().requires_grad_(), x64.clone().requires_grad_()
    _pre(xr, Kr, br, utype, s).backward(dpre)
    Ka, ba, xa = K64.abs().requires_grad_(), b64.abs().requires_grad_(), x64.abs().requires_grad_()
    _pre(xa, Ka, ba, utype, s).backward(dpre.abs())
    dK = torch.full(ks, NAN, device=DEV)
    db = torch.full(bs, NAN, device=DEV)
    acc = torch.zeros(dK.numel() + db.numel(), dtype=torch.int64, device=DEV)
    launch(UP_BWD_PARAM, [xd, out, doutd, dK, db, acc], B, C, W, s, utype, act, alpha)
    r_dk = check("dK %s %s s%d" % (utype, act, s), dK.cpu(), Kr.grad, 1e-5 * Ka.grad + 1e-9)
    r_db = check("db %s %s s%d" % (utype, act, s), db.cpu(), br.grad, 1e-5 * ba.grad + 1e-9)
    din = torch.full((B, C, W), NAN, device=DEV)
    launch(UP_BWD_INPUT, [out, doutd, Kd, din], B, C, W, s, utype, act, alpha)
    r_dx = check("din %s %s s%d" % (utype, act, s), din.cpu(), xr.grad, 1e-5 * xa.grad + 1e-30)
    # the weight-gradient sums are reproducible
    dK2, db2 = torch.empty_like(dK), torch.empty_like(db)
    launch(UP_BWD_PARAM, [xd, out, doutd, dK2, db2, acc], B, C, W, s, utype, act, alpha)
    assert torch.equal(dK, dK2) and torch.equal(db, db2)
    return max(r_fwd, r_dk, r_db, r_dx)


@pytest.mark.parametrize("utype", ["SubPixel", "2D", "1D"])
@pytest.mark.parametrize("act", ["Relu", "LeakyRelu", None])
def test_kernel_sweep(utype, act):
    """C = 80, the stock scales 11 (first layer, W = 37 frames) and 25 (second layer, W = 37 * 11), and a scale of 3 over a width
    that leaves a partial 32-position tile"""
    worst = 0.0
    for s, B, W in ((11, 2, 37), (25, 2, 407), (3, 3, 45)):
        worst = max(worst, _sweep_case(utype, act, s, B, 80, W, 100 + s))
    print("MEASURED upsample kernels %s / %s worst err / bound %.3g" % (utype, act, worst))


@pytest.mark.parametrize("C", [1, 6, 13, 128])
def test_1d_kernels_at_other_widths(C):
    """the hook takes any 1 <= C <= 128: odd widths use the scalar loops, 128 the largest shared-memory footprint"""
    print("MEASURED upsample 1D C=%d worst err / bound %.3g" % (C, _sweep_case("1D", "LeakyRelu", 5, 2, C, 40, 200 + C)))


def test_1d_split_rows():
    _sweep_case("1D", "Relu", 4, 2, 80, 33, 300, split=1)
    _sweep_case("SubPixel", "LeakyRelu", 4, 2, 80, 33, 301, split=1)


# ------------------------------------------------------------------------------------------------------------------------------
# pinned to the executed reference (ce_1d)
# ------------------------------------------------------------------------------------------------------------------------------
def test_executed_reference_ce_1d():
    R = np.load(GOLDEN)
    hp = hparams.copy()
    for keys, values in (("small_hparams_keys", "small_hparams_values"), ("ce_1d_hparams_keys", "ce_1d_hparams_values")):
        for k, v in zip(R[keys], R[values]):
            setattr(hp, str(k), eval(str(v)))
    assert hp.upsample_type == "1D" and list(hp.upsample_scales) == [2, 3] and hp.cin_channels == 6
    params = {tb.engine_name("WaveNet_model/" + str(n)): torch.from_numpy(R["ce_1d_var/" + str(n)]) for n in R["ce_1d_var_names"]}
    c = torch.from_numpy(R["c"])                                                   # [2, 6, 4]
    B, C, W0 = c.shape
    K = [params["local_conditioning_upsampling_%d/kernel" % (i + 1)].to(DEV) for i in range(2)]
    bias = [params["local_conditioning_upsampling_%d/bias" % (i + 1)].to(DEV) for i in range(2)]
    act = hp.upsample_activation
    outs, W, x = [], W0, c.to(DEV)
    for i, s in enumerate(hp.upsample_scales):
        o = torch.full((B, C, W * s), NAN, device=DEV)
        launch(UP_FWD, [x, K[i], bias[i], o, None], B, C, W, s, "1D", act)
        outs.append(o)
        x, W = o, W * s
    err_up = np.abs(outs[1].cpu().numpy() - R["ce_1d_upsampled_c"]).max()
    assert err_up <= 2e-6
    # d loss / d c_up from the oracle on the same fixture (recorded dropout masks), fed into the backward launches
    cu = ow.upsample(c, params, hp).detach().requires_grad_(True)
    masks = [torch.from_numpy(R["ce_1d_mask_%d" % l]) for l in range(hp.layers)]
    y_hat = ow.step(torch.from_numpy(R["ce_1d_x"]), cu, params, hp, dropout_masks=masks, c_is_upsampled=True)
    y = torch.from_numpy(R["ce_1d_y"])[:, :, 0].long()
    ow.loss_fn(y_hat, y, torch.from_numpy(R["input_lengths"]).long(), hp).backward()
    dout = cu.grad.contiguous().to(DEV)
    grads = {}
    for i in (1, 0):
        s, Wi = hp.upsample_scales[i], outs[i].shape[2] // hp.upsample_scales[i]
        layer_in = outs[0] if i == 1 else c.to(DEV)
        dK, db = torch.full_like(K[i], NAN), torch.full_like(bias[i], NAN)
        acc = torch.zeros(dK.numel() + db.numel(), dtype=torch.int64, device=DEV)
        launch(UP_BWD_PARAM, [layer_in, outs[i], dout, dK, db, acc], B, C, Wi, s, "1D", act)
        grads[i] = (dK.cpu(), db.cpu())
        if i == 1:
            din = torch.full((B, C, Wi), NAN, device=DEV)
            launch(UP_BWD_INPUT, [outs[i], dout, K[i], din], B, C, Wi, s, "1D", act)
            dout = din
    floor = 1e-3 * max(np.abs(R[k]).max() for k in R.files if k.startswith("ce_1d_grad/"))
    worst = 0.0
    for i in (0, 1):
        for j, leaf in enumerate(("kernel", "bias")):
            ref = R["ce_1d_grad/inference/ConvTranspose1D_layer_%d/%s" % (i, leaf)]
            tol = 2e-4 * max(np.abs(ref).max(), floor)
            e = np.abs(grads[i][j].numpy() - ref).max()
            worst = max(worst, e / tol)
            assert e <= tol, (i, leaf, e, tol)
    print("MEASURED ce_1d upsampled_c max err %.3g; upsampler gradients worst err / bound %.3g" % (err_up, worst))


# ------------------------------------------------------------------------------------------------------------------------------
# end to end (Cfg-2 widths: R256 / G512 / S256)
# ------------------------------------------------------------------------------------------------------------------------------
def _hp(**kw):
    hp = hparams.copy()
    hp.parse("layers=4,stacks=2,residual_channels=256,gate_channels=512,skip_out_channels=256,upsample_scales=[4,4],hop_size=16,"
             "wavenet_dropout=0.0,upsample_type=1D")
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


CE = dict(input_type="mulaw-quantize", quantize_channels=256, out_channels=256)
MOL = dict(input_type="raw", out_channels=30, legacy=False, residual_legacy=False)


def _params(hp, seed):
    """oracle init with random biases; the upsampler kernels leave their NN_init identity so that the activation sees both signs"""
    p = ow.init_params(hp, seed=seed, random_bias=True)
    g = torch.Generator().manual_seed(seed + 1)
    for k in p:
        if k.startswith("local_conditioning_upsampling") and k.endswith("kernel"):
            p[k] = p[k] + 0.2 * torch.randn(p[k].shape, generator=g) / math.sqrt(p[k].shape[-1])
    return p


def _inputs(hp, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    hop = math.prod(hp.upsample_scales)
    c = torch.rand(B, hp.cin_channels, T // hop, generator=g) * 2 - 1
    w = (torch.sin(torch.arange(T) * 0.05)[None] * 0.5 + 0.05 * torch.randn(B, T, generator=g)).clamp(-0.95, 0.95)
    if ow.is_mulaw_quantize(hp.input_type):
        from oracle import audio as oa
        idx = torch.from_numpy(oa.mulaw_quantize(w.numpy()))
        x = torch.nn.functional.one_hot(idx, hp.quantize_channels).float().transpose(1, 2)
        y, xd = idx, idx.int()
    else:
        x, y, xd = w.unsqueeze(1), w, w.clone()
    lengths = torch.tensor([T] + [max(T - 37 * (i + 1), 2) for i in range(B - 1)])
    return x, c, y, lengths, xd


def _run(m, hp, B, T, xd, c, y, lengths, backward=True):
    ldo = 256 if ow.is_mulaw_quantize(hp.input_type) else 32
    logits = torch.zeros(B, T, ldo, device=DEV)
    m.forward(xd.cuda(), c.cuda(), y.int().cuda() if ow.is_mulaw_quantize(hp.input_type) else y.cuda(), lengths.int().cuda(),
              logits=logits, save_for_backward=backward)
    if backward:
        m.backward()
    torch.cuda.synchronize()
    return m.loss_value(), logits[:, :, :hp.out_channels].cpu(), (m.export_grads() if backward else None)


def _compare(tag, hp, B, T, seed, loss_tol, own_dcup=False):
    """own_dcup: the upsampler gradients are checked against float64 autograd of the oracle's upsampler fed the engine's own
    d loss / d c_up (workspace "dc_up") within 2e-3 relative, the other tensors against the fp32 oracle as usual"""
    params = _params(hp, seed)
    x, c, y, lengths, xd = _inputs(hp, B, T, seed)
    m = t2.wavenet.WaveNet(hp, B, T)
    m.load_params(params)
    loss, logits, grads = _run(m, hp, B, T, xd, c, y, lengths)
    loss_ref, grads_ref, yhat_ref = ow.train_step(params, x, c, y, lengths, hp)
    if own_dcup:
        dcup = m.workspace_tensor("dc_up", (B, T, hp.cin_channels)).cpu().to(F64).transpose(1, 2)
        p64 = {k: v.to(F64).requires_grad_(k.startswith("local_conditioning")) for k, v in params.items()}
        ow.upsample(c.to(F64), p64, hp).backward(dcup)
        up_ref = {k: v.grad for k, v in p64.items() if k.startswith("local_conditioning")}
        up_rel = {k: ((grads[k].to(F64) - g).norm() / g.norm()).item() for k, g in up_ref.items()}
        print("MEASURED %s upsampler gradients vs float64 on the engine's dc_up: worst rel %.3g" % (tag, max(up_rel.values())))
        assert max(up_rel.values()) < 2e-3, up_rel
        grads_ref = {k: v for k, v in grads_ref.items() if k not in up_ref}
    gtol = 1e-1
    pre = ow.upsample(c, {k: v for k, v in params.items()}, types.SimpleNamespace(**{**hp.values(), "upsample_activation": "none"}))
    neg = (pre < 0).float().mean().item()
    cup = m.workspace_tensor("c_up", (B, T, hp.cin_channels)).float().cpu()
    cup_err = (cup - ow.upsample(c, params, hp).transpose(1, 2)).abs().max().item()
    err = (logits - yhat_ref.transpose(1, 2)).abs()
    worst, bad = {}, []
    for name, gr in grads_ref.items():
        den = gr.norm().item()
        rel = (grads[name] - gr).norm().item() / max(den, 1e-12)
        if den >= 1e-7:
            worst[name] = rel
            if rel >= gtol:
                bad.append("%s rel %.4g |ref| %.3g" % (name, rel, den))
    up_worst = max([v for k, v in worst.items() if k.startswith("local_conditioning")] or [0.0])
    print("MEASURED %s loss err %.3g logits max %.3g mean %.3g c_up max %.3g worst grad rel %.4g (upsampler %.4g) vs the fp32 oracle; "
          "%.2f of the pre-activations < 0" % (tag, abs(loss - loss_ref.item()), err.max().item(), err.mean().item(), cup_err,
                                               max(worst.values()), up_worst, neg))
    assert 0.05 < neg < 0.95
    assert cup_err < 1e-2
    assert abs(loss - loss_ref.item()) < loss_tol
    assert err.max().item() < 8e-3 and err.mean().item() < 1.5e-3
    assert not bad, bad
    assert sum(k.startswith("local_conditioning") for k in worst) == (0 if own_dcup else 2 * len(hp.upsample_scales))
    return m, params, (x, c, y, lengths, xd), grads


@pytest.mark.parametrize("kind,utype,act", [("ce", "1D", "Relu"), ("mol", "1D", "Relu"), ("ce", "1D", "LeakyRelu"), ("mol", "1D", None)])
def test_training_matches_oracle(kind, utype, act):
    hp = _hp(upsample_type=utype, upsample_activation=act, **(CE if kind == "ce" else MOL))
    _compare("upsample_%s_%s_%s_B3xT512" % (kind, utype, act), hp, 3, 512, 51, 1e-4 if kind == "ce" else 6e-4)


@pytest.mark.parametrize("kind,utype,act", [("ce", "SubPixel", "LeakyRelu"), ("mol", "2D", None)])
def test_training_new_activations_on_subpixel_and_2d(kind, utype, act):
    """The SubPixel / 2D bias gradients are sums over every position of one phase. Without ReLU zeroing half of the terms they cancel
    heavily, so the bf16 rounding of the gradient chain upstream shows in full (measured on an H100: the last layer's SubPixel bias
    gradient under LeakyReLU is 0.106 relative to the fp32 oracle and 0.063 relative to the bf16-storage oracle, norm 1.4e-3). The
    upsampler gradients are therefore checked on the engine's own d loss / d c_up, which isolates the path this change adds."""
    hp = _hp(upsample_type=utype, upsample_activation=act, **(CE if kind == "ce" else MOL))
    _compare("upsample_%s_%s_%s_B3xT512" % (kind, utype, act), hp, 3, 512, 51, 1e-4 if kind == "ce" else 6e-4, own_dcup=True)


def test_backward_is_reproducible_and_adam_matches_oracle():
    hp = _hp(upsample_activation="LeakyRelu", **CE)
    B, T = 3, 512
    m, params, (x, c, y, lengths, xd), grads = _compare("upsample_ce_1D_leaky_adam", hp, B, T, 52, 1e-4)
    _, _, again = _run(m, hp, B, T, xd, c, y, lengths)
    for k in grads:
        assert torch.equal(grads[k], again[k]), k
    # the phased backward (data-parallel overlap: the conditioning path on the side stream) gives the same bits
    m.backward(0, 2)
    m.backward(100, 2)
    for gi in range(2):
        m.backward(1 + gi, 2)
    torch.cuda.synchronize()
    phased = m.export_grads()
    for k in grads:
        assert torch.equal(grads[k], phased[k]), k
    state, p_ref = {}, {k: v.clone() for k, v in params.items()}
    ow.adam_step(p_ref, grads, state, hp, 0)
    m.optimizer_step()
    torch.cuda.synchronize()
    p_new, ema = m.export_params(), m.unflatten(m.ema)
    for k in p_ref:
        assert (p_new[k] - p_ref[k]).abs().max().item() < 2e-6, k
        assert (ema[k] - state["ema"][k]).abs().max().item() < 2e-6, k


def test_fp32_class_forward():
    hp = _hp(upsample_activation="LeakyRelu", **MOL)
    B, T = 2, 256
    params = _params(hp, 53)
    x, c, y, lengths, xd = _inputs(hp, B, T, 53)
    m = t2.wavenet.WaveNet(hp, B, T, precision="fp32-class")
    m.load_params(params)
    loss, logits, _ = _run(m, hp, B, T, xd, c, y, lengths, backward=False)
    loss_ref, _, yhat = ow.train_step(params, x, c, y, lengths, hp)
    err = (logits - yhat.transpose(1, 2)).abs().max().item()
    print("MEASURED upsample 1D fp32-class logits max err %.3g loss err %.3g" % (err, abs(loss - loss_ref.item())))
    assert err < 1e-4 and abs(loss - loss_ref.item()) < 1e-4


def test_ar_conditioning_equals_training_and_teacher_forced_ar_matches_oracle():
    hp = _hp(upsample_activation="LeakyRelu", **CE)
    B, T = 3, 48
    g = torch.Generator().manual_seed(54)
    params = _params(hp, 54)
    idx = torch.randint(90, 166, (B, T), generator=g)
    c = torch.rand(B, 80, T // 16, generator=g) * 2 - 1
    syn = t2.wavenet.WaveNetSynthesizer(hp, B, T, cluster_size=8)
    syn.load_params(params)
    ti = torch.cat([idx[:, 1:], idx[:, -1:]], dim=1).int().cuda()
    _, raw = syn.generate(c.cuda(), idx[:, 0].int().cuda(), test_inputs=ti, u_a=torch.rand(B, T, generator=g).cuda(), return_raw=True)
    torch.cuda.synchronize()
    # c_up is the first buffer of the synthesis workspace (bf16 [B][T][cin]); the training forward builds it with the same launches
    cup_ar = syn.workspace[:B * T * 80 * 2].view(torch.bfloat16).reshape(B, T, 80).clone()
    m = t2.wavenet.WaveNet(hp, B, T)
    m.load_params(params)
    _run(m, hp, B, T, idx.int(), c, idx, torch.full((B,), T), backward=False)
    assert torch.equal(cup_ar, m.workspace_tensor("c_up", (B, T, 80)))
    onehot = torch.nn.functional.one_hot(idx, 256).float()
    _, ref = ow.incremental(onehot[:, :1], c, params, hp, T, test_inputs=torch.cat([onehot[:, 1:], onehot[:, -1:]], 1),
                            u_cat=torch.full((B, T), 0.5))
    err = (raw.cpu() - ref).abs()
    print("MEASURED upsample 1D LeakyReLU AR mulaw raw max err %.3g mean %.3g" % (err.max().item(), err.mean().item()))
    assert err.max().item() < 4e-2 and err.mean().item() < 6e-3


def test_dropin_model_trains_with_1d_leaky():
    from wavenet_vocoder.models import create_model
    from wavenet_vocoder.util import mulaw_quantize
    hp = _hp(residual_channels=128, gate_channels=256, skip_out_channels=128, wavenet_dropout=0.05, upsample_activation="LeakyRelu", **CE)
    model = create_model("WaveNet", hp)
    g = torch.Generator().manual_seed(0)
    B, T = 2, 512
    wav = (torch.sin(torch.arange(T) * 0.05)[None] * 0.5 + 0.02 * torch.randn(B, T, generator=g)).clamp(-1, 1)
    idx = torch.from_numpy(mulaw_quantize(wav.numpy())).cuda()
    x = torch.nn.functional.one_hot(idx.long(), 256).float().transpose(1, 2)
    c = (torch.rand(B, 80, T // 16, generator=g) * 2 - 1).cuda()
    lengths = torch.tensor([T, T - 40]).cuda()
    losses = []
    for step in range(30):
        model.initialize(idx.unsqueeze(-1), c, None, lengths, x=x)
        losses.append(float(model.add_loss()))
        model.add_optimizer(step)
    print("MEASURED upsample 1D LeakyReLU drop-in loss %.4f -> %.4f" % (losses[0], losses[-1]))
    assert losses[-1] < 0.9 * losses[0], losses
    model.initialize(None, c[:, :, :2].transpose(1, 2).contiguous(), None, None)
    assert model.tower_y_hat[0].shape == (B, 32)
