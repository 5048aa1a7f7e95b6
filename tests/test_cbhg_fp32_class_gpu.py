"""The fp32-class (split bf16) mode of the CBHG post-processing net + linear head against the fp32 oracle (oracle.tacotron.linear_head):
the engine alone on a given mel (training and inference), stage by stage, through Tacotron.linear_from_mel, chained behind the
fp32-class Tacotron at Cfg-3 widths (deterministic and with the device's dropout / zoneout masks), after free-running synthesis, and
the changed kernels one launch at a time (split gru_fwd_kernel against a float64 recurrence re-anchored every step on the kernel's own
outputs, split max-pool exactly, split highway). The linear gate is the 1e-3 mean |error| parity target wherever the oracle sees the same
input; the other bounds are about twice the values measured on an H100."""
import ctypes

import pytest
import torch

from hparams import hparams
from oracle import tacotron as ot
from parity_util import record
from t2_import import t2
from test_parity_full_gpu import taco_batch, taco_masks
from test_tacotron_gpu import _trained_like_stats

pytestmark = pytest.mark.gpu
L = t2.lib
F64 = torch.float64
LIN_L1 = 1e-3          # BASELINE.json parity target, applied to the linear spectrogram
HU, RU = 128, 128
U, SF = 2.0 ** -24, 2.0 ** -16          # fp32 unit roundoff; relative error of a hi + lo pair
POOL_FWD, HIGHWAY_FWD, GRU_FWD = 3, 5, 7


def _hp(stochastic=False, **kw):
    hp = hparams.copy()
    hp.parse("predict_linear=True" + ("" if stochastic else ",tacotron_dropout_rate=0.0,tacotron_zoneout_rate=0.0"))
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


def _pairs(t, n):
    """recombine rows [hi(n) | lo(n)] (split workspace tensors) into fp32 [..., n]"""
    t = t.reshape(-1, 2 * n).float()
    return t[:, :n] + t[:, n:]


def _ws(cfg, ws, name):
    p, cnt = ctypes.c_void_p(), ctypes.c_longlong()
    L.check(L.load().t2_cbhg_workspace_tensor(ctypes.byref(cfg), L.ptr(ws), name.encode(), ctypes.byref(p), ctypes.byref(cnt)))
    off = p.value - ws.data_ptr()
    return ws[off:off + cnt.value * 2].view(torch.bfloat16)


def _engine(hp, params, mel, lin_t, tl, training, B, T):
    """the CBHG engine of an fp32-class Tacotron model driven directly on `mel`; returns (model, linear outputs, linear loss)"""
    model = t2.tacotron.Tacotron(hp, B, 16, T, precision="fp32-class")
    model.load_params(params)
    model.pack()
    lib, cfg = model.lib, ctypes.byref(model.cbhg)
    mel_d, lin_d = mel.cuda().contiguous(), lin_t.cuda().contiguous()     # held until the forward has run
    if tl is not None:
        tl_d = tl.int().cuda()
        L.check(lib.t2_cbhg_set_target_lengths(cfg, L.ptr(model.cb_workspace), L.ptr(tl_d), L.stream_ptr()))
    L.check(lib.t2_cbhg_forward(cfg, L.ptr(model.params[model.n_taco:]), L.ptr(model.cb_packed), L.ptr(model.cb_workspace),
                                L.ptr(mel_d), L.ptr(lin_d), L.ptr(model.cb_loss), int(training), L.stream_ptr()))
    torch.cuda.synchronize()
    return model, model.linear_outputs().cpu(), model.cb_loss[0].item()


def _inputs(hp, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    mel = (torch.randn(B, T, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    lin_t = (torch.randn(B, T, hp.num_freq, generator=g) * 1.5 - 1).clamp(-4, 4)
    tl = torch.tensor([T] + [max(T - 6 * (i + 1), 4) for i in range(B - 1)])
    return mel, lin_t, tl


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("B,T,mask,stock", [(5, 37, False, False), (8, 64, True, False), (32, 200, False, True)])
def test_engine_matches_oracle(B, T, mask, stock, training):
    hp = _hp(mask_decoder=mask) if stock else _hp(mask_decoder=mask, num_freq=513)
    params = ot.init_params(hp, seed=11, random_bias=True)
    if not training:
        params = _trained_like_stats(params, 11)
    mel, lin_t, tl = _inputs(hp, B, T, 5)
    with torch.no_grad():
        ref = ot.linear_head(mel, params, hp, training)
        loss_ref = ot.linear_loss(lin_t, ref, hp, tl if mask else None).item()
    _, lin, loss = _engine(hp, params, mel, lin_t, tl if mask else None, training, B, T)
    m = record("cbhg_fp32_class_engine_B%d_T%d_%s" % (B, T, "train" if training else "eval"), lin_l1=(lin - ref).abs().mean().item(),
               lin_max=(lin - ref).abs().max().item(), loss_err=abs(loss - loss_ref))
    assert m["lin_l1"] <= LIN_L1 and m["lin_max"] < 5e-5 and m["loss_err"] < 1.1e-5, m


def test_stages():
    """bank (after batch norm), pooled, GRU input (last highway output) and GRU outputs of one training forward, pairs recombined"""
    hp = _hp(num_freq=513)
    B, T = 8, 64
    params = ot.init_params(hp, seed=12, random_bias=True)
    mel, lin_t, _ = _inputs(hp, B, T, 6)
    model, _, _ = _engine(hp, params, mel, lin_t, None, True, B, T)
    P = "CBHG_postnet/"
    with torch.no_grad():
        bank = torch.cat([ot.conv_block(mel, params, P + "conv_bank/conv1d_%d/" % k, "relu", True, 0.0) for k in range(1, hp.cbhg_kernels + 1)], dim=-1)
        pooled = torch.maximum(bank, torch.cat([bank[:, 1:], torch.full_like(bank[:, :1], float("-inf"))], dim=1))
        p1 = ot.conv_block(pooled, params, P + "proj1/", "relu", True, 0.0)
        h = ot.conv_block(p1, params, P + "proj2/", None, True, 0.0) + mel
        h = h @ params[P + "dense/kernel"] + params[P + "dense/bias"]
        for i in range(hp.cbhg_highwaynet_layers):
            q = P + "highwaynet_%d/" % (i + 1)
            Tt = torch.sigmoid(h @ params[q + "T/kernel"] + params[q + "T/bias"])
            h = torch.relu(h @ params[q + "H/kernel"] + params[q + "H/bias"]) * Tt + h * (1.0 - Tt)
        rnn = ot.cbhg(mel, params, hp, True)
    KC = hp.cbhg_kernels * hp.cbhg_conv_channels
    cfg, ws = model.cbhg, model.cb_workspace
    got = {k: _pairs(_ws(cfg, ws, k).cpu(), n).reshape(B, T, n) for k, n in
           (("bank_outputs", KC), ("pooled_outputs", KC), ("gru_input", HU), ("rnn_outputs", 2 * RU))}
    m = record("cbhg_fp32_class_stages", bank_max=(got["bank_outputs"] - bank).abs().max().item(),
               pooled_max=(got["pooled_outputs"] - pooled).abs().max().item(), gru_in_max=(got["gru_input"] - h).abs().max().item(),
               rnn_max=(got["rnn_outputs"] - rnn).abs().max().item())
    assert m["bank_max"] < 3.6e-4 and m["pooled_max"] < 3.6e-4 and m["gru_in_max"] < 1e-4 and m["rnn_max"] < 2.7e-5, m


def test_linear_from_mel_with_moving_statistics():
    """B = 6 (not a multiple of 4): the inference engine linear_from_mel builds, with non-trivial moving statistics"""
    hp = _hp(num_freq=513)
    params = _trained_like_stats(ot.init_params(hp, seed=13, random_bias=True), 13)
    mel, _, _ = _inputs(hp, 6, 45, 7)
    model = t2.tacotron.Tacotron(hp, 6, 16, 45, precision="fp32-class")
    model.load_params(params)
    lin = model.linear_from_mel(mel.cuda()).cpu()
    with torch.no_grad():
        ref = ot.linear_head(mel, params, hp, False)
    m = record("cbhg_fp32_class_linear_from_mel", lin_l1=(lin - ref).abs().mean().item(), lin_max=(lin - ref).abs().max().item())
    assert m["lin_l1"] <= LIN_L1 and m["lin_max"] < 5e-5, m


@pytest.mark.parametrize("stochastic", [False, True])
def test_chained_cfg3(stochastic):
    """Tacotron(precision='fp32-class') with predict_linear at Cfg-3 widths, B = 32, T_in 160, T_out 200; stochastic: dropout 0.5 and
    zoneout 0.1 with the device's masks injected into the oracle. mel_outputs within the bounds of the Tacotron fp32-class tests."""
    hp = _hp(stochastic)
    B, T_in, T_out = 32, 160, 200
    params = ot.init_params(hp, seed=61, random_bias=True)
    inputs, lens, mel, stop = taco_batch(hp, B, T_in, T_out, 61)
    lin_t = (torch.randn(B, T_out, hp.num_freq, generator=torch.Generator().manual_seed(61)) * 1.5 - 1).clamp(-4, 4)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out, precision="fp32-class")
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=True, seed=99, linear_targets=lin_t.cuda())
    torch.cuda.synchronize()
    masks = taco_masks(model, hp, B, T_in, T_out)
    with torch.no_grad():
        ref = ot.forward(params, inputs, lens, mel, hp, training=True, masks=masks)
        loss_ref = ot.linear_loss(lin_t, ref["linear_outputs"], hp).item()
    melo = model.workspace_tensor("mel_outputs", (B, T_out, hp.num_mels)).cpu()
    lin = model.linear_outputs().cpu()
    m = record("cbhg_fp32_class_chained_cfg3_%s" % ("stochastic" if stochastic else "deterministic"),
               mel_l1=(melo - ref["mel_outputs"]).abs().mean().item(), lin_l1=(lin - ref["linear_outputs"]).abs().mean().item(),
               lin_max=(lin - ref["linear_outputs"]).abs().max().item(), loss_err=abs(model.cb_loss[0].item() - loss_ref))
    assert m["mel_l1"] <= 1e-3 and m["mel_l1"] < 1.3e-4 and m["lin_l1"] <= LIN_L1 and m["lin_max"] < 1.3e-4 and m["loss_err"] < 2.1e-5, m


def test_backward_fails_in_the_library():
    hp = _hp(num_freq=513)
    B, T_in, T_out = 4, 24, 20
    params = ot.init_params(hp, seed=63, random_bias=True)
    inputs, lens, mel, stop = taco_batch(hp, B, T_in, T_out, 63)
    model = t2.tacotron.Tacotron(hp, B, T_in, T_out, precision="fp32-class")
    model.load_params(params)
    model.forward(inputs.int().cuda(), lens.int().cuda(), mel.cuda(), stop.cuda(), training=True,
                  linear_targets=torch.zeros(B, T_out, hp.num_freq).cuda())
    with pytest.raises(L.T2Error, match="no backward pass"):
        model.backward()


def test_synthesis_then_linear_from_mel():
    """120 free-running synthesis steps (stop bias held low), then linear_from_mel on the synthesised mel_outputs; the oracle runs the
    linear head on the same synthesised frames (its input), and on its own synthesis for the end-to-end figure"""
    hp = _hp(tacotron_zoneout_rate=0.1)
    B, T_in, steps = 8, 120, 120
    params = _trained_like_stats(ot.init_params(hp, seed=66, random_bias=True), 66)
    params["stop_token_projection/bias"] = torch.full((1,), -20.0)
    inputs, lens, _, _ = taco_batch(hp, B, T_in, steps, 66)
    model = t2.tacotron.Tacotron(hp, B, T_in, steps, precision="fp32-class")
    model.load_params(params)
    out = model.synthesize(inputs.int().cuda(), lens.int().cuda(), chunk=32)
    assert out["T"] == steps
    lin = model.linear_from_mel(out["mel_outputs"]).cpu()
    with torch.no_grad():
        ref = ot.synthesize(params, inputs, lens, hp, max_iters=steps)
        ref_same = ot.linear_head(out["mel_outputs"].cpu().float(), params, hp, False)
        ref_own = ot.linear_head(ref["mel_outputs"], params, hp, False)
    m = record("cbhg_fp32_class_synthesis_120", mel_l1=(out["mel_outputs"].cpu() - ref["mel_outputs"]).abs().mean().item(),
               lin_l1=(lin - ref_same).abs().mean().item(), lin_max=(lin - ref_same).abs().max().item(),
               lin_l1_end_to_end=(lin - ref_own).abs().mean().item())
    assert m["mel_l1"] < 2e-5 and m["lin_l1"] <= LIN_L1 and m["lin_max"] < 7e-6 and m["lin_l1_end_to_end"] <= LIN_L1, m


# ---- one launch at a time --------------------------------------------------------------------------------------------------------
def _launch(kernel, p, i):
    c = L.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate(i):
        c.i[k] = int(v)
    L.check(L.load().t2_dbg_cbhg_kernel(ctypes.byref(c), L.stream_ptr()))
    torch.cuda.synchronize()


def _split(x):
    """fp32 [..., n] -> rows [hi(n) | lo(n)] as the kernels store them"""
    hi = x.to(torch.bfloat16)
    return torch.cat([hi, (x - hi.float()).to(torch.bfloat16)], dim=-1)


def test_split_maxpool_is_exact():
    B, T, C = 5, 37, 1024
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B * T, C, generator=g)
    x[::7] = x[1::7][:x[::7].shape[0]]              # ties between neighbours
    xs = _split(x).cuda()
    out = torch.full_like(xs, float("nan"))
    _launch(POOL_FWD, [xs, out], [B * T, T, C, 1])
    v = _pairs(xs.cpu(), C).reshape(B, T, C)
    nxt = torch.cat([v[:, 1:], torch.full_like(v[:, :1], float("-inf"))], dim=1)
    take = (nxt > v).reshape(B * T, C)
    xr = xs.cpu().reshape(B, T, 2 * C)
    ref = torch.where(torch.cat([take, take], dim=-1), torch.cat([xr[:, 1:], xr[:, :1]], dim=1).reshape(B * T, 2 * C), xs.cpu())
    assert torch.equal(out.cpu().view(torch.int16), ref.view(torch.int16))


def test_split_highway():
    N = 8 * 37
    g = torch.Generator().manual_seed(4)
    pre, h = torch.randn(N, 2 * HU, generator=g) * 2, torch.randn(N, HU, generator=g)
    bh, bt = torch.randn(HU, generator=g) * 0.5, torch.randn(HU, generator=g) * 0.5
    hf = torch.full((N, HU), float("nan"), device="cuda")
    hb = torch.full((N, 2 * HU), float("nan"), device="cuda").to(torch.bfloat16)
    _launch(HIGHWAY_FWD, [pre.cuda(), bh.cuda(), bt.cuda(), h.cuda(), hf, hb, None], [N, HU, 1])
    p64 = pre.to(F64)
    Hh = torch.relu(p64[:, :HU] + bh.to(F64))
    Tt = torch.sigmoid(p64[:, HU:] + bt.to(F64))
    ref = Hh * Tt + h.to(F64) * (1 - Tt)
    bound = 2 * (Tt * (1 - Tt) * (Hh - h.to(F64)).abs() * 2.0 ** -20 * (1 + (p64[:, HU:] + bt.to(F64)).abs()) + 16 * U * (Hh.abs() + h.to(F64).abs())) + 1e-30
    err_f = (hf.cpu().to(F64) - ref).abs()
    got_b = _pairs(hb.cpu(), HU).to(F64)
    err_b = (got_b - ref).abs()
    m = record("cbhg_fp32_class_highway", hf_ratio=(err_f / bound).max().item(), hb_ratio=(err_b / (bound + SF * ref.abs())).max().item())
    assert m["hf_ratio"] <= 1.0 and m["hb_ratio"] <= 1.0, m
    assert torch.equal(_split(hf.cpu()).view(torch.int16), hb.cpu().view(torch.int16)), "hb must be the split of hf"


def _gru_reference(XP, Ws, anchor):
    """float64 GRU with the exact fp32 recurrent weights, re-anchored every step on the kernel's own recombined output of the previous
    step (known to 2^-16 relative). Per step: dots 130 u sum|terms| + 2^-16 sum|h W| (the hi + lo weights) + the carried anchor error;
    sigmoid / tanh / update as tests/gru_reference.py; the stored pair 2^-16 |h|; a factor-2 margin."""
    B, T, _ = XP.shape
    X = XP.to(F64)
    out = torch.zeros(B, T, 2 * RU, dtype=F64)
    bnd = torch.zeros_like(out)
    for d in range(2):
        W = Ws[d]
        Wg, Wc = W["gk"][HU:].to(F64), W["ck"][HU:].to(F64)
        Wga, Wca = Wg.abs(), Wc.abs()
        bg, bc = W["gb"].to(F64), W["cb"].to(F64)
        order = range(T) if d == 0 else range(T - 1, -1, -1)
        prev = None
        for t in order:
            h = torch.zeros(B, RU, dtype=F64) if prev is None else anchor[:, prev, d * RU:(d + 1) * RU].to(F64)
            dh = h.abs() * SF
            xg, xc = X[:, t, d * 3 * RU:d * 3 * RU + 2 * RU], X[:, t, d * 3 * RU + 2 * RU:(d + 1) * 3 * RU]
            a = xg + bg + h @ Wg
            da = 130 * U * (xg.abs() + bg.abs() + h.abs() @ Wga) + SF * (h.abs() @ Wga) + dh @ Wga
            gt = torch.sigmoid(a)
            dg = gt * (1 - gt) * (da + 2.0 ** -21 * (1 + a.abs())) + 2 * U * gt
            r, u, dr, du = gt[:, :RU], gt[:, RU:], dg[:, :RU], dg[:, RU:]
            rh = r * h
            drh = h.abs() * dr + r * dh + U * rh.abs()
            pc = xc + bc + rh @ Wc
            dpc = 130 * U * (xc.abs() + bc.abs() + rh.abs() @ Wca) + SF * (rh.abs() @ Wca) + drh @ Wca
            c = torch.tanh(pc)
            dc = (1 - c * c) * dpc + 4 * U * c.abs()
            hn = u * h + (1 - u) * c
            dhn = (h - c).abs() * du + u * dh + (1 - u) * dc + 8 * U * ((u * h).abs() + ((1 - u) * c).abs())
            out[:, t, d * RU:(d + 1) * RU] = hn
            bnd[:, t, d * RU:(d + 1) * RU] = 2 * dhn + 2 * SF * hn.abs() + 1e-30
            prev = t
    return out, bnd


@pytest.mark.parametrize("B,T", [(1, 2), (5, 37), (9, 200)])
def test_split_gru_fwd(B, T):
    g = torch.Generator().manual_seed(B * 100 + T)
    p = ot.init_params(_hp(), seed=B + T, random_bias=True)
    parts, offs, Ws, o = [], [], [], 0
    for n in ("forward", "backward"):
        q = "CBHG_postnet/%s_RNN/" % n
        W = dict(gk=p[q + "gates/kernel"], ck=p[q + "candidate/kernel"], gb=torch.randn(2 * RU, generator=g) * 0.3, cb=torch.randn(RU, generator=g) * 0.3)
        Ws.append(W)
        d = {}
        for k in ("gk", "ck", "gb", "cb"):
            d[k] = o
            parts.append(W[k].reshape(-1))
            o += W[k].numel()
        offs.append(d)
    flat = torch.cat(parts).cuda()
    XP = torch.randn(B, T, 6 * RU, generator=g)
    N = B * T
    out = torch.full((N + 3, 4 * RU), float("nan"), device="cuda").to(torch.bfloat16)
    ints = [B, T, HU, RU]
    for d in range(2):
        ints += [offs[d]["gk"], offs[d]["ck"], offs[d]["gb"], offs[d]["cb"]]
    _launch(GRU_FWD, [flat, XP.cuda(), out] + [None] * 8, ints + [1])
    got = _pairs(out[:N].cpu(), 2 * RU).reshape(B, T, 2 * RU)
    assert torch.isnan(out[N:].float()).all(), "written past row N"
    ref, bnd = _gru_reference(XP, Ws, got)
    m = record("cbhg_fp32_class_gru_fwd_B%d_T%d" % (B, T), worst_err_over_bound=((got.to(F64) - ref).abs() / bnd).max().item(),
               max_err=(got.to(F64) - ref).abs().max().item())
    assert m["worst_err_over_bound"] <= 1.0, m
