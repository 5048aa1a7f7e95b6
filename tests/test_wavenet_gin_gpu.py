"""Global (speaker) conditioning on the H100: training forward / backward / Adam, the fp32-class forward and AR synthesis against the
fp32 CPU oracle with speaker ids (tests/wavenet_gin_oracle.py), plus exact properties of the per-item gate bias.

Bounds, and why they are those of the gin-off tests:
  The speaker term enters every layer as a per-item gate bias b_gin + W_gin^T emb[id] computed in fp32 and added in fp32 inside the
  gate epilogue, the same way as the fused b_dil + b_cin. It adds no bf16 rounding of its own, so the bf16-path deviation from the fp32
  oracle is that of tests/test_wavenet_gpu.py: loss <= 1e-4 (CE) / 6e-4 (MoL), logits max <= 8e-3 and mean <= 1.5e-3, and every
  gradient tensor within 1e-1 relative (L2) of the fp32 oracle. The gin gradients are sums of the same d gate pre-activations that the
  gate-bias gradients sum (their bound is met there), weighted by the fp32 embedding, so they carry the same relative error.
  dW_gin and d gc_embedding are finished in fp32 from 64-bit fixed-point sums in a fixed order: two backward runs are bit-identical.
  With zero gin weights and a zero embedding the per-item bias is bias_g + (0 + 0) == bias_g exactly, so logits and gradients equal
  the gin-off engine bit for bit (the loss is a float atomic sum: equal up to its last bits).
  fp32-class forward: logits <= 1e-4 (tests/test_precision_modes_gpu.py). AR: the bounds of tests/test_wavenet_ar_gpu.py.
MEASURED lines are printed for the record."""
import math

import pytest
import torch

from hparams import hparams
from oracle import wavenet as ow
from t2_import import t2
from wavenet_gin_oracle import incremental_g, train_step_g

pytestmark = pytest.mark.gpu


def _hp(**kw):
    hp = hparams.copy()
    hp.parse("layers=4,stacks=2,residual_channels=256,gate_channels=512,skip_out_channels=256,upsample_scales=[4,4],hop_size=16,"
             "wavenet_dropout=0.0,gin_channels=16,n_speakers=4,use_speaker_embedding=True")
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


CE = dict(input_type="mulaw-quantize", quantize_channels=256, out_channels=256)
MOL = dict(input_type="raw", out_channels=30, legacy=False, residual_legacy=False, upsample_type="2D")


def _inputs(hp, B, T, seed, same_items=False):
    g = torch.Generator().manual_seed(seed)
    hop = math.prod(hp.upsample_scales)
    c = torch.rand(B, hp.cin_channels, T // hop, generator=g)
    w = (torch.sin(torch.arange(T) * 0.05)[None] * 0.5 + 0.05 * torch.randn(B, T, generator=g)).clamp(-0.95, 0.95)
    if same_items:
        c, w = c[:1].expand_as(c).contiguous(), w[:1].expand_as(w).contiguous()
    if ow.is_mulaw_quantize(hp.input_type):
        from oracle import audio as oa
        idx = torch.from_numpy(oa.mulaw_quantize(w.numpy()))
        x = torch.nn.functional.one_hot(idx, hp.quantize_channels).float().transpose(1, 2)
        y, xd = idx, idx.int()
    else:
        x, y, xd = w.unsqueeze(1), w, w.clone()
    lengths = torch.full((B,), T) if same_items else torch.tensor([T] + [max(T - 37 * (i + 1), 2) for i in range(B - 1)])
    return x, c, y, lengths, xd


def _params(hp, seed):
    p = ow.init_params(hp, seed=seed, random_bias=True)
    p["gc_embedding"] = p["gc_embedding"] * 4          # speaker terms of the size of the other gate inputs
    return p


def _engine(hp, B, T, params, **kw):
    m = t2.wavenet.WaveNet(hp, B, T, **kw)
    m.load_params(params)
    return m


def _run(m, hp, B, T, xd, c, y, lengths, speakers=None, seed=None, backward=True):
    ldo = 256 if ow.is_mulaw_quantize(hp.input_type) else 32
    logits = torch.zeros(B, T, ldo, device="cuda")
    if speakers is not None:
        m.set_speakers(speakers)
    m.forward(xd.cuda(), c.cuda(), y.int().cuda() if ow.is_mulaw_quantize(hp.input_type) else y.cuda(), lengths.int().cuda(),
              logits=logits, save_for_backward=backward, seed=seed)
    if backward:
        m.backward()
    torch.cuda.synchronize()
    return m.loss_value(), logits[:, :, :hp.out_channels].cpu(), (m.export_grads() if backward else None)


def _compare(tag, hp, B, T, seed, ids, loss_tol):
    params = _params(hp, seed)
    x, c, y, lengths, xd = _inputs(hp, B, T, seed)
    m = _engine(hp, B, T, params)
    loss, logits, grads = _run(m, hp, B, T, xd, c, y, lengths, speakers=ids, seed=77)
    masks = None
    if hp.wavenet_dropout > 0:        # the masks the kernels drew, read back from the dropped-activation stash
        keep = 1.0 - hp.wavenet_dropout
        xs = m.workspace_tensor("x", (hp.layers, B, T, hp.residual_channels))
        xds = m.workspace_tensor("xd", (hp.layers, B, T, hp.residual_channels))
        kept = (xds != 0) | (xs == 0)
        masks = [(kept[l].float() / keep).transpose(1, 2).cpu() for l in range(hp.layers)]
    g = torch.tensor(ids).reshape(B, 1)
    loss_ref, grads_ref, yhat_ref = train_step_g(params, x, c, y, lengths, hp, g=g, dropout_masks=masks)
    err = (logits - yhat_ref.transpose(1, 2)).abs()
    worst, bad = {}, []
    for name, gr in grads_ref.items():
        den = gr.norm().item()
        rel = (grads[name] - gr).norm().item() / max(den, 1e-12)
        if den >= 1e-7:
            worst[name] = rel
            if rel >= 1e-1:
                bad.append("%s rel %.4g |ref| %.3g" % (name, rel, den))
    gin_worst = max(v for k, v in worst.items() if "gin" in k or k == "gc_embedding")
    print("MEASURED %s loss err %.3g logits max %.3g mean %.3g worst grad rel %.4g (gin tensors %.4g)" % (
        tag, abs(loss - loss_ref.item()), err.max().item(), err.mean().item(), max(worst.values()), gin_worst))
    assert abs(loss - loss_ref.item()) < loss_tol
    assert err.max().item() < 8e-3 and err.mean().item() < 1.5e-3
    assert not bad, bad
    for name in ["gc_embedding"] + ["ResidualConv1DGLU_%d/residual_block_gin_conv/%s" % (l, k) for l in range(hp.layers)
                                    for k in ("kernel", "bias")]:
        assert name in worst, name            # every speaker tensor has a gradient the check covered
    return m, params, grads, grads_ref


@pytest.mark.parametrize("kind", ["ce", "mol"])
def test_training_matches_oracle(kind):
    hp = _hp(wavenet_dropout=0.05, **(CE if kind == "ce" else MOL))
    _compare("gin_%s_B4xT512" % kind, hp, 4, 512, 31, [2, 0, 3, 1], 1e-4 if kind == "ce" else 6e-4)


def test_training_matches_oracle_ragged_T():
    hp = _hp(upsample_scales=[5, 4], hop_size=20, **CE)
    _compare("gin_ce_B3xT400", hp, 3, 400, 32, [3, 1, 0], 1e-4)


def test_shared_speaker_rows_sum_and_unused_rows_are_zero():
    hp = _hp(**CE)
    m, params, grads, grads_ref = _compare("gin_ce_shared_speakers", hp, 4, 256, 33, [1, 3, 1, 3], 1e-4)
    d = grads["gc_embedding"]
    assert (d[0] == 0).all() and (d[2] == 0).all()
    assert (d[1] != 0).any() and (d[3] != 0).any()
    # both items of speaker 1 add into its row: the row differs from what either item alone gives
    x, c, y, lengths, xd = _inputs(hp, 4, 256, 33)
    _, _, g_one = _run(m, hp, 4, 256, xd, c, y, lengths, speakers=[1, 3, 0, 2], seed=77)
    assert (g_one["gc_embedding"][1] - d[1]).abs().max() > 0


def test_zero_speaker_weights_and_no_ids_equal_gin_off_bitwise():
    hp = _hp(**CE)
    hp_off = _hp(gin_channels=-1, **CE)
    B, T = 2, 384
    params = _params(hp, 34)
    off_params = {k: v for k, v in params.items() if "gin" not in k and k != "gc_embedding"}
    x, c, y, lengths, xd = _inputs(hp, B, T, 34)
    ref_loss, ref_logits, ref_grads = _run(_engine(hp_off, B, T, off_params), hp, B, T, xd, c, y, lengths)
    zero = {k: (torch.zeros_like(v) if ("gin" in k or k == "gc_embedding") else v) for k, v in params.items()}
    for label, p, ids in (("zero weights", zero, [3, 1]), ("no ids", params, None)):
        m = _engine(hp, B, T, p)
        if ids is None:
            m.set_speakers(None)
        loss, logits, grads = _run(m, hp, B, T, xd, c, y, lengths, speakers=ids)
        assert abs(loss - ref_loss) <= 1e-6 * abs(ref_loss), label
        assert torch.equal(logits, ref_logits), label
        for k, g in ref_grads.items():
            assert torch.equal(grads[k], g), (label, k)
        if ids is None:
            assert all(float(grads[k].abs().max()) == 0 for k in grads if "gin" in k or k == "gc_embedding")


def test_swapping_ids_swaps_logits_and_backward_is_reproducible():
    hp = _hp(**MOL)
    B, T = 2, 256
    params = _params(hp, 35)
    x, c, y, lengths, xd = _inputs(hp, B, T, 35, same_items=True)
    m = _engine(hp, B, T, params)
    _, la, ga = _run(m, hp, B, T, xd, c, y, lengths, speakers=[0, 2])
    _, lb, gb = _run(m, hp, B, T, xd, c, y, lengths, speakers=[2, 0])
    assert (la[0] - la[1]).abs().max() > 1e-3
    assert torch.equal(la[0], lb[1]) and torch.equal(la[1], lb[0])
    _, lc, gc = _run(m, hp, B, T, xd, c, y, lengths, speakers=[0, 2])
    for k in ga:
        assert torch.equal(ga[k], gc[k]), k


def test_out_of_range_ids_raise_before_launch_and_are_guarded_in_the_kernel():
    hp = _hp(**CE)
    B, T = 2, 256
    params = _params(hp, 36)
    x, c, y, lengths, xd = _inputs(hp, B, T, 36)
    m = _engine(hp, B, T, params)
    with pytest.raises(ValueError):
        m.forward(xd.cuda(), c.cuda(), y.int().cuda(), lengths.int().cuda(), speakers=[0, 4])
    bad = torch.tensor([0, 7], dtype=torch.int32, device="cuda")          # past the host check: the kernel guards the index
    t2.lib.check(m.lib.t2_wn_set_speakers(t2.wavenet.ctypes.byref(m.cfg), t2.lib.ptr(m.workspace), t2.lib.ptr(bad), t2.lib.stream_ptr()))
    _run(m, hp, B, T, xd, c, y, lengths, backward=False)
    z = m.workspace_tensor("z", (hp.layers, B, T, hp.gate_channels // 2)).float()
    assert torch.isnan(z[:, 1]).all() and torch.isfinite(z[:, 0]).all()     # item 1's gate biases are NaN, item 0 is untouched


def test_adam_step_matches_oracle():
    hp = _hp(**CE)
    m, params, grads, _ = _compare("gin_ce_adam", hp, 4, 512, 31, [1, 2, 0, 3], 1e-4)
    state, p_ref = {}, {k: v.clone() for k, v in params.items()}
    ow.adam_step(p_ref, grads, state, hp, 0)
    m.optimizer_step()
    torch.cuda.synchronize()
    p_new, ema = m.export_params(), m.unflatten(m.ema)
    for k in p_ref:
        assert (p_new[k] - p_ref[k]).abs().max().item() < 2e-6, k
        assert (ema[k] - state["ema"][k]).abs().max().item() < 2e-6, k


def test_fp32_class_forward():
    hp = _hp(**MOL)
    B, T = 2, 256
    params = _params(hp, 38)
    x, c, y, lengths, xd = _inputs(hp, B, T, 38)
    m = _engine(hp, B, T, params, precision="fp32-class")
    loss, logits, _ = _run(m, hp, B, T, xd, c, y, lengths, speakers=[3, 0], backward=False)
    loss_ref, _, yhat = train_step_g(params, x, c, y, lengths, hp, g=torch.tensor([[3], [0]]))
    err = (logits - yhat.transpose(1, 2)).abs().max().item()
    print("MEASURED gin fp32-class logits max err %.3g loss err %.3g" % (err, abs(loss - loss_ref.item())))
    assert err < 1e-4 and abs(loss - loss_ref.item()) < 1e-4


@pytest.mark.parametrize("cs", [1, 8, 16])
def test_ar_teacher_forced_mulaw(cs):
    hp = _hp(**CE)
    B, T = 3, 48
    g = torch.Generator().manual_seed(41)
    params = _params(hp, 41)
    idx = torch.randint(90, 166, (B, T), generator=g)
    c = torch.rand(B, 80, T // 16, generator=g)
    ids = [2, 0, 3]
    onehot = torch.nn.functional.one_hot(idx, 256).float()
    init = onehot[:, :1]
    _, ref = incremental_g(init, c, params, hp, T, ids, test_inputs=torch.cat([onehot[:, 1:], onehot[:, -1:]], 1),
                           u_cat=torch.full((B, T), 0.5))
    syn = t2.wavenet.WaveNetSynthesizer(hp, B, T, cluster_size=cs)
    syn.load_params(params)
    ti = torch.cat([idx[:, 1:], idx[:, -1:]], dim=1).int().cuda()
    _, raw = syn.generate(c.cuda(), idx[:, 0].int().cuda(), test_inputs=ti, u_a=torch.rand(B, T, generator=g).cuda(), return_raw=True,
                          speakers=ids)
    torch.cuda.synchronize()
    err = (raw.cpu() - ref).abs()
    print("MEASURED gin AR mulaw cs=%d raw max err %.3g mean %.3g" % (cs, err.max().item(), err.mean().item()))
    assert err.max().item() < 4e-2 and err.mean().item() < 6e-3
    # without ids the speaker term is gone: item outputs change
    _, raw0 = syn.generate(c.cuda(), idx[:, 0].int().cuda(), test_inputs=ti, return_raw=True)
    torch.cuda.synchronize()
    assert (raw0.cpu() - raw.cpu()).abs().max() > 1e-2


@pytest.mark.parametrize("cs", [1, 8])
def test_ar_teacher_forced_mol_and_free_running(cs):
    hp = _hp(**MOL)
    B, T = 2, 48
    g = torch.Generator().manual_seed(42)
    params = _params(hp, 42)
    w = torch.rand(B, T, generator=g) - 0.5
    c = torch.rand(B, 80, T // 16, generator=g)
    ids = [3, 1]
    syn = t2.wavenet.WaveNetSynthesizer(hp, B, T, cluster_size=cs)
    syn.load_params(params)
    ti = torch.cat([w[:, 1:], w[:, -1:]], dim=1)
    _, ref = incremental_g(w[:, :1, None], c, params, hp, T, ids, test_inputs=ti[:, :, None],
                           u_mix=torch.full((B, T, 10), 0.5), u_logistic=torch.full((B, T), 0.5))
    _, raw = syn.generate(c.cuda(), w[:, 0].contiguous().cuda(), test_inputs=ti.contiguous().cuda(), return_raw=True, speakers=ids)
    torch.cuda.synchronize()
    err = (raw.cpu() - ref).abs()
    print("MEASURED gin AR MoL cs=%d raw max err %.3g mean %.3g" % (cs, err.max().item(), err.mean().item()))
    assert err.max().item() < 4e-2 and err.mean().item() < 6e-3
    # free running with injected uniforms: the oracle, fed the samples the kernel drew, draws the same samples from the same uniforms
    ua = torch.rand(B, T, 10, generator=g).clamp(1e-5, 1 - 1e-5)
    ub = torch.rand(B, T, generator=g).clamp(1e-5, 1 - 1e-5)
    out = syn.generate(c.cuda(), torch.zeros(B).cuda(), u_a=ua.cuda(), u_b=ub.cuda(), speakers=ids).cpu()
    torch.cuda.synchronize()
    outs, _ = incremental_g(torch.zeros(B, 1, 1), c, params, hp, T, ids, test_inputs=out[:, :, None], u_mix=ua, u_logistic=ub)
    agree = ((outs.reshape(B, T) - out).abs() < 2e-2).float().mean().item()
    print("MEASURED gin AR MoL cs=%d free-running agreement %.4f" % (cs, agree))
    assert agree > 0.95


def test_dropin_model_with_speakers_trains():
    from wavenet_vocoder.models import create_model
    from wavenet_vocoder.util import mulaw_quantize
    hp = _hp(residual_channels=128, gate_channels=256, skip_out_channels=128, wavenet_dropout=0.05, **CE)
    model = create_model("WaveNet", hp)
    g = torch.Generator().manual_seed(0)
    B, T = 2, 512
    wav = (torch.sin(torch.arange(T) * 0.05)[None] * 0.5 + 0.02 * torch.randn(B, T, generator=g)).clamp(-1, 1)
    idx = torch.from_numpy(mulaw_quantize(wav.numpy())).cuda()
    x = torch.nn.functional.one_hot(idx.long(), 256).float().transpose(1, 2)
    c = torch.rand(B, 80, T // 16, generator=g).cuda()
    lengths = torch.tensor([T, T - 40]).cuda()
    spk = torch.tensor([[2], [0]], dtype=torch.int32)
    losses = []
    for step in range(30):
        model.initialize(idx.unsqueeze(-1), c, spk, lengths, x=x)
        losses.append(float(model.add_loss()))
        model.add_optimizer(step)
    print("MEASURED gin drop-in loss %.4f -> %.4f" % (losses[0], losses[-1]))
    assert losses[-1] < 0.9 * losses[0], losses
    model.initialize(None, c[:, :, :2].transpose(1, 2).contiguous(), spk[:, 0], None)
    assert model.tower_y_hat[0].shape == (B, 32)
