"""CPU checks of the float64 AR-synthesis reference (tests/wavenet_ar_reference.py) that test_wavenet_ar_batch_gpu.py trusts:
without bf16 rounding it is the oracle's incremental pass under teacher forcing and the oracle's parallel forward (with the legacy skip
scale folded into the skip weights), and with rounding it rounds exactly the kernels ar_pack_kernel stores as bf16. Also pins the
mirror of the host's launch plan on a 132-SM device."""
import pytest
import torch

from hparams import hparams
from oracle import wavenet as ow
from wavenet_ar_reference import batch_for_ipc, launch_plan, reference_raw
from wavenet_gin_oracle import incremental_g

HEADS = {"mulaw": dict(input_type="mulaw-quantize", quantize_channels=16, out_channels=16),
         "mol": dict(input_type="raw", out_channels=6),
         "gauss": dict(input_type="raw", out_channels=2)}


def _hp(head, **kw):
    hp = hparams.copy()
    hp.parse("layers=6,stacks=2,residual_channels=16,gate_channels=32,skip_out_channels=16,cin_channels=8,hop_size=4,"
             "upsample_type=NearestNeighbor,wavenet_dropout=0.0")
    for k, v in dict(HEADS[head], **kw).items():
        hp.set_hparam(k, v)
    return hp


def _case(hp, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    params = {k: v.double() for k, v in ow.init_params(hp, seed=seed, random_bias=True).items()}
    if ow.is_mulaw_quantize(hp.input_type):
        x = torch.randint(0, hp.quantize_channels, (B, T), generator=g)
        xin = torch.nn.functional.one_hot(x, hp.quantize_channels).double()          # [B, T, Q]
    else:
        x = (torch.rand(B, T, generator=g, dtype=torch.float64) * 2 - 1) * 0.8
        xin = x.unsqueeze(-1)
    c = torch.rand(B, hp.cin_channels, T // hp.hop_size, generator=g, dtype=torch.float64)
    return params, x, xin, c


def _c_up(c, hp):
    return c.repeat_interleave(hp.hop_size, dim=-1).transpose(1, 2)


@pytest.mark.parametrize("head", sorted(HEADS))
@pytest.mark.parametrize("legacy", [True, False])
def test_reference_is_incremental_under_teacher_forcing(head, legacy):
    hp = _hp(head, legacy=legacy, residual_legacy=legacy)
    B, T = 3, 40
    params, x, xin, c = _case(hp, B, T, 5)
    ti = torch.cat([xin[:, 1:], xin[:, -1:]], dim=1)          # step t + 1 is fed input t + 1
    kw = dict(normal=torch.zeros(B, T)) if head == "gauss" else {}
    _, raw = ow.incremental(xin[:, :1], c, params, hp, T, test_inputs=ti, **kw)
    ref = reference_raw(x, _c_up(c, hp), params, hp, bf16=False)
    assert ref.dtype == torch.float64 and raw.dtype == torch.float64
    assert (ref - raw).abs().max().item() < 1e-10


@pytest.mark.parametrize("legacy,residual_legacy", [(True, True), (True, False), (False, True), (False, False)])
def test_folded_skip_scale_reproduces_step(legacy, residual_legacy):
    hp = _hp("mol", legacy=legacy, residual_legacy=residual_legacy, layers=8, stacks=2)
    params, x, xin, c = _case(hp, 2, 48, 6)
    y = ow.step(xin.transpose(1, 2), c, params, hp).transpose(1, 2)
    ref = reference_raw(x, _c_up(c, hp), params, hp, bf16=False)
    assert (ref - y).abs().max().item() < 1e-10


def test_speaker_reference_is_incremental():
    hp = _hp("gauss", gin_channels=4, n_speakers=3)
    B, T = 3, 32
    params, x, xin, c = _case(hp, B, T, 7)
    spk = torch.tensor([2, 0, 1])
    ti = torch.cat([xin[:, 1:], xin[:, -1:]], dim=1)
    _, raw = incremental_g(xin[:, :1], c, params, hp, T, spk, test_inputs=ti, normal=torch.zeros(B, T))
    ref = reference_raw(x, _c_up(c, hp), params, hp, speakers=spk, bf16=False)
    assert (ref - raw).abs().max().item() < 1e-10


@pytest.mark.parametrize("legacy", [True, False])
def test_bf16_rounding_is_where_the_kernel_stores_bf16(legacy):
    """the rounded reference equals the unrounded one on parameters whose bf16-stored kernels are pre-rounded: the dilated, cin, out
    and final kernels as they are, the skip kernel after its fp32 scaling (so it is rounded here with the scale applied)"""
    hp = _hp("mol", legacy=legacy, residual_legacy=legacy)
    params, x, xin, c = _case(hp, 2, 40, 8)
    params = {k: v.float() for k, v in params.items()}
    r = lambda t: t.to(torch.bfloat16).float()
    pre = dict(params)
    from wavenet_ar_reference import skip_scales
    sc = skip_scales(hp)
    for l in range(hp.layers):
        p = "ResidualConv1DGLU_%d/" % l
        for n in ("causal_conv", "cin_conv", "out_conv"):
            pre[p + "residual_block_%s/kernel" % n] = r(params[p + "residual_block_%s/kernel" % n])
        s32 = torch.tensor(sc[l], dtype=torch.float32)
        pre[p + "residual_block_skip_conv/kernel"] = r(params[p + "residual_block_skip_conv/kernel"] * s32).double() / sc[l]
    for n in ("final_convolution_1/kernel", "final_convolution_2/kernel"):
        pre[n] = r(params[n])
    got = reference_raw(x, _c_up(c, hp), params, hp)
    want = reference_raw(x, _c_up(c, hp), pre, hp, bf16=False)
    assert (got - want).abs().max().item() < 1e-10
    assert (got - reference_raw(x, _c_up(c, hp), params, hp, bf16=False)).abs().max().item() > 1e-4   # the rounding is there


@pytest.mark.parametrize("cs", [1, 2, 4, 8, 16])
def test_launch_plan_reaches_every_instantiation(cs):
    """on a 132-SM H100: the batch sizes chosen for ipc 1, 2, 3, 4 and waves give the <1>, <2> and <4> kernels, partly filled last
    clusters, and more clusters than fit"""
    hp = _hp("mol")
    plans = [launch_plan(hp, batch_for_ipc(k, cs, 132), cs, 132) for k in (1, 2, 3, 4, 5)]
    assert [p["ipc"] for p in plans] == [1, 2, 3, 4, 4]
    assert [p["NI"] for p in plans] == [1, 2, 4, 4, 4]
    assert [p["ragged"] for p in plans] == [False, True, True, False, True]
    assert [p["waves"] for p in plans] == [False, False, False, False, True]
    assert all(p["clusters"] * cs <= 132 for p in plans[:4]) and plans[4]["clusters"] == 132 // cs + 1
    assert all(p["clusters"] * p["ipc"] >= p["B"] > (p["clusters"] - 1) * p["ipc"] for p in plans)


def test_launch_plan_prefetch_and_rings():
    hp = hparams.copy()
    hp.parse("layers=6,stacks=2,residual_channels=128,gate_channels=256,skip_out_channels=128")
    assert [launch_plan(hp, 3, cs, 132)["prefetch"] for cs in (1, 2, 4, 8, 16)] == [False, False, True, True, True]
    assert not launch_plan(hp, 3, 8, 132, prefetch_env=False)["prefetch"]
    paper = hparams.copy()
    paper.parse("layers=24,stacks=4,residual_channels=256,gate_channels=512,skip_out_channels=256,out_channels=30")
    assert not launch_plan(paper, 2, 8, 132)["prefetch"] and launch_plan(paper, 2, 16, 132)["prefetch"]
    assert launch_plan(hparams, 20, 16, 132)["ring_slots"] == 2048          # 20 layers, 2 stacks: dilation 512
    assert launch_plan(hparams, 20, 16, 132)["ipc"] == 3 and launch_plan(hparams, 20, 16, 132)["ragged"]
