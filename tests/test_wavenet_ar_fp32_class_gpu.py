"""Fast-WaveNet AR synthesis in the fp32-class mode (WaveNetSynthesizer(precision="fp32-class"): fp32 synthesis weights and fp32
conditioning in wn_ar_kernel) against float64 references with UNROUNDED weights (reference_raw(..., bf16=False)).

Teacher forcing makes the raw outputs a function of the fed inputs, so they are compared directly; what is left between the kernel and
the reference is fp32 accumulation order and the fast tanh / sigmoid, as in the bf16 mode against its bf16-rounded reference
(test_wavenet_ar_batch_gpu.py). The conditioning is plain fp32 (not bf16-representable): the fp32-class mode never rounds it. Free
running, the mu-law samples are compared with oracle.wavenet.incremental on the same injected draws: they must agree up to the first
step whose draw lies within 2e-6 of a step of the reference CDF, where fp32 rounding may legitimately part them.

Every test prints MEASURED lines. Bounds are about three times what an H100 80GB HBM3 (132 SMs, 700 W power limit) measured:
  - 6 layers, every head, cluster size 1 / 8 / 16, one to four items per cluster and waves, kernel_size 2 and 4, speakers: at most
    4.6e-7 (MoL; 1.6e-7 Gaussian, 1.3e-7 mu-law), mean 1.3e-8 to 7.0e-8. Bound 1.5e-6;
  - learnable upsamplers (SubPixel, 2D, 1D x ReLU / LeakyReLU / none): at most 2.5e-7 where the bf16 mode measures 3.2e-3 to 3.8e-3
    against the same reference. Bound 1.5e-6 (the bf16 mode keeps the 4e-2 bound of test_wavenet_ar_gpu.py);
  - paper model (24 layers, 4 stacks, MoL 30), B 2, T 320: 1.3e-6 at cluster size 8, 1.2e-6 at 16, mean 2.3e-7. Bound 4e-6;
  - free running, mu-law, B 2, T 2048: the fp32-class samples equal the oracle's for the whole utterance; the bf16 ones for 1388 and
    281 steps (the first draws within 2e-6 of a reference CDF step come at 1388 and 261)."""
import pytest
import torch

from hparams import hparams
from oracle import wavenet as ow
from t2_import import t2
from test_wavenet_ar_fp32_class_cpu import launch_plan_fp32
from wavenet_ar_kernel_size_reference import reference_raw as reference_raw_ks
from wavenet_ar_reference import batch_for_ipc, reference_raw

pytestmark = pytest.mark.gpu

TOL = 1.5e-6            # 6 layers, any head, cluster size, batch shape, kernel_size, speakers, learnable upsampler
TOL_PAPER_DEEP = 4e-6   # 24 layers, 4 stacks, paper widths
NEAR = 2e-6             # a draw this close to a step of the reference CDF may pick either side

HEADS = {"mulaw": dict(input_type="mulaw-quantize", quantize_channels=256, out_channels=256),
         "mol": dict(input_type="raw", out_channels=30, legacy=False, residual_legacy=False),
         "gauss": dict(input_type="raw", out_channels=2)}
CHEAP = "layers=6,stacks=2,residual_channels=128,gate_channels=256,skip_out_channels=128"
PAPER_DEEP = "layers=24,stacks=4,residual_channels=256,gate_channels=512,skip_out_channels=256"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _hp(head, widths=CHEAP, **kw):
    hp = hparams.copy()
    hp.parse(widths + ",cin_channels=80,hop_size=16,upsample_type=NearestNeighbor,upsample_scales=[4,4],wavenet_dropout=0.0")
    for k, v in dict(HEADS[head], **kw).items():
        hp.set_hparam(k, v)
    return hp


def _head(hp):
    return "mulaw" if ow.is_mulaw_quantize(hp.input_type) else ("gauss" if hp.out_channels == 2 else "mol")


def _data(hp, B, T, seed):
    """distinct per-item inputs, fp32 conditioning frames and sampling draws"""
    g = torch.Generator().manual_seed(seed)
    if _head(hp) == "mulaw":
        x = torch.randint(40, 216, (B, T), generator=g).int()
    else:
        x = (torch.rand(B, T, generator=g) * 2 - 1) * 0.8
    c = torch.rand(B, hp.cin_channels, -(-T // hp.hop_size), generator=g)
    nm = hp.out_channels // 3
    draws = {"mulaw": lambda: dict(u_a=torch.rand(B, T, generator=g)),
             "mol": lambda: dict(u_a=torch.rand(B, T, nm, generator=g).clamp(1e-5, 1 - 1e-5),
                                 u_b=torch.rand(B, T, generator=g).clamp(1e-5, 1 - 1e-5)),
             "gauss": lambda: dict(u_b=torch.randn(B, T, generator=g))}[_head(hp)]()
    return x, c, draws


def _synth(hp, B, T, cs, params, precision="fp32-class"):
    syn = t2.wavenet.WaveNetSynthesizer(hp, B, T, cluster_size=cs, precision=precision)
    syn.load_params(params)
    return syn


def _generate(syn, x, c, draws, speakers=None):
    """teacher forced: step 0 is fed x[:, 0] and step t + 1 is fed x[:, t + 1]"""
    ti = torch.cat([x[:, 1:], x[:, -1:]], dim=1).contiguous().cuda()
    out, raw = syn.generate(c.cuda(), x[:, 0].contiguous().cuda(), test_inputs=ti, return_raw=True, speakers=speakers,
                            **{k: v.cuda() for k, v in draws.items()})
    torch.cuda.synchronize()
    return out.cpu(), raw.cpu()


def _c_up(hp, c, T, params):
    """the conditioning as the reference network sees it, [B, T, cin]: the nearest-neighbour repeat, or the oracle's fp32 upsampling"""
    if hp.upsample_type == "NearestNeighbor":
        return t2.wavenet.nn_upsample(hp, c, T)
    return ow.upsample(c, params, hp).transpose(1, 2)


def _err(name, hp, params, x, c, raw, speakers=None):
    T = x.shape[1]
    c_up = _c_up(hp, c, T, params).cuda()
    if hp.kernel_size != 3:
        ref = reference_raw_ks(x.cuda(), c_up, params, hp, bf16=False).cpu()
    else:
        ref = reference_raw(x.cuda(), c_up, params, hp, speakers=speakers, bf16=False).cpu()
    err = (raw.double() - ref).abs()
    print("MEASURED AR fp32-class %s: max abs %.3e, mean %.3e" % (name, err.max().item(), err.mean().item()))
    assert torch.isfinite(raw).all()
    return err.max().item()


def _check_draws(name, hp, draws, out, raw):
    """the samples are the head's sampling function of the kernel's own raw outputs with the injected draws"""
    head = _head(hp)
    if head == "mulaw":
        cdf = torch.softmax(raw.double(), -1).cumsum(-1)
        u = draws["u_a"].double().unsqueeze(-1)
        want = (cdf < u).sum(-1).clamp(max=255)
        near = (cdf - u).abs().amin(-1) < NEAR
        assert ((out.long() == want) | near).all(), name
    elif head == "mol":
        want = ow.sample_from_discretized_mix_logistic(raw.transpose(1, 2), hp.log_scale_min, draws["u_a"], draws["u_b"])
        assert (out - want).abs().max().item() < 1e-4, name
    else:
        want = ow.sample_from_gaussian(raw.transpose(1, 2), hp.log_scale_min_gauss, draws["u_b"])
        assert (out - want).abs().max().item() < 1e-4, name


def _case(name, hp, B, T, cs, seed, tol, speakers=None):
    params = ow.init_params(hp, seed=seed, random_bias=True)
    x, c, draws = _data(hp, B, T, seed)
    out, raw = _generate(_synth(hp, B, T, cs, params), x, c, draws, speakers=speakers)
    err = _err(name, hp, params, x, c, raw, speakers=speakers)
    assert err < tol, (name, err)
    _check_draws(name, hp, draws, out, raw)


# ---- 1. teacher forced against the unrounded float64 reference -------------------------------------------------------------------
_TARGETS = (1, 2, 4, 5)           # items per cluster; 5: more clusters than fit (waves)
_MATRIX = [(head, cs, k) for head in HEADS for cs in (1, 8, 16) for k in _TARGETS]


@pytest.mark.parametrize("head,cs,target", _MATRIX, ids=["%s-cs%d-ipc%d" % m for m in _MATRIX])
def test_teacher_forced_matrix(head, cs, target):
    hp = _hp(head)
    B = batch_for_ipc(target, cs, _sms())
    plan = launch_plan_fp32(hp, B, cs, _sms())
    assert plan["ipc"] == min(target, 4)
    _case("%s CS=%d B=%d ipc=%d NI=%d prefetch=%s" % (head, cs, B, plan["ipc"], plan["NI"], plan["prefetch"]),
          hp, B, 64, cs, 500 + 10 * cs + target, TOL)


@pytest.mark.parametrize("k,head", [(2, "mulaw"), (2, "mol"), (4, "gauss"), (4, "mulaw")])
def test_teacher_forced_kernel_size(k, head):
    hp = _hp(head, kernel_size=k)
    cs = 8
    B = batch_for_ipc(3, cs, _sms())
    _case("kernel_size %d %s" % (k, head), hp, B, 64, cs, 600 + k, TOL)


def test_teacher_forced_speakers():
    """per-item gate biases from t2_wn_ar_set_speakers, read through the fp32-class bias block"""
    hp = _hp("gauss", gin_channels=16, n_speakers=7)
    cs = 8
    B = batch_for_ipc(3, cs, _sms())
    _case("speakers", hp, B, 64, cs, 61, TOL, speakers=torch.arange(B) * 3 % 7)


@pytest.mark.parametrize("cs", [8, 16])
def test_teacher_forced_paper_model(cs):
    """24 layers in 4 stacks at paper widths, MoL head: the fp32 slices stream from L2 at both cluster sizes"""
    hp = _hp("mol", PAPER_DEEP)
    assert not launch_plan_fp32(hp, 2, cs, _sms())["prefetch"]
    _case("paper model cs=%d" % cs, hp, 2, 320, cs, 62, TOL_PAPER_DEEP)


# ---- 2. learnable upsamplers: the last upsampling layer's fp32 output is the conditioning ----------------------------------------
_UPS = [(t, a) for t in ("SubPixel", "2D", "1D") for a in ("Relu", "LeakyRelu", None)]


@pytest.mark.parametrize("utype,act", _UPS, ids=["%s-%s" % u for u in _UPS])
def test_learnable_upsampler(utype, act):
    """both modes on the same case against the float64 reference fed the oracle's fp32 upsampling"""
    hp = _hp("mol", upsample_type=utype, upsample_activation=act)
    cs, T = 4, 64
    B = batch_for_ipc(3, cs, _sms())
    params = ow.init_params(hp, seed=63, random_bias=True)
    x, c, draws = _data(hp, B, T, 63)
    errs = {}
    for precision in ("bf16", "fp32-class"):
        out, raw = _generate(_synth(hp, B, T, cs, params, precision), x, c, draws)
        errs[precision] = _err("%s %s upsampler (%s)" % (utype, act, precision), hp, params, x, c, raw)
        _check_draws(utype, hp, draws, out, raw)
    assert errs["fp32-class"] < TOL, errs
    assert errs["bf16"] < 4e-2, errs


# ---- 3. free running against the oracle's incremental forward with the same draws -----------------------------------------------
def _prefix(a, b):
    """per item: the number of leading steps on which the index sequences a and b [B, T] agree"""
    diff = a != b
    T = a.shape[1]
    return [int(d.nonzero()[0]) if d.any() else T for d in diff]


def test_free_running_mulaw_follows_the_oracle():
    hp = _hp("mulaw")
    B, T, cs = 2, 2048, 8
    params = ow.init_params(hp, seed=64, random_bias=True)
    g = torch.Generator().manual_seed(64)
    c = torch.rand(B, hp.cin_channels, T // hp.hop_size, generator=g)
    u = torch.rand(B, T, generator=g)
    init = torch.full((B,), 127, dtype=torch.int32)
    outs, raws = ow.incremental(torch.nn.functional.one_hot(init.long(), 256).float().unsqueeze(1), c, params, hp, T, u_cat=u)
    want = outs.argmax(-1)                                                  # [B, T]
    cdf = torch.softmax(raws.double(), -1).cumsum(-1)
    near = (cdf - u.double().unsqueeze(-1)).abs().amin(-1) < NEAR           # on the reference's own path
    first_near = [int(n.nonzero()[0]) if n.any() else T for n in near]
    prefix = {}
    for precision in ("bf16", "fp32-class"):
        syn = _synth(hp, B, T, cs, params, precision)
        got = syn.generate(c.cuda(), init.cuda(), u_a=u.cuda()).cpu().long()
        prefix[precision] = _prefix(got, want)
        print("MEASURED AR free-running %s: identical prefix %s of %d steps (first draw within %.0e of a CDF step: %s)" % (
            precision, prefix[precision], T, NEAR, first_near))
    for p, n in zip(prefix["fp32-class"], first_near):
        assert p >= n, (prefix, first_near)
    fp32, bf16 = min(prefix["fp32-class"]), min(prefix["bf16"])
    assert fp32 == T or fp32 >= 10 * bf16, prefix


@pytest.mark.parametrize("head", ["mol", "gauss"])
def test_free_running_scalar_heads_are_finite_and_in_range(head):
    hp = _hp(head)
    B, T, cs = 3, 1024, 8
    params = ow.init_params(hp, seed=65, random_bias=True)
    c = torch.rand(B, hp.cin_channels, T // hp.hop_size, generator=torch.Generator().manual_seed(65))
    out = _synth(hp, B, T, cs, params).generate(c.cuda(), torch.zeros(B).cuda(), seed=4).cpu()
    print("MEASURED AR free-running fp32-class %s: range [%.4f, %.4f], std %.4f" % (head, out.min(), out.max(), out.std()))
    assert torch.isfinite(out).all() and out.min() >= -1 and out.max() <= 1 and out.std() > 0


# ---- 4. determinism --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("head", ["mol", "mulaw"])
def test_item_does_not_depend_on_its_batch_or_instantiation(head):
    """the first items of batches that run the <4>, <2> and <1> instantiations get the same bits, teacher forced and free running,
    and a repeated call gives the same bits again"""
    hp = _hp(head)
    cs, T = 8, 48
    sms = _sms()
    sizes = [batch_for_ipc(k, cs, sms) for k in (3, 2, 1)]
    assert [launch_plan_fp32(hp, b, cs, sms)["NI"] for b in sizes] == [4, 2, 1]
    params = ow.init_params(hp, seed=66, random_bias=True)
    x, c, draws = _data(hp, sizes[0], T, 66)
    res = []
    for b in sizes:
        syn = _synth(hp, b, T, cs, params)
        forced = _generate(syn, x[:b], c[:b], {k: v[:b] for k, v in draws.items()})
        free = tuple(t.cpu() for t in syn.generate(c[:b].cuda(), x[:b, 0].contiguous().cuda(), seed=9, return_raw=True))
        again = tuple(t.cpu() for t in syn.generate(c[:b].cuda(), x[:b, 0].contiguous().cuda(), seed=9, return_raw=True))
        assert all(torch.equal(p, q) for p, q in zip(free, again)), b
        res.append((forced, free))
    for (forced, free), b in zip(res[1:], sizes[1:]):
        for got, want in zip(forced + free, res[0][0] + res[0][1]):
            assert torch.equal(got, want[:b]), b
    print("MEASURED AR fp32-class %s: batches %s bit-identical on their shared items" % (head, sizes))


@pytest.mark.parametrize("cs", [8, 16])
def test_prefetch_off_is_bitwise(cs, monkeypatch):
    """the shared-memory prefetch of the fp32 slices and the L2-streaming path read the same weight bits and do the same arithmetic"""
    hp = _hp("mol")
    B = batch_for_ipc(3, cs, _sms())
    assert launch_plan_fp32(hp, B, cs, _sms())["prefetch"]
    T = 48
    params = ow.init_params(hp, seed=67, random_bias=True)
    x, c, draws = _data(hp, B, T, 67)
    syn = _synth(hp, B, T, cs, params)
    out_a, raw_a = _generate(syn, x, c, draws)
    monkeypatch.setenv("T2_AR_PREFETCH", "0")
    out_b, raw_b = _generate(syn, x, c, draws)
    print("MEASURED AR fp32-class cs %d: prefetch on / off bit-identical %s" % (cs, torch.equal(raw_a, raw_b)))
    assert torch.equal(raw_a, raw_b) and torch.equal(out_a, out_b)
