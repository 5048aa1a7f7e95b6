"""WaveNet at dilated-convolution kernel_size 2 and 4 on the GPU, through every path that runs the dilated convolution.

  - Training step against the oracle with the methods and bounds of test_wavenet_gpu.py (bf16-emulating step_sim and plain fp32):
    mu-law CE at R 128 / G 256 / S 128, MoL and Gaussian heads at R 256 / G 512 / S 256; and with dropout on, the masks the kernels
    drew injected into the fp32 oracle, at the bounds of test_parity_full_gpu.py.
  - Two backward runs bit-identical; the phased backward equal to the monolithic one.
  - The persistent layer chains bit-identical to the per-layer launches, up to the full-depth stack of dilation 512, where the taps'
    reach (k-1) d spans 4 (k = 2) and 12 (k = 4) 128-row tiles.
  - The fp32-class forward at the bound of test_precision_modes_gpu.py.
  - AR synthesis teacher forced against the float64 kernel_size-general reference (wavenet_ar_kernel_size_reference.py): mu-law, MoL
    and Gaussian heads, one, two and four items per cluster, paper widths, and full-depth dilation rings that wrap; and against the
    training forward's outputs on the same inputs.
  - train.py / synthesize.py --model WaveNet with --hparams kernel_size=2 on a toy corpus, through a TF-bundle checkpoint.
Every measured error is printed as a MEASURED line (parity_util.record). Measured on an H100 80GB HBM3 (700 W power limit): training
logits max 1.2e-3 .. 3.5e-3, worst gradient tensor 0.9 % .. 3.5 % rel vs step_sim and 1.8 % .. 5.6 % vs fp32 (the raw heads use
test_wavenet_gpu.py's seeds; with another seed the k = 2 Gaussian case put the small-norm SubPixel bias gradient at 7.4 % vs step_sim,
the random-walk cancellation test_wavenet_gpu.py describes); with dropout masks, loss 2e-5, logits max 1.9e-3; fp32-class logits max 2.9e-6 .. 1.2e-5; AR against the float64 reference max 8.8e-8 .. 4.2e-7 (bound 2e-6),
4e-6 for the full-depth rings (measured 1.5e-7); AR against the training forward max 1.6e-3, mean 3.8e-4."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import t2_checkpoint
import t2_tf_bundle as tb
import test_parity_full_gpu as parity
import test_precision_modes_gpu as modes
import test_wavenet_ar_batch_gpu as arb
import test_wavenet_gpu as wg
import test_wavenet_persistent_gpu as pers
from hparams import hparams
from oracle import wavenet as ow
from parity_util import record
from t2_import import t2
from wavenet_ar_kernel_size_reference import launch_plan, reference_raw
from wavenet_ar_reference import batch_for_ipc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CE = dict(input_type="mulaw-quantize", quantize_channels=256, out_channels=256)
MOL = dict(input_type="raw", out_channels=30, legacy=False, residual_legacy=False, upsample_type="2D")
GAUSS = dict(input_type="raw", out_channels=2)
PAPER_W = dict(residual_channels=256, gate_channels=512, skip_out_channels=256)


# ---------------------------------------------------------------------------------------------- training step against the oracle
@pytest.mark.parametrize("k", [2, 4])
def test_training_step_ce(k):
    wg._run(wg._hp(kernel_size=k, **CE), B=2, T=512, seed=60 + k)


@pytest.mark.parametrize("k,head", [(2, "mol"), (4, "mol"), (2, "gauss"), (4, "gauss")])
def test_training_step_raw_heads_paper_widths(k, head):
    """test_wavenet_gpu.py's MoL / ConvTranspose2D and Gaussian / SubPixel cases (same batch, seed and bounds) with kernel_size k"""
    hp = wg._hp(kernel_size=k, **dict(MOL if head == "mol" else GAUSS, **PAPER_W))
    if head == "mol":
        wg._run(hp, B=3, T=256, seed=13, loss_tol=6e-4)
    else:
        wg._run(hp, B=2, T=256, seed=16, loss_tol=3e-3)


@pytest.mark.parametrize("k", [2, 4])
def test_training_step_with_dropout_masks(k):
    """dropout 0.05 on, 8 layers up to dilation 8 at paper widths: the masks the kernels drew are read back and given to the oracle"""
    hp = parity._wn_hp("input_type=mulaw-quantize,quantize_channels=256,out_channels=256,wavenet_dropout=0.05,layers=8,stacks=2,"
                       "kernel_size=%d" % k)
    parity._wn_compare("wavenet_k%d_8L_2x2048_ce_dropout" % k, hp, 2, 2048, 80 + k,
                       dict(loss=1e-4, logits_max=4e-3, logits_mean=6e-4, grad_rel=0.15, grad_cos=0.99))


@pytest.mark.parametrize("k", [2, 4])
def test_backward_is_reproducible_and_phased_backward_matches(k):
    hp = pers._hp("wavenet_ce", kernel_size=k)
    B, T = 2, 4096
    m = t2.wavenet.WaveNet(hp, B, T)
    m.init_variables(seed=5)
    x, c, y, ln = pers._inputs(hp, B, T, 9)
    m.forward(x, c, y, ln, seed=3)
    m.backward()
    torch.cuda.synchronize()
    first = m.grads.clone()
    m.forward(x, c, y, ln, seed=3)
    m.backward()
    torch.cuda.synchronize()
    assert torch.equal(first, m.grads), "two backward runs differ"
    n_groups = 3
    m.backward(0, n_groups)
    m.backward(100, n_groups)
    for g in range(n_groups):
        m.backward(1 + g, n_groups)
    torch.cuda.synchronize()
    assert torch.equal(first, m.grads), "phased backward differs from the monolithic one"
    assert m.chain_errors() == 0 and float(first.abs().sum()) > 0


# ---------------------------------------------------------------------------------------------- persistent chains
CHAINS = {"cfg2_k2": ("wavenet_ce", 2, 7680, 2), "cfg2_k4": ("wavenet_ce", 2, 7680, 4),
          "full_depth_k2": ("wavenet_default", 2, 8192, 2), "full_depth_k4": ("wavenet_default", 2, 8192, 4)}


@pytest.mark.parametrize("case", sorted(CHAINS))
def test_persistent_chain_matches_per_layer_launches_bit_for_bit(case):
    base, B, T, k = CHAINS[case]
    hp = pers._hp(base, kernel_size=k)
    ref = pers._run(hp, B, T, True)
    new = pers._run(hp, B, T, False)
    pers._check_chains_ran(hp, ref, new)
    for name in pers.STASHES:
        assert torch.equal(ref["stash"][name], new["stash"][name]), "stash %s differs" % name
    assert torch.equal(ref["grads"], new["grads"]), "gradients differ"
    s_ref, s_new = ref["scalars"].view(torch.float32), new["scalars"].view(torch.float32)
    assert torch.allclose(s_ref[:2], s_new[:2], rtol=1e-5, atol=0)


def test_persistent_chain_with_t_not_a_tile_multiple_k4():
    hp = pers._hp("wavenet_default", kernel_size=4, upsample_scales=[4, 4], hop_size=16, wavenet_dropout=0.05)
    ref = pers._run(hp, 2, 5136, True)
    new = pers._run(hp, 2, 5136, False)
    pers._check_chains_ran(hp, ref, new)
    for name in pers.STASHES:
        assert torch.equal(ref["stash"][name], new["stash"][name]), "stash %s differs" % name
    assert torch.equal(ref["grads"], new["grads"])


# ---------------------------------------------------------------------------------------------- fp32-class forward
@pytest.mark.parametrize("k,shape", [(2, "small_ce"), (4, "small_ce"), (2, "small_gauss"), (4, "small_gauss")])
def test_fp32_class_forward(k, shape):
    hp = hparams.copy()
    if shape == "small_ce":
        hp.parse("input_type=mulaw-quantize,quantize_channels=256,out_channels=256,layers=6,stacks=2,residual_channels=128,gate_channels=256,"
                 "skip_out_channels=128,upsample_scales=[4,4],hop_size=16,wavenet_dropout=0.0")
        B, T = 2, 400
    else:
        hp.parse("input_type=raw,out_channels=2,layers=6,stacks=2,residual_channels=256,gate_channels=512,skip_out_channels=256,"
                 "upsample_scales=[4,4],hop_size=16,wavenet_dropout=0.0,legacy=False,residual_legacy=False,upsample_type=2D")
        B, T = 2, 256
    hp.set_hparam("kernel_size", k)
    out = {}
    for precision in ("fp32-class", "bf16"):
        mx, mean, dl, model = modes._forward(hp, B, T, 31, precision)
        out[precision] = (mx, mean, dl)
        del model
        torch.cuda.empty_cache()
    record("wavenet_k%d_precision_modes_%s" % (k, shape), fp32_class_logits_max=out["fp32-class"][0],
           fp32_class_logits_mean=out["fp32-class"][1], fp32_class_loss_err=out["fp32-class"][2], bf16_logits_max=out["bf16"][0],
           bf16_loss_err=out["bf16"][2])
    assert out["fp32-class"][0] <= 1e-4 and out["fp32-class"][2] <= 1e-4, out
    assert out["bf16"][0] <= 5e-3 and out["bf16"][2] <= (3e-3 if shape == "small_gauss" else 1e-3), out


# ---------------------------------------------------------------------------------------------- AR synthesis
TOL_AR = 2e-6            # at kernel_size 3 the same shapes measure 1.3e-7 .. 1.3e-6 (test_wavenet_ar_batch_gpu.py)
TOL_AR_DEEP = 4e-6


def _ar_check(name, hp, params, x, c, draws, out, raw, tol):
    T = x.shape[1]
    ref = reference_raw(x.cuda(), t2.wavenet.nn_upsample(hp, c, T).cuda(), params, hp).cpu()
    err = (raw.double() - ref).abs()
    record("wavenet_ar_k%d_%s" % (hp.kernel_size, name), max_abs=err.max().item(), mean_abs=err.mean().item())
    assert torch.isfinite(raw).all()
    assert err.max().item() < tol, (name, err.max().item())
    head = arb._head(hp)
    if head == "mulaw":
        cdf = torch.softmax(raw.double(), -1).cumsum(-1)
        want = (cdf < draws["u_a"].double().unsqueeze(-1)).sum(-1).clamp(max=255)
        assert (out.long() == want).float().mean().item() > 0.97, name
    elif head == "mol":
        want = ow.sample_from_discretized_mix_logistic(raw.transpose(1, 2), hp.log_scale_min, draws["u_a"], draws["u_b"])
        assert (out - want).abs().max().item() < 1e-4, name
    else:
        want = ow.sample_from_gaussian(raw.transpose(1, 2), hp.log_scale_min_gauss, draws["u_b"])
        assert (out - want).abs().max().item() < 1e-4, name


def _ar_case(hp, B, T, cs, seed, tol, name):
    plan = launch_plan(hp, B, cs, arb._sms())
    print("AR plan k=%d: %s" % (hp.kernel_size, plan))
    params = ow.init_params(hp, seed=seed, random_bias=True)
    x, c, draws = arb._data(hp, B, T, seed)
    out, raw = arb._generate(arb._synth(hp, B, T, cs, params), x, c, draws)
    _ar_check(name, hp, params, x, c, draws, out, raw, tol)
    return plan


_AR_MATRIX = [(k, head, ipc) for k in (2, 4) for head in ("mulaw", "mol", "gauss") for ipc in (1, 2, 4)]


@pytest.mark.parametrize("k,head,ipc", _AR_MATRIX, ids=["k%d-%s-ipc%d" % m for m in _AR_MATRIX])
def test_ar_teacher_forced(k, head, ipc):
    hp = arb._hp(head, kernel_size=k)
    cs = 8
    B = batch_for_ipc(ipc, cs, arb._sms())
    plan = _ar_case(hp, B, 64, cs, 200 + 10 * k + ipc, TOL_AR, "%s_ipc%d" % (head, ipc))
    assert plan["ipc"] == ipc and plan["NI"] == ipc


@pytest.mark.parametrize("k,cs", [(2, 16), (4, 16), (4, 8)])
def test_ar_paper_widths(k, cs):
    """R 256 / G 512 / S 256: stage-1 width K1 = k R + 80 per CTA slice; the weight slices are prefetched into shared memory where
    they fit (launch_plan mirrors the host's condition) and stream from L2 otherwise"""
    hp = arb._hp("mol", arb.PAPER, kernel_size=k)
    _ar_case(hp, batch_for_ipc(3, cs, arb._sms()), 48, cs, 230 + k + cs, TOL_AR, "paper_cs%d" % cs)


@pytest.mark.parametrize("k", [2, 4])
def test_ar_default_model_rings_wrap(k):
    """20 layers in 2 stacks (dilation up to 512), Gaussian head, T = 2200 longer than the deepest ring ((k-1) 512 + 1 slots rounded up
    to a power of two: 1024 at k = 2, 2048 at k = 4), so every ring wraps"""
    hp = hparams.copy()
    hp.parse("upsample_type=NearestNeighbor,wavenet_dropout=0.0,kernel_size=%d" % k)
    B, T, cs = 4, 2200, 16
    assert launch_plan(hp, B, cs, arb._sms())["ring_slots"] == {2: 1024, 4: 2048}[k] < T
    _ar_case(hp, B, T, cs, 240 + k, TOL_AR_DEEP, "default_model_T2200")


@pytest.mark.parametrize("k,head", [(2, "mulaw"), (4, "mulaw"), (2, "gauss"), (4, "gauss")])
def test_ar_teacher_forced_matches_the_training_forward(k, head):
    """the same parameters and fed inputs through the training forward (bf16 operands) and the AR kernel (bf16 weights, fp32
    activations): the raw outputs agree within the training path's bound against the fp32 oracle (test_wavenet_gpu.py)"""
    hp = arb._hp(head, kernel_size=k)
    B, T = 2, 512
    params = ow.init_params(hp, seed=250 + k, random_bias=True)
    x, c, draws = arb._data(hp, B, T, 250 + k)
    out, raw = arb._generate(arb._synth(hp, B, T, 8, params), x, c, draws)
    m = t2.wavenet.WaveNet(hp, B, T, dropout=0.0)
    m.load_params(params)
    no = 256 if head == "mulaw" else 32
    logits = torch.zeros(B, T, no, device="cuda")
    xd = x.int().cuda() if head == "mulaw" else x.float().cuda()
    m.forward(xd, c.cuda(), xd, torch.full((B,), T, dtype=torch.int32, device="cuda"), logits=logits, save_for_backward=False)
    torch.cuda.synchronize()
    err = (logits[:, :, :hp.out_channels].cpu() - raw).abs()
    record("wavenet_ar_k%d_%s_vs_training_forward" % (k, head), max_abs=err.max().item(), mean_abs=err.mean().item())
    assert err.max().item() < 8e-3 and err.mean().item() < 1.5e-3, (err.max().item(), err.mean().item())


# ---------------------------------------------------------------------------------------------- command-line workflow
HP = ("input_type=mulaw-quantize,quantize_channels=256,out_channels=256,layers=4,stacks=2,residual_channels=128,gate_channels=256,"
      "skip_out_channels=128,wavenet_batch_size=2,wavenet_test_size=2,wavenet_test_batches=None,max_time_steps=4400,"
      "wavenet_synthesis_batch_size=2,trim_silence=False,train_with_GTA=False,kernel_size=2")


def _cli(args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT, T2_CHECKPOINT_FORMAT="tf")
    r = subprocess.run([sys.executable] + args, cwd=cwd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "%s\nSTDOUT:\n%s\nSTDERR:\n%s" % (" ".join(args), r.stdout[-3000:], r.stderr[-3000:])
    return r.stdout


def test_cli_train_and_synthesize_at_kernel_size_2(tmp_path):
    from scipy.io import wavfile
    base = str(tmp_path)
    wavs = os.path.join(base, "wavs")
    os.makedirs(wavs)
    rng = np.random.default_rng(2)
    for i in range(6):
        n = int(rng.integers(9000, 14000))
        t = np.arange(n) / 22050.0
        w = 0.4 * np.sin(2 * np.pi * (180 + 50 * i) * t) + 0.02 * rng.standard_normal(n)
        wavfile.write(os.path.join(wavs, "LJ%03d.wav" % i), 22050, (w * 32767).astype(np.int16))
    _cli([os.path.join(ROOT, "wavenet_preprocess.py"), "--base_dir", base, "--input_dir", wavs, "--hparams", HP], base)
    gta = os.path.join(base, "tacotron_output", "gta")
    common = ["--base_dir", base, "--hparams", HP, "--name", "k2", "--checkpoint_interval", "3", "--eval_interval", "3",
              "--wavenet_input", os.path.join(gta, "map.txt")]
    _cli([os.path.join(ROOT, "train.py"), "--model", "WaveNet", "--wavenet_train_steps", "3"] + common, base)
    ckpt_dir = os.path.join(base, "logs-k2", "wave_pretrained")
    prefix = os.path.join(ckpt_dir, "wavenet_model.ckpt-3")
    shapes = tb.list_bundle(prefix)
    kernel = shapes[tb.wavenet_tf_name("ResidualConv1DGLU_0/residual_block_causal_conv/kernel", hparams.upsample_type)]
    assert tuple(kernel["shape"]) == (2, 128, 256), kernel
    # resume from the TF bundle: the step counter continues
    out = _cli([os.path.join(ROOT, "train.py"), "--model", "WaveNet", "--wavenet_train_steps", "5"] + common, base)
    assert "Loading checkpoint" in out and os.path.isfile(os.path.join(ckpt_dir, "wavenet_model.ckpt-5.index"))
    variables, _ = t2_checkpoint.load(os.path.join(ckpt_dir, "wavenet_model.ckpt-5"))
    assert tuple(variables["ResidualConv1DGLU_3/residual_block_causal_conv/kernel"].shape) == (2, 128, 256)
    mels = os.path.join(base, "mels_in")
    os.makedirs(mels)
    for f in sorted(os.listdir(os.path.join(gta, "mels")))[:2]:
        np.save(os.path.join(mels, f), np.load(os.path.join(gta, "mels", f))[:24])
    _cli([os.path.join(ROOT, "synthesize.py"), "--model", "WaveNet", "--name", "k2", "--hparams", HP, "--mels_dir", mels], base)
    out_dir = os.path.join(base, "wavenet_output", "wavs")
    written = [f for f in os.listdir(out_dir) if f.endswith(".wav")]
    assert len(written) == 2
    for f in written:
        rate, data = wavfile.read(os.path.join(out_dir, f))
        assert rate == 22050 and data.dtype == np.int16 and 0 < len(data) <= 24 * 275 and len(data) % 275 == 0
