"""The persistent layer chains (one launch for all forward gate / out GEMMs, one for all backward dz / dx GEMMs) against the
per-layer launches they replace (t2_dbg_wn_per_layer): every tile runs the same arithmetic, and bias sums are order-independent
fixed-point atomics, so every stash, the losses and every gradient must agree bit for bit."""
import ctypes
import math

import pytest
import torch

from bench import workload_hparams
from t2_import import t2

pytestmark = pytest.mark.gpu

STASHES = ("x", "xd", "ta", "sb", "z", "dg", "dxin")


def _hp(base, **kw):
    hp = workload_hparams(base)
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


def _inputs(hp, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    hop = math.prod(hp.upsample_scales)
    Tc = T // hop
    c = torch.rand(B, hp.cin_channels, Tc, generator=g)
    w = (torch.sin(torch.arange(T) * 0.05)[None] * 0.5 + 0.05 * torch.randn(B, T, generator=g)).clamp(-0.95, 0.95)
    lengths = torch.tensor([T] + [max(T - 301 * (i + 1), 2) for i in range(B - 1)], dtype=torch.int32)
    if hp.input_type == "mulaw-quantize":
        x = t2.audio.mulaw_quantize(w.cuda()).int()
        return x, c.cuda(), x, lengths.cuda()
    return w.cuda(), c.cuda(), w.cuda(), lengths.cuda()


def _ws(m, name):
    p, n, eb = ctypes.c_void_p(), ctypes.c_longlong(), ctypes.c_int()
    t2.lib.check(m.lib.t2_wn_workspace_tensor(ctypes.byref(m.cfg), t2.lib.ptr(m.workspace), name.encode(), ctypes.byref(p),
                                              ctypes.byref(n), ctypes.byref(eb)))
    off = p.value - m.workspace.data_ptr()
    return m.workspace[off:off + n.value * eb.value].clone()


def _run(hp, B, T, per_layer, speakers=None):
    m = t2.wavenet.WaveNet(hp, B, T)
    m.init_variables(seed=3)
    if speakers is not None:
        m.set_speakers(speakers)
    x, c, y, ln = _inputs(hp, B, T, 7)
    m.lib.t2_dbg_wn_per_layer(1 if per_layer else 2)
    try:
        n0 = m.lib.t2_launch_count()
        m.forward(x, c, y, ln)
        m.backward()
        torch.cuda.synchronize()
        launches = m.lib.t2_launch_count() - n0
    finally:
        m.lib.t2_dbg_wn_per_layer(0)
    assert m.chain_errors() == 0, "a layer-chain dependency wait timed out"
    return {"stash": {k: _ws(m, k) for k in STASHES}, "scalars": _ws(m, "scalars"), "grads": m.grads.clone(), "launches": launches}


def _check_chains_ran(hp, ref, new):
    # the 2L - 1 forward and 2L backward per-layer GEMM launches became one launch per direction
    assert ref["launches"] - new["launches"] == 4 * hp.layers - 3, (ref["launches"], new["launches"])


CASES = {
    "cfg2": ("wavenet_ce", 2, 7680, {}),                                      # 120 M tiles, fewer than the SMs
    "more_tiles_than_sms": ("wavenet_ce", 4, 8192, {}),
    "B3_no_dropout": ("wavenet_ce", 3, 5120, {"wavenet_dropout": 0.0}),
    "default_widths": ("wavenet_default", 2, 8192, {}),                       # dilation 512: taps span 8 tiles
    "mol": ("wavenet_mol", 2, 4096, {}),
    "gin": ("wavenet_ce", 2, 4096, {"gin_channels": 16, "n_speakers": 4, "use_speaker_embedding": True}),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_persistent_chain_matches_per_layer_launches_bit_for_bit(case):
    base, B, T, kw = CASES[case]
    hp = _hp(base, **kw)
    spk = torch.arange(B, dtype=torch.int32, device="cuda") % 4 if "gin_channels" in kw else None
    ref = _run(hp, B, T, True, spk)
    new = _run(hp, B, T, False, spk)
    _check_chains_ran(hp, ref, new)
    for k in STASHES:
        assert torch.equal(ref["stash"][k], new["stash"][k]), "stash %s differs" % k
    assert torch.equal(ref["grads"], new["grads"]), "gradients differ"
    # the loss is a float atomic sum: its last bits depend on the order the head's tiles finish in
    s_ref, s_new = ref["scalars"].view(torch.float32), new["scalars"].view(torch.float32)
    assert torch.allclose(s_ref[:2], s_new[:2], rtol=1e-5, atol=0)


def test_persistent_chain_with_t_not_a_tile_multiple():
    # T = 16 * 321: the last M tile of every item is partly past the sequence end (hop 16 keeps T a multiple of the hop)
    hp = _hp("wavenet_ce", upsample_scales=[4, 4], hop_size=16, wavenet_dropout=0.05)
    ref = _run(hp, 2, 5136, True)
    new = _run(hp, 2, 5136, False)
    _check_chains_ran(hp, ref, new)
    for k in STASHES:
        assert torch.equal(ref["stash"][k], new["stash"][k]), "stash %s differs" % k
    assert torch.equal(ref["grads"], new["grads"])
