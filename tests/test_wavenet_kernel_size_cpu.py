"""WaveNet dilated-convolution kernel_size 2 and 4 without a GPU.

  - The oracle against the reference's own graph code executed at kernel_size 2 and 4 (tests/golden/reference_wavenet_kernel_size.npz,
    make_reference_wavenet_kernel_size_vectors.py): training output, loss and gradients with the recorded dropout masks, the
    teacher-forced incremental pass of the evaluation branch, free-running synthesis with the recorded draws, and the variable names and
    shapes against wavenet_tf_name and the library's parameter table. The checks are those of test_reference_wavenet_graph.py at k = 3.
  - The accepted range (2 <= kernel_size <= 4) in the hparam check, the config check and the library's layout.
  - The parameter table, a TF-bundle checkpoint round trip, and the persistent layer-chain tickets at the new sizes."""
import ctypes
import os

import numpy as np
import pytest
import torch

import t2_tf_bundle as tb
import test_reference_wavenet_graph as base
from bench import workload_hparams
from oracle import wavenet as ow
from t2_import import t2

PATH = os.path.join(os.path.dirname(__file__), "golden", "reference_wavenet_kernel_size.npz")
TAGS = ["%s_k%d" % (t, k) for k in (2, 4) for t in ("ce_subpixel", "mol_2d", "gauss_nn")]


@pytest.fixture(scope="module")
def R():
    return np.load(PATH)


# ---------------------------------------------------------------------------------------------- the executed reference at k = 2, 4
@pytest.mark.parametrize("tag", TAGS)
def test_fixture_runs_the_kernel_size_it_is_named_for(R, tag):
    hp = base._hp(R, tag)
    assert hp.kernel_size == int(tag[-1])
    assert R["%s_var/inference/ResidualConv1DGLU_0/residual_block_causal_conv_ResidualConv1DGLU_0/kernel" % tag].shape[0] == hp.kernel_size


@pytest.mark.parametrize("tag", TAGS)
def test_variable_names_and_shapes_match_the_name_map_and_the_library_table(R, tag):
    """the library refuses the fixture's SMALL widths, so its table is taken at the smallest product widths (R 128, G 256, S 128, 8
    conditioning channels): the same names, and every shape equal to the oracle's at those widths"""
    base.test_variable_names_match_the_checkpoint_name_map(R, tag)
    hp = base._hp(R, tag)
    for n, v in dict(residual_channels=128, gate_channels=256, skip_out_channels=128, cin_channels=8, num_mels=8).items():
        setattr(hp, n, v)
    table, _ = t2.wavenet.param_table(t2.wavenet.make_config(hp, 2, 4 * hp.hop_size, dropout=0.0))
    names = {"WaveNet_model/" + str(n) for n in R[tag + "_var_names"]}
    assert {tb.wavenet_tf_name(name, hp.upsample_type) for name, _, _ in table} == names
    assert {name: tuple(shape) for name, _, shape in table} == {name: tuple(s) for name, s in ow.param_shapes(hp).items()}
    for l in range(hp.layers):
        name = "ResidualConv1DGLU_%d/residual_block_causal_conv/kernel" % l
        ref = R["%s_var/%s" % (tag, tb.wavenet_tf_name(name, hp.upsample_type)[len("WaveNet_model/"):])].shape
        assert dict((n, s) for n, _, s in table)[name] == (ref[0], 128, 256) and ref[0] == hp.kernel_size


@pytest.mark.parametrize("tag", TAGS)
def test_training_graph_output_loss_and_gradients(R, tag):
    base.test_training_graph_output_loss_and_gradients(R, tag)


@pytest.mark.parametrize("tag", TAGS)
def test_evaluation_branch_teacher_forced_incremental_pass(R, tag):
    base.test_evaluation_branch_teacher_forced_incremental_pass(R, tag)


@pytest.mark.parametrize("tag", TAGS)
def test_synthesis_branch_free_running_with_the_recorded_draws(R, tag):
    base.test_synthesis_branch_free_running_with_the_recorded_draws(R, tag)


# ---------------------------------------------------------------------------------------------- accepted range
def _hp(k, **kw):
    hp = workload_hparams("wavenet_default")
    hp.set_hparam("kernel_size", k)
    for n, v in kw.items():
        hp.set_hparam(n, v)
    return hp


@pytest.mark.parametrize("k", [1, 5])
def test_kernel_size_outside_2_to_4_is_refused_with_one_reason(k):
    bad = t2.wavenet.unsupported_hparams(_hp(k))
    assert len(bad) == 1 and bad[0].startswith("kernel_size=%d" % k) and "2, 3 or 4" in bad[0], bad
    with pytest.raises(t2.lib.T2Error, match="kernel_size"):
        t2.wavenet.make_config(_hp(k), 2, 4096)


@pytest.mark.parametrize("k", [1, 5, 0, -3])
def test_library_layout_refuses_kernel_size_outside_2_to_4(k):
    lib = t2.lib.load()
    cfg = t2.wavenet.make_config(_hp(3), 2, 4096)
    cfg.kernel_size = k
    sz = t2.wavenet.WnSizes()
    assert lib.t2_wn_sizes(ctypes.byref(cfg), ctypes.byref(sz)) != 0
    msg = lib.t2_last_error().decode()
    assert "kernel_size must be 2, 3 or 4" in msg and ("got %d" % k) in msg, msg


@pytest.mark.parametrize("k", [2, 3, 4])
def test_kernel_sizes_2_to_4_are_accepted(k):
    hp = _hp(k)
    assert t2.wavenet.unsupported_hparams(hp) == []
    for precision in ("bf16", "fp32-class"):
        cfg = t2.wavenet.make_config(hp, 2, 4096, dropout=0.0 if precision == "fp32-class" else None, precision=precision)
        sz = t2.wavenet.WnSizes()
        t2.lib.check(t2.lib.load().t2_wn_sizes(ctypes.byref(cfg), ctypes.byref(sz)))
        pb, wb = ctypes.c_longlong(), ctypes.c_longlong()
        t2.lib.check(t2.lib.load().t2_wn_ar_sizes(ctypes.byref(cfg), 8, ctypes.byref(pb), ctypes.byref(wb)))


@pytest.mark.parametrize("k", [2, 4])
@pytest.mark.parametrize("variant", [dict(), dict(input_type="raw", out_channels=30, upsample_type="2D"),
                                     dict(gin_channels=16, n_speakers=4, use_speaker_embedding=True)])
def test_parameter_table_matches_the_oracle(k, variant):
    hp = _hp(k, **variant)
    table, _ = t2.wavenet.param_table(t2.wavenet.make_config(hp, 2, 4096))
    assert {name: tuple(shape) for name, _, shape in table} == {name: tuple(s) for name, s in ow.param_shapes(hp).items()}
    assert dict((name, shape) for name, _, shape in table)["ResidualConv1DGLU_3/residual_block_causal_conv/kernel"] == (
        k, hp.residual_channels, hp.gate_channels)


def test_tf_bundle_checkpoint_round_trip_at_kernel_size_2(tmp_path):
    """t2_checkpoint.save(fmt='tf') of an engine whose table is the library's at kernel_size 2 -> load: every variable, EMA shadow and
    Adam slot comes back with the [2, R, G] causal-conv shape and the same bits"""
    import t2_checkpoint
    from test_tf_bundle_cpu import _FakeEngine
    hp = _hp(2, upsample_type="2D")
    table, _ = t2.wavenet.param_table(t2.wavenet.make_config(hp, 2, 4096))
    a = _FakeEngine([(name, shape) for name, _, shape in table], 7)
    a.ema, a.hp, a.global_step = a.params * 0.5, hp, 1234
    path = t2_checkpoint.save(str(tmp_path), "wavenet_model.ckpt", a, fmt="tf")
    entry = tb.list_bundle(path)[tb.wavenet_tf_name("ResidualConv1DGLU_0/residual_block_causal_conv/kernel", hp.upsample_type)]
    assert tuple(entry["shape"]) == (2, hp.residual_channels, hp.gate_channels), entry
    variables, state = t2_checkpoint.load(path)
    assert state["global_step"] == 1234 and set(variables) == {name for name, _, _ in table}
    for name, off, shape, _ in a.tensors:
        n = int(np.prod(shape))
        assert tuple(variables[name].shape) == tuple(shape), name
        assert torch.equal(variables[name].reshape(-1), a.params[off:off + n])
        assert torch.equal(state["ema"][name].reshape(-1), a.ema[off:off + n])
        assert torch.equal(state["adam_m"][name].reshape(-1), a.m[off:off + n])
    b = _FakeEngine([(name, shape) for name, _, shape in table], 8)
    b.hp = hp
    loaded, missing = tb.import_tf(path, "WaveNet", b)
    assert not missing and torch.equal(a.params, b.params)


# ---------------------------------------------------------------------------------------------- persistent layer chains
# (name, B, T, kernel_size); wavenet_default reaches dilation 512, so (k-1) d spans 4 (k = 2) and 12 (k = 4) 128-row tiles
CHAIN_SHAPES = [("wavenet_ce", 2, 7680, 2), ("wavenet_ce", 2, 7680, 4), ("wavenet_default", 2, 8192, 2), ("wavenet_default", 2, 8192, 4),
                ("wavenet_default", 2, 5136, 4), ("wavenet_ce", 3, 5136, 2), ("wavenet_mol", 2, 4096, 4)]


def _tickets(cfg, d):
    lib = t2.lib.load()
    n = lib.t2_dbg_wn_chain(ctypes.byref(cfg), d, None, 0)
    assert n > 0, lib.t2_last_error()
    buf = (ctypes.c_int * (8 * n))()
    assert lib.t2_dbg_wn_chain(ctypes.byref(cfg), d, buf, n) == n
    return np.frombuffer(buf, dtype=np.int32).reshape(n, 8)


@pytest.mark.parametrize("name,B,T,k", CHAIN_SHAPES)
def test_chain_tickets_wait_for_exactly_the_rows_they_read(name, B, T, k):
    """test_wavenet_chain_cpu.py's property with the taps' reach (k-1) d: a gate tile reads xd_l rows [t0 - (k-1)d, t0 + 128), a dx
    tile dg_l rows [t0, t0 + 128 + (k-1)d)"""
    hp = workload_hparams(name)
    hp.set_hparam("kernel_size", k)
    if T % 256:
        hp.set_hparam("upsample_scales", [4, 4])
        hp.set_hparam("hop_size", 16)
    cfg = t2.wavenet.make_config(hp, B, T)
    L, G = hp.layers, hp.gate_channels
    Gh = G // 2
    tpb = -(-T // 128)
    MT = B * tpb
    reach = lambda l: (k - 1) * (1 << (l % (L // hp.stacks)))
    idx = lambda kind, l, m: (kind * L + l) * MT + m
    for d in (0, 1):
        tk = _tickets(cfg, d)
        n0 = G // 256 if d == 0 else Gh // (256 if Gh >= 256 else 128)
        order = []
        for l in (range(L) if d == 0 else range(L - 1, -1, -1)):
            order += [(0, l, m, n) for n in range(n0) for m in range(MT)]
            if d == 1 or l + 1 < L:
                order += [(1, l, m, 0) for m in range(MT)]
        assert [tuple(r[:4]) for r in tk] == order
        finished_before = {}
        for i, (kind, l, m, n, lo, hi, target, done) in enumerate(tk):
            assert done == idx(kind, l, m)
            finished_before.setdefault(done, []).append(i)
            b, t0 = m // tpb, (m % tpb) * 128
            if d == 0 and kind == 0:
                rows, dep_kind, dep_l, need = (max(0, t0 - reach(l)), min(T, t0 + 128)), 1, l - 1, 1
            elif d == 0:
                rows, dep_kind, dep_l, need = (t0, min(T, t0 + 128)), 0, l, n0
            elif kind == 0:
                rows, dep_kind, dep_l, need = (t0, min(T, t0 + 128)), 1, l + 1, 1
            else:
                rows, dep_kind, dep_l, need = (t0, min(T, t0 + 128 + reach(l))), 0, l, n0
            if (d == 0 and kind == 0 and l == 0) or (d == 1 and kind == 0 and l == L - 1):
                assert hi < lo
                continue
            want = (idx(dep_kind, dep_l, b * tpb + rows[0] // 128), idx(dep_kind, dep_l, b * tpb + (rows[1] - 1) // 128))
            assert (lo, hi) == want and target == need
            for c in range(lo, hi + 1):
                assert len([j for j in finished_before.get(c, []) if j < i]) == need
