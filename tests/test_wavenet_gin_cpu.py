"""Global (speaker) conditioning of the WaveNet vocoder, host side and oracle: no GPU needed.

The mol_gin scenario of tests/golden/reference_wavenet_graph.npz was produced by executing the reference's own WaveNet graph with
speaker ids (gc_embedding + residual_block_gin_conv). Its optimizer step is checked here through the speaker-aware oracle training
step with the bounds of tests/test_reference_wavenet_graph.py; the engine's parameter table, checkpoint names, configuration checks,
gradient buckets, feeder and id validation are checked against the same reference."""
import os

import numpy as np
import pytest
import torch

import t2_tf_bundle as tb
from hparams import hparams
from oracle import wavenet as ow
from t2_import import t2
from wavenet_gin_oracle import incremental_g, train_step_g

PATH = os.path.join(os.path.dirname(__file__), "golden", "reference_wavenet_graph.npz")
TAG = "mol_gin"


@pytest.fixture(scope="module")
def R():
    return np.load(PATH)


def _hp(R):
    hp = hparams.copy()
    for keys, values in (("small_hparams_keys", "small_hparams_values"), (TAG + "_hparams_keys", TAG + "_hparams_values")):
        for k, v in zip(R[keys], R[values]):
            setattr(hp, str(k), eval(str(v)))
    return hp


def _eng(name):
    return tb.engine_name("WaveNet_model/" + str(name))


def _params(R):
    return {_eng(n): torch.from_numpy(R["%s_var/%s" % (TAG, n)]).clone() for n in R[TAG + "_var_names"]}


def test_gc_embedding_names_map_both_ways():
    assert tb.wavenet_tf_name("gc_embedding") == "WaveNet_model/gc_embedding"
    assert tb.engine_name("WaveNet_model/gc_embedding") == "gc_embedding"
    n = "ResidualConv1DGLU_3/residual_block_gin_conv/kernel"
    assert tb.wavenet_tf_name(n) == "WaveNet_model/inference/ResidualConv1DGLU_3/residual_block_gin_conv_ResidualConv1DGLU_3/kernel"
    assert tb.engine_name(tb.wavenet_tf_name(n)) == n


def test_mol_gin_optimizer_step_of_the_executed_reference(R):
    """train_step with speaker ids + adam_step land on the reference's updated variables and EMA shadows (bounds of
    test_reference_wavenet_graph.test_one_optimizer_step_of_the_executed_reference)"""
    hp = _hp(R)
    params = _params(R)
    x, c = torch.from_numpy(R[TAG + "_x"]), torch.from_numpy(R["c"])
    lengths = torch.from_numpy(R["input_lengths"]).long()
    masks = [torch.from_numpy(R["%s_mask_%d" % (TAG, l)]) for l in range(hp.layers)]
    y = torch.from_numpy(R[TAG + "_y"])[:, :, 0]
    g = torch.from_numpy(R[TAG + "_g"])
    step = int(R[TAG + "_global_step"])
    loss, grads, _ = train_step_g(params, x, c, y, lengths, hp, g=g, dropout_masks=masks)
    assert abs(float(loss) - float(R[TAG + "_loss"])) <= 1e-5 * abs(float(R[TAG + "_loss"]))
    assert float(grads["gc_embedding"].abs().max()) > 0
    new, state = {k: v.clone() for k, v in params.items()}, {}
    lr = ow.adam_step(new, grads, state, hp, step)
    for name in R[TAG + "_var_names"]:
        eng = _eng(name)
        old = R["%s_var/%s" % (TAG, name)]
        key = "%s_new/%s" % (TAG, name)
        if key not in R.files:
            assert eng.startswith("ResidualConv1DGLU_%d/residual_block_out_conv" % (hp.layers - 1)) and float(grads[eng].abs().max()) == 0.0
            delta_ref = np.zeros_like(old)
        else:
            delta_ref = R[key] - old
        delta = new[eng].numpy() - params[eng].numpy()
        tol = 5e-3 * lr + 2e-7 * np.abs(old).max()
        assert np.abs(delta - delta_ref).max() <= tol, eng
        ema_ref = R["%s_ema/%s" % (TAG, name)] - old
        ema = state["ema"][eng].numpy() - params[eng].numpy()
        assert np.abs(ema - ema_ref).max() <= (1 - hp.wavenet_ema_decay) * tol + 1.2e-7 * np.abs(old).max(), eng


def test_teacher_forced_incremental_with_speakers_equals_parallel_step(R):
    hp = _hp(R)
    params = _params(R)
    c = torch.from_numpy(R["c"])
    B = c.shape[0]
    n = ow.upsample(c, params, hp).shape[-1]
    gen = torch.Generator().manual_seed(5)
    y0 = torch.rand(B, n, 1, generator=gen) * 1.6 - 0.8
    g = torch.tensor([[(b * 2 + 1) % hp.n_speakers] for b in range(B)])
    initial = torch.zeros(B, 1, 1)
    c_up = ow.upsample(c, params, hp)
    _, raws = incremental_g(initial, c_up, params, hp, n, g, test_inputs=y0, c_is_upsampled=True,
                            u_mix=torch.full((B, n, hp.out_channels // 3), 0.5), u_logistic=torch.full((B, n), 0.5))
    x_par = torch.cat([initial, y0[:, :-1]], dim=1).transpose(1, 2)
    par = ow.step(x_par, c_up, params, hp, c_is_upsampled=True, g=g).transpose(1, 2)
    assert (raws - par).abs().max() <= 5e-5 * max(1.0, float(par.abs().max()))
    swapped = ow.step(x_par, c_up, params, hp, c_is_upsampled=True, g=g.flip(0)).transpose(1, 2)
    assert (swapped - par).abs().max() > 1e-3          # the speaker term reaches the output


def _gin_hp(**kw):
    hp = hparams.copy()
    hp.parse("layers=4,stacks=2,residual_channels=128,gate_channels=256,skip_out_channels=128,upsample_scales=[4,4],hop_size=16,"
             "gin_channels=16,n_speakers=4,use_speaker_embedding=True")
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


def test_config_checks():
    wn = t2.wavenet
    assert wn.unsupported_hparams(_gin_hp()) == []
    cfg = wn.make_config(_gin_hp(), 2, 256)
    assert (cfg.gin_channels, cfg.n_speakers) == (16, 4)
    bad = wn.unsupported_hparams(_gin_hp(use_speaker_embedding=False))
    assert len(bad) == 1 and "use_speaker_embedding" in bad[0] and "wavenet.py:151-158" in bad[0]
    bad = wn.unsupported_hparams(_gin_hp(n_speakers=0))
    assert len(bad) == 1 and "n_speakers" in bad[0]
    with pytest.raises(t2.lib.T2Error):
        wn.make_config(_gin_hp(n_speakers=0), 2, 256)
    stock = hparams.copy()
    assert wn.unsupported_hparams(stock) == [] and wn.make_config(stock, 2, 275 * 4).gin_channels == 0


def test_engine_parameter_table_is_the_reference_variable_set(R):
    """the mol_gin configuration at engine-supported widths: the table through wavenet_tf_name names exactly the reference's variables,
    with the per-layer gin convolution inside the layer's range and the embedding outside the residual stack"""
    hp = _hp(R)
    for k, v in (("residual_channels", 128), ("gate_channels", 256), ("skip_out_channels", 128), ("cin_channels", 8)):
        hp.set_hparam(k, v)
    cfg = t2.wavenet.make_config(hp, 2, 64 * int(np.prod(hp.upsample_scales)))
    table, n_params = t2.wavenet.param_table(cfg)
    got = {tb.wavenet_tf_name(n, hp.upsample_type) for n, _, _ in table}
    want = {"WaveNet_model/" + str(n) for n in R[TAG + "_var_names"]}
    assert got == want
    shapes = {n: s for n, _, s in table}
    assert shapes["gc_embedding"] == (hp.n_speakers, hp.gin_channels)
    assert shapes["ResidualConv1DGLU_0/residual_block_gin_conv/kernel"] == (1, hp.gin_channels, 256)
    off = {n: o for n, o, _ in table}
    for l in range(hp.layers):
        lo = off["ResidualConv1DGLU_%d/residual_block_causal_conv/kernel" % l]
        hi = off["ResidualConv1DGLU_%d/residual_block_causal_conv/kernel" % (l + 1)] if l + 1 < hp.layers else off["final_convolution_1/kernel"]
        assert lo < off["ResidualConv1DGLU_%d/residual_block_gin_conv/kernel" % l] < hi
    assert off["gc_embedding"] > off["final_convolution_2/bias"]
    for G in range(1, hp.layers + 1):
        groups, rest = t2.wavenet.grad_buckets(table, hp.layers, n_params, G)
        covered = np.zeros(n_params, dtype=np.int64)
        for a, b in groups + rest:
            covered[a:b] += 1
        assert (covered == 1).all(), G


def test_gin_off_table_is_unchanged():
    """gin_channels off: the table has no speaker tensors; on: exactly the embedding and one gin convolution per layer more"""
    hp = _gin_hp()
    on, _ = t2.wavenet.param_table(t2.wavenet.make_config(hp, 2, 256))
    hp.set_hparam("gin_channels", -1)
    off, n_off = t2.wavenet.param_table(t2.wavenet.make_config(hp, 2, 256))
    assert {n for n, _, _ in on} - {n for n, _, _ in off} == {"gc_embedding"} | {
        "ResidualConv1DGLU_%d/residual_block_gin_conv/%s" % (l, k) for l in range(4) for k in ("kernel", "bias")}


def test_tf_bundle_round_trip_with_speaker_tensors(tmp_path):
    hp = _gin_hp()
    table, n = t2.wavenet.param_table(t2.wavenet.make_config(hp, 2, 256))

    class Eng(object):
        def __init__(self, seed):
            self.tensors, self.n_params, self.device, self.global_step, self.hp = table, n, torch.device("cpu"), 7, hp
            self.params = torch.randn(n, generator=torch.Generator().manual_seed(seed))
            self.m = self.v = self.ema = None

        def unflatten(self, buf):
            return {k: buf[o:o + int(np.prod(s))].reshape(s).clone() for k, o, s in self.tensors}

        def export_params(self):
            return self.unflatten(self.params)

        def load_params(self, params):
            for k, o, s in self.tensors:
                self.params[o:o + int(np.prod(s))] = params[k].reshape(-1)

    a, b = Eng(1), Eng(2)
    prefix = str(tmp_path / "wavenet_model.ckpt-7")
    names = tb.export_tf(prefix, "WaveNet", a)
    assert "WaveNet_model/gc_embedding" in names
    assert "WaveNet_model/inference/ResidualConv1DGLU_2/residual_block_gin_conv_ResidualConv1DGLU_2/bias" in names
    loaded, missing = tb.import_tf(prefix, "WaveNet", b)
    assert not missing
    pa, pb = a.export_params(), b.export_params()
    for k in pa:
        assert torch.equal(pa[k], pb[k]), k
    variables, _ = tb.load_as_engine_dicts(prefix)
    assert set(variables) == set(pa)


def _map(tmp_path, speaker_col):
    hop = 16
    rng = np.random.default_rng(0)
    os.makedirs(tmp_path / "audio", exist_ok=True)
    os.makedirs(tmp_path / "mels", exist_ok=True)
    rows = []
    for i in range(12):
        frames = int(rng.integers(10, 30))
        np.save(tmp_path / "audio" / ("a%d.npy" % i), rng.integers(0, 256, frames * hop).astype(np.int16))
        np.save(tmp_path / "mels" / ("m%d.npy" % i), rng.uniform(-4, 4, (frames, 80)).astype(np.float32))
        rows.append("audio/a%d.npy|mels/m%d.npy|mels/m%d.npy|%s|t" % (i, i, i, speaker_col(i)))
    mp = str(tmp_path / "map.txt")
    open(mp, "w").write("\n".join(rows) + "\n")
    return mp


def _feeder_hp():
    return _gin_hp(input_type="mulaw-quantize", quantize_channels=256, out_channels=256, wavenet_batch_size=4, wavenet_test_size=4,
                   wavenet_test_batches=None, max_time_steps=None, train_with_GTA=False, num_mels=80)


def test_feeder_yields_speaker_ids(tmp_path):
    from wavenet_vocoder.feeder import Feeder
    mp = _map(tmp_path, lambda i: i % 4)
    f = Feeder(mp, str(tmp_path), _feeder_hp())
    rows = {r[0]: int(r[3]) for r in (l.split("|") for l in open(mp).read().split("\n") if l)}
    for b in f.train_group() + f.test_batches():
        g = b["global_condition_features"]
        assert g.dtype == np.int32 and g.shape == (4, 1) and ((g >= 0) & (g < 4)).all()
    ex = [f._load(m) for m in f._train_meta[:4]]
    assert [e[2] for e in ex] == [rows[m[0]] for m in f._train_meta[:4]]
    assert f.prepare_batch(ex)["global_condition_features"][:, 0].tolist() == [e[2] for e in ex]


def test_feeder_rejects_rows_without_speaker(tmp_path):
    from wavenet_vocoder.feeder import Feeder
    f = Feeder(_map(tmp_path, lambda i: "<no_g>"), str(tmp_path), _feeder_hp())
    with pytest.raises(RuntimeError, match="global condition features"):
        f.train_group()


def test_out_of_range_speaker_ids_raise_before_any_launch():
    ids = t2.wavenet.speaker_ids(torch.tensor([[3], [0]]), 2, 4)
    assert ids.dtype == torch.int32 and ids.tolist() == [3, 0]
    for bad in ([4, 0], [0, -1], [0, 1, 2], [0.0, 1.0]):
        with pytest.raises(ValueError):
            t2.wavenet.speaker_ids(bad, 2, 4)
