"""ConvTranspose1D conditioning upsampler and the LeakyReLU / linear upsampling activations of the WaveNet engine, host side (no GPU):
config checks of tacotron-2_b200/wavenet.py, the t2_wn_config_t mirror, the library's range checks (rejected before any launch), the
parameter table against the oracle and the executed reference's variable names, the product's NN_init kernel against the kernels the
reference's ConvTranspose1D._init_kernel produced (tests/golden/reference_wavenet_graph.npz, scenario ce_1d), and a TF-bundle round
trip under the reference's ConvTranspose1D names."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import t2_tf_bundle as tb
from hparams import hparams
from oracle import wavenet as ow
from t2_import import t2

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_wavenet_graph.npz")
WN = t2.wavenet


def _hp(**kw):
    hp = hparams.copy()
    hp.parse("layers=4,stacks=2,residual_channels=256,gate_channels=512,skip_out_channels=256,input_type=mulaw-quantize,"
             "quantize_channels=256,out_channels=256,upsample_type=1D,upsample_scales=[4,4],hop_size=16")
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


def _lib():
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    lib.t2_launch_count.restype = ctypes.c_longlong
    return lib


def test_config_checks_accept_the_new_variants_and_keep_the_rest():
    for kw in (dict(), dict(upsample_activation="LeakyRelu"), dict(upsample_activation="LeakyRelu", leaky_alpha=0.0),
               dict(upsample_activation="LeakyRelu", leaky_alpha=1.0), dict(upsample_activation=None),
               dict(upsample_type="SubPixel", upsample_activation="LeakyRelu"), dict(upsample_type="2D", upsample_activation=None),
               dict(freq_axis_kernel_size=3)):
        assert WN.unsupported_hparams(_hp(**kw)) == [], kw
    for name, value in (("upsample_type", "Resize"), ("upsample_activation", "Elu"), ("upsample_activation", "relu6")):
        bad = WN.unsupported_hparams(_hp(**{name: value}))
        assert len(bad) == 1 and bad[0].startswith(name + "="), (name, bad)
    for alpha in (-0.1, 1.5, float("nan")):
        bad = WN.unsupported_hparams(_hp(upsample_activation="LeakyRelu", leaky_alpha=alpha))
        assert len(bad) == 1 and bad[0].startswith("leaky_alpha="), (alpha, bad)
    assert WN.unsupported_hparams(_hp(leaky_alpha=1.5)) == []          # the slope is read only under LeakyRelu
    # the shipped configurations are unchanged: ReLU, alpha 0 in the struct
    import paper_hparams
    for hp in (hparams, paper_hparams.hparams):
        assert WN.unsupported_hparams(hp) == []
        cfg = WN.make_config(hp, 2, 4 * math.prod(hp.upsample_scales))
        assert (cfg.upsample_activation, cfg.leaky_alpha) == (0, 0.0)
        assert cfg.upsample_type == {"SubPixel": 0, "2D": 1}[hp.upsample_type]


def test_make_config_fills_the_new_fields():
    cfg = WN.make_config(_hp(upsample_activation="LeakyRelu", leaky_alpha=0.25), 2, 64)
    assert (cfg.upsample_type, cfg.upsample_activation, cfg.leaky_alpha) == (2, 1, 0.25)
    cfg = WN.make_config(_hp(upsample_activation=None, freq_axis_kernel_size=5), 2, 64)
    assert (cfg.upsample_type, cfg.upsample_activation, cfg.leaky_alpha, cfg.freq_axis_kernel_size) == (2, 2, 0.0, 5)
    sz = WN.WnSizes()
    t2.lib.check(_lib().t2_wn_sizes(ctypes.byref(cfg), ctypes.byref(sz)))        # 1D does not read freq_axis_kernel_size
    cfg.upsample_type = 0
    assert _lib().t2_wn_sizes(ctypes.byref(cfg), ctypes.byref(sz)) == -2         # ... SubPixel still does
    with pytest.raises(t2.lib.T2Error):
        WN.make_config(_hp(upsample_type="Resize"), 2, 64)


def test_struct_mirror_matches_the_library():
    lib = _lib()
    lib.t2_struct_size.argtypes = [ctypes.c_char_p]
    assert lib.t2_struct_size(b"t2_wn_config_t") == ctypes.sizeof(WN.WnConfig)
    names = [f[0] for f in WN.WnConfig._fields_]
    assert names[-3:] == ["n_speakers", "upsample_activation", "leaky_alpha"]
    assert WN.WnConfig.leaky_alpha.offset == ctypes.sizeof(WN.WnConfig) - 4


def test_range_checks_reject_before_any_launch():
    """bad codes and slopes: -1 (T2_ERR_INVALID_ARG) from the size query and from forward / backward / AR with null buffers; the
    launch counter does not move"""
    lib = _lib()
    sz = WN.WnSizes()
    n0 = lib.t2_launch_count()
    for field, value in (("upsample_type", 3), ("upsample_type", -1), ("upsample_activation", 3), ("upsample_activation", -1),
                         ("leaky_alpha", -0.01), ("leaky_alpha", 1.01), ("leaky_alpha", float("nan")), ("leaky_alpha", float("inf"))):
        cfg = WN.make_config(_hp(upsample_activation="LeakyRelu"), 2, 64)
        setattr(cfg, field, value)
        assert lib.t2_wn_sizes(ctypes.byref(cfg), ctypes.byref(sz)) == -1, (field, value)
        assert lib.t2_wn_init(ctypes.byref(cfg), None, None, None) == -1
        assert lib.t2_wn_forward(ctypes.byref(cfg), None, None, None, None, None, None, None, None, None, 1, ctypes.c_ulonglong(0),
                                 None, None) == -1
        assert lib.t2_wn_backward(ctypes.byref(cfg), None, None, None, None, None, None, ctypes.c_ulonglong(0), None, None) == -1
        assert lib.t2_wn_ar_generate(ctypes.byref(cfg), 8, None, None, None, None, None, None, None, None, ctypes.c_ulonglong(0),
                                     None, None, None) == -1
        assert len(lib.t2_last_error()) > 0
    # the kernel hook checks every argument before any driver call
    fake = 1 << 20
    ok = dict(p=[fake] * 6, i=[2, 80, 8, 4, 2, 1, 0], f=0.4)
    for kernel, change in ((1, ("i", 1, 0)), (1, ("i", 1, 129)), (1, ("i", 4, 3)), (1, ("i", 5, 3)), (1, ("f", 0, 1.5)),
                           (1, ("f", 0, float("nan"))), (1, ("p", 0, 0)), (1, ("i", 6, 2)), (2, ("p", 5, 0)), (3, ("p", 3, 0)),
                           (2, ("i", 4, 0)), (9, None)):
        c = t2.lib.DbgKernel()
        c.kernel = kernel
        for k, v in enumerate(ok["p"]):
            c.p[k] = v
        for k, v in enumerate(ok["i"]):
            c.i[k] = v
        c.f[0] = ok["f"]
        if change is not None:
            arr, k, v = change
            getattr(c, arr)[k] = v
            if (kernel, change) == (2, ("i", 4, 0)):
                c.i[3] = 33                                    # SubPixel weight gradient: scale <= 32
        rc = lib.t2_dbg_wn_kernel(ctypes.byref(c), None)
        assert rc in (-1, -2), (kernel, change, rc)
    assert lib.t2_launch_count() == n0


def test_parameter_table_matches_oracle_and_reference_names():
    cfg_hp = _hp(upsample_activation="LeakyRelu")
    tensors, n = WN.param_table(WN.make_config(cfg_hp, 2, 64))
    assert [(t[0], t[2]) for t in tensors] == [(k, tuple(v)) for k, v in ow.param_shapes(cfg_hp).items()]
    assert dict((t[0], t[2]) for t in tensors)["local_conditioning_upsampling_2/kernel"] == (1, 4, 80, 80)
    # the executed reference's ce_1d scenario (cin 6, scales [2, 3]): its upsampler variables are what wavenet_tf_name gives the
    # engine's upsampler tensors, with the engine's shape rule
    R = np.load(GOLDEN)
    ref = {"WaveNet_model/" + str(k): tuple(R["ce_1d_var/" + str(k)].shape) for k in R["ce_1d_var_names"] if "ConvTranspose1D" in str(k)}
    hp6 = _hp(upsample_scales=[2, 3], hop_size=6)
    eng = [t for t in WN.param_table(WN.make_config(hp6, 2, 60))[0] if t[0].startswith("local_conditioning_upsampling")]
    got = {tb.wavenet_tf_name(name, "1D"): (shape[0], shape[1], 6, 6) if name.endswith("kernel") else (6,) for name, _, shape in eng}
    assert got == ref and len(ref) == 4
    for name, _, shape in eng:
        assert tb.engine_name(tb.wavenet_tf_name(name, "1D")) == name


def test_nn_init_matches_the_executed_reference():
    R = np.load(GOLDEN)
    hp = hparams.copy()
    for keys, values in (("small_hparams_keys", "small_hparams_values"), ("ce_1d_hparams_keys", "ce_1d_hparams_values")):
        for k, v in zip(R[keys], R[values]):
            setattr(hp, str(k), eval(str(v)))
    assert hp.upsample_type == "1D" and hp.NN_init
    tensors = [(k, 0, tuple(v)) for k, v in ow.param_shapes(hp).items()]
    got = t2.init.wavenet_variables(hp, tensors, 5)
    keys = [k for k in R.files if k.startswith("ce_1d_init/")]
    assert len(keys) == 2
    for k in keys:
        eng = tb.engine_name("WaveNet_model/" + k.split("/", 1)[1])
        assert np.abs(got[eng].numpy() - R[k]).max() <= 1e-7, eng
    # the full-size product initialiser agrees with the oracle's NN_init at the stock width
    hp = _hp()
    tensors = [(k, 0, tuple(v)) for k, v in ow.param_shapes(hp).items()]
    a, b = t2.init.wavenet_variables(hp, tensors, 7), ow.init_params(hp, seed=7)
    for k in a:
        if "upsampling" in k:
            assert torch.equal(a[k], b[k]), k


class _FakeWaveNet:
    """the attributes export_tf / import_tf read from a WaveNet engine, on the host"""

    def __init__(self, hp, seed):
        self.hp = hp
        self.tensors, n = WN.param_table(WN.make_config(hp, 2, 64))
        self.n_params, self.device = n, torch.device("cpu")
        g = torch.Generator().manual_seed(seed)
        self.params, self.m, self.v = (torch.randn(n, generator=g) for _ in range(3))
        self.ema = self.params * 0.5
        self.global_step = 17

    def unflatten(self, flat):
        return {k: flat[o:o + int(np.prod(s))].reshape(s).clone() for k, o, s in self.tensors}

    def export_params(self):
        return self.unflatten(self.params)

    def load_params(self, params):
        for k, o, s in self.tensors:
            self.params[o:o + int(np.prod(s))] = torch.as_tensor(params[k]).reshape(-1)


def test_tf_bundle_round_trip(tmp_path):
    hp = _hp(upsample_activation="LeakyRelu")
    a = _FakeWaveNet(hp, 1)
    prefix = str(tmp_path / "wavenet_model.ckpt-17")
    names = tb.export_tf(prefix, "WaveNet", a)
    assert "WaveNet_model/inference/ConvTranspose1D_layer_1/kernel" in names
    assert "WaveNet_model/inference/ConvTranspose1D_layer_0/bias/ExponentialMovingAverage" in names
    variables, state = tb.load_as_engine_dicts(prefix)
    assert set(variables) == {t[0] for t in a.tensors} and state["global_step"] == 17
    for k, v in a.export_params().items():
        assert np.array_equal(variables[k].reshape(v.shape), v.numpy()), k
    b = _FakeWaveNet(hp, 2)
    loaded, missing = tb.import_tf(prefix, "WaveNet", b)
    assert not missing and b.global_step == 17
    for k, o, s in a.tensors:                  # the alignment padding between tensors is not part of a checkpoint
        n = int(np.prod(s))
        for buf in ("params", "m", "v", "ema"):
            assert torch.equal(getattr(a, buf)[o:o + n], getattr(b, buf)[o:o + n]), (buf, k)
