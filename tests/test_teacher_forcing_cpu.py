"""Teacher-forcing ratio below 1 ('constant' mode, helpers.py:115-128) without a GPU: the hparam checks, the ratio each engine is
built with, the ctypes mirror of t2_taco_config_t and the library's range check, which runs before any driver call (the null
buffers passed here are never touched)."""
import ctypes
import math

import numpy as np
import pytest

from hparams import hparams
from t2_import import t2

import mask_hash as mh


def _hp(**kw):
    hp = hparams.copy()
    hp.set_hparam("predict_linear", False)
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


@pytest.mark.parametrize("ratio", [0.0, 0.3, 1.0])
def test_constant_ratios_in_range_are_accepted(ratio):
    hp = _hp(tacotron_teacher_forcing_ratio=ratio)
    assert t2.tacotron.unsupported_hparams(hp) == []
    cfg = t2.tacotron.make_config(hp, 4, 40, 80)
    assert cfg.teacher_forcing_ratio == pytest.approx(ratio)


def test_scheduled_mode_is_still_rejected_with_one_reason():
    hp = _hp(tacotron_teacher_forcing_mode="scheduled", tacotron_teacher_forcing_ratio=0.5)
    bad = t2.tacotron.unsupported_hparams(hp)
    assert len(bad) == 1 and bad[0].startswith("tacotron_teacher_forcing_mode="), bad


@pytest.mark.parametrize("ratio", [-0.1, 1.5])
def test_ratios_outside_the_unit_interval_are_rejected(ratio):
    hp = _hp(tacotron_teacher_forcing_ratio=ratio)
    bad = t2.tacotron.unsupported_hparams(hp)
    assert len(bad) == 1 and bad[0].startswith("tacotron_teacher_forcing_ratio="), bad
    with pytest.raises(t2.lib.T2Error):
        t2.tacotron.make_config(hp, 4, 40, 80)
    with pytest.raises(t2.lib.T2Error):
        t2.tacotron.make_config(_hp(), 4, 40, 80, teacher_forcing_ratio=ratio)


def test_gta_engines_feed_the_targets_and_training_uses_the_hparam():
    from tacotron.models.tacotron import engine_teacher_forcing_ratio
    hp = _hp(tacotron_teacher_forcing_ratio=0.5)
    assert engine_teacher_forcing_ratio(hp, gta=True) == 1.0
    assert engine_teacher_forcing_ratio(hp, gta=False) == 0.5
    cfg = t2.tacotron.make_config(hp, 4, 40, 80, teacher_forcing_ratio=engine_teacher_forcing_ratio(hp, gta=True))
    assert cfg.teacher_forcing_ratio == 1.0
    assert t2.tacotron.make_config(hp, 4, 40, 80).teacher_forcing_ratio == 0.5


def test_struct_mirror_ends_with_the_ratio():
    lib = t2.lib.load()
    lib.t2_struct_size.argtypes = [ctypes.c_char_p]
    C = t2.tacotron.TacoConfig
    assert lib.t2_struct_size(b"t2_taco_config_t") == ctypes.sizeof(C)
    assert C._fields_[-1] == ("teacher_forcing_ratio", ctypes.c_float)
    assert C.teacher_forcing_ratio.offset + 4 == ctypes.sizeof(C)


@pytest.mark.parametrize("ratio", [-0.1, 1.5, math.nan])
def test_library_rejects_a_ratio_outside_the_unit_interval_before_any_launch(ratio):
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    cfg = t2.tacotron.make_config(_hp(), 2, 40, 8)
    cfg.teacher_forcing_ratio = ratio
    null = ctypes.c_void_p(0)
    n, pb, wb, nt = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    rcs = [lib.t2_taco_sizes(ctypes.byref(cfg), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(nt)),
           lib.t2_taco_forward(ctypes.byref(cfg), null, null, null, null, null, null, null, null, 1, ctypes.c_ulonglong(0), null, null),
           lib.t2_taco_forward(ctypes.byref(cfg), null, null, null, null, null, null, null, null, 0, ctypes.c_ulonglong(0), null, null),
           lib.t2_taco_backward(ctypes.byref(cfg), null, null, null, null, null, null, null, null, ctypes.c_ulonglong(0), null, null)]
    for rc in rcs:
        assert rc == -1, (ratio, rc, lib.t2_last_error())
        assert b"teacher_forcing_ratio" in lib.t2_last_error()


def test_sizes_accept_the_unit_interval():
    lib = t2.lib.load()
    for ratio in (0.0, 0.5, 1.0):
        cfg = t2.tacotron.make_config(_hp(), 2, 40, 8, teacher_forcing_ratio=ratio)
        n, pb, wb, nt = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
        assert lib.t2_taco_sizes(ctypes.byref(cfg), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(nt)) == 0


def test_host_copy_of_the_draw_is_uniform_and_seed_dependent():
    """the per-step draw is element t of hash stream 40 (include/t2b200.h); the GPU tests choose their seeds with this host copy"""
    u = mh.hash_uniform32(mh.hash_seed(5, 40), np.arange(1 << 16, dtype=np.uint64))
    assert abs(float((u < 0.5).mean()) - 0.5) < 1e-2 and abs(float((u < 0.3).mean()) - 0.3) < 1e-2
    u2 = mh.hash_uniform32(mh.hash_seed(6, 40), np.arange(1 << 16, dtype=np.uint64))
    assert abs(float(((u < 0.5) == (u2 < 0.5)).mean()) - 0.5) < 1e-2
