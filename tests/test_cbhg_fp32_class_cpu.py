"""The fp32-class (split bf16) mode of the CBHG engine without a GPU: the CbhgConfig mirror, the split_bf16 argument checks of
t2_cbhg_sizes / t2_cbhg_forward / t2_cbhg_backward, the bf16-mode sizes, and the split arguments of the CBHG kernel hooks. Every call
that is expected to fail does so before any driver call, so the device pointers passed here are never dereferenced."""
import ctypes

import pytest

from hparams import hparams
from t2_import import t2

L = t2.lib
HU, RU = 128, 128
FAKE = 4096                                         # a non-null device pointer that the checks never dereference
POOL_FWD, HIGHWAY_FWD, GRU_FWD, BN_FWD = 3, 5, 7, 1
INVALID_ARG = -1                                    # T2_ERR_INVALID_ARG
# (B, T) -> (n_params, packed bytes, workspace bytes) of the bf16 mode at the stock CBHG widths (num_freq 1025)
BF16_SIZES = {(4, 37): (1826580, 8028160, 5771008), (32, 200): (1826580, 8028160, 234543616)}


def _hp():
    hp = hparams.copy()
    hp.parse("predict_linear=True")
    return hp


def _lib():
    lib = L.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    return lib


def _sizes(cfg):
    n, pb, wb, nt = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    rc = _lib().t2_cbhg_sizes(ctypes.byref(cfg), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(nt))
    return rc, (n.value, pb.value, wb.value)


def test_cbhg_config_mirror():
    lib = _lib()
    assert lib.t2_struct_size(b"t2_cbhg_config_t") == ctypes.sizeof(t2.tacotron.CbhgConfig)
    names = [f[0] for f in t2.tacotron.CbhgConfig._fields_]
    assert names[-1] == "split_bf16"
    hp = _hp()
    assert t2.tacotron.make_cbhg_config(hp, 4, 37, 0.0).split_bf16 == 0
    assert t2.tacotron.make_cbhg_config(hp, 4, 37, 0.0, "fp32-class").split_bf16 == 1
    with pytest.raises(L.T2Error):
        t2.tacotron.make_cbhg_config(hp, 4, 37, 0.0, "fp16")


@pytest.mark.parametrize("B,T", sorted(BF16_SIZES))
def test_bf16_sizes_are_unchanged(B, T):
    rc, sizes = _sizes(t2.tacotron.make_cbhg_config(_hp(), B, T, 0.0))
    assert rc == 0 and sizes == BF16_SIZES[(B, T)]


def test_split_sizes_grow_only_the_split_buffers():
    hp = _hp()
    rc0, (n0, pb0, wb0) = _sizes(t2.tacotron.make_cbhg_config(hp, 32, 200, 0.0))
    rc1, (n1, pb1, wb1) = _sizes(t2.tacotron.make_cbhg_config(hp, 32, 200, 0.0, "fp32-class"))
    assert rc0 == 0 and rc1 == 0 and n1 == n0
    assert pb0 < pb1 < 3 * pb0 and wb0 < wb1 < 2 * wb0


@pytest.mark.parametrize("value", [2, -1, 1 << 20])
def test_split_values_other_than_0_1_are_rejected(value):
    lib = _lib()
    cfg = t2.tacotron.make_cbhg_config(_hp(), 4, 37, 0.0)
    cfg.split_bf16 = value
    rc, _ = _sizes(cfg)
    assert rc == INVALID_ARG and b"split_bf16" in lib.t2_last_error()
    rc = lib.t2_cbhg_forward(ctypes.byref(cfg), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE),
                             None, None, 0, None)
    assert rc == INVALID_ARG and b"split_bf16" in lib.t2_last_error()
    rc = lib.t2_cbhg_backward(ctypes.byref(cfg), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE),
                              ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE), None)
    assert rc == INVALID_ARG and b"split_bf16" in lib.t2_last_error()


def test_backward_rejects_the_split_mode_before_any_launch():
    lib = _lib()
    cfg = t2.tacotron.make_cbhg_config(_hp(), 4, 37, 0.0, "fp32-class")
    rc = lib.t2_cbhg_backward(ctypes.byref(cfg), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE),
                              ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE), None)
    assert rc == INVALID_ARG and b"no backward pass" in lib.t2_last_error()


def _hook(kernel, p, i):
    lib = _lib()
    c = L.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = v
    for k, v in enumerate(i):
        c.i[k] = v
    return lib.t2_dbg_cbhg_kernel(ctypes.byref(c), None), lib.t2_last_error()


def _ptrs(n):
    return [FAKE * (k + 1) for k in range(n)]


GRU_I = [5, 37, HU, RU, 0, 1000, 2000, 3000, 4000, 5000, 6000, 7000]


@pytest.mark.parametrize("kernel,n_p,ints,slot", [
    (POOL_FWD, 2, [8 * 37, 37, 1024], 3),
    (HIGHWAY_FWD, 7, [8 * 37, HU], 2),
    (GRU_FWD, 3, GRU_I, 12),
    (BN_FWD, 9, [8 * 37, 128, 1024, 0, 1024, 1, 1, 128], 8),
])
@pytest.mark.parametrize("value", [2, -1])
def test_hook_split_argument_is_checked_before_any_launch(kernel, n_p, ints, slot, value):
    i = list(ints) + [0] * (slot + 1 - len(ints))
    i[slot] = value
    rc, err = _hook(kernel, _ptrs(n_p), i)
    assert rc == INVALID_ARG and b"split" in err and b"not 0 or 1" in err, err


def test_split_gru_hook_requires_null_stashes():
    rc, err = _hook(GRU_FWD, _ptrs(11), GRU_I + [1])
    assert rc == INVALID_ARG and b"no stashes" in err, err
