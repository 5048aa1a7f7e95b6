"""Host side of the audio front-end at every supported n_fft (512, 1024, 2048, 4096): plan sizing, the rejection of every other
size, Griffin-Lim workspace sizing, the mel filterbank against the oracle and the win_size=None default. No GPU compute."""
import ctypes

import numpy as np
import pytest

from audio_nfft_points import POINTS, hp_for, point_id
from oracle import audio as oa
from t2_import import t2

T2_ERR_UNSUPPORTED_SHAPE = -2


def _plan_bytes(hp):
    lib = t2.lib.load()
    cfg = t2.audio.make_config(hp)
    nb = ctypes.c_longlong(-1)
    return lib.t2_stft_mel_plan_bytes(ctypes.byref(cfg), ctypes.byref(nb)), nb.value


@pytest.mark.parametrize("point", POINTS, ids=point_id)
def test_plan_accepts_power_of_two_sizes(point):
    rc, nb = _plan_bytes(hp_for(*point))
    assert rc == 0, t2.lib.load().t2_last_error()
    n = point[1] // 2
    assert nb >= n * 16 + (n // 2 + 1) * 16 + point[3] * 8    # twiddles W_N, W_n_fft (half range) and the window


@pytest.mark.parametrize("n_fft", [256, 8192, 1100, 1200, 2000])
def test_plan_rejects_other_sizes(n_fft):
    hp = hp_for(22050, 2048, 275, 256)
    hp.set_hparam("n_fft", n_fft)
    rc, _ = _plan_bytes(hp)
    assert rc == T2_ERR_UNSUPPORTED_SHAPE
    msg = t2.lib.load().t2_last_error().decode()
    assert "512, 1024, 2048 or 4096" in msg and "got %d" % n_fft in msg and "hparams.py:52" in msg
    with pytest.raises(t2.lib.T2Error):
        t2.audio.MelFrontEnd(hp, device="cpu")                 # the plan is sized before any device memory is touched


def test_plan_keeps_its_other_checks():
    for kw in (dict(win_size=1200, n_fft=1024), dict(num_mels=129), dict(fmax=4001, sample_rate=8000, n_fft=512, win_size=400)):
        hp = hp_for(22050, 2048, 275, 1100)
        for k, v in kw.items():
            hp.set_hparam(k, v)
        rc, _ = _plan_bytes(hp)
        assert rc < 0, kw


@pytest.mark.parametrize("n_fft", [512, 1024, 2048, 4096])
def test_griffin_lim_workspace_scales_with_n_fft(n_fft):
    lib = t2.lib.load()
    hp = hp_for(16000, n_fft, 200, 400)
    cfg = t2.audio.make_config(hp)
    B, frames = 3, 37
    nb = ctypes.c_longlong()
    assert lib.t2_griffin_lim_bytes(ctypes.byref(cfg), B, frames, ctypes.byref(nb)) == 0
    al = lambda v: (v + 255) // 256 * 256
    assert nb.value == al(B * frames * (n_fft // 2 + 1) * 8) + al(B * frames * 400 * 4)   # float2 phases + windowed frames


@pytest.mark.parametrize("point", POINTS, ids=point_id)
def test_mel_basis_matches_oracle(point):
    hp = hp_for(*point)
    lib = t2.lib.load()
    cfg = t2.audio.make_config(hp)
    out = np.zeros((hp.num_mels, hp.n_fft // 2 + 1), dtype=np.float64)
    assert lib.t2_mel_basis_f64(ctypes.byref(cfg), out.ctypes.data_as(ctypes.c_void_p)) == 0
    ref = oa.build_mel_basis(hp)
    assert out.shape == ref.shape
    assert np.abs(out - ref).max() <= 1e-12 * np.abs(ref).max()


def test_win_size_none_means_n_fft():
    for n_fft in (512, 4096):
        hp = hp_for(16000, n_fft, 200, None)
        cfg = t2.audio.make_config(hp)
        assert cfg.win_size == n_fft
        assert _plan_bytes(hp)[0] == 0


# t2_dbg_audio_kernel (tests/test_audio_kernels_gpu.py): each call breaks one argument of an otherwise valid launch and is refused before
# any driver call; the fake pointers are never dereferenced and nothing is launched
_FAKE = [256 * (k + 1) for k in range(4)]
_HOOK_GOOD = {1: (_FAKE, [3, 5000, 1]), 2: (_FAKE[:1], [1000]), 3: (_FAKE, [3, 40]), 4: (_FAKE[:3], [3, 40]), 5: (_FAKE[:3], [3, 40])}


def _audio_hook(kernel, p, i, f=(0.97, 1.0), n_fft=1024):
    lib = t2.lib.load()
    hp = hp_for(16000, 1024, 200, 800)
    hp.set_hparam("n_fft", n_fft)
    cfg = t2.audio.make_config(hp)
    c = t2.lib.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = v
    for k, v in enumerate(i):
        c.i[k] = v
    for k, v in enumerate(f):
        c.f[k] = v
    return lib.t2_dbg_audio_kernel(ctypes.byref(cfg), ctypes.byref(c), None), lib.t2_last_error()


@pytest.mark.parametrize("kernel,change,msg", [
    (9, None, b"unknown kernel id"), (0, None, b"unknown kernel id"),
    (1, ("p", 0), b"STFT_MEL: null"), (1, ("p", 1), b"STFT_MEL: null"), (1, ("p", 2), b"STFT_MEL: null"),
    (1, ("i", 0, 0), b"STFT_MEL: B"), (1, ("i", 1, 0), b"STFT_MEL: B"), (1, ("i", 2, 2), b"time_major"), (1, ("i", 2, -1), b"time_major"),
    (1, ("f", 0, float("nan")), b"finite"), (1, ("f", 1, float("inf")), b"finite"),
    (2, ("p", 0), b"GL_INIT_PHASE"), (2, ("i", 0, 0), b"GL_INIT_PHASE"),
    (3, ("p", 0), b"GL_ISTFT: null"), (3, ("p", 3), b"GL_ISTFT: null"), (3, ("i", 0, 0), b"GL_ISTFT: B"), (3, ("i", 1, 1), b"GL_ISTFT: B"),
    (4, ("p", 2), b"GL_OLA: null"), (4, ("i", 0, 0), b"GL_OLA: B"), (4, ("i", 1, 1), b"GL_OLA: B"),
    (5, ("p", 1), b"GL_STFT: null"), (5, ("i", 0, 0), b"GL_STFT: B"), (5, ("i", 1, 1), b"GL_STFT: B")])
def test_audio_hook_refuses_bad_arguments_before_any_launch(kernel, change, msg):
    lib = t2.lib.load()
    n0 = lib.t2_launch_count()
    p, i = _HOOK_GOOD.get(kernel, (_FAKE, [1, 1]))
    p, i, f = list(p), list(i), [0.97, 1.0]
    if change is not None:
        if change[0] == "p":
            p[change[1]] = 0
        else:
            {"i": i, "f": f}[change[0]][change[1]] = change[2]
    rc, err = _audio_hook(kernel, p, i, f)
    assert rc in (-1, -2) and msg in err, (rc, err)
    assert lib.t2_launch_count() == n0


@pytest.mark.parametrize("kernel", [1, 2, 3, 4, 5])
def test_audio_hook_refuses_an_unsupported_n_fft(kernel):
    p, i = _HOOK_GOOD[kernel]
    rc, err = _audio_hook(kernel, list(p), list(i), n_fft=8192)
    assert rc == T2_ERR_UNSUPPORTED_SHAPE and b"got 8192" in err, err
