"""Host side of the audio front-end kernels (csrc/t2_audio.cu): plans, batched GPU calls on torch tensors."""
import ctypes

import torch

from . import lib as L


class AudioConfig(ctypes.Structure):
    _fields_ = [
        ("sample_rate", ctypes.c_int), ("n_fft", ctypes.c_int), ("hop_size", ctypes.c_int),
        ("win_size", ctypes.c_int), ("num_mels", ctypes.c_int), ("fmin", ctypes.c_float), ("fmax", ctypes.c_float),
        ("magnitude_power", ctypes.c_float), ("min_level_db", ctypes.c_float), ("ref_level_db", ctypes.c_float),
        ("max_abs_value", ctypes.c_float), ("symmetric_mels", ctypes.c_int),
        ("allow_clipping_in_normalization", ctypes.c_int), ("signal_normalization", ctypes.c_int),
    ]


def make_config(hp):
    hop = hp.hop_size
    if hop is None:
        hop = int(hp.frame_shift_ms / 1000 * hp.sample_rate)
    win = hp.win_size
    if win is None:  # librosa.stft(win_length=None): the window spans the whole frame (reference hparams.py:81)
        win = hp.n_fft
    c = AudioConfig()
    c.sample_rate, c.n_fft, c.hop_size, c.win_size, c.num_mels = hp.sample_rate, hp.n_fft, hop, win, hp.num_mels
    c.fmin, c.fmax, c.magnitude_power = hp.fmin, hp.fmax, hp.magnitude_power
    c.min_level_db, c.ref_level_db, c.max_abs_value = hp.min_level_db, hp.ref_level_db, hp.max_abs_value
    c.symmetric_mels = int(hp.symmetric_mels)
    c.allow_clipping_in_normalization = int(hp.allow_clipping_in_normalization)
    c.signal_normalization = int(hp.signal_normalization)
    return c


class MelFrontEnd(object):
    """Fused STFT -> |.|^p -> mel -> dB -> normalise on the GPU for batches of equal-length clips."""

    def __init__(self, hparams, device="cuda"):
        self.lib = L.load()
        self.cfg = make_config(hparams)
        self.device = torch.device(device)
        nbytes = ctypes.c_longlong()
        L.check(self.lib.t2_stft_mel_plan_bytes(ctypes.byref(self.cfg), ctypes.byref(nbytes)))
        self.plan = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            L.check(self.lib.t2_stft_mel_plan_init(ctypes.byref(self.cfg), L.ptr(self.plan), L.stream_ptr()))

    def frames(self, n_samples):
        return 1 + n_samples // self.cfg.hop_size

    def __call__(self, wav, preemphasis=0.0, gain=1.0, time_major=True, linear=False, out=None, out_linear=None):
        """wav: fp32 CUDA tensor [B, n] -> mel fp32 [B, frames, num_mels] (time_major) or [B, num_mels, frames]."""
        assert wav.is_cuda and wav.dtype == torch.float32 and wav.dim() == 2 and wav.is_contiguous()
        B, n = wav.shape
        fr = self.frames(n)
        nm, bins = self.cfg.num_mels, self.cfg.n_fft // 2 + 1
        if out is None:
            out = torch.empty((B, fr, nm) if time_major else (B, nm, fr), dtype=torch.float32, device=wav.device)
        if linear and out_linear is None:
            out_linear = torch.empty((B, fr, bins) if time_major else (B, bins, fr), dtype=torch.float32, device=wav.device)
        L.check(self.lib.t2_stft_mel_f32(ctypes.byref(self.cfg), L.ptr(self.plan), L.ptr(wav), B, n,
                                         ctypes.c_float(preemphasis), ctypes.c_float(gain), L.ptr(out),
                                         L.ptr(out_linear if linear else None), int(time_major), L.stream_ptr()))
        return (out, out_linear) if linear else out


    def mel_basis(self):
        """dense [num_mels, n_fft/2+1] float64 filterbank of the fused kernel (host copy)"""
        import numpy as np
        out = np.zeros((self.cfg.num_mels, self.cfg.n_fft // 2 + 1), dtype=np.float64)
        L.check(self.lib.t2_mel_basis_f64(ctypes.byref(self.cfg), out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def griffin_lim(self, mag, iters, seed=0, phase=None):
        """mag: fp32 CUDA [B, frames, bins] magnitudes -> waveform fp32 [B, hop * (frames - 1)] after `iters` Griffin-Lim rounds
        (datasets/audio.py:151-161). phase: optional fp32 [B, frames, bins, 2] initial unit phases (updated in place)."""
        assert mag.is_cuda and mag.dtype == torch.float32 and mag.dim() == 3 and mag.is_contiguous() and mag.shape[2] == self.cfg.n_fft // 2 + 1
        B, frames = int(mag.shape[0]), int(mag.shape[1])
        nb = ctypes.c_longlong()
        L.check(self.lib.t2_griffin_lim_bytes(ctypes.byref(self.cfg), B, frames, ctypes.byref(nb)))
        ws = torch.empty(nb.value, dtype=torch.uint8, device=mag.device)
        wav = torch.empty(B, self.cfg.hop_size * (frames - 1), dtype=torch.float32, device=mag.device)
        if phase is not None:
            assert phase.is_cuda and phase.dtype == torch.float32 and phase.is_contiguous() and tuple(phase.shape) == (B, frames, mag.shape[2], 2)
        L.check(self.lib.t2_griffin_lim_f32(ctypes.byref(self.cfg), L.ptr(self.plan), L.ptr(mag), L.ptr(phase), B, frames, int(iters),
                                            ctypes.c_ulonglong(seed), L.ptr(ws), L.ptr(wav), L.stream_ptr()))
        return wav


def _eltwise(fn_name, x, out_dtype):
    lib = L.load()
    assert x.is_cuda and x.is_contiguous()
    out = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    L.check(getattr(lib, fn_name)(L.ptr(x), L.ptr(out), ctypes.c_longlong(x.numel()), L.stream_ptr()))
    return out


def mulaw_quantize(x):
    """fp32 CUDA tensor in [-1, 1] -> int32 mu-law indices (wavenet_vocoder/util.py:71-102)."""
    assert x.dtype == torch.float32
    return _eltwise("t2_mulaw_quantize_f32_i32", x, torch.int32)


def inv_mulaw_quantize(q):
    assert q.dtype == torch.int32
    return _eltwise("t2_inv_mulaw_quantize_i32_f32", q, torch.float32)


def mulaw(x):
    assert x.dtype == torch.float32
    return _eltwise("t2_mulaw_f32", x, torch.float32)


def inv_mulaw(y):
    assert y.dtype == torch.float32
    return _eltwise("t2_inv_mulaw_f32", y, torch.float32)


def preemphasis(x, k):
    lib = L.load()
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.is_contiguous()
    y = torch.empty_like(x)
    L.check(lib.t2_preemphasis_f32(L.ptr(x), L.ptr(y), x.shape[0], x.shape[1], ctypes.c_float(k), L.stream_ptr()))
    return y
