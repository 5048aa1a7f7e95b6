"""Drop-in for the reference's datasets/audio.py: same free functions taking (array, hparams), numpy in / numpy out,
computed by the sm_90a kernels of libt2b200.so (host<->device copies inside each call). No CPU fallback: without
a CUDA device or the built library these functions raise.

Covered (reference datasets/audio.py line numbers): preemphasis :22-25, get_hop_size :54-59, linearspectrogram
:61-68, melspectrogram :70-77, librosa_pad_lr :210-219; plus the mu-law family of wavenet_vocoder/util.py.
Inversion: inv_linear_spectrogram :118-133 / inv_mel_spectrogram :97-112 through a GPU Griffin-Lim (:151-161); the LWS option
(`use_lws`, an external C library) is not provided.
"""
import numpy as np
import torch

from t2_import import t2

_front_ends = {}


def get_hop_size(hparams):
    hop_size = hparams.hop_size
    if hop_size is None:
        assert hparams.frame_shift_ms is not None
        hop_size = int(hparams.frame_shift_ms / 1000 * hparams.sample_rate)
    return hop_size


def _fe(hparams):
    key = (hparams.sample_rate, hparams.n_fft, get_hop_size(hparams), hparams.win_size, hparams.num_mels, hparams.fmin,
           hparams.fmax, hparams.magnitude_power, hparams.min_level_db, hparams.ref_level_db, hparams.max_abs_value,
           hparams.symmetric_mels, hparams.allow_clipping_in_normalization, hparams.signal_normalization)
    if key not in _front_ends:
        _front_ends[key] = t2.audio.MelFrontEnd(hparams)
    return _front_ends[key]


def _to_dev(wav):
    w = torch.from_numpy(np.ascontiguousarray(wav, dtype=np.float32))
    return w.reshape(1, -1).cuda() if w.dim() == 1 else w.cuda()


def preemphasis(wav, k, preemphasize=True):
    if not preemphasize:
        return wav
    return t2.audio.preemphasis(_to_dev(wav), k)[0].cpu().numpy()


def melspectrogram(wav, hparams):
    """wav: 1-D float array -> [num_mels, frames] float32 (audio.py:70-77)."""
    return _fe(hparams)(_to_dev(wav), time_major=False)[0].cpu().numpy()


def linearspectrogram(wav, hparams):
    """wav: 1-D float array -> [n_fft/2+1, frames] float32 (audio.py:61-68)."""
    _, lin = _fe(hparams)(_to_dev(wav), time_major=False, linear=True)
    return lin[0].cpu().numpy()


def _denormalize(D, hparams):
    """inverse of the [-max_abs, max_abs] (symmetric) / [0, max_abs] scaling of the dB spectrogram (audio.py:272-284)"""
    m, floor = hparams.max_abs_value, hparams.min_level_db
    if hparams.allow_clipping_in_normalization:
        D = np.clip(D, -m if hparams.symmetric_mels else 0, m)
    if hparams.symmetric_mels:
        return (D + m) * -floor / (2 * m) + floor
    return D * -floor / m + floor


def _db_to_amp(x):
    return np.power(10.0, x * 0.05)


def _griffin_lim(S, hparams, seed=0):
    """S: [bins, frames] magnitudes -> waveform (audio.py:151-161); phases are re-estimated hparams.griffin_lim_iters times on the GPU"""
    mag = torch.from_numpy(np.ascontiguousarray(np.abs(S).T, dtype=np.float32))[None].cuda()
    return _fe(hparams).griffin_lim(mag, hparams.griffin_lim_iters, seed=seed)[0].cpu().numpy()


def _lin_to_wav(S, hparams):
    if getattr(hparams, "use_lws", False):
        raise NotImplementedError("use_lws: the LWS phase reconstruction library is not part of this repo (datasets/audio.py:126-130)")
    return inv_preemphasis(_griffin_lim(S ** hparams.power, hparams), hparams.preemphasis, hparams.preemphasize)


def inv_linear_spectrogram(linear_spectrogram, hparams):
    """[n_fft/2+1, frames] normalised dB spectrogram -> waveform (audio.py:118-133)"""
    D = _denormalize(linear_spectrogram, hparams) if hparams.signal_normalization else linear_spectrogram
    return _lin_to_wav(_db_to_amp(D + hparams.ref_level_db) ** (1 / hparams.magnitude_power), hparams)


_inv_mel = {}


def _mel_to_linear(mel, hparams):
    """pseudo-inverse of the mel filterbank, floored at 1e-10 (audio.py:231-241)"""
    fe = _fe(hparams)
    if id(fe) not in _inv_mel:
        _inv_mel[id(fe)] = np.linalg.pinv(fe.mel_basis())
    return np.maximum(1e-10, np.dot(_inv_mel[id(fe)], mel))


def inv_mel_spectrogram(mel_spectrogram, hparams):
    """[num_mels, frames] normalised dB mel spectrogram -> waveform (audio.py:97-112)"""
    D = _denormalize(mel_spectrogram, hparams) if hparams.signal_normalization else mel_spectrogram
    return _lin_to_wav(_mel_to_linear(_db_to_amp(D + hparams.ref_level_db) ** (1 / hparams.magnitude_power), hparams), hparams)


def melspectrogram_batch(wavs, hparams, preemphasis_coef=0.0, gain=1.0):
    """Batched variant used by the preprocessor: wavs [B, n] -> [B, frames, num_mels] (the on-disk layout)."""
    return _fe(hparams)(_to_dev(wavs), preemphasis=preemphasis_coef, gain=gain, time_major=True).cpu().numpy()


def librosa_pad_lr(x, fsize, fshift, pad_sides=1):
    assert pad_sides in (1, 2)
    pad = (x.shape[0] // fshift + 1) * fshift - x.shape[0]
    if pad_sides == 1:
        return 0, pad
    return pad // 2, pad // 2 + pad % 2


def mulaw_quantize(x, mu=256):
    return t2.audio.mulaw_quantize(_to_dev(x).reshape(-1)).cpu().numpy().reshape(np.shape(x)).astype(np.int64)


def inv_mulaw_quantize(y, mu=256):
    q = torch.from_numpy(np.ascontiguousarray(y, dtype=np.int32)).reshape(-1).cuda()
    return t2.audio.inv_mulaw_quantize(q).cpu().numpy().reshape(np.shape(y))


def mulaw(x, mu=256):
    return t2.audio.mulaw(_to_dev(x).reshape(-1)).cpu().numpy().reshape(np.shape(x))


def inv_mulaw(y, mu=256):
    return t2.audio.inv_mulaw(_to_dev(y).reshape(-1)).cpu().numpy().reshape(np.shape(y))


# ---- wav IO and silence trimming (reference datasets/audio.py:11-52): host-side plumbing around the kernels --------------------
def load_wav(path, sr):
    """librosa.core.load(path, sr)[0] without librosa: float32 mono in [-1, 1], polyphase-resampled to `sr` when needed."""
    from scipy.io import wavfile
    from scipy.signal import resample_poly
    rate, data = wavfile.read(path)
    if data.dtype.kind == "i":
        data = data.astype(np.float32) / float(np.iinfo(data.dtype).max + 1)
    elif data.dtype.kind == "u":
        data = (data.astype(np.float32) - 128.0) / 128.0
    data = data.astype(np.float32)
    if data.ndim == 2:
        data = data.mean(axis=1)
    if rate != sr:
        from math import gcd
        g = gcd(int(rate), int(sr))
        data = resample_poly(data, sr // g, rate // g).astype(np.float32)
    return data


def save_wav(wav, path, sr):
    from scipy.io import wavfile
    wav = np.asarray(wav)
    wav = wav * (32767 / max(0.01, np.max(np.abs(wav)) if wav.size else 0.0))          # an empty signal (a 0-frame mel) writes an empty file
    wavfile.write(path, sr, wav.astype(np.int16))


def save_wavenet_wav(wav, path, sr, inv_preemphasize=False, k=0.97):
    save_wav(np.asarray(wav, dtype=np.float32), path, sr)


def inv_preemphasis(wav, k, inv_preemphasize=True):
    if not inv_preemphasize:
        return wav
    from scipy import signal
    return signal.lfilter([1], [1, -k], wav)


def start_and_end_indices(quantized, silence_threshold=2):
    """first / last sample whose mu-law index is more than `silence_threshold` away from 127 (audio.py:33-44)"""
    q = np.asarray(quantized).astype(np.int64)
    loud = np.nonzero(np.abs(q - 127) > silence_threshold)[0]
    assert loud.size > 0
    start = int(loud[0])
    tail = loud[loud >= 2]
    end = int(tail[-1]) if tail.size else start
    return start, end


def trim_silence(wav, hparams):
    """librosa.effects.trim(wav, top_db, frame_length, hop_length)[0] (audio.py:46-52): keep from the first to the last frame whose
    RMS power is within trim_top_db of the loudest frame; start = first_frame * hop, end = min(len, (last_frame + 1) * hop).
    UNPINNED (librosa is not installable here). Frames are CENTRED on t * hop with reflect padding - librosa's rmse from 0.6 on. The
    reference's requirements.txt says librosa 0.5.1, but its call passes `frame_length=`, a keyword effects.trim only has from 0.6 (0.5.x
    named it n_fft and framed the unpadded signal), so the code as written needs the centred variant."""
    n, hop, top_db = hparams.trim_fft_size, hparams.trim_hop_size, hparams.trim_top_db
    y = np.pad(np.asarray(wav, dtype=np.float64), n // 2, mode="reflect")
    frames = 1 + (len(y) - n) // hop
    idx = np.arange(n)[None, :] + hop * np.arange(frames)[:, None]
    mse = np.mean(y[idx] ** 2, axis=1)
    db = 10.0 * np.log10(np.maximum(1e-10, mse)) - 10.0 * np.log10(np.maximum(1e-10, mse.max()))
    keep = np.nonzero(db > -top_db)[0]
    if keep.size == 0:
        return wav[:0]
    return wav[int(keep[0]) * hop:min(len(wav), (int(keep[-1]) + 1) * hop)]
