"""The audio front-end kernels (tacotron-2_b200/csrc/t2_audio.cu), one launch at a time through t2_dbg_audio_kernel (STFT_MEL,
GL_INIT_PHASE, GL_ISTFT, GL_OLA, GL_STFT) and the public pre-emphasis call, against float64 references computed here from the exact
fp32 inputs the kernels read (oracle/audio.py stays the end-to-end reference of tests/test_audio_gpu.py). Every n_fft (512, 1024,
2048, 4096) runs with a window shorter than n_fft and with one spanning it. The frame-parallel kernels run F = 4096 / (n_fft / 2)
frames per CTA on at most 2 CTAs per SM, so the main shapes hold more than 2 SMs F frames (the SM count read at run time) over
B = 3 items of a frame count that is not a multiple of F: every CTA makes a second trip, some of its slots leave the loop while their
neighbours go on, and CTAs hold frames of two items. Outputs start as NaN with a NaN guard past their end: every owned element must be
written, the guard must stay NaN.

Bounds (u = 2^-24, the fp32 unit roundoff; e = 2^-53; E = 5 log2(n_fft) e sum |x_w|, a bound on the error of one float64 FFT of the
windowed frame x_w per component, which covers the radix-4/8/16 butterflies with table twiddles, the real-FFT untangle step, and
numpy's pocketfft; kernel and reference each carry one E):
  STFT_MEL   The reference builds each frame as the kernel does (pre-emphasis and gain in float64, the float64 periodic Hann), takes a
             float64 rfft, rounds the components to complex64, and takes np.abs and ** p in float32. Kernel and reference components each
             sit within u |X| + E of the exact X, so |m_kernel - m| <= dm = 4u m + 3E, with m the float64 modulus of the complex64
             components (2u m for the two complex64 roundings, 2 sqrt(2) E < 3E for the two FFTs, 2u m for float(|X|^2) and sqrtf).
             Both values of |X|^p lie in [lo, hi] = [max(m - dm, 0)^p (1 - 12u), (m + dm)^p (1 + 12u)]: 12u covers powf (4 ulp <= 8u)
             or the fp32 square, float(v) in finish() and numpy's own float32 rounding. The mel value is the float64 dot of these with
             the non-negative basis of t2_mel_basis_f64, so its interval is the dot of the intervals (widened by 2^-40 for the float64
             sums). dB = 20 log10(max(min_level, v)) - ref_level_db is monotone in v, so both dB values lie within
             20 log10(max(ml, hi) / max(ml, lo)) of each other, plus log10f (2 ulp <= 4u |log10 v|, times 20), the fp32 product by 20
             (20 u |log10 v|) and the subtraction (u |dB|): bound = 20 log10(hi' / lo') + 100u |log10 v| + 2u |dB|. The raw checks use
             signal_normalization = 0 and min_level_db = -300, so only true zeros reach the floor. Normalisation is affine with slope
             s = (2 if symmetric_mels else 1) max_abs_value / -min_level_db, then clipping (1-Lipschitz): bound = s bound_dB + 8u
             (max_abs_value + |ref|) for its four fp32 operations.
  GL_INIT    sincospif(2u') of the exact fp32 u' = (hash_u32(seed, index) >> 8) 2^-24: within 2^-23 absolute of float64 cos / sin(2 pi u').
  GL_ISTFT   float64 irfft (np.fft.irfft, which ignores the imaginary parts of the DC and Nyquist bins) of S e^(i phi) from the fp32
             magnitudes and phase components, times the float64 window, rounded to fp32: 2u |ref| + 2E', E' = 5 log2(n_fft) e (2 / n_fft)
             sum_k |X_k| (the l1 bound on every output sample sets the scale of the FFT error).
  GL_OLA     m <= ceil(win / hop) frames cover a sample. The kernel adds the m fp32 terms ((m - 1) u sum |t|) and the m fp32 squares of the
             fp32 window (m u wss: each square and each add rounds once, all terms positive), then divides (u): |y - ref| <= (2m + 1) u
             sum |t| / wss where wss > fp32 tiny, (m - 1) u sum |t| where it is not (the plain sum: Hann w[0] = 0, and the gaps of
             hop > win_size, where the result is exactly 0). The frames are arbitrary random values, not the frames of any signal.
  GL_STFT    unit phases z / |z| of the complex64 STFT. The kernel's and the reference's complex64 values differ by <= 2 sqrt(2) (u m + E)
             (m the reference modulus), and |a / |a| - b / |b|| <= 2 |a - b| / |b|, so the phases differ by <= 4 sqrt(2) (u + E / m),
             plus 4u for the fp32 modulus and division: bound 16u + 6E / m, checked where m > 8E (the excluded bins, whose phase is
             not determined by the data, are counted and reported). An all-zero item gives exactly (1, 0) in every bin (np.angle(0) = 0).
  preemphasis, and MelFrontEnd / griffin_lim against the same launches issued through the hook: bit for bit.
Every check records its worst err / bound through parity_util.record. Measured on an H100 80GB HBM3 (132 SMs) at its 700 W power limit:
0.32 for the raw dB spectra, 0.17 normalised, 0.27 for the short clips, 0.29 at 128 mels, 0.41 for the initial phases, 0.50 for GL_ISTFT
(the fp32 rounding), 0.65 for GL_OLA, 0.14 for GL_STFT with no bin excluded; pre-emphasis and both compositions are bit-identical."""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

import mask_hash as mh
from audio_nfft_points import hp_for
from parity_util import record
from t2_import import t2

pytestmark = pytest.mark.gpu
L = t2.lib
DEV = "cuda"
F64 = np.float64
NAN = float("nan")
U = 2.0 ** -24
EPS = 2.0 ** -53
TINY = float(np.finfo(np.float32).tiny)
PAD = 61                                   # NaN guard elements past every output
IDS = dict(STFT_MEL=1, GL_INIT_PHASE=2, GL_ISTFT=3, GL_OLA=4, GL_STFT=5)
# (sample rate, n_fft, hop, win_size): at every n_fft one window shorter than n_fft and one spanning it
POINTS = [(8000, 512, 100, 400), (8000, 512, 128, 512), (16000, 1024, 200, 800), (16000, 1024, 256, 1024), (24000, 2048, 300, 1200),
          (24000, 2048, 512, 2048), (44100, 4096, 551, 2205), (48000, 4096, 1024, 4096)]
RAW = dict(signal_normalization=0, min_level_db=-300.0)


def pid(p):
    return "nfft%d-win%d" % (p[1], p[3])


@functools.lru_cache(maxsize=None)
def front(point, num_mels=None):
    hp = hp_for(*point)
    if num_mels is not None:
        hp.set_hparam("num_mels", num_mels)
        hp.set_hparam("fmin", 0)
    return t2.audio.MelFrontEnd(hp)


def config(fe, **fields):
    c = t2.audio.AudioConfig.from_buffer_copy(fe.cfg)
    for k, v in fields.items():
        setattr(c, k, v)
    return c


def hook(cfg, kernel, p=(), i=(), f=(), seed=0):
    c = L.DbgKernel()
    c.kernel = IDS[kernel]
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate(i):
        c.i[k] = int(v)
    for k, v in enumerate(f):
        c.f[k] = float(v)
    c.seed = seed
    L.check(L.load().t2_dbg_audio_kernel(ctypes.byref(cfg), ctypes.byref(c), L.stream_ptr()))
    torch.cuda.synchronize()


def nan_out(n):
    return torch.full((n + PAD,), NAN, device=DEV)


def body(name, buf, n):
    """the n owned elements of a nan_out buffer as float64 numpy; all written, the guard untouched"""
    assert torch.isnan(buf[n:]).all().item(), "%s: written past its end" % name
    out = buf[:n].cpu().numpy().astype(F64)
    assert not np.isnan(out).any(), "%s: %d elements not written" % (name, int(np.isnan(out).sum()))
    return out


def check(name, got, ref, bound, **info):
    err = np.abs(np.asarray(got, dtype=F64) - ref)
    ratio = np.where(err == 0, 0.0, err / np.where(bound > 0, bound, 1e-300))
    worst = float(np.nan_to_num(ratio, nan=np.inf).max()) if ratio.size else 0.0
    record(name, worst_err_over_bound=worst, **info)
    assert worst <= 1.0, "%s: worst err / bound %.3g at %s" % (name, worst, np.unravel_index(np.argmax(ratio), ratio.shape))


def grid_frames(n_fft):
    """frames per item for B = 3 items: past one full wave of the frame grid (2 CTAs per SM, F frames each), with a partial second
    wave, and not a multiple of F"""
    F = 4096 // (n_fft // 2)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    fr = -(-(2 * sms * F + 5 * F + 3) // 3)
    while fr % F == 0:
        fr += 1
    assert 3 * fr > 2 * sms * F and (3 * fr) % (2 * sms * F) != 0
    return fr


def hann(win):
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win) / win)


def frames64(x32, n_fft, hop, win, pre=0.0, gain=1.0):
    """[B, 1 + n // hop, n_fft] float64 frames as the STFT kernels build them: centred, zero padded, pre-emphasis and gain in float64,
    times the float64 periodic Hann placed in the middle of the n_fft frame"""
    B, n = x32.shape
    x = x32.astype(F64)
    if pre != 0.0:
        x = x - F64(np.float32(pre)) * np.concatenate([np.zeros((B, 1)), x[:, :-1]], axis=1)
    x = x * F64(np.float32(gain))
    lpad = (n_fft - win) // 2
    w = np.zeros(n_fft)
    w[lpad:lpad + win] = hann(win)
    si = np.arange(1 + n // hop)[:, None] * hop - n_fft // 2 + np.arange(n_fft)[None, :]
    ok = (si >= 0) & (si < n)
    return np.where(ok[None], x[:, np.clip(si, 0, n - 1)], 0.0) * w


def fft_err(n_fft, l1):
    return 5 * math.log2(n_fft) * EPS * l1


def spectrum_ref(frames, n_fft, p):
    """(float32 |X|^p as float64, float64 modulus of the complex64 components, per-frame FFT error E)"""
    Xc = np.fft.rfft(frames, axis=-1).astype(np.complex64)
    v = (np.abs(Xc) ** np.float32(p)).astype(F64)
    m = np.abs(Xc.astype(np.complex128))
    return v, m, fft_err(n_fft, np.abs(frames).sum(-1, keepdims=True))


def db_bound(v, lo, hi, ml, ref_db):
    lv = np.log10(np.maximum(ml, v))
    y = 20 * lv - ref_db
    return y, 20 * np.log10(np.maximum(ml, hi) / np.maximum(ml, lo)) + 100 * U * np.abs(lv) + 2 * U * np.abs(y)


def normalize(cfg, y, b):
    M, mdb = cfg.max_abs_value, cfg.min_level_db
    s = (2 * M if cfg.symmetric_mels else M) / -mdb
    r = s * (y - mdb) - (M if cfg.symmetric_mels else 0.0)
    if cfg.allow_clipping_in_normalization:
        r = np.clip(r, -M if cfg.symmetric_mels else 0.0, M)
    return r, s * b + 8 * U * (M + np.abs(r))


def expected(fe, cfg, wav, pre, gain):
    """(mel, lin) references and bounds, [B, frames, nm] / [B, frames, bins]"""
    p = cfg.magnitude_power
    v, m, E = spectrum_ref(frames64(wav, cfg.n_fft, cfg.hop_size, cfg.win_size, pre, gain), cfg.n_fft, p)
    dm = 4 * U * m + 3 * E
    lo, hi = np.maximum(m - dm, 0.0) ** p * (1 - 12 * U), (m + dm) ** p * (1 + 12 * U)
    W = fe.mel_basis().T
    ml = float(np.float32(math.exp(cfg.min_level_db / 20.0 * math.log(10.0))))
    lin = db_bound(v, lo, hi, ml, cfg.ref_level_db)
    mel = db_bound(v @ W, (lo @ W) * (1 - 2.0 ** -40), (hi @ W) * (1 + 2.0 ** -40), ml, cfg.ref_level_db)
    if cfg.signal_normalization:
        lin, mel = normalize(cfg, *lin), normalize(cfg, *mel)
    return mel, lin


def stft_mel(fe, cfg, wav, pre=0.0, gain=1.0, time_major=1, linear=True):
    """one STFT_MEL launch -> (mel [B, frames, nm], lin [B, frames, bins] or None), read back time-major"""
    B, n = wav.shape
    fr, nm, bins = 1 + n // cfg.hop_size, cfg.num_mels, cfg.n_fft // 2 + 1
    mel = nan_out(B * fr * nm)
    lin = nan_out(B * fr * bins) if linear else None
    hook(cfg, "STFT_MEL", p=(fe.plan, torch.from_numpy(wav).to(DEV), mel, lin), i=(B, n, time_major), f=(pre, gain))
    out = []
    for name, buf, c in (("mel", mel, nm), ("lin", lin, bins)):
        if buf is None:
            out.append(None)
            continue
        a = body(name, buf, B * fr * c)
        out.append(a.reshape(B, fr, c) if time_major else a.reshape(B, c, fr).transpose(0, 2, 1))
    return out


def chirp(rng, n, sr, amp):
    """chirp from 100 Hz to 0.4 sr plus noise at a tenth of its amplitude, fp32"""
    t = np.arange(n) / float(sr)
    w = amp * np.sin(2 * np.pi * (100 + 0.2 * sr * t / max(t[-1], 1.0 / sr)) * t) + rng.normal(0, 0.1 * amp, n)
    return w.astype(np.float32)


# ---- STFT_MEL ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("point", POINTS, ids=pid)
def test_stft_mel_raw_db(point):
    """dB spectra without normalisation at magnitude_power 2 and 1, pre-emphasis / gain off and on, both layouts, on the grid-stride
    shape: a loud chirp, a silent item (the floor, reached only by true zeros) and a quiet chirp"""
    fe = front(point)
    sr, n_fft, hop = point[:3]
    fr = grid_frames(n_fft)
    n = (fr - 1) * hop + hop // 2
    rng = np.random.default_rng(n_fft + point[3])
    wav = np.stack([chirp(rng, n, sr, 0.5), np.zeros(n, np.float32), chirp(rng, n, sr, 0.02)])
    for power, pre, gain, tm in ((2.0, 0.0, 1.0, 1), (2.0, 0.97, 1.7, 0), (1.0, 0.0, 1.0, 0), (1.0, 0.97, 0.6, 1)):
        cfg = config(fe, magnitude_power=power, **RAW)
        mel, lin = stft_mel(fe, cfg, wav, pre, gain, tm)
        (rm, bm), (rl, bl) = expected(fe, cfg, wav, pre, gain)
        info = dict(n_fft=n_fft, win=point[3], power=power, preemphasis=pre, time_major=tm, frames=3 * fr)
        check("stft_mel_raw_mel", mel, rm, bm, **info)
        check("stft_mel_raw_lin", lin, rl, bl, **info)
        assert (rl[1] == rl[1].min()).all() and rl[0].max() > rl[1].max() + 200       # the silent item sits on the floor


@pytest.mark.parametrize("point", POINTS, ids=pid)
def test_stft_mel_normalisation(point):
    """signal_normalization at the four (symmetric_mels, clipping) combinations: a loud sinusoid clips at +max_abs_value, a silent item
    at the bottom end, a mid-level chirp in noise (noise power per bin about -15 dB, 50 dB above the floor) lands inside the range"""
    fe = front(point)
    sr, n_fft, hop, win = point
    n = 37 * hop + 11
    rng = np.random.default_rng(sr)
    t = np.arange(n) / float(sr)
    loud = 0.9 * np.sin(2 * np.pi * 440.0 * t)
    mid = 0.02 * np.sin(2 * np.pi * (100 + 0.2 * sr * t / t[-1]) * t) + rng.normal(0, math.sqrt(0.03 / (0.375 * win)), n)
    wav = np.stack([loud, np.zeros(n), mid]).astype(np.float32)
    for sym in (1, 0):
        for clip in (1, 0):
            cfg = config(fe, symmetric_mels=sym, allow_clipping_in_normalization=clip)
            mel, lin = stft_mel(fe, cfg, wav, time_major=sym)
            (rm, bm), (rl, bl) = expected(fe, cfg, wav, 0.0, 1.0)
            M = cfg.max_abs_value
            bottom = -M if sym else 0.0
            for r in (rm, rl):
                if clip:
                    assert (r[0] == M).any() and (r[1] == bottom).all()
                else:
                    assert r[0].max() > M and r[1].max() < bottom
                inside = (r[2] > bottom + 0.1) & (r[2] < M - 0.1)
                assert inside.mean() > 0.3, inside.mean()
            check("stft_mel_norm_mel", mel, rm, bm, n_fft=n_fft, win=point[3], symmetric=sym, clip=clip)
            check("stft_mel_norm_lin", lin, rl, bl, n_fft=n_fft, win=point[3], symmetric=sym, clip=clip)


@pytest.mark.parametrize("point", POINTS, ids=pid)
def test_stft_mel_short_clips_layouts_and_no_linear(point):
    """n_samples of 1, below hop and below n_fft, B = 2, both layouts, with and without the linear output"""
    fe = front(point)
    sr, n_fft, hop = point[:3]
    rng = np.random.default_rng(hop)
    cfg = config(fe, **RAW)
    for n in (1, hop - 1, n_fft - 3):
        wav = np.stack([chirp(rng, n, sr, 0.3), chirp(rng, n, sr, 0.05)])
        (rm, bm), (rl, bl) = expected(fe, cfg, wav, 0.97, 1.0)
        for tm, linear in ((1, True), (0, False)):
            mel, lin = stft_mel(fe, cfg, wav, 0.97, 1.0, tm, linear)
            check("stft_mel_short_mel", mel, rm, bm, n_fft=n_fft, n=n, time_major=tm)
            if linear:
                check("stft_mel_short_lin", lin, rl, bl, n_fft=n_fft, n=n)


def test_stft_mel_128_mels_at_512():
    """num_mels = 128 at n_fft = 512 (8 kHz, fmin 0): the low filters span two or three bins"""
    point = (8000, 512, 100, 400)
    fe = front(point, num_mels=128)
    W = fe.mel_basis()
    widths = (W != 0).sum(1)
    assert fe.cfg.num_mels == 128 and widths.min() <= 2
    fr = grid_frames(512)
    n = (fr - 1) * 100 + 3
    wav = np.stack([chirp(np.random.default_rng(s), n, 8000, a) for s, a in ((1, 0.5), (2, 0.05), (3, 0.2))])
    cfg = config(fe, **RAW)
    mel, lin = stft_mel(fe, cfg, wav, 0.0, 1.0, 1)
    (rm, bm), (rl, bl) = expected(fe, cfg, wav, 0.0, 1.0)
    check("stft_mel_128_mel", mel, rm, bm, min_filter_bins=int(widths.min()))
    check("stft_mel_128_lin", lin, rl, bl)


@pytest.mark.parametrize("point", POINTS, ids=pid)
def test_mel_front_end_is_the_hook_launch(point):
    """MelFrontEnd.__call__ (the product path) equals the STFT_MEL launch bit for bit"""
    fe = front(point)
    sr, n_fft, hop = point[:3]
    n = 23 * hop + 5
    wav = np.stack([chirp(np.random.default_rng(s), n, sr, 0.4) for s in range(2)])
    x = torch.from_numpy(wav).to(DEV)
    for tm in (1, 0):
        mel, lin = fe(x, preemphasis=0.97, gain=1.3, time_major=bool(tm), linear=True)
        fr, nm, bins = 1 + n // hop, fe.cfg.num_mels, n_fft // 2 + 1
        hm, hl = nan_out(2 * fr * nm), nan_out(2 * fr * bins)
        hook(fe.cfg, "STFT_MEL", p=(fe.plan, x, hm, hl), i=(2, n, tm), f=(0.97, 1.3))
        assert torch.equal(mel.reshape(-1), hm[:2 * fr * nm]) and torch.equal(lin.reshape(-1), hl[:2 * fr * bins])


# ---- Griffin-Lim --------------------------------------------------------------------------------------------------------------------
def test_gl_init_phase():
    """exp(2 pi i u) from the counter hash, n not a multiple of 256"""
    fe = front(POINTS[0])
    n = 3 * 37 * 257 + 5
    for seed in (7, 0x1234_5678_9ABC_DEF0):
        ph = nan_out(2 * n)
        hook(fe.cfg, "GL_INIT_PHASE", p=(ph,), i=(n,), seed=seed)
        got = body("phase", ph, 2 * n).reshape(n, 2)
        u = (mh.hash_u32(seed, np.arange(n, dtype=np.uint64)) >> np.uint32(8)).astype(F64) * 2.0 ** -24
        bound = np.full(n, 2.0 ** -23)
        check("gl_init_phase_cos", got[:, 0], np.cos(2 * np.pi * u), bound, seed=seed)
        check("gl_init_phase_sin", got[:, 1], np.sin(2 * np.pi * u), bound, seed=seed)


def random_spectrum(rng, B, fr, bins):
    """fp32 magnitudes in [0, 1) and fp32 (cos, sin) of random angles: the DC and Nyquist bins get non-zero imaginary parts too"""
    S = rng.random((B, fr, bins)).astype(np.float32)
    a = rng.random((B, fr, bins)) * 2 * np.pi
    ph = np.stack([np.cos(a), np.sin(a)], axis=-1).astype(np.float32)
    assert np.abs(ph[:, :, [0, -1], 1]).mean() > 0.3
    return S, ph


@pytest.mark.parametrize("point", POINTS, ids=pid)
def test_gl_istft(point):
    fe = front(point)
    n_fft, hop, win = point[1:]
    bins = n_fft // 2 + 1
    fr = grid_frames(n_fft)
    S, ph = random_spectrum(np.random.default_rng(n_fft + win), 3, fr, bins)
    out = nan_out(3 * fr * win)
    hook(fe.cfg, "GL_ISTFT", p=(fe.plan, torch.from_numpy(S).to(DEV), torch.from_numpy(ph).to(DEV), out), i=(3, fr))
    got = body("frames", out, 3 * fr * win).reshape(3, fr, win)
    X = S.astype(F64) * (ph[..., 0].astype(F64) + 1j * ph[..., 1].astype(F64))
    lpad = (n_fft - win) // 2
    ref = np.fft.irfft(X, n=n_fft, axis=-1)[..., lpad:lpad + win] * hann(win)
    E = fft_err(n_fft, 2.0 / n_fft * np.abs(X).sum(-1, keepdims=True))
    check("gl_istft", got, ref, 2 * U * np.abs(ref) + 2 * E, n_fft=n_fft, win=win, frames=3 * fr)


def ola_hops(win):
    d = next(k for k in (4, 5, 3, 7) if win % k == 0)
    h = win // 3 + 1
    while win % h == 0:
        h += 1
    return (win // d, h, win + 37)          # divides win_size, does not, exceeds it


@pytest.mark.parametrize("point", POINTS, ids=pid)
def test_gl_ola(point):
    fe = front(point)
    n_fft, _, win = point[1:]
    rng = np.random.default_rng(win)
    B, fr = 2, 37
    lpad = (n_fft - win) // 2
    w2 = np.float32(hann(win)).astype(F64) ** 2            # the fp32 window the kernel squares
    for hop in ola_hops(win):
        cfg = config(fe, hop_size=hop)
        frames = rng.standard_normal((B, fr, win)).astype(np.float32)
        n_out = hop * (fr - 1)
        y = nan_out(B * n_out)
        hook(cfg, "GL_OLA", p=(fe.plan, torch.from_numpy(frames).to(DEV), y), i=(B, fr))
        got = body("y", y, B * n_out).reshape(B, n_out)
        pos = np.arange(n_out) + n_fft // 2 - lpad
        acc, l1, wss, m = np.zeros((B, n_out)), np.zeros((B, n_out)), np.zeros(n_out), np.zeros(n_out)
        for k in range(fr):
            wi = pos - k * hop
            ok = (wi >= 0) & (wi < win)
            t = np.where(ok[None], frames[:, k, np.clip(wi, 0, win - 1)].astype(F64), 0.0)
            acc, l1 = acc + t, l1 + np.abs(t)
            wss, m = wss + np.where(ok, w2[np.clip(wi, 0, win - 1)], 0.0), m + ok
        div = wss > TINY
        ref = np.where(div, acc / np.where(div, wss, 1.0), acc)
        bound = np.where(div, (2 * m + 1) * U * l1 / np.where(div, wss, 1.0), np.maximum(m - 1, 0) * U * l1)
        if hop > win:
            assert (m == 0).any() and (got[:, m == 0] == 0).all()        # the gaps between frames are exactly 0
        assert (~div & (m > 0)).any() or hop <= win
        check("gl_ola", got, ref, bound, n_fft=n_fft, win=win, hop=hop, plain_sum_samples=int((~div).sum()))


@pytest.mark.parametrize("point", POINTS, ids=pid)
def test_gl_stft(point):
    fe = front(point)
    n_fft, hop, win = point[1:]
    bins = n_fft // 2 + 1
    fr = grid_frames(n_fft)
    n_out = hop * (fr - 1)
    rng = np.random.default_rng(hop)
    y = (0.3 * rng.standard_normal((3, n_out))).astype(np.float32)
    y[1] = 0.0
    ph = nan_out(3 * fr * bins * 2)
    hook(fe.cfg, "GL_STFT", p=(fe.plan, torch.from_numpy(y).to(DEV), ph), i=(3, fr))
    got = body("phase", ph, 3 * fr * bins * 2).reshape(3, fr, bins, 2)
    assert (got[1, ..., 0] == 1).all() and (got[1, ..., 1] == 0).all()              # np.angle(0) = 0
    frames = frames64(y, n_fft, hop, win)
    Xc = np.fft.rfft(frames, axis=-1).astype(np.complex64).astype(np.complex128)
    m = np.abs(Xc)
    E = fft_err(n_fft, np.abs(frames).sum(-1, keepdims=True))
    keep = m > 8 * E
    keep[1] = False
    excluded = int((~keep[[0, 2]]).sum())
    ref = Xc / np.where(m > 0, m, 1.0)
    bound = (16 * U + 6 * E / np.where(m > 0, m, 1.0))[keep]
    for c, part in enumerate((ref.real, ref.imag)):
        check("gl_stft", got[..., c][keep], part[keep], bound, n_fft=n_fft, win=win, frames=3 * fr, excluded_bins=excluded)
    assert excluded <= 2 * fr * bins // 1000


@pytest.mark.parametrize("point", POINTS, ids=pid)
def test_griffin_lim_is_the_hook_launches(point):
    """MelFrontEnd.griffin_lim equals init / istft / ola / stft / ... issued one launch at a time, bit for bit: the waveform, and the
    final phases left in phase_io"""
    fe = front(point)
    n_fft, hop, win = point[1:]
    bins, B, fr = n_fft // 2 + 1, 2, 45
    S, ph = random_spectrum(np.random.default_rng(3), B, fr, bins)
    mag = torch.from_numpy(S).to(DEV)
    for iters, seed in ((2, None), (1, 7)):
        ph_a = torch.from_numpy(ph).to(DEV)
        wav = fe.griffin_lim(mag, iters, seed=seed or 0, phase=None if seed else ph_a)
        ph_b = torch.from_numpy(ph).to(DEV).reshape(-1) if seed is None else torch.empty(B * fr * bins * 2, device=DEV)
        frames, y = torch.empty(B * fr * win, device=DEV), torch.empty(B, hop * (fr - 1), device=DEV)
        if seed is not None:
            hook(fe.cfg, "GL_INIT_PHASE", p=(ph_b,), i=(B * fr * bins,), seed=seed)
        for it in range(iters + 1):
            hook(fe.cfg, "GL_ISTFT", p=(fe.plan, mag, ph_b, frames), i=(B, fr))
            hook(fe.cfg, "GL_OLA", p=(fe.plan, frames, y), i=(B, fr))
            if it < iters:
                hook(fe.cfg, "GL_STFT", p=(fe.plan, y, ph_b), i=(B, fr))
        assert torch.equal(wav, y), (iters, seed)
        if seed is None:
            assert torch.equal(ph_a.reshape(-1), ph_b)


# ---- pre-emphasis -------------------------------------------------------------------------------------------------------------------
def test_preemphasis_restarts_every_row():
    rng = np.random.default_rng(11)
    x = rng.uniform(-1, 1, (4, 1237)).astype(np.float32)
    k = 0.97
    got = t2.audio.preemphasis(torch.from_numpy(x).to(DEV), k).cpu().numpy()
    prev = np.concatenate([np.zeros((4, 1)), x[:, :-1].astype(F64)], axis=1)
    ref = (x.astype(F64) - F64(np.float32(k)) * prev).astype(np.float32)
    record("preemphasis", mismatches=int((got != ref).sum()))
    assert np.array_equal(got, ref)
