"""The (sample rate, n_fft, hop, window) points the audio front-end is tested at: the reference's advice (hparams.py:43-54) of a
50 ms window, a 12.5 ms hop and n_fft the first power of two above the window, from 8 to 48 kHz."""
from hparams import hparams

POINTS = [(8000, 512, 100, 400), (16000, 1024, 200, 800), (24000, 2048, 300, 1200), (44100, 4096, 551, 2205), (48000, 4096, 600, 2400)]


def hp_for(sample_rate, n_fft, hop, win):
    hp = hparams.copy()
    hp.set_hparam("sample_rate", sample_rate)
    hp.set_hparam("n_fft", n_fft)
    hp.set_hparam("num_freq", n_fft // 2 + 1)
    hp.set_hparam("hop_size", hop)
    hp.set_hparam("win_size", win)
    hp.set_hparam("fmax", min(hparams.fmax, sample_rate // 2))   # the stock 7600 Hz is above Nyquist at 8 kHz
    return hp


def point_id(p):
    return "%dHz-nfft%d-win%s" % (p[0], p[1], p[3])
