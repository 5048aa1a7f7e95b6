"""Config 1 (BASELINE.json): fused STFT + 80-band mel on 1 s clips of 22.05 kHz audio, batch of 4096 clips on one H100.
Reports clip-seconds/s, achieved algorithmic HBM GB/s (114 120 B per clip-second at the defaults, SURVEY.md §8d) against
MEASURED_PEAKS.json, the numpy oracle on the host cores (bounded sample), the time of one Griffin-Lim round, and the card's name
and power limit read in the same run.

--sample_rate / --n_fft time another corpus: the window and hop default to the reference's advice (hparams.py:43-54), 50 ms and
12.5 ms, and to the stock hparams at 22.05 kHz."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from hparams import hparams
from oracle import audio as oa
from t2_import import t2


def card():
    """name and power limit of the current device (nvidia-smi query; the limit is part of every time measured on it)"""
    dev = torch.cuda.current_device()
    info = {"name": torch.cuda.get_device_name(dev)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in r.stdout.strip().split(",")]
    except Exception as e:      # the measurement stands without it; say so instead of guessing
        info["power_limit"] = "unknown (%s)" % type(e).__name__
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sample_rate", type=int, default=hparams.sample_rate)
    ap.add_argument("--n_fft", type=int, default=hparams.n_fft)
    ap.add_argument("--batch", type=int, default=4096, help="1 s clips per fused STFT / mel call")
    ap.add_argument("--gl_batch", type=int, default=16, help="5 s clips per Griffin-Lim call")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    hp = hparams.copy()
    sr = args.sample_rate
    stock = sr == hparams.sample_rate
    hp.set_hparam("sample_rate", sr)
    hp.set_hparam("n_fft", args.n_fft)
    hp.set_hparam("win_size", hparams.win_size if stock else int(0.05 * sr))
    hp.set_hparam("hop_size", hparams.hop_size if stock else int(0.0125 * sr))
    hp.set_hparam("fmax", min(hparams.fmax, sr // 2))
    hop = hp.hop_size

    B, n = args.batch, sr
    g = torch.Generator(device="cuda").manual_seed(1)
    wav = (torch.rand(B, n, device="cuda", generator=g) * 2 - 1) * 0.5
    fe = t2.audio.MelFrontEnd(hp)
    out = fe(wav)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = args.reps
    e0.record()
    for _ in range(reps):
        fe(wav, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    algo_bytes = B * 4 * (n + (n // hop + 1) * hp.num_mels)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", 6650.0))
    res = {"metric": "stft_mel_clip_seconds_per_sec", "value": B / (ms * 1e-3), "unit": "clip-s/s", "ms_per_batch": ms, "batch": B,
           "sample_rate": sr, "n_fft": hp.n_fft, "hop": hop, "win": hp.win_size,
           "roofline": {"bound": "hbm", "achieved": algo_bytes / (ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                        "frac": algo_bytes / (ms * 1e-3) / 1e9 / peak, "note": "fp64 FFT in shared memory: the kernel is FP64/smem-latency bound, not HBM bound"}}

    # one Griffin-Lim round (inverse STFT + overlap-add + STFT): the difference of `iters` and 0 rounds over `iters`
    frames = 1 + 5 * sr // hop
    mag = torch.rand(args.gl_batch, frames, hp.n_fft // 2 + 1, device="cuda", generator=g)
    iters = 20
    fe.griffin_lim(mag, iters)
    fe.griffin_lim(mag, 0)
    torch.cuda.synchronize()
    t = {}
    for it in (0, iters):
        e0.record()
        for _ in range(reps):
            fe.griffin_lim(mag, it)
        e1.record()
        torch.cuda.synchronize()
        t[it] = e0.elapsed_time(e1) / reps
    res["griffin_lim"] = {"ms_per_round": (t[iters] - t[0]) / iters, "batch": args.gl_batch, "clip_seconds": 5, "frames": frames,
                          "ms_0_rounds": t[0]}

    w = wav[:32].cpu().numpy()
    t0 = time.perf_counter()
    for i in range(32):
        oa.melspectrogram(w[i], hp)
    dt = time.perf_counter() - t0
    res["cpu_baseline"] = {"value": 32 / dt, "unit": "clip-s/s", "cores": 1, "kind": "port", "sample": "32 clips, numpy oracle, single thread"}
    res["card"] = card()
    print(json.dumps(res))

if __name__ == "__main__":
    main()
