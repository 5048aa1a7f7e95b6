"""Config 1 (BASELINE.json): fused STFT + 80-band mel on 1 s clips of 22.05 kHz audio, batch of 4096 clips on one H100.
Reports clip-seconds/s, achieved algorithmic HBM GB/s (114 120 B per clip-second, SURVEY.md §8d) against
MEASURED_PEAKS.json, and the numpy oracle on the host cores (bounded sample)."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from hparams import hparams
from oracle import audio as oa
from t2_import import t2

def main():
    B, n = 4096, 22050
    g = torch.Generator(device="cuda").manual_seed(1)
    wav = (torch.rand(B, n, device="cuda", generator=g) * 2 - 1) * 0.5
    fe = t2.audio.MelFrontEnd(hparams)
    out = fe(wav)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 5
    e0.record()
    for _ in range(reps):
        fe(wav, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    algo_bytes = B * 4 * (n + 81 * 80)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", 6650.0))
    res = {"metric": "stft_mel_clip_seconds_per_sec", "value": B / (ms * 1e-3), "unit": "clip-s/s", "ms_per_batch": ms, "batch": B,
           "roofline": {"bound": "hbm", "achieved": algo_bytes / (ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                        "frac": algo_bytes / (ms * 1e-3) / 1e9 / peak, "note": "fp64 FFT in shared memory: the kernel is FP64/smem-latency bound, not HBM bound"}}
    w = wav[:32].cpu().numpy()
    t0 = time.perf_counter()
    for i in range(32):
        oa.melspectrogram(w[i], hparams)
    dt = time.perf_counter() - t0
    res["cpu_baseline"] = {"value": 32 / dt, "unit": "clip-s/s", "cores": 1, "kind": "port", "sample": "32 clips, numpy oracle, single thread"}
    print(json.dumps(res))

if __name__ == "__main__":
    main()
