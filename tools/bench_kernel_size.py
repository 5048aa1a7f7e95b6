"""WaveNet cost per dilated-convolution kernel_size on one GPU: the Cfg-2 training step (bench.py's wavenet_ce workload: 24 layers /
4 stacks, R256 / G512 / S256, mu-law CE, 2 x 7680 samples, CUDA graph, fwd + bwd + clip + Adam + EMA) and the AR time per sample step
(tools/bench_ar.py's shapes: paper widths, mu-law, one utterance of 22000 samples, cluster size 16), at kernel_size 2, 3 and 4.

The kernel sizes alternate within each round (the order rotates from round to round) and every round times all of them, so a drift of
the shared machine shows as spread between rounds rather than as a difference between sizes. Prints the card's name, power limit and
maximum SM clock, one JSON line per measurement, then the median and spread per kernel size.

  python tools/bench_kernel_size.py [--rounds 3] [--steps 50] [--warmup 5] [--ar-samples 22000]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bench import synth_batch, workload_hparams, WN_SHAPES  # noqa: E402
from hparams import hparams  # noqa: E402
from t2_import import t2  # noqa: E402

KERNEL_SIZES = (2, 3, 4)


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in r.stdout.strip().split(",")] if r.returncode == 0 else (torch.cuda.get_device_name(), "?", "?")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock, "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def gate_gflop(hp, B, T):
    """2 B T G (k R + C): one layer's forward gate GEMM"""
    return 2.0 * B * T * hp.gate_channels * (hp.kernel_size * hp.residual_channels + hp.cin_channels) / 1e9


class Train(object):
    def __init__(self, k):
        self.hp = workload_hparams("wavenet_ce")
        self.hp.set_hparam("kernel_size", k)
        self.B, self.T = WN_SHAPES["wavenet_ce"]
        self.model = t2.wavenet.WaveNet(self.hp, self.B, self.T)
        self.model.init_variables(seed=5339)
        q = lambda w: t2.audio.mulaw_quantize(torch.from_numpy(w).cuda()).cpu().numpy()
        x, c, lengths = synth_batch(self.hp, self.B, self.T, 2, q)
        self.model.capture(*[torch.from_numpy(a).cuda() for a in (x, c, x, lengths)])

    def time_ms(self, steps, warmup):
        for _ in range(warmup):
            self.model.train_step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            self.model.train_step()
        e1.record()
        torch.cuda.synchronize()
        loss = self.model.loss_value()
        assert loss == loss, "NaN loss"
        return e0.elapsed_time(e1) / steps


class Synth(object):
    def __init__(self, k, T):
        hp = hparams.copy()
        hp.parse("layers=24,stacks=4,residual_channels=256,gate_channels=512,skip_out_channels=256,upsample_scales=[11,25],"
                 "input_type=mulaw-quantize,quantize_channels=256,out_channels=256")
        hp.set_hparam("kernel_size", k)
        self.T = T // 275 * 275
        self.syn = t2.wavenet.WaveNetSynthesizer(hp, 1, self.T, cluster_size=16)
        self.syn.init_variables(seed=5)
        self.c = torch.rand(1, 80, self.T // 275, device="cuda")
        self.init = torch.full((1,), 127, dtype=torch.int32, device="cuda")
        self.syn.generate(self.c, self.init, seed=1)      # warm-up: module load, kernel attributes

    def time_us_per_step(self):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        self.syn.generate(self.c, self.init, seed=2)
        e1.record()
        torch.cuda.synchronize()
        return 1e3 * e0.elapsed_time(e1) / self.T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ar-samples", type=int, default=22000)
    args = ap.parse_args()
    info = card()
    print(json.dumps(dict(info, kind="card")), flush=True)
    train = {k: Train(k) for k in KERNEL_SIZES}
    synth = {k: Synth(k, args.ar_samples) for k in KERNEL_SIZES}
    res = {k: {"train_ms": [], "ar_us": []} for k in KERNEL_SIZES}
    for r in range(args.rounds):
        order = KERNEL_SIZES[r % len(KERNEL_SIZES):] + KERNEL_SIZES[:r % len(KERNEL_SIZES)]
        for k in order:
            ms = train[k].time_ms(args.steps, args.warmup)
            us = synth[k].time_us_per_step()
            res[k]["train_ms"].append(ms)
            res[k]["ar_us"].append(us)
            print(json.dumps({"kind": "round", "round": r, "kernel_size": k, "train_ms_per_step": ms, "ar_us_per_sample_step": us}),
                  flush=True)
    hp = workload_hparams("wavenet_ce")
    B, T = WN_SHAPES["wavenet_ce"]
    print("\n%s, power limit %s, max SM clock %s" % (info["gpu"], info["power_limit"], info["max_sm_clock"]))
    print("| kernel_size | gate GEMM per layer (GFLOP) | train step ms (median, min-max) | AR us / sample step (median, min-max) |")
    print("|---|---|---|---|")
    for k in KERNEL_SIZES:
        hp.set_hparam("kernel_size", k)
        t, a = res[k]["train_ms"], res[k]["ar_us"]
        print("| %d | %.2f | %.3f (%.3f-%.3f) | %.2f (%.2f-%.2f) |" % (k, gate_gflop(hp, B, T), statistics.median(t), min(t), max(t),
                                                                   statistics.median(a), min(a), max(a)))
        print(json.dumps({"kind": "summary", "kernel_size": k, "train_ms_median": statistics.median(t), "train_ms": t,
                          "ar_us_median": statistics.median(a), "ar_us": a}), flush=True)


if __name__ == "__main__":
    main()
