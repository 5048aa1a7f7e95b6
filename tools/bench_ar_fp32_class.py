"""Fast-WaveNet AR synthesis: time per sample step of the bf16 and fp32-class (fp32 synthesis weights and conditioning) modes.

Workloads: the default widths (20 layers, R 128 / G 256 / S 128) and the paper widths (24 layers, R 256 / G 512 / S 256), each with
the mu-law (256-way softmax) and the MoL (30 outputs) heads, at B 1 and 20 and cluster sizes 8 and 16. Free-running generation of
--T samples from random conditioning. One synthesizer per (workload, mode) is built and warmed up first; then --rounds rounds run every
workload once in each mode, the two modes back to back, with CUDA events around each generate call. Prints one JSON line per workload
(median and min-max microseconds per sample step over the rounds, the fp32-class / bf16 ratio of the medians, and whether the host
prefetches each CTA's weight slices into shared memory), then a markdown table and the card's name, power limit and max SM clock read
in the same run.

    python tools/bench_ar_fp32_class.py [--T 5500] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hparams import hparams  # noqa: E402
from t2_import import t2  # noqa: E402

WIDTHS = {"default": "layers=20,stacks=2,residual_channels=128,gate_channels=256,skip_out_channels=128",
          "paper": "layers=24,stacks=4,residual_channels=256,gate_channels=512,skip_out_channels=256"}
HEADS = {"mulaw": "input_type=mulaw-quantize,quantize_channels=256,out_channels=256",
         "mol": "input_type=raw,quantize_channels=65536,out_channels=30"}
MODES = ("bf16", "fp32-class")
SMEM_LIMIT = 232448 - 1024          # shared memory per CTA t2_wn_ar_generate lets the kernel use


def card():
    """name, power limit and max SM clock of the current device (part of every time measured on it)"""
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def prefetch(hp, B, cs, esize, sms):
    """t2_wn_ar_generate's choice: both per-layer weight slots (esize bytes per weight) fit next to the activations"""
    R, G, S, C, L, k = hp.residual_channels, hp.gate_channels, hp.skip_out_channels, hp.cin_channels, hp.layers, hp.kernel_size
    Gh = G // 2
    n = max(1, min(sms // cs, B))
    ipc = -(-B // n)
    while ipc > 4:
        n += 1
        ipc = -(-B // n)
    ni = 1 if ipc <= 1 else (2 if ipc <= 2 else 4)
    ZC, RC, SC, OC, K1 = Gh // cs, R // cs, S // cs, -(-hp.out_channels // cs), k * R + C
    per_rank_layer = 2 * ZC * K1 + (RC + SC) * Gh
    smem = 4 * (ni * (((K1 + 3) & ~3) + Gh + R + ZC + RC + max(2 * ZC, RC + SC) + SC + S + cs * OC + ((C + 3) & ~3) + 1)
                + L * (2 * ZC + RC) + ((2 * L + 1 + 3) & ~3)) + 64
    return (per_rank_layer * esize) % 16 == 0 and smem + 2 * per_rank_layer * esize + 64 <= SMEM_LIMIT


def workload(widths, head, B, cs, T, precision):
    hp = hparams.copy()
    hp.parse(WIDTHS[widths] + "," + HEADS[head] + ",upsample_scales=[11,25]")
    syn = t2.wavenet.WaveNetSynthesizer(hp, B, T, cluster_size=cs, precision=precision)
    syn.init_variables(seed=5)
    c = torch.rand(B, hp.cin_channels, T // 275, device="cuda", generator=torch.Generator("cuda").manual_seed(7))
    init = (torch.full((B,), 127, dtype=torch.int32) if head == "mulaw" else torch.zeros(B)).cuda()
    syn.generate(c, init, seed=1)         # warm-up: module load, kernel attributes
    return hp, syn, c, init


def time_us_per_step(syn, c, init, T):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    syn.generate(c, init, seed=2)
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=5500, help="samples per utterance (a multiple of the hop size 275)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    assert args.T % 275 == 0 and args.rounds >= 3
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    keys = [(w, h, B, cs) for w in WIDTHS for h in HEADS for B in (1, 20) for cs in (8, 16)]
    runs = {(k, m): workload(*k, args.T, m) for k in keys for m in MODES}
    torch.cuda.synchronize()
    times = {(k, m): [] for k in keys for m in MODES}
    for _ in range(args.rounds):
        for k in keys:
            for m in MODES:
                _, syn, c, init = runs[(k, m)]
                times[(k, m)].append(time_us_per_step(syn, c, init, args.T))
    gpu = card()
    rows = []
    for k in keys:
        hp = runs[(k, MODES[0])][0]
        r = {"widths": k[0], "head": k[1], "B": k[2], "cluster_size": k[3], "T": args.T, "rounds": args.rounds}
        for m, esize in zip(MODES, (2, 4)):
            t = times[(k, m)]
            r[m] = {"us_per_step_median": statistics.median(t), "min": min(t), "max": max(t),
                    "prefetch": bool(prefetch(hp, k[2], k[3], esize, sms))}
        r["fp32_class_over_bf16"] = r["fp32-class"]["us_per_step_median"] / r["bf16"]["us_per_step_median"]
        r["card"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    print("\n| widths | head | B | CS | bf16 us/step (min-max) | prefetch | fp32-class us/step (min-max) | prefetch | ratio |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        a, b = r["bf16"], r["fp32-class"]
        print("| %s | %s | %d | %d | %.1f (%.1f-%.1f) | %s | %.1f (%.1f-%.1f) | %s | %.2f |" % (
            r["widths"], r["head"], r["B"], r["cluster_size"], a["us_per_step_median"], a["min"], a["max"],
            "on" if a["prefetch"] else "off", b["us_per_step_median"], b["min"], b["max"], "on" if b["prefetch"] else "off",
            r["fp32_class_over_bf16"]))
    print("\ncard (name, power limit, max SM clock): %s; T = %d, %d rounds" % (gpu, args.T, args.rounds))


if __name__ == "__main__":
    main()
