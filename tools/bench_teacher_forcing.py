"""Cost of a teacher-forcing ratio below 1 on the Tacotron training step at Cfg-3 (default widths, B = 32, T_in = 160, T_out = 800,
dropout 0.5, zoneout 0.1, predict_linear off): the captured step (pack + forward + backward) plus Adam at ratio 1.0 (batched prenet
and projections), 0.5 and 0.0 (per-step prenet, projections and their backward), alternated in one process so all see the same card
state. Prints one JSON line per run and a summary with the card name and power limit.

  python tools/bench_teacher_forcing.py [--steps 20] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from hparams import hparams
from t2_import import t2

B, T_IN, T_OUT = 32, 160, 800


def make(ratio):
    hp = hparams.copy()
    hp.parse("predict_linear=False")
    m = t2.tacotron.Tacotron(hp, B, T_IN, T_OUT, teacher_forcing_ratio=ratio)
    m.init_variables(seed=3)
    g = torch.Generator().manual_seed(1)
    inputs = torch.randint(2, 66, (B, T_IN), generator=g).int().cuda()
    lens = torch.full((B,), T_IN, dtype=torch.int32).cuda()
    mel = (torch.randn(B, T_OUT, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4).cuda()
    stop = torch.zeros(B, T_OUT)
    stop[:, -3:] = 1
    m.capture(inputs, lens, mel, stop.cuda())
    return m


def time_steps(m, steps):
    for _ in range(3):
        m.train_step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m.train_step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    models = {"ratio_1.0": make(1.0), "ratio_0.5": make(0.5), "ratio_0.0": make(0.0)}
    res = {k: [] for k in models}
    for r in range(args.rounds):
        for k, m in models.items():
            ms = time_steps(m, args.steps)
            res[k].append(ms)
            print(json.dumps({"round": r, "config": k, "ms_per_step": round(ms, 3), "loss": m.losses()["total"],
                              "launches_per_step": m.launches_per_step}), flush=True)
    print(json.dumps({"card": card, "B": B, "T_in": T_IN, "T_out": T_OUT, "steps": args.steps,
                      "ms_per_step": {k: [round(v, 3) for v in vs] for k, vs in res.items()}}), flush=True)


if __name__ == "__main__":
    main()
