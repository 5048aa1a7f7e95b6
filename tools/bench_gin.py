"""Cost of global (speaker) conditioning on the WaveNet training step at Cfg-2 (24 layers / 4 stacks, R256/G512/S256, mu-law-256,
B = 2 x T = 7680, dropout 0.05): the captured step (pack + forward + backward) plus Adam, with gin_channels = 16 / n_speakers = 8
and with global conditioning off, alternated in one process so both see the same card state. Prints one JSON line per run and a
summary with the card name and power limit.

  python tools/bench_gin.py [--steps 100] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from hparams import hparams
from t2_import import t2

B, T = 2, 7680


def make(gin):
    hp = hparams.copy()
    hp.parse("layers=24,stacks=4,residual_channels=256,gate_channels=512,skip_out_channels=256,upsample_scales=[16,16],hop_size=256,"
             "input_type=mulaw-quantize,quantize_channels=256,out_channels=256,wavenet_dropout=0.05")
    if gin:
        hp.parse("gin_channels=16,n_speakers=8,use_speaker_embedding=True")
    m = t2.wavenet.WaveNet(hp, B, T)
    m.init_variables(seed=3)
    g = torch.Generator().manual_seed(1)
    x = torch.randint(0, 256, (B, T), generator=g).int().cuda()
    c = torch.rand(B, 80, T // 256, generator=g).cuda()
    lengths = torch.full((B,), T, dtype=torch.int32).cuda()
    if gin:
        m.set_speakers([3, 6])
    m.capture(x, c, x, lengths)
    return m


def time_steps(m, steps):
    for _ in range(5):
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
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    models = {"gin_off": make(False), "gin_16x8": make(True)}
    res = {k: [] for k in models}
    for r in range(args.rounds):
        for k, m in models.items():
            ms = time_steps(m, args.steps)
            res[k].append(ms)
            print(json.dumps({"round": r, "config": k, "ms_per_step": round(ms, 4), "loss": m.loss_value()}), flush=True)
    print(json.dumps({"card": card, "B": B, "T": T, "steps": args.steps,
                      "ms_per_step": {k: [round(v, 4) for v in vs] for k, vs in res.items()}}), flush=True)


if __name__ == "__main__":
    main()
