"""Cost of the ConvTranspose1D conditioning upsampler with LeakyReLU against the SubPixel / ReLU default, on the two WaveNet training
workloads of bench.py: wavenet_ce (Cfg-2: 24 layers / 4 stacks, R256/G512/S256, mu-law-256, B = 2 x T = 7680) and wavenet_mol (same
stack, raw input + MoL-10, B = 8 x T = 16128), both with upsample_scales [16, 16]. Prints:
  - the captured training step (pack + forward + backward) plus Adam, both upsamplers alternated in one process, `--rounds` times;
  - each upsampler launch on its own at the step's shapes (forward, weight gradient, input gradient per layer), through
    t2_dbg_wn_kernel captured `--reps` times into one CUDA graph and timed with CUDA events, and the same at the reference's
    stock scales [11, 25] (hop 275);
  - the FLOP each ConvTranspose1D launch needs (counted from shapes: 2 B W s C^2 per layer and pass) and its rate;
  - the card name and power limit.
The backward upsampler launches run on the library's side stream, under the residual stack's weight-gradient GEMM, so their share of
the step is an upper bound on what they add to it.

  python tools/bench_upsample.py [--steps 50] [--rounds 3] [--reps 50] [--workloads wavenet_ce,wavenet_mol] [--out FILE]"""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bench import WN_SHAPES, workload_hparams
from t2_import import t2

L = t2.lib
CONFIGS = {"subpixel_relu": ("SubPixel", "Relu"), "1d_leaky": ("1D", "LeakyRelu")}
TYPES, ACTS = {"SubPixel": 0, "2D": 1, "1D": 2}, {"Relu": 0, "LeakyRelu": 1, None: 2}


def make(workload, utype, act):
    hp = workload_hparams(workload)
    hp.set_hparam("upsample_type", utype)
    hp.set_hparam("upsample_activation", act)
    B, T = WN_SHAPES[workload]
    m = t2.wavenet.WaveNet(hp, B, T)
    m.init_variables(seed=3)
    g = torch.Generator().manual_seed(1)
    if hp.input_type == "mulaw-quantize":
        x = torch.randint(0, 256, (B, T), generator=g).int().cuda()
    else:
        x = ((torch.rand(B, T, generator=g) * 2 - 1) * 0.5).cuda()
    c = (torch.rand(B, 80, T // 256, generator=g) * 8 - 4).cuda()          # symmetric mels in [-4, 4]
    lengths = torch.full((B,), T, dtype=torch.int32).cuda()
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


def _call(kernel, p, B, C, W, s, utype, act, alpha):
    c = L.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate((B, C, W, s, TYPES[utype], ACTS[act], 0)):
        c.i[k] = int(v)
    c.f[0] = alpha
    L.check(L.load().t2_dbg_wn_kernel(ctypes.byref(c), L.stream_ptr()))


def time_launch(fn, reps):
    """device time per call: `reps` calls captured into one CUDA graph, replayed once warm and then timed"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_times(B, T, scales, utype, act, reps):
    """per layer: forward, weight gradient (+ its fixed-point finalisation), input gradient (layers > 0) in ms, with the FLOP of 1D"""
    C, alpha = 80, 0.4 if act == "LeakyRelu" else 0.0
    g = torch.Generator().manual_seed(0)
    W = T // math.prod(scales)
    x = (torch.rand(B, C, W, generator=g) * 8 - 4).cuda()
    out = []
    for i, s in enumerate(scales):
        ks = {"SubPixel": (3, 3, 1, s), "2D": (3, s, 1, 1), "1D": (1, s, C, C)}[utype]
        nb = {"SubPixel": s, "2D": 1, "1D": C}[utype]
        K = (torch.randn(ks, generator=g) * 0.1).cuda()
        b = (torch.randn(nb, generator=g) * 0.1).cuda()
        y = torch.empty(B, C, W * s, device="cuda")
        dy = torch.randn(B, C, W * s, generator=g).cuda()
        dK, db = torch.empty_like(K), torch.empty_like(b)
        acc = torch.empty(K.numel() + b.numel(), dtype=torch.int64, device="cuda")
        dx = torch.empty(B, C, W, device="cuda")
        args = (B, C, W, s, utype, act, alpha)
        row = {"layer": i, "W": W, "s": s,
               "fwd_ms": time_launch(lambda: _call(1, [x, K, b, y, None], *args), reps),
               "wgrad_ms": time_launch(lambda: _call(2, [x, y, dy, dK, db, acc], *args), reps)}
        if i > 0:
            row["dgrad_ms"] = time_launch(lambda: _call(3, [y, dy, K, dx], *args), reps)
        if utype == "1D":
            row["gflop_per_pass"] = 2.0 * B * W * s * C * C / 1e9
            row["fwd_tflops"] = row["gflop_per_pass"] / row["fwd_ms"]          # GFLOP per ms = TFLOP/s
        out.append(row)
        x, W = y, W * s
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--workloads", default="wavenet_ce,wavenet_mol")
    ap.add_argument("--out", default=None, help="also write the summary as JSON to this file")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    summary = {"card": card}
    for wl in args.workloads.split(","):
        B, T = WN_SHAPES[wl]
        models = {k: make(wl, *v) for k, v in CONFIGS.items()}
        res = {k: [] for k in models}
        for r in range(args.rounds):
            for k, m in models.items():
                ms = time_steps(m, args.steps)
                res[k].append(ms)
                print(json.dumps({"workload": wl, "round": r, "config": k, "ms_per_step": round(ms, 4), "loss": m.loss_value()}), flush=True)
        del models
        torch.cuda.empty_cache()
        kt = {k: kernel_times(B, T, [16, 16], *v, args.reps) for k, v in CONFIGS.items()}
        step = {k: min(v) for k, v in res.items()}
        share = {k: sum(r["fwd_ms"] + r["wgrad_ms"] + r.get("dgrad_ms", 0.0) for r in kt[k]) / step[k] for k in kt}
        summary[wl] = {"B": B, "T": T, "ms_per_step": {k: [round(v, 4) for v in vs] for k, vs in res.items()},
                       "upsampler_kernels": kt, "upsampler_share_of_step": share}
        print(json.dumps({wl: summary[wl]}), flush=True)
    # the reference's stock scales (hop 275) at the wavenet_ce batch
    summary["stock_scales_B2xT7700"] = {k: kernel_times(2, 7700, [11, 25], *v, args.reps) for k, v in CONFIGS.items()}
    print(json.dumps({"card": card, "stock_scales_B2xT7700": summary["stock_scales_B2xT7700"]}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
