"""CBHG post-processing net + linear head: forward time and linear error of the bf16 and fp32-class (split_bf16) modes.

Runs t2_cbhg_forward at stock widths (num_freq 1025) on one random mel batch in both modes, alternating the two modes over --reps
rounds of --iters forwards each (CUDA events around the whole round, after --warmup forwards per mode), and compares each mode's linear
outputs with the fp32 oracle (oracle.tacotron.linear_head) on the same input. Prints one JSON line with the per-forward medians, the
linear mean / max |error| of both modes and the card name and power limit read in the same run.

    python tools/bench_cbhg_fp32_class.py --B 32 --T 800 [--training 1]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hparams import hparams  # noqa: E402
from oracle import tacotron as ot  # noqa: E402
from t2_import import t2  # noqa: E402

L = t2.lib


def card():
    """name and power limit of the current device (the limit is part of every time measured on it)"""
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


class Engine:
    def __init__(self, hp, params, B, T, precision):
        lib = L.load()
        self.lib = lib
        self.cfg = t2.tacotron.make_cbhg_config(hp, B, T, 0.0, precision)
        pb, wb, n = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong()
        L.check(lib.t2_cbhg_sizes(ctypes.byref(self.cfg), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), None))
        self.packed = torch.empty(pb.value, dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(wb.value, dtype=torch.uint8, device="cuda")
        self.prm = torch.zeros(n.value, dtype=torch.float32, device="cuda")
        for i in range(self._count(lib)):
            name = ctypes.create_string_buffer(256)
            off, nd, sh, tr = ctypes.c_longlong(), ctypes.c_int(), (ctypes.c_int * 4)(), ctypes.c_int()
            L.check(lib.t2_cbhg_param_info(ctypes.byref(self.cfg), i, name, 256, ctypes.byref(off), ctypes.byref(nd), sh, ctypes.byref(tr)))
            v = params[name.value.decode()].reshape(-1)
            self.prm[off.value:off.value + v.numel()] = v.cuda()
        L.check(lib.t2_cbhg_init(ctypes.byref(self.cfg), L.ptr(self.packed), L.ptr(self.ws), L.stream_ptr()))
        L.check(lib.t2_cbhg_pack_weights(ctypes.byref(self.cfg), L.ptr(self.prm), L.ptr(self.packed), L.ptr(self.ws), L.stream_ptr()))

    def _count(self, lib):
        nt = ctypes.c_int()
        L.check(lib.t2_cbhg_sizes(ctypes.byref(self.cfg), None, None, None, ctypes.byref(nt)))
        return nt.value

    def forward(self, mel, lin_t, training):
        L.check(self.lib.t2_cbhg_forward(ctypes.byref(self.cfg), L.ptr(self.prm), L.ptr(self.packed), L.ptr(self.ws), L.ptr(mel), L.ptr(lin_t),
                                         L.ptr(None), int(training), L.stream_ptr()))

    def linear(self, B, T, NF):
        p, cnt = ctypes.c_void_p(), ctypes.c_longlong()
        L.check(self.lib.t2_cbhg_workspace_tensor(ctypes.byref(self.cfg), L.ptr(self.ws), b"linear_outputs", ctypes.byref(p), ctypes.byref(cnt)))
        off = p.value - self.ws.data_ptr()
        nfp = (NF + 7) // 8 * 8
        return self.ws[off:off + cnt.value * 4].view(torch.float32).reshape(B, T, nfp)[:, :, :NF].clone()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--T", type=int, default=800)
    ap.add_argument("--training", type=int, default=0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle", type=int, default=1, help="compare both modes with the fp32 oracle (CPU, slow at T = 800)")
    a = ap.parse_args()
    hp = hparams.copy()
    hp.parse("predict_linear=True")
    params = ot.init_params(hp, seed=7, random_bias=True)
    g = torch.Generator().manual_seed(7)
    mel = (torch.randn(a.B, a.T, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    lin_t = (torch.randn(a.B, a.T, hp.num_freq, generator=g) * 1.5 - 1).clamp(-4, 4)
    mel_d, lin_d = mel.cuda(), lin_t.cuda()
    eng = {p: Engine(hp, params, a.B, a.T, p) for p in ("bf16", "fp32-class")}
    # moving statistics change in training mode: the error comparison runs once per mode, from the initial parameters, before the timing
    res = {"B": a.B, "T": a.T, "training": a.training, "card": card()}
    if a.oracle:
        with torch.no_grad():
            ref = ot.linear_head(mel, {k: v.clone() for k, v in params.items()}, hp, bool(a.training))
        for p, e in eng.items():
            e.forward(mel_d, lin_d, a.training)
            torch.cuda.synchronize()
            err = (e.linear(a.B, a.T, hp.num_freq).cpu() - ref).abs()
            res["lin_l1_" + p], res["lin_max_" + p] = err.mean().item(), err.max().item()
    for e in eng.values():
        for _ in range(a.warmup):
            e.forward(mel_d, lin_d, a.training)
    torch.cuda.synchronize()
    times = {p: [] for p in eng}
    for _ in range(a.reps):
        for p, e in eng.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.iters):
                e.forward(mel_d, lin_d, a.training)
            t1.record()
            t1.synchronize()
            times[p].append(t0.elapsed_time(t1) / a.iters)
    for p in eng:
        res["ms_" + p] = statistics.median(times[p])
        res["ms_all_" + p] = times[p]
    res["ratio"] = res["ms_fp32-class"] / res["ms_bf16"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
