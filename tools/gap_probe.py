"""Debug tool (GPU box): where does the time of the WaveNet residual-stack GEMM chain go in the captured Cfg-2 step?

Every act_gemm CTA stamps %globaltimer at entry / after griddepcontrol.wait / at exit, and every ticket of a persistent layer chain
stamps its start / dependencies met / end and SM (t2_dbg_set_timing_buffer); each launch of the captured graph has its own slice.
  --per-layer   run the gate / out and dz / dx GEMMs as per-layer launches: per launch, the exit spread (slowest minus fastest CTA)
                and the gap from the previous launch's last exit to this launch's first CTA past its wait; sums per chain
  (default)     the layer chains as the step runs them: span, busy and dependency-wait totals, per-SM timeline, per-layer spans
  --json PATH   also write the rows
"""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from t2_import import t2
from bench import workload_hparams, synth_batch, B_PER_GPU, T_STEP

SLOTS = 16
ap = argparse.ArgumentParser()
ap.add_argument("--per-layer", action="store_true")
ap.add_argument("--json", default=None)
args = ap.parse_args()

L = t2.lib
lib = L.load()
hp = workload_hparams()
m = t2.wavenet.WaveNet(hp, B_PER_GPU, T_STEP)
m.init_variables(seed=1)
idx, c, lengths = synth_batch(hp, B_PER_GPU, T_STEP, 2, lambda w: t2.audio.mulaw_quantize(torch.from_numpy(w).cuda()).cpu().numpy())
x = torch.from_numpy(idx).cuda(); cc = torch.from_numpy(c).cuda(); ln = torch.from_numpy(lengths).cuda()
lib.t2_dbg_wn_per_layer(1 if args.per_layer else 0)
for _ in range(2):
    m.forward(x, cc, x, ln); m.backward()
torch.cuda.synchronize()

NL, MT = hp.layers, B_PER_GPU * -(-T_STEP // 128)
ng, nz = hp.gate_channels // 256, (hp.gate_channels // 2) // (256 if hp.gate_channels >= 512 else 128)
n_tix = [lib.t2_dbg_wn_chain(ctypes.byref(m.cfg), d, None, 0) for d in (0, 1)]
# the slices of one step's launches in enqueue order: (name, slots), where a slot is one CTA (act_gemm) or one ticket (chain)
launches = []
if args.per_layer:
    for l in range(NL):
        launches.append(("gate%02d" % l, MT * ng))
        if l + 1 < NL:
            launches.append(("out%02d" % l, MT))
else:
    launches.append(("chain_fwd", n_tix[0]))
launches += [("skip", MT), ("final1", MT), ("ce_head", MT), ("dh2", MT), ("dskip", MT)]
if args.per_layer:
    for l in range(NL - 1, -1, -1):
        launches += [("dz%02d" % l, MT * nz), ("dx%02d" % l, MT)]
else:
    launches.append(("chain_bwd", n_tix[1]))
launches.append(("dcond", MT))
step_slots = sum(n for _, n in launches)
buf = torch.zeros(3 * step_slots * SLOTS, dtype=torch.int64, device="cuda")
lib.t2_dbg_set_timing_buffer(L.ptr(buf))
m.capture(x, cc, x, ln)            # warm-up pass = slices [0, step), captured pass = slices [step, 2 step)
lib.t2_dbg_set_timing_buffer(None)
for _ in range(3):
    m._graph.replay()
torch.cuda.synchronize()
lib.t2_dbg_wn_per_layer(0)
t = buf.view(-1, SLOTS)[step_slots:2 * step_slots].cpu().double()
card = torch.cuda.get_device_name()
out = {"card": card, "mode": "per-layer" if args.per_layer else "chains", "launches": []}
o = 0
sl = {}
for name, n in launches:
    sl[name] = t[o:o + n]
    o += n
t0 = min(float(v[:, 8].min()) for k, v in sl.items() if not k.startswith("chain")) if args.per_layer else float(sl["chain_fwd"][:, 0].min())
print("%s, %s; times in us from the first stamp" % (card, out["mode"]))
if args.per_layer:
    print("%-8s %6s %9s %9s %9s %9s %8s %8s" % ("launch", "ctas", "entry_min", "wait_min", "exit_min", "exit_max", "spread", "gap"))
    prev_exit = None
    sums = {"fwd": [0.0, 0.0], "bwd": [0.0, 0.0]}
    for name, n in launches:
        v = sl[name]
        e, w, xx = (v[:, 8] - t0) / 1e3, (v[:, 9] - t0) / 1e3, (v[:, 10] - t0) / 1e3
        spread = float(xx.max() - xx.min())
        gap = None if prev_exit is None else float(w.min()) - prev_exit
        prev_exit = float(xx.max())
        part = "fwd" if name.startswith(("gate", "out")) else "bwd" if name.startswith(("dz", "dx")) else None
        if part:
            sums[part][0] += spread
            sums[part][1] += gap or 0.0
        out["launches"].append({"launch": name, "ctas": n, "entry_min_us": float(e.min()), "wait_min_us": float(w.min()),
                                "exit_min_us": float(xx.min()), "exit_max_us": float(xx.max()), "exit_spread_us": spread, "gap_us": gap})
        print("%-8s %6d %9.2f %9.2f %9.2f %9.2f %8.2f %8s" % (name, n, e.min(), w.min(), xx.min(), xx.max(), spread,
                                                           "-" if gap is None else "%.2f" % gap))
    for part in ("fwd", "bwd"):
        print("%s chain: exit spreads %.1f us + launch gaps %.1f us = %.1f us per step" % (part, sums[part][0], sums[part][1],
                                                                                         sum(sums[part])))
    out["sums_us"] = sums
else:
    for name in ("chain_fwd", "chain_bwd"):
        v = sl[name]
        s, d, e, sm = (v[:, 0] - t0) / 1e3, (v[:, 1] - t0) / 1e3, (v[:, 2] - t0) / 1e3, v[:, 3].long()
        span = float(e.max() - s.min())
        wait = float((d - s).sum())
        busy = float((e - d).sum())
        nsm = int(sm.unique().numel())
        per_sm = [(int(q), float((e - d)[sm == q].sum()), float((d - s)[sm == q].sum())) for q in sm.unique()]
        idle = nsm * span - busy - wait
        print("%s: %d tickets on %d SMs, span %.1f us | busy %.1f SM-us, dependency wait %.1f SM-us (%.1f us per SM), "
              "between tickets / tail %.1f SM-us" % (name, len(v), nsm, span, busy, wait, wait / max(nsm, 1), idle))
        rows = []
        kinds = ("gate", "out") if name == "chain_fwd" else ("dz", "dx")
        tk = (ctypes.c_int * (8 * len(v)))()
        lib.t2_dbg_wn_chain(ctypes.byref(m.cfg), 0 if name == "chain_fwd" else 1, tk, len(v))
        tk = torch.tensor(list(tk)).view(-1, 8)
        for l in range(NL):
            for kd in (0, 1):
                sel = (tk[:, 0] == kd) & (tk[:, 1] == l)
                if sel.any():
                    rows.append({"gemm": "%s%02d" % (kinds[kd], l), "first_start_us": float(s[sel].min()), "last_end_us": float(e[sel].max()),
                                 "wait_us": float((d - s)[sel].sum())})
        print("  per GEMM (first start .. last end, summed wait): " + "  ".join(
            "%s %.0f..%.0f w%.0f" % (r["gemm"], r["first_start_us"], r["last_end_us"], r["wait_us"]) for r in rows[:6]) + " ...")
        print("  SM timeline (busy / wait us per SM, first 8): " + "  ".join("sm%d %.0f/%.0f" % p for p in per_sm[:8]))
        out[name] = {"tickets": len(v), "sms": nsm, "span_us": span, "busy_sm_us": busy, "wait_sm_us": wait, "idle_sm_us": idle,
                     "per_gemm": rows, "per_sm": per_sm}
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump(out, open(args.json, "w"), indent=1)
