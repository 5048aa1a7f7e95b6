"""Config 5 (BASELINE.json): Fast-WaveNet autoregressive synthesis real-time factor on one H100.
RTF = wall time / audio duration (T / 22050 s); < 1 is faster than real time. Paper widths, 1 s of audio."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hparams import hparams
from t2_import import t2

def run(input_type, B, cs, T=22000, precision="bf16"):
    hp = hparams.copy()
    hp.parse("layers=24,stacks=4,residual_channels=256,gate_channels=512,skip_out_channels=256,upsample_scales=[11,25]")
    if input_type == "mulaw-quantize":
        hp.parse("input_type=mulaw-quantize,quantize_channels=256,out_channels=256")
    else:
        hp.parse("input_type=raw,quantize_channels=65536,out_channels=30")
    syn = t2.wavenet.WaveNetSynthesizer(hp, B, T, cluster_size=cs, precision=precision)
    syn.init_variables(seed=5)
    c = torch.rand(B, 80, T // 275, device="cuda")
    init = (torch.full((B,), 127, dtype=torch.int32) if input_type == "mulaw-quantize" else torch.zeros(B)).cuda()
    syn.generate(c, init, seed=1)  # warm-up (module load, attribute set)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = syn.generate(c, init, seed=2)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    return {"input_type": input_type, "batch": B, "cluster_size": cs, "samples": T, "ms": ms, "us_per_step": 1e3 * ms / T,
            "rtf_per_utterance": ms / 1e3 / (T / 22050.0), "aggregate_x_realtime": B * (T / 22050.0) / (ms / 1e3)}

if __name__ == "__main__":
    res = []
    if len(sys.argv) > 1:          # profiling: one short run (python tools/bench_ar.py <T>)
        print(json.dumps(run("mulaw-quantize", 1, 16, T=int(sys.argv[1]) // 275 * 275 or 275)), flush=True)
        sys.exit(0)
    for it in ("mulaw-quantize", "raw"):
        for B, cs in ((1, 8), (1, 16), (20, 8), (20, 16)):
            r = run(it, B, cs)
            res.append(r)
            print(json.dumps(r), flush=True)
