"""Cost of the attention-state flags (mask_encoder=False: energies and softmax over all T_in positions; cumulative_weights=False) on
the Tacotron path at Cfg-3 (default widths, B = 32, T_in = 160, dropout 0.5, zoneout 0.1, predict_linear off). Input lengths fall
linearly from T_in to T_in / 4, so the un-masked attention does real extra work on the short rows. For each of the four flag
combinations, alternated in rounds in one process so all see the same card state:
  * the captured training step (pack + forward + backward) plus Adam at T_out = 800;
  * free-running synthesis: the decoder steps of t2_taco_infer_steps (prenet, LSTMs, attention, projections), per step.
Prints one JSON line per run and a summary with the card name and power limit.

  python tools/bench_attention_state.py [--steps 10] [--rounds 3] [--synth-steps 400]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from hparams import hparams
from t2_import import t2

B, T_IN, T_OUT = 32, 160, 800
COMBOS = {"masked_cumulative": {}, "unmasked": dict(mask_encoder=False), "noncumulative": dict(cumulative_weights=False),
          "unmasked_noncumulative": dict(mask_encoder=False, cumulative_weights=False)}


def _hp(flags):
    hp = hparams.copy()
    hp.parse("predict_linear=False")
    for k, v in flags.items():
        hp.set_hparam(k, v)
    return hp


def _batch(hp, T_out):
    g = torch.Generator().manual_seed(1)
    inputs = torch.randint(2, 66, (B, T_IN), generator=g).int()
    lens = torch.linspace(T_IN, T_IN // 4, B).round().int()
    for b in range(B):
        inputs[b, lens[b]:] = 0
    mel = (torch.randn(B, T_out, hp.num_mels, generator=g) * 1.5 - 1).clamp(-4, 4)
    stop = torch.zeros(B, T_out)
    stop[:, -3:] = 1
    return inputs.cuda(), lens.cuda(), mel.cuda(), stop.cuda()


def make_train(flags):
    hp = _hp(flags)
    m = t2.tacotron.Tacotron(hp, B, T_IN, T_OUT)
    m.init_variables(seed=3)
    m.capture(*_batch(hp, T_OUT))
    return m


def time_train(m, steps):
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


def make_synth(flags, n):
    hp = _hp(flags)
    m = t2.tacotron.Tacotron(hp, B, T_IN, n)
    m.init_variables(seed=3)
    m.pack()
    inputs, lens, _, _ = _batch(hp, n)
    return m, inputs, lens


def time_synth(m, inputs, lens, n):
    """begin (encoder, decoder reset) once, then all n decoder steps in one t2_taco_infer_steps call; the stop rule is not consulted"""
    cfg = ctypes.byref(m.cfg)
    L = t2.lib
    args = (L.ptr(m.params), L.ptr(m.packed), L.ptr(m.workspace))
    ms = []
    for _ in range(2):
        L.check(m.lib.t2_taco_infer_begin(cfg, *args, L.ptr(inputs), L.ptr(lens), L.stream_ptr()))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        L.check(m.lib.t2_taco_infer_steps(cfg, *args, L.ptr(lens), 0, n, ctypes.c_ulonglong(0), L.stream_ptr()))
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / n)
    return ms[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--synth-steps", type=int, default=400)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    train = {k: make_train(f) for k, f in COMBOS.items()}
    synth = {k: make_synth(f, args.synth_steps) for k, f in COMBOS.items()}
    res = {k: {"train_ms_per_step": [], "synth_ms_per_decoder_step": []} for k in COMBOS}
    for r in range(args.rounds):
        for k in COMBOS:
            ms = time_train(train[k], args.steps)
            res[k]["train_ms_per_step"].append(round(ms, 3))
            print(json.dumps({"round": r, "config": k, "train_ms_per_step": round(ms, 3), "loss": train[k].losses()["total"],
                              "launches_per_step": train[k].launches_per_step}), flush=True)
        for k in COMBOS:
            ms = time_synth(*synth[k], args.synth_steps)
            res[k]["synth_ms_per_decoder_step"].append(round(ms, 4))
            print(json.dumps({"round": r, "config": k, "synth_ms_per_decoder_step": round(ms, 4)}), flush=True)
    print(json.dumps({"card": card, "B": B, "T_in": T_IN, "T_out": T_OUT, "synth_steps": args.synth_steps,
                      "input_lengths": [T_IN, T_IN // 4], "results": res}), flush=True)


if __name__ == "__main__":
    main()
