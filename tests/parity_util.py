"""Shared helpers of the GPU parity tests: every measured error is printed as a `MEASURED {json}` line and, when T2_PARITY_LOG
names a file, appended to it, so that the tolerances in the tests (<= 2x the measured value) can be audited against a run."""
import json
import os

_OUT = os.environ.get("T2_PARITY_LOG")


def record(test, **values):
    vals = {k: (float(v) if hasattr(v, "__float__") else v) for k, v in values.items()}
    line = {"test": test}
    line.update(vals)
    print("MEASURED " + json.dumps(line))
    if _OUT:
        with open(_OUT, "a") as f:
            f.write(json.dumps(line) + "\n")
    return vals


def grad_report(grads, grads_ref, min_norm=1e-7):
    """per-tensor (relative L2 error, cosine) of two {name: tensor} dicts -> (rows, worst_rel, worst_cos)"""
    rows, worst_rel, worst_cos = [], 0.0, 1.0
    for name, g_ref in grads_ref.items():
        g = grads[name]
        den = g_ref.norm().item()
        rel = (g - g_ref).norm().item() / max(den, 1e-30)
        cos = (g * g_ref).sum().item() / max(den * g.norm().item(), 1e-30)
        rows.append((name, rel, cos, den))
        if den >= min_norm:
            worst_rel, worst_cos = max(worst_rel, rel), min(worst_cos, cos)
    return rows, worst_rel, worst_cos
