"""The ticket / dependency tables of the persistent WaveNet layer chains (t2_dbg_wn_chain), checked without a GPU: every ticket
waits only for earlier tickets of its batch item, and the tiles it waits for cover exactly the rows its GEMM reads."""
import ctypes

import numpy as np
import pytest

from bench import workload_hparams, WN_SHAPES
from t2_import import t2

SHAPES = [(name,) + WN_SHAPES[name] for name in ("wavenet_ce", "wavenet_mol", "wavenet_default")] + [
    ("wavenet_ce", 4, 8192), ("wavenet_ce", 3, 5120), ("wavenet_ce", 2, 5136), ("wavenet_default", 2, 8192)]


def _cfg(name, B, T):
    hp = workload_hparams(name)
    if T % 256:
        hp.set_hparam("upsample_scales", [4, 4])
        hp.set_hparam("hop_size", 16)
    return t2.wavenet.make_config(hp, B, T), hp


def _tickets(cfg, d):
    lib = t2.lib.load()
    n = lib.t2_dbg_wn_chain(ctypes.byref(cfg), d, None, 0)
    assert n > 0, lib.t2_last_error()
    buf = (ctypes.c_int * (8 * n))()
    assert lib.t2_dbg_wn_chain(ctypes.byref(cfg), d, buf, n) == n
    return np.frombuffer(buf, dtype=np.int32).reshape(n, 8)


@pytest.mark.parametrize("name,B,T", SHAPES)
def test_chain_tickets_wait_for_exactly_the_rows_they_read(name, B, T):
    cfg, hp = _cfg(name, B, T)
    L, G, R = hp.layers, hp.gate_channels, hp.residual_channels
    Gh = G // 2
    tpb = -(-T // 128)
    MT = B * tpb
    dil = lambda l: 1 << (l % (L // hp.stacks))
    idx = lambda kind, l, m: (kind * L + l) * MT + m
    for d in (0, 1):
        tk = _tickets(cfg, d)
        n0 = G // 256 if d == 0 else Gh // (256 if Gh >= 256 else 128)
        # launch order of the per-layer loop: forward gate (m fastest, then n), out; backward from the top layer: dz, dx
        order = []
        for l in (range(L) if d == 0 else range(L - 1, -1, -1)):
            order += [(0, l, m, n) for n in range(n0) for m in range(MT)]
            if d == 1 or l + 1 < L:
                order += [(1, l, m, 0) for m in range(MT)]
        assert [tuple(r[:4]) for r in tk] == order
        finished_before = {}
        for i, (kind, l, m, n, lo, hi, target, done) in enumerate(tk):
            assert done == idx(kind, l, m)
            finished_before.setdefault(done, []).append(i)
            b, t0 = m // tpb, (m % tpb) * 128
            if d == 0 and kind == 0:         # gate: xd_l rows [t0 - 2d, t0 + 128), written by out(l-1)
                rows, dep_kind, dep_l, need = (max(0, t0 - 2 * dil(l)), min(T, t0 + 128)), 1, l - 1, 1
            elif d == 0:                     # out: z_l rows of its own tile, written by every N tile of gate(l)
                rows, dep_kind, dep_l, need = (t0, min(T, t0 + 128)), 0, l, n0
            elif kind == 0:                  # dz: dxin_{l+1} rows of its own tile, written by dx(l+1)
                rows, dep_kind, dep_l, need = (t0, min(T, t0 + 128)), 1, l + 1, 1
            else:                            # dx: dg_l rows [t0, t0 + 128 + 2d), written by dz(l)
                rows, dep_kind, dep_l, need = (t0, min(T, t0 + 128 + 2 * dil(l))), 0, l, n0
            if (d == 0 and kind == 0 and l == 0) or (d == 1 and kind == 0 and l == L - 1):
                assert hi < lo, "a chain's first GEMM reads only what was written before the launch"
                continue
            want = (idx(dep_kind, dep_l, b * tpb + rows[0] // 128), idx(dep_kind, dep_l, b * tpb + (rows[1] - 1) // 128))
            assert (lo, hi) == want and target == need
            for c in range(lo, hi + 1):      # every awaited counter is completed by `need` EARLIER tickets
                assert len([j for j in finished_before.get(c, []) if j < i]) == need
