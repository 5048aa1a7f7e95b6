"""Every fused epilogue of the wgmma GEMM engine (tacotron-2_b200/csrc/t2_gemm.cuh), its split-K, cluster-multicast and segment
mechanics, the weight-gradient tile table and the fixed-point column sums, each against a float64 reference computed from the exact
bf16 inputs (and, for the masks, from the host copy of the counter hash in mask_hash.py).

Tolerances are per element against the float64 reference:
  fp32 accumulator outputs    |err| <= 2^-20 (|A|.|W|)[elem] + 2^-23 |ref| + 1e-7   (fp32 accumulation, then one fp32 rounding
                              for the bias add)
  bf16 outputs                the same + 2^-8 |ref|
  tanh.approx / sigmoid       + 1e-3 absolute (bf16 gate outputs)
  fast-intrinsic scalar math  loss / count sums within 1e-5 relative; gradients and states within 1e-4 max|ref| (+ bf16 rounding)
Every check prints the worst err / bound ratio through parity_util.record. Output buffers are pre-filled with NaN: padding columns and
rows past the end must still be NaN afterwards, and NaN in the unaddressed channels of every input proves they are not read."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import mask_hash as mh
from parity_util import record
from t2_import import t2

pytestmark = pytest.mark.gpu
L = t2.lib
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
F64 = torch.float64
NAN = float("nan")
EPI = dict(GATE=0, RES=1, BIAS_ACT=2, CE=3, MOL=4, SCALE_RELUMASK=5, GATE_BWD=6, DX=7, LSTM=8, TOUT=9)
E20, E23 = 2.0 ** -20, 2.0 ** -23


# ------------------------------------------------------------------------------------------------------------------------------
# plumbing
# ------------------------------------------------------------------------------------------------------------------------------
def _lib():
    lib = L.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    return lib


def act_map(Lyr, B, T, C, ld=None, scale=0.5, gen=None):
    """bf16 activation [L, B, T, ld]; channels >= C are NaN (the engine must never read them)"""
    ld = ld or (C + 7) // 8 * 8
    a = (torch.randn(Lyr, B, T, ld, generator=gen) * scale).bfloat16()
    a[..., C:] = NAN
    return {"t": a.to(DEV), "C": C, "ld": ld, "L": Lyr}


def weight(wL, N, K, gen=None):
    return (torch.randn(wL, N, K, generator=gen) / math.sqrt(K)).bfloat16().to(DEV)


def nan_buf(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


def call(epi, BN, maps, segs, W, T, B, n_tiles, ptr=None, f=None, i=None, seed=0, w_layer=0, w_k0=0, ksplit=0, cluster=0, sync=True):
    """one t2_dbg_act_gemm launch; returns the cluster size that was launched"""
    lib = _lib()
    c = L.DbgGemm()
    for j, m in enumerate(maps):
        c.a[j] = L.DbgAct(m["t"].data_ptr(), m["C"], T, B, m["L"], m["ld"])
    c.na = len(maps)
    for j, s in enumerate(segs):
        c.seg[j] = L.DbgSeg(*s)
    c.nseg = len(segs)
    c.w = W.data_ptr()
    c.wL, c.wN, c.wK = W.shape
    c.w_layer, c.w_k0 = w_layer, w_k0
    c.T, c.B, c.n_tiles, c.ksplit, c.epi, c.BN, c.cluster = T, B, n_tiles, ksplit, EPI[epi], BN, cluster
    for k, v in (ptr or {}).items():
        c.ptr[k] = None if v is None else v.data_ptr()
    for k, v in (f or {}).items():
        c.f[k] = v
    for k, v in (i or {}).items():
        c.i[k] = v
    c.seed = seed
    L.check(lib.t2_dbg_act_gemm(ctypes.byref(c), L.stream_ptr()))
    if sync:
        torch.cuda.synchronize()
    return c.cluster_used


def gemm_ref(maps, segs, W, T, B, w_layer=0, w_k0=0):
    """float64 D[B, T, wN] = sum_seg sum_layer sum_k A[l, b, t + shift, k0 + k] W[w_layer, n, w_k0 + kofs + k] and |A|.|W| of the same
    contraction; rows outside [0, T) of the same item, channels >= C and weight columns >= wK are zero (TMA out-of-bounds fill)"""
    Wd = W[w_layer].to(F64)
    N, wK = Wd.shape
    D = torch.zeros(B, T, N, dtype=F64, device=DEV)
    Da = torch.zeros_like(D)
    kofs = w_k0
    for (m, sh, k0, nkb, l0, nl) in segs:
        A, C = maps[m]["t"], maps[m]["C"]
        width = nkb * 64
        for lyr in range(l0, l0 + nl):
            a = torch.zeros(B, T, width, dtype=F64, device=DEV)
            nch = max(0, min(width, C - k0))
            lo, hi = max(0, -sh), min(T, T - sh)
            if nch > 0 and hi > lo:
                a[:, lo:hi, :nch] = A[lyr, :, lo + sh:hi + sh, k0:k0 + nch].to(F64)
            w = torch.zeros(N, width, dtype=F64, device=DEV)
            ncol = max(0, min(width, wK - kofs))
            if ncol > 0:
                w[:, :ncol] = Wd[:, kofs:kofs + ncol]
            D += a @ w.t()
            Da += a.abs() @ w.abs().t()
            kofs += width
    return D, Da


def check(name, got, ref, bound, **info):
    err = (got.to(F64) - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=float("inf")).max().item() if err.numel() else 0.0
    record(name, worst_err_over_bound=ratio, **info)
    assert ratio <= 1.0, "%s: worst err / bound %.3g" % (name, ratio)


def all_nan(name, t):
    assert t.numel() == 0 or torch.isnan(t.float()).all().item(), "%s: written outside its bounds" % name


def fx_total(acc):
    """host copy of fx_value: int64 fixed point (2^-40) -> float64, NaN for a poisoned / out-of-range total"""
    a = acc.to(torch.int64)
    v = a.to(F64) * 2.0 ** -40
    return torch.where(a.abs() < 2 ** 62, v, torch.full_like(v, NAN))


def seed_offset(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# the mask hash
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,stream,i0", [(0, 0, 0), (12345, 7, 2 ** 32 - 5000), (2 ** 63 + 99, 2 ** 31 + 3, 3 * 2 ** 32 + 11)])
def test_host_hash_matches_device(seed, stream, i0):
    """the host copy reproduces t2_rng_uniform_f32 bit for bit, over indices that cross 2^32"""
    lib = _lib()
    n = 10000
    out = torch.empty(n, dtype=torch.float32, device=DEV)
    L.check(lib.t2_rng_uniform_f32(ctypes.c_ulonglong(seed), ctypes.c_uint(stream), ctypes.c_longlong(i0), ctypes.c_longlong(n),
                                   L.ptr(out), L.stream_ptr()))
    torch.cuda.synchronize()
    idx = np.arange(i0, i0 + n, dtype=np.uint64)
    host = mh.hash_uniform32(mh.hash_seed(seed, stream), idx)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), host.view(np.uint32))
    # pair form: both halves of one 32-bit hash, thresholds from the float rate
    hs = mh.hash_seed(seed, stream)
    bits = mh.hash_bits32(hs, idx >> np.uint64(1))
    thr = mh.keep_threshold16(0.25)
    keep = mh.hash_keep16(hs, idx, thr)
    expect = np.where(idx % 2 == 1, bits >> 16, bits & 0xFFFF) >= thr
    assert np.array_equal(keep, expect) and 0.2 < 1 - keep.mean() < 0.3


# ------------------------------------------------------------------------------------------------------------------------------
# EPI_BIAS_ACT
# ------------------------------------------------------------------------------------------------------------------------------
BIAS_ACT_CASES = [
    # BN, T, act, nvalid, bias, outs ("b", "f", "bf"), pdrop, seed_off, split
    (128, 1, 1, 81, True, "bf", 0.0, False, False),
    (128, 31, 0, 200, True, "bf", 0.0, False, False),
    (128, 200, 2, 200, False, "b", 0.0, False, False),
    (128, 385, 1, 81, True, "f", 0.25, True, False),
    (256, 33, 2, 200, True, "bf", 0.0, False, False),
    (256, 128, 1, 81, True, "bf", 0.25, False, False),
    (256, 385, 0, 512, True, "bf", 0.1, True, False),
    (128, 200, 1, 81, True, "bf", 0.0, False, True),
    (256, 33, 2, 200, True, "bf", 0.0, False, True),
    (128, 31, 0, 84, False, "bf", 0.0, False, True),     # ldo = 88: the last 32-column group crosses ldo (element path)
]


@pytest.mark.parametrize("BN,T,act,nvalid,has_bias,outs,pdrop,use_off,split", BIAS_ACT_CASES)
def test_bias_act(BN, T, act, nvalid, has_bias, outs, pdrop, use_off, split):
    g = torch.Generator().manual_seed(T * 7 + nvalid)
    B, C = 2, 200
    maps = [act_map(1, B, T, C, gen=g)]
    segs = [(0, -3, 0, 4, 0, 1), (0, 0, 0, 4, 0, 1), (0, 5, 0, 4, 0, 1)]
    W = weight(1, nvalid, 3 * 256, g)
    bias = torch.randn(nvalid, generator=g).to(DEV) if has_bias else None
    ldo = (nvalid + 7) // 8 * 8 + (0 if split else 8)
    rows, slack = B * T, 3
    ob = nan_buf((rows + slack, (2 if split else 1) * ldo), torch.bfloat16) if "b" in outs else None
    of = nan_buf((rows + slack, ldo), torch.float32) if "f" in outs else None
    seed, off = 777, 1234
    so = seed_offset(off) if use_off else None
    call("BIAS_ACT", BN, maps, segs, W, T, B, (nvalid + BN - 1) // BN,
         ptr={0: ob, 1: bias, 2: of, 7: so}, f={1: pdrop}, i={0: ldo, 1: act, 2: nvalid, 3: 5, 11: int(split)}, seed=seed)
    D, Da = gemm_ref(maps, segs, W, T, B)
    v = D + (bias.to(F64) if has_bias else 0)
    v = v.relu() if act == 1 else torch.tanh(v) if act == 2 else v
    bound = E20 * Da + E23 * v.abs() + 1e-7 + (2e-7 if act == 2 else 0)    # tanhf_: ex2.approx + rcp.approx
    if pdrop > 0:
        hs = mh.hash_seed(seed + (off if use_off else 0), 5)
        idx = (np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(ldo) + np.arange(nvalid, dtype=np.uint64)[None, :])
        keep = torch.from_numpy(mh.hash_uniform32(hs, idx) >= np.float32(pdrop)).to(DEV).view(B, T, nvalid)
        kinv = float(np.float32(1) / (np.float32(1) - np.float32(pdrop)))
        v = torch.where(keep, v * kinv, torch.zeros_like(v))
        bound = bound * kinv
    v, bound = v.reshape(rows, nvalid), bound.reshape(rows, nvalid)
    name = "bias_act_BN%d_T%d_act%d_n%d_%s_p%g_split%d" % (BN, T, act, nvalid, outs, pdrop, split)
    if of is not None:
        check(name + "_f32", of[:rows, :nvalid], v, bound)
        all_nan(name + " f32 padding", of[:rows, nvalid:])
        all_nan(name + " f32 tail", of[rows:])
    if ob is not None:
        if split:
            got = ob[:rows, :nvalid].to(F64) + ob[:rows, ldo:ldo + nvalid].to(F64)
            check(name + "_split", got, v, bound + 2.0 ** -16 * v.abs())
            check(name + "_split_hi", ob[:rows, :nvalid], v, bound + 2.0 ** -8 * v.abs())
            # columns of the last 32-column group past nvalid (up to ldo) hold zeros, the rest stays untouched
            zc = min(ldo, (nvalid + 31) // 32 * 32)
            assert (ob[:rows, nvalid:zc] == 0).all() and (ob[:rows, ldo + nvalid:ldo + zc] == 0).all()
            all_nan(name + " split padding", ob[:rows, zc:ldo])
        else:
            check(name + "_bf16", ob[:rows, :nvalid], v, bound + 2.0 ** -8 * v.abs())
            all_nan(name + " bf16 padding", ob[:rows, nvalid:])
        all_nan(name + " bf16 tail", ob[rows:])


# ------------------------------------------------------------------------------------------------------------------------------
# EPI_RES
# ------------------------------------------------------------------------------------------------------------------------------
RES_CASES = [(128, 1, 0.0, False, False), (128, 33, 0.25, True, False), (128, 385, 0.25, False, False), (256, 31, 0.25, False, False),
             (256, 200, 0.25, True, False), (256, 128, 0.0, False, False), (128, 200, 0.0, False, True), (256, 33, 0.0, False, True)]


def res_ref(maps, segs, W, x, bias, rs, p, T, B, R, seed, layer):
    D, Da = gemm_ref(maps, segs, W, T, B)
    xo = (D + bias.to(F64) + x) * rs
    bound = (E20 * Da + E23 * xo.abs() + 1e-7) * abs(rs)
    keep = None
    if p > 0:
        hs = mh.hash_seed(seed, layer)
        idx = np.arange(B * T, dtype=np.uint64)[:, None] * np.uint64(R) + np.arange(R, dtype=np.uint64)[None, :]
        keep = torch.from_numpy(mh.hash_keep16(hs, idx, mh.keep_threshold16(p))).to(DEV).view(B, T, R)
    return xo, bound, keep


@pytest.mark.parametrize("R,T,p,use_off,split", RES_CASES)
def test_res(R, T, p, use_off, split):
    g = torch.Generator().manual_seed(R + T)
    B, Gh = 2, 200
    maps = [act_map(1, B, T, Gh, gen=g)]
    segs = [(0, 0, 0, 4, 0, 1)]
    W = weight(1, R, 256, g)
    bias = torch.randn(R, generator=g).to(DEV)
    rows, slack = B * T, 5
    rs, seed, off, layer = 0.7071, 99, 31337, 3
    xv = (torch.randn(rows, R, generator=g) * 0.5).to(DEV)
    if split:
        hi = xv.bfloat16()
        x_in = torch.cat([hi, (xv - hi.float()).bfloat16()], 1)
        x = (x_in[:, :R].to(F64) + x_in[:, R:].to(F64)).view(B, T, R)
    else:
        x_in = xv.bfloat16()
        x = x_in.to(F64).view(B, T, R)
    x_out = nan_buf((rows + slack, (2 if split else 1) * R), torch.bfloat16)
    xd = None if split else nan_buf((rows + slack, R), torch.bfloat16)
    call("RES", R, maps, segs, W, T, B, 1, ptr={0: x_in, 1: x_out, 2: xd, 3: bias, 7: seed_offset(off) if use_off else None},
         f={0: rs, 1: p}, i={1: layer, 11: int(split)}, seed=seed)
    xo, bound, keep = res_ref(maps, segs, W, x, bias, rs, p, T, B, R, seed + (off if use_off else 0), layer)
    name = "res_R%d_T%d_p%g_off%d_split%d" % (R, T, p, use_off, split)
    xo, bound = xo.view(rows, R), bound.view(rows, R)
    if split:
        check(name + "_split", x_out[:rows, :R].to(F64) + x_out[:rows, R:].to(F64), xo, bound + 2.0 ** -16 * xo.abs())
    else:
        check(name + "_xout", x_out[:rows], xo, bound + 2.0 ** -8 * xo.abs())
        kinv = float(np.float32(1) / (np.float32(1) - np.float32(p)))
        xdr = xo * kinv if keep is None else torch.where(keep.view(rows, R), xo * kinv, torch.zeros_like(xo))
        check(name + "_xd", xd[:rows], xdr, bound * kinv + 2.0 ** -8 * xdr.abs())
        all_nan(name + " xd tail", xd[rows:])
    all_nan(name + " tail", x_out[rows:])


# ------------------------------------------------------------------------------------------------------------------------------
# EPI_GATE (BN 256): 3 dilated taps of x + the conditioning, as the real gate GEMM
# ------------------------------------------------------------------------------------------------------------------------------
GATE_BN = 256
GATE_CASES = [(128, 33, True, False), (256, 200, True, False), (512, 128, False, False), (256, 385, True, False),
              (128, 1, True, False), (256, 31, False, True)]


@pytest.mark.parametrize("Gh,T,stash,split", GATE_CASES)
def test_gate(Gh, T, stash, split):
    g = torch.Generator().manual_seed(Gh + T)
    B, R, Cc, d = 2, 128, 80, 4
    maps = [act_map(2, B, T, R, gen=g), act_map(1, B, T, R, gen=g), act_map(1, B, T, R, gen=g), act_map(1, B, T, Cc, gen=g)]
    segs = [(0, -2 * d, 0, 2, 1, 1), (1, -d, 0, 2, 0, 1), (2, 0, 0, 2, 0, 1), (3, 0, 0, 2, 0, 1)]
    K = 3 * 128 + 128
    W = weight(2, 2 * Gh, K, g)                   # rows interleaved per 128-channel tile: [a(128) | b(128)] per n_tile
    bias = torch.randn(2 * Gh, generator=g).to(DEV)
    rows, slack = B * T, 3
    z = nan_buf((rows + slack, (2 if split else 1) * Gh), torch.bfloat16)
    ta = nan_buf((rows + slack, Gh), torch.bfloat16) if stash else None
    sb = nan_buf((rows + slack, Gh), torch.bfloat16) if stash else None
    call("GATE", GATE_BN, maps, segs, W, T, B, Gh // 128, ptr={0: ta, 1: sb, 2: z, 3: bias}, i={0: Gh, 11: int(split)}, w_layer=1)
    D, Da = gemm_ref(maps, segs, W, T, B, w_layer=1)
    D, Da = D.view(rows, Gh // 128, 2, 128), Da.view(rows, Gh // 128, 2, 128)
    a = D[:, :, 0].reshape(rows, Gh) + bias[:Gh].to(F64)
    s = D[:, :, 1].reshape(rows, Gh) + bias[Gh:].to(F64)
    ba, bs = E20 * Da[:, :, 0].reshape(rows, Gh) + E23 * a.abs() + 1e-7, E20 * Da[:, :, 1].reshape(rows, Gh) + E23 * s.abs() + 1e-7
    tr, sr = torch.tanh(a), torch.sigmoid(s)
    zr = tr * sr
    name = "gate_Gh%d_T%d_stash%d_split%d" % (Gh, T, stash, split)
    if split:
        check(name + "_z_split", z[:rows, :Gh].to(F64) + z[:rows, Gh:].to(F64), zr, ba + bs + 2.0 ** -16 * zr.abs() + 1e-6)
    else:
        check(name + "_z", z[:rows], zr, ba + bs + 2.0 ** -8 * zr.abs() + 1e-3)
    all_nan(name + " z tail", z[rows:])
    if stash:
        check(name + "_tanh", ta[:rows], tr, ba + 2.0 ** -8 * tr.abs() + 1e-3)
        check(name + "_sigmoid", sb[:rows], sr, bs + 2.0 ** -8 * sr.abs() + 1e-3)
        all_nan(name + " stash tails", torch.cat([ta[rows:], sb[rows:]]))


# ------------------------------------------------------------------------------------------------------------------------------
# EPI_SCALE_RELUMASK / EPI_GATE_BWD / EPI_DX: the backward epilogues with fixed-point column sums
# ------------------------------------------------------------------------------------------------------------------------------
def colsum_bound(elem_bound, ref_vals):
    """fx column sums: the elements' own bounds, the 5-level float tree of warp_colsum32 and the 2^-41 rounding of each addend"""
    n_add = ref_vals.shape[0] // 32 + 1
    return elem_bound.sum(0) + 2.0 ** -21 * ref_vals.abs().sum(0) + n_add * 4 * 2.0 ** -41 + 1e-9


def twice(launch):
    """run an fx-producing launch twice on fresh accumulators: the int64 totals must be bitwise equal"""
    first = launch()
    second = launch()
    for a, b in zip(first, second):
        if a.dtype == torch.int64:
            assert torch.equal(a, b), "fixed-point column sums differ between two identical runs"
        else:
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "outputs differ between two identical runs"
    return first


SCALE_RELUMASK_CASES = [(128, 33, 2, True), (256, 200, 1, True), (128, 385, 1, False), (256, 1, 2, True)]


@pytest.mark.parametrize("BN,T,ntile,use_div", SCALE_RELUMASK_CASES)
def test_scale_relumask(BN, T, ntile, use_div):
    g = torch.Generator().manual_seed(BN + T)
    B, C = 2, 136
    ldo = ntile * BN
    maps = [act_map(1, B, T, C, gen=g)]
    segs = [(0, 0, 0, 3, 0, 1), (0, 1, 0, 3, 0, 1)]
    W = weight(1, ldo, 384, g)
    rows, slack = B * T, 2
    h = (torch.randn(rows + slack, ldo, generator=g)).relu().bfloat16().to(DEV)     # half of h is exactly zero
    h[rows:] = NAN
    div = torch.tensor([3.5], device=DEV)
    scale = 0.75

    def launch():
        out = nan_buf((rows + slack, ldo), torch.bfloat16)
        fx = torch.zeros(ldo, dtype=torch.int64, device=DEV)
        call("SCALE_RELUMASK", BN, maps, segs, W, T, B, ntile, ptr={0: out, 1: h, 2: div if use_div else None, 3: fx},
             f={0: scale}, i={0: ldo})
        return out, fx
    out, fx = twice(launch)
    D, Da = gemm_ref(maps, segs, W, T, B)
    s = float(np.float32(scale) / np.float32(3.5)) if use_div else scale
    m = (h[:rows].to(F64) > 0)
    v = torch.where(m, D.view(rows, ldo) * s, torch.zeros(rows, ldo, dtype=F64, device=DEV))
    bound = torch.where(m, (E20 * Da.view(rows, ldo) + 1e-7) * s + E23 * v.abs(), torch.zeros_like(v))
    name = "scale_relumask_BN%d_T%d_nt%d_div%d" % (BN, T, ntile, use_div)
    check(name + "_out", out[:rows], v, bound + 2.0 ** -8 * v.abs() + 1e-30)
    all_nan(name + " tail", out[rows:])
    check(name + "_colsum", fx_total(fx), v.sum(0), colsum_bound(bound, v))


GATE_BWD_CASES = [(128, 384, 33), (256, 256, 200), (256, 512, 1), (128, 128, 385)]


@pytest.mark.parametrize("BN,Gh,T", GATE_BWD_CASES)
def test_gate_bwd(BN, Gh, T):
    g = torch.Generator().manual_seed(BN + Gh + T)
    B, S = 2, 136
    maps = [act_map(1, B, T, S, gen=g)]
    segs = [(0, 0, 0, 3, 0, 1)]
    W = weight(1, Gh, 192, g)
    rows, slack = B * T, 2
    ta = torch.tanh(torch.randn(rows + slack, Gh, generator=g)).bfloat16().to(DEV)
    sb = torch.sigmoid(torch.randn(rows + slack, Gh, generator=g)).bfloat16().to(DEV)
    ta[rows:] = NAN
    sb[rows:] = NAN

    def launch():
        dg = nan_buf((rows + slack, 2 * Gh), torch.bfloat16)
        f3 = torch.zeros(2 * Gh, dtype=torch.int64, device=DEV)
        f4 = torch.zeros(2 * Gh, dtype=torch.int64, device=DEV)
        call("GATE_BWD", BN, maps, segs, W, T, B, Gh // BN, ptr={0: ta, 1: sb, 2: dg, 3: f3, 4: f4}, i={0: Gh})
        return dg, f3, f4
    dg, f3, f4 = twice(launch)
    assert torch.equal(f3, f4)
    D, Da = gemm_ref(maps, segs, W, T, B)
    dz, bz = D.view(rows, Gh), E20 * Da.view(rows, Gh) + 1e-7
    a, s = ta[:rows].to(F64), sb[:rows].to(F64)
    da, db = dz * (1 - a * a) * s, dz * a * s * (1 - s)
    ba = bz * ((1 - a * a) * s).abs() + 4 * 2.0 ** -24 * da.abs()
    bb = bz * (a * s * (1 - s)).abs() + 5 * 2.0 ** -24 * db.abs()
    ref, bound = torch.cat([da, db], 1), torch.cat([ba, bb], 1)
    name = "gate_bwd_BN%d_Gh%d_T%d" % (BN, Gh, T)
    check(name + "_dg", dg[:rows], ref, bound + 2.0 ** -8 * ref.abs() + 1e-30)
    all_nan(name + " tail", dg[rows:])
    check(name + "_colsum", fx_total(f3), ref.sum(0), colsum_bound(bound, ref))


DX_CASES = [(128, 33, True, 0.25, True), (256, 200, False, 0.25, False), (128, 1, True, 0.0, False),
            (256, 385, True, 0.1, False), (128, 128, False, 0.0, False)]


@pytest.mark.parametrize("R,T,with_dxo,p,use_off", DX_CASES)
def test_dx(R, T, with_dxo, p, use_off):
    g = torch.Generator().manual_seed(R + T + 1)
    B, Gh = 2, 200
    maps = [act_map(1, B, T, Gh, gen=g)]
    segs = [(0, 0, 0, 4, 0, 1)]
    W = weight(1, R, 256, g)
    rows, slack = B * T, 2
    dxo = (torch.randn(rows + slack, R, generator=g) * 0.5).bfloat16().to(DEV) if with_dxo else None
    if with_dxo:
        dxo[rows:] = NAN
    rs, fscale, seed, off, layer = 0.7071, 0.5, 4242, 77, 6

    def launch():
        dx = nan_buf((rows + slack, R), torch.bfloat16)
        fx = torch.zeros(R, dtype=torch.int64, device=DEV)
        call("DX", R, maps, segs, W, T, B, 1, ptr={0: dxo, 1: dx, 2: fx, 7: seed_offset(off) if use_off else None},
             f={0: rs, 1: p, 2: fscale}, i={1: layer}, seed=seed)
        return dx, fx
    dx, fx = twice(launch)
    D, Da = gemm_ref(maps, segs, W, T, B)
    acc, bacc = D.view(rows, R), E20 * Da.view(rows, R) + 1e-7
    kinv = float(np.float32(1) / (np.float32(1) - np.float32(p)))
    if p > 0:
        hs = mh.hash_seed(seed + (off if use_off else 0), layer)
        idx = np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(R) + np.arange(R, dtype=np.uint64)[None, :]
        keep = torch.from_numpy(mh.hash_keep16(hs, idx, mh.keep_threshold16(p))).to(DEV)
        acc, bacc = torch.where(keep, acc * kinv, torch.zeros_like(acc)), torch.where(keep, bacc * kinv, torch.zeros_like(bacc))
    ref = acc + (rs * dxo[:rows].to(F64) if with_dxo else 0)
    bound = bacc + 2 * E23 * ref.abs() + 1e-30
    name = "dx_R%d_T%d_dxo%d_p%g" % (R, T, with_dxo, p)
    check(name + "_dx", dx[:rows], ref, bound + 2.0 ** -8 * ref.abs())
    all_nan(name + " tail", dx[rows:])
    check(name + "_colsum", fx_total(fx), fscale * ref.sum(0), fscale * colsum_bound(bound, ref))


# ------------------------------------------------------------------------------------------------------------------------------
# EPI_TOUT (swapped GEMM, transposed fp32 output) and split-K
# ------------------------------------------------------------------------------------------------------------------------------
TOUT_BN = 32
TOUT_CASES = [(1, (0, 1)), (1, (1, 0)), (1, (2, 2)), (4, (2, 2)), (8, (2, 2))]


@pytest.mark.parametrize("ksplit,modes", TOUT_CASES)
def test_tout_and_split_k(ksplit, modes):
    g = torch.Generator().manual_seed(ksplit * 10 + modes[0])
    K, H4, nb = 200, 13 * 64, 33                       # 13 k-blocks: not divisible by 4 or 8
    rows0, ld0, ld1 = 120, 128, 96
    A = {"t": (torch.randn(1, 1, K, H4, generator=g) * 0.5).bfloat16().to(DEV), "C": H4, "ld": H4, "L": 1}
    W = weight(1, nb, H4, g)
    d0 = (torch.randn(nb + 1, ld0, generator=g)).to(DEV) if modes[0] else nan_buf((nb + 1, ld0), torch.float32)
    d1 = (torch.randn(nb + 1, ld1, generator=g)).to(DEV) if modes[1] else nan_buf((nb + 1, ld1), torch.float32)
    p0, p1 = d0.clone(), d1.clone()
    call("TOUT", TOUT_BN, [A], [(0, 0, 0, 13, 0, 1)], W, K, 1, 2, ptr={0: d0, 1: d1},
         i={0: rows0, 1: ld0, 2: modes[0], 3: K, 4: ld1, 5: modes[1], 6: nb}, ksplit=ksplit)
    D, Da = gemm_ref([A], [(0, 0, 0, 13, 0, 1)], W, K, 1)
    D, Da = D[0].t(), Da[0].t()                          # [nb, K]
    name = "tout_ks%d_modes%d%d" % (ksplit, *modes)
    for dst, pre, lo, hi, ld, mode in ((d0, p0, 0, rows0, ld0, modes[0]), (d1, p1, rows0, K, ld1, modes[1])):
        ref = D[:, lo:hi] + (pre[:nb, :hi - lo].to(F64) if mode else 0)
        check(name + "_rows%d" % lo, dst[:nb, :hi - lo], ref, E20 * Da[:, lo:hi] + E23 * ref.abs() + 1e-7 + (2 * E23 * ref.abs() if mode else 0))
        if mode == 0:
            all_nan(name + " padding", torch.cat([dst[:nb, hi - lo:].flatten(), dst[nb:].flatten()]))
        else:
            assert torch.equal(dst[:nb, hi - lo:], pre[:nb, hi - lo:]) and torch.equal(dst[nb:], pre[nb:])


# ------------------------------------------------------------------------------------------------------------------------------
# EPI_CE
# ------------------------------------------------------------------------------------------------------------------------------
CE_BN = 256
CE_CASES = [(200, [200, 1, 2, 131]), (33, [33, 2, 1, 30]), (385, [385, 384, 2, 129])]


@pytest.mark.parametrize("T,lengths", CE_CASES)
def test_cross_entropy(T, lengths):
    from oracle import wavenet as ow
    g = torch.Generator().manual_seed(T)
    B, C, ld = len(lengths), 136, 520
    maps = [act_map(1, B, T, C, gen=g)]
    segs = [(0, -1, 0, 3, 0, 1), (0, 0, 0, 3, 0, 1)]
    W = weight(1, 256, 384, g)
    bias = (torch.randn(256, generator=g) * 0.5).to(DEV)
    tgt = torch.randint(0, 256, (B, T), generator=g, dtype=torch.int32).to(DEV)
    lens = torch.tensor(lengths, dtype=torch.int32, device=DEV)
    rows, slack = B * T, 2
    sums = torch.zeros(2, device=DEV)
    dl = nan_buf((rows + slack, ld), torch.bfloat16)
    logits = nan_buf((rows + slack, 256), torch.float32)
    call("CE", CE_BN, maps, segs, W, T, B, 1, ptr={0: tgt, 1: lens, 2: bias, 3: sums[0:1], 4: sums[1:2], 5: dl, 6: logits}, i={1: ld})
    D, Da = gemm_ref(maps, segs, W, T, B)
    z = (D + bias.to(F64)).cpu().requires_grad_(True)
    y = tgt.long().cpu()
    mask = ow.sequence_mask(lens.cpu(), T)[:, 1:]
    per = torch.nn.functional.cross_entropy(z[:, :-1].reshape(-1, 256), y[:, 1:].reshape(-1), reduction="none").view(B, T - 1) * mask
    cnt = torch.count_nonzero(per).item()
    mean = ow.masked_cross_entropy(z.transpose(1, 2), y, lens.cpu())
    (mean * cnt).backward()
    name = "ce_T%d_len%s" % (T, "-".join(map(str, lengths)))
    loss_sum = mean.item() * cnt
    record(name + "_loss", rel=abs(sums[0].item() - loss_sum) / abs(loss_sum), count=sums[1].item(), count_ref=cnt)
    assert abs(sums[0].item() - loss_sum) <= 1e-5 * abs(loss_sum) and sums[1].item() == cnt
    zf = z.detach().to(DEV).view(rows, 256)
    check(name + "_logits", logits[:rows], zf, E20 * Da.view(rows, 256) + E23 * zf.abs() + 1e-7)
    gr = z.grad.to(DEV).view(rows, 256)
    check(name + "_dlogits", dl[:rows, :256].to(F64) + dl[:rows, 256:512].to(F64), gr, torch.full_like(gr, 2.0 ** -16))
    all_nan(name + " padding", torch.cat([dl[:rows, 512:].flatten(), dl[rows:].flatten(), logits[rows:].flatten()]))


# ------------------------------------------------------------------------------------------------------------------------------
# EPI_MOL (mixture of logistics and the single-Gaussian heads)
# ------------------------------------------------------------------------------------------------------------------------------
MOL_BN = 32
MOL_CASES = [("mol", 10, 65536), ("mol", 3, 256), ("gauss", 1, 65536), ("gauss", 2, 65536)]


@pytest.mark.parametrize("head,nm,nc", MOL_CASES)
def test_mol(head, nm, nc):
    from oracle import wavenet as ow
    g = torch.Generator().manual_seed(nm + nc)
    B, T, C, ld = 3, 200, 136, 40
    lengths = [200, 2, 150]
    nout = 3 * nm if head == "mol" else 2
    maps = [act_map(1, B, T, C, gen=g)]
    segs = [(0, 0, 0, 3, 0, 1)]
    W = weight(1, nout, 192, g)
    lsm, lsg = -7.0, -7.0
    if head == "mol":
        bias = torch.cat([torch.randn(nm, generator=g), torch.randn(nm, generator=g) * 0.3, torch.full((nm,), -6.5)])
    else:
        bias = torch.tensor([0.0, -6.8])                   # log-scale straddles the clamp
    bias = bias.to(DEV)
    choices = torch.tensor([-1.0, 1.0, 0.9995, -0.9995])
    tgt = torch.where(torch.rand(B, T, generator=g) < 0.2, choices[torch.randint(0, 4, (B, T), generator=g)],
                      torch.rand(B, T, generator=g) * 1.98 - 0.99).float().to(DEV)
    lens = torch.tensor(lengths, dtype=torch.int32, device=DEV)
    rows, slack = B * T, 2
    sums = torch.zeros(2, device=DEV)
    dy = nan_buf((rows + slack, ld), torch.bfloat16)
    yo = nan_buf((rows + slack, 32), torch.float32)
    call("MOL", MOL_BN, maps, segs, W, T, B, 1, ptr={0: tgt, 1: lens, 2: bias, 3: sums[0:1], 4: sums[1:2], 5: dy, 6: yo},
         f={0: lsm, 1: 1.0 / (nc - 1), 2: math.log((nc - 1) / 2.0), 3: lsg},
         i={0: nm, 1: ld, 2: 0 if head == "mol" else nm})
    D, Da = gemm_ref(maps, segs, W, T, B)
    yh = (D + bias.to(F64)).cpu().requires_grad_(True)     # [B, T, nout]
    mask = ow.sequence_mask(lens.cpu(), T)[:, 1:].to(F64)
    yt = tgt.to(F64).cpu()[:, 1:].unsqueeze(-1)
    if head == "mol":
        per = ow.discretized_mix_logistic_loss(yh[:, :-1].transpose(1, 2), yt, num_classes=nc, log_scale_min=lsm, reduce=False)
    else:
        per = ow.gaussian_maximum_likelihood_estimation_loss(yh[:, :-1].transpose(1, 2), yt, lsg, nc, use_cdf=(nm == 2), reduce=False)
    loss = (per[..., 0] * mask).sum()
    loss.backward()
    name = "%s_nm%d_nc%d" % (head, nm, nc)
    rel = abs(sums[0].item() - loss.item()) / abs(loss.item())
    record(name + "_loss", rel=rel, count=sums[1].item())
    assert rel <= 1e-5 and sums[1].item() == mask.sum().item()
    yref = torch.zeros(rows, 32, dtype=F64, device=DEV)
    yref[:, :nout] = yh.detach().to(DEV).view(rows, nout)
    ybound = torch.zeros_like(yref)
    ybound[:, :nout] = E20 * Da.view(rows, nout) + E23 * yref[:, :nout].abs() + 1e-7
    check(name + "_yhat", yo[:rows], yref, ybound + 1e-30)
    gref = torch.zeros(rows, 32, dtype=F64, device=DEV)
    gref[:, :nout] = yh.grad.to(DEV).view(rows, nout)
    check(name + "_dyhat", dy[:rows, :32], gref, 1e-4 * gref.abs().max() + 2.0 ** -8 * gref.abs())
    all_nan(name + " padding", torch.cat([dy[:rows, 32:].flatten(), dy[rows:].flatten(), yo[rows:].flatten()]))


# ------------------------------------------------------------------------------------------------------------------------------
# EPI_LSTM (swapped GEMM + LSTM cell + zoneout)
# ------------------------------------------------------------------------------------------------------------------------------
LSTM_BN = 32
LSTM_CASES = [(32, 3, True), (32, 33, False), (256, 32, True), (256, 33, True), (256, 3, False)]


@pytest.mark.parametrize("H,B,training", LSTM_CASES)
def test_lstm(H, B, training):
    from oracle import tacotron as ot
    g = torch.Generator().manual_seed(H + B)
    K = (H + 63) // 64 * 64
    Wh = (torch.randn(4, H, K, generator=g) / math.sqrt(K)).bfloat16()     # gate g, unit u, k
    wrec = torch.empty(4 * H, K, dtype=torch.bfloat16)
    for r in range(4 * H):                                                   # tile row p: gate p / 32, unit 32 m_tile + p % 32
        mt, p = divmod(r, 128)
        wrec[r] = Wh[p // 32, mt * 32 + p % 32]
    A = {"t": wrec.view(1, 1, 4 * H, K).to(DEV), "C": K, "ld": K, "L": 1}
    state = (torch.randn(1, B, K, generator=g) * 0.5).bfloat16().to(DEV)
    ps, lhp, lhs, lho = 4 * H + 8, H + 8, H + 16, H
    pre = torch.randn(B, ps, generator=g).to(DEV)
    bias = torch.randn(4 * H, generator=g).to(DEV) * 0.5
    c_prev = torch.randn(B, H, generator=g).to(DEV)
    h_prev = (torch.randn(B, lhp, generator=g) * 0.5).bfloat16().to(DEV)
    t, stream, z, seed, off = 5, 27, 0.1, 2024, 9
    lens = torch.tensor([(7 if b % 3 else 3) for b in range(B)], dtype=torch.int32, device=DEV)     # some items already ended
    c_out = nan_buf((B + 1, H), torch.float32)
    h_state = nan_buf((B + 1, lhs), torch.bfloat16)
    h_out = nan_buf((B + 1, lho), torch.bfloat16)
    gst = nan_buf((B + 1, 4 * H), torch.bfloat16)
    tst = nan_buf((B + 1, H), torch.bfloat16)
    call("LSTM", LSTM_BN, [A], [(0, 0, 0, K // 64, 0, 1)], state, 4 * H, 1, (B + 31) // 32,
         ptr={0: pre, 1: bias, 2: c_prev, 3: c_out, 4: h_prev, 5: h_state, 6: h_out, 7: gst, 8: tst, 9: lens, 10: seed_offset(off)},
         f={0: z}, i={0: H, 1: B, 3: ps, 4: lhp, 5: lhs, 6: lho, 7: t, 8: stream, 9: int(training)}, seed=seed)
    kern = Wh.to(F64).permute(2, 0, 1).reshape(K, 4 * H).to(DEV)             # [K, 4H], column g*H + u
    x = state[0].to(F64)
    b_all = bias.to(F64) + pre[:, :4 * H].to(F64)
    cp, hp = c_prev.to(F64), h_prev[:, :H].to(F64)
    zz = x @ kern + b_all
    cn, hn = ot.lstm_cell(x, cp, torch.zeros(B, 0, dtype=F64, device=DEV), kern, b_all)
    if training:
        idx = (np.uint64(t) * np.uint64(B) + np.arange(B, dtype=np.uint64)[:, None]) * np.uint64(H) + np.arange(H, dtype=np.uint64)[None, :]
        mc = torch.from_numpy(mh.hash_uniform32(mh.hash_seed(seed + off, stream * 2), idx) >= np.float32(z)).to(DEV).to(F64)
        mhm = torch.from_numpy(mh.hash_uniform32(mh.hash_seed(seed + off, stream * 2 + 1), idx) >= np.float32(z)).to(DEV).to(F64)
        cs, hs = ot.zoneout(cp, cn, z, True, mc), ot.zoneout(hp, hn, z, True, mhm)
    else:
        cs, hs = ot.zoneout(cp, cn, z, False), ot.zoneout(hp, hn, z, False)
    live = (t < lens).to(DEV)[:, None]
    gates = torch.cat([torch.sigmoid(zz[:, :H]), torch.tanh(zz[:, H:2 * H]), torch.sigmoid(zz[:, 2 * H:3 * H] + 1), torch.sigmoid(zz[:, 3 * H:])], 1)
    cs, hs = torch.where(live, cs, cp), torch.where(live, hs, hp)
    ho, tc = torch.where(live, hn, torch.zeros_like(hn)), torch.where(live, torch.tanh(cn), torch.zeros_like(cn))
    gates = torch.where(live, gates, torch.zeros_like(gates))
    name = "lstm_H%d_B%d_train%d" % (H, B, training)
    tol = lambda r: 1e-4 * r.abs().max() + 1e-30
    check(name + "_c", c_out[:B], cs, tol(cs))
    check(name + "_hstate", h_state[:B, :H], hs, tol(hs) + 2.0 ** -8 * hs.abs())
    check(name + "_hout", h_out[:B], ho, tol(ho) + 2.0 ** -8 * ho.abs())
    check(name + "_gates", gst[:B], gates, tol(gates) + 2.0 ** -8 * gates.abs())
    check(name + "_tanhc", tst[:B], tc, tol(tc) + 2.0 ** -8 * tc.abs())
    all_nan(name + " padding", torch.cat([c_out[B:].flatten(), h_state[:, H:].flatten(), h_out[B:].flatten(), gst[B:].flatten(),
                                           tst[B:].flatten()]))


# ------------------------------------------------------------------------------------------------------------------------------
# engine mechanics
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [33, 200])
def test_segments_layers_offsets_and_channel_slices(T):
    """K over the layer axis (nlayers > 1 on L > 1 maps), w_layer / w_k0, k0 > 0 on a map with ld > C, 4 distinct maps"""
    g = torch.Generator().manual_seed(T)
    B, N = 3, 256
    maps = [act_map(3, B, T, 128, gen=g), act_map(1, B, T, 200, ld=264, gen=g), act_map(2, B, T, 72, gen=g), act_map(1, B, T, 64, gen=g)]
    segs = [(0, -2, 0, 2, 0, 3), (1, 3, 64, 3, 0, 1), (2, 0, 0, 2, 1, 1), (3, -40, 0, 1, 0, 1), (0, 1, 64, 1, 2, 1)]
    ktot = (6 + 3 + 2 + 1 + 1) * 64
    W = weight(3, N, ktot + 128 + 40, g)
    out = nan_buf((B * T + 1, N), torch.float32)
    call("BIAS_ACT", 128, maps, segs, W, T, B, 2, ptr={2: out}, i={0: N, 1: 0, 2: N}, w_layer=2, w_k0=128)
    D, Da = gemm_ref(maps, segs, W, T, B, w_layer=2, w_k0=128)
    check("segments_T%d" % T, out[:B * T], D.view(-1, N), E20 * Da.view(-1, N) + 1e-7)
    all_nan("segments tail", out[B * T:])


@pytest.mark.parametrize("epi,BN", [("BIAS_ACT", 128), ("BIAS_ACT", 256), ("RES", 128), ("RES", 256)])
def test_cluster_multicast_is_bitwise_equal(epi, BN):
    """the weight feed changes (one TMA multicast per cluster), the MMA order does not: outputs must be bitwise equal"""
    g = torch.Generator().manual_seed(BN)
    B, T, C = 2, 1024, 200                      # 16 M tiles: divisible by every cluster size
    maps = [act_map(1, B, T, C, gen=g)]
    segs = [(0, -1, 0, 4, 0, 1), (0, 0, 0, 4, 0, 1)]
    N = 2 * BN if epi == "BIAS_ACT" else BN
    W = weight(1, N, 512, g)
    bias = torch.randn(N, generator=g).to(DEV)
    rows = B * T
    x_in = (torch.randn(rows, BN, generator=g) * 0.5).bfloat16().to(DEV)

    def run(cs):
        if epi == "BIAS_ACT":
            o = nan_buf((rows, N), torch.float32)
            ob = nan_buf((rows, N), torch.bfloat16)
            used = call(epi, BN, maps, segs, W, T, B, 2, ptr={0: ob, 1: bias, 2: o}, i={0: N, 1: 1, 2: N}, cluster=cs)
            return used, (o, ob)
        xo = nan_buf((rows, BN), torch.bfloat16)
        xd = nan_buf((rows, BN), torch.bfloat16)
        used = call(epi, BN, maps, segs, W, T, B, 1, ptr={0: x_in, 1: xo, 2: xd, 3: bias}, f={0: 0.5, 1: 0.25}, i={1: 2}, seed=5,
                    cluster=cs)
        return used, (xo, xd)
    used1, base = run(1)
    assert used1 == 1
    for cs in (2, 4, 8):
        try:
            used, got = run(cs)
        except L.T2Error as e:
            if cs == 8 and "cannot be scheduled" in str(e):
                continue
            raise
        assert used == cs, "asked for a cluster of %d, launched %d" % (cs, used)
        for a, b in zip(base, got):
            assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                               b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32)), "cluster %d differs" % cs
    D, Da = gemm_ref(maps, segs, W, T, B)
    if epi == "BIAS_ACT":
        v = (D + bias.to(F64)).relu().view(rows, N)
        check("cluster_%s_%d" % (epi, BN), base[0], v, E20 * Da.view(rows, N) + E23 * v.abs() + 1e-7)


def test_dependent_launch_chain():
    """kernel 2 reads kernel 1's output as its A operand and as EPI_RES's prefetched x_in, launched back to back on one stream:
    the programmatic-dependent-launch wait must precede every global read"""
    g = torch.Generator().manual_seed(11)
    B, T, C, R = 2, 385, 200, 128
    maps1 = [act_map(1, B, T, C, gen=g)]
    segs1 = [(0, 0, 0, 4, 0, 1)]
    W1 = weight(1, R, 256, g)
    W2 = weight(1, R, 128, g)
    b1, b2 = torch.randn(R, generator=g).to(DEV), torch.randn(R, generator=g).to(DEV)
    rows = B * T
    for rep in range(3):
        y = nan_buf((rows, R), torch.bfloat16)         # stale reads of y would be NaN
        x_out = nan_buf((rows, R), torch.bfloat16)
        call("BIAS_ACT", 128, maps1, segs1, W1, T, B, 1, ptr={0: y, 1: b1}, i={0: R, 1: 2, 2: R}, sync=False)
        m2 = [{"t": y.view(1, B, T, R), "C": R, "ld": R, "L": 1}]
        call("RES", R, m2, [(0, -1, 0, 2, 0, 1)], W2, T, B, 1, ptr={0: y, 1: x_out, 3: b2}, f={0: 1.0, 1: 0.0}, i={1: 0})
        xo, bound, _ = res_ref(m2, [(0, -1, 0, 2, 0, 1)], W2, y.to(F64).view(B, T, R), b2, 1.0, 0.0, T, B, R, 0, 0)
        assert not torch.isnan(y.float()).any()
        check("pdl_chain_rep%d" % rep, x_out, xo.view(rows, R), bound.view(rows, R) + 2.0 ** -8 * xo.abs().view(rows, R))


# ------------------------------------------------------------------------------------------------------------------------------
# fixed-point column sums (bias gradients)
# ------------------------------------------------------------------------------------------------------------------------------
def _fx_colsum(addends):
    lib = _lib()
    out = nan_buf((addends.shape[1],), torch.float32)
    L.check(lib.t2_dbg_fx_colsum(L.ptr(addends), addends.shape[0], addends.shape[1], L.ptr(out), L.stream_ptr()))
    return out


def test_fx_colsum_non_finite_and_overflow():
    """a NaN or Inf addend, or a column whose sum leaves the fixed-point range, must finalise to a non-finite gradient: never to a
    finite or sign-flipped value"""
    g = torch.Generator().manual_seed(3)
    n = 1000
    cols = torch.randn(n, 9, generator=g) * 0.01
    cols[17, 0] = NAN
    cols[3, 1] = float("inf")
    cols[5, 2] = -float("inf")
    cols[:, 3] = 0
    cols[[10, 900], 3] = 5e6                      # each in range, the sum (1e7) is not
    cols[:, 4] = 0
    cols[[1, 2], 4] = -5e6
    cols[:, 5] = 0
    cols[[7, 8], 5] = 3e6                          # sum 6e6 > 2^22
    cols[40, 6] = 2.0 ** 22                        # one out-of-range addend
    d = cols.to(DEV)
    out = _fx_colsum(d)
    record("fx_edge_cases", values=[float(v) for v in out.cpu()])
    for c in range(7):
        assert not math.isfinite(out[c].item()), "column %d finalised to %r" % (c, out[c].item())
    # ordinary columns: deterministic and within n * 2^-41 of the float64 sum
    ref = cols[:, 7:].to(F64).sum(0)
    again = _fx_colsum(d)
    assert torch.equal(out[7:].view(torch.int32), again[7:].view(torch.int32))
    err = (out[7:].to(F64).cpu() - ref).abs()
    assert (err <= n * 2.0 ** -41 + 2.0 ** -24 * ref.abs()).all(), err


def test_fx_colsum_exact_for_representable_addends():
    """addends on the 2^-40 grid sum exactly, whatever the atomic order"""
    g = torch.Generator().manual_seed(4)
    a = (torch.randint(-2 ** 20, 2 ** 20, (4096, 64), generator=g).to(torch.float64) * 2.0 ** -30).float()
    out = _fx_colsum(a.to(DEV))
    ref = a.to(F64).sum(0)
    assert torch.equal(out.cpu(), ref.float())


# ------------------------------------------------------------------------------------------------------------------------------
# weight-gradient tile table
# ------------------------------------------------------------------------------------------------------------------------------
def _wg_ref(maps, tile, T, B):
    A, Bm = maps[tile["a_map"]], maps[tile["b_map"]]
    m, n = tile["m_valid"], tile["n_valid"]

    def rows(mp, ch0, sh, lyr, width):
        out = torch.zeros(B, T, width, dtype=F64, device=DEV)
        nch = max(0, min(width, mp["C"] - ch0))
        lo, hi = max(0, -sh), min(T, T - sh)
        if nch > 0 and hi > lo:
            out[:, lo:hi, :nch] = mp["t"][lyr, :, lo + sh:hi + sh, ch0:ch0 + nch].to(F64)
        return out.reshape(B * T, width)
    a = rows(A, tile["a_ch0"], tile["a_shift"], tile["a_layer"], m)
    b = rows(Bm, tile["b_ch0"], tile["b_shift"], tile["b_layer"], n)
    return a.t() @ b, a.abs().t() @ b.abs()


@pytest.mark.parametrize("T", [33, 200])
def test_wgrad_tiles(T):
    g = torch.Generator().manual_seed(T + 5)
    B = 2
    maps = [act_map(2, B, T, 200, ld=208, gen=g), act_map(1, B, T, 64, gen=g), act_map(3, B, T, 130, ld=136, gen=g),
            act_map(1, B, T, 256, gen=g), act_map(1, B, T, 72, ld=80, gen=g), act_map(2, B, T, 320, gen=g)]
    div0 = torch.zeros(1, device=DEV)
    div4 = torch.full((1,), 4.0, device=DEV)
    # (tile fields, divisor) - out regions are disjoint except the two accumulate-2 tiles, which share one
    spec = [
        (dict(a_map=0, a_ch0=0, a_shift=0, a_layer=1, b_map=5, b_ch0=0, b_shift=0, b_layer=1, ldc=300, m_valid=128, n_valid=256,
              scale=0.5, accumulate=0), None),
        (dict(a_map=2, a_ch0=64, a_shift=-5, a_layer=2, b_map=4, b_ch0=0, b_shift=2, b_layer=0, ldc=70, m_valid=40, n_valid=65,
              scale=1.0, accumulate=0), None),
        (dict(a_map=1, a_ch0=0, a_shift=3, a_layer=0, b_map=3, b_ch0=0, b_shift=0, b_layer=0, ldc=8, m_valid=64, n_valid=1,
              scale=2.0, accumulate=1), None),
        (dict(a_map=0, a_ch0=64, a_shift=-1, a_layer=0, b_map=2, b_ch0=0, b_shift=0, b_layer=0, ldc=64, m_valid=100, n_valid=63,
              scale=1.0, accumulate=2), None),
        (dict(a_map=0, a_ch0=64, a_shift=-1, a_layer=0, b_map=2, b_ch0=0, b_shift=0, b_layer=1, ldc=64, m_valid=100, n_valid=63,
              scale=1.0, accumulate=2), None),
        (dict(a_map=4, a_ch0=0, a_shift=0, a_layer=0, b_map=5, b_ch0=64, b_shift=-3, b_layer=0, ldc=200, m_valid=72, n_valid=192,
              scale=1e-18, accumulate=0), div0),
        (dict(a_map=3, a_ch0=128, a_shift=1, a_layer=0, b_map=0, b_ch0=0, b_shift=0, b_layer=0, ldc=260, m_valid=128, n_valid=200,
              scale=1.0, accumulate=1), div4),
    ]
    offs, total = [], 0
    shared = None
    for k, (t, _) in enumerate(spec):
        if t["accumulate"] == 2 and shared is not None:
            offs.append(shared)
            continue
        offs.append(total)
        if t["accumulate"] == 2:
            shared = total
        total += t["m_valid"] * t["ldc"] + 16
    out = nan_buf((total + 64,), torch.float32)
    pre = torch.randn(total + 64, generator=g).to(DEV)
    for k, (t, _) in enumerate(spec):            # prefill: accumulate 1 on random values, accumulate 2 on zeros
        if t["accumulate"]:
            reg = out[offs[k]:offs[k] + t["m_valid"] * t["ldc"]].view(t["m_valid"], t["ldc"])
            reg[:, :t["n_valid"]] = pre[offs[k]:offs[k] + t["m_valid"] * t["ldc"]].view(t["m_valid"], t["ldc"])[:, :t["n_valid"]] \
                if t["accumulate"] == 1 else 0
    before = out.clone()
    tiles = (L.DbgWgradTile * len(spec))()
    for k, (t, dv) in enumerate(spec):
        for key, v in t.items():
            setattr(tiles[k], key, v)
        tiles[k].out_off = offs[k]
        tiles[k].div = None if dv is None else dv.data_ptr()
    amaps = (L.DbgAct * 6)(*[L.DbgAct(m["t"].data_ptr(), m["C"], T, B, m["L"], m["ld"]) for m in maps])
    L.check(_lib().t2_dbg_wgrad_tiles(amaps, 6, tiles, len(spec), L.ptr(out), T, B, L.stream_ptr()))
    torch.cuda.synchronize()
    covered = torch.zeros_like(out, dtype=torch.bool)
    done = set()
    for k, (t, dv) in enumerate(spec):
        if offs[k] in done:
            continue
        m, n, ldc = t["m_valid"], t["n_valid"], t["ldc"]
        ref, refa = torch.zeros(m, n, dtype=F64, device=DEV), torch.zeros(m, n, dtype=F64, device=DEV)
        for j, (t2_, dv2) in enumerate(spec):
            if offs[j] == offs[k]:
                r, ra = _wg_ref(maps, t2_, T, B)
                sc = float(np.float32(t2_["scale"]) / max(np.float32(dv2.item()), np.float32(1e-20))) if dv2 is not None else t2_["scale"]
                ref, refa = ref + sc * r, refa + abs(sc) * ra
        if t["accumulate"]:
            ref = ref + before[offs[k]:offs[k] + m * ldc].view(m, ldc)[:, :n].to(F64)
        done.add(offs[k])
        reg = out[offs[k]:offs[k] + m * ldc].view(m, ldc)
        check("wgrad_T%d_tile%d_acc%d_m%d_n%d" % (T, k, t["accumulate"], m, n), reg[:, :n], ref,
              E20 * refa + 3 * E23 * ref.abs() + 1e-7 * (1 + abs(ref).max()))
        covered[offs[k]:offs[k] + m * ldc].view(m, ldc)[:, :n] = True
    assert torch.equal(out[~covered].isnan(), before[~covered].isnan()), "wgrad wrote outside its tiles"
    all_nan("wgrad untouched", out[~covered & before.isnan()])


# ------------------------------------------------------------------------------------------------------------------------------
# coverage of the kernel table
# ------------------------------------------------------------------------------------------------------------------------------
# (epilogue, BN) of every parametrized case: the column-tile width comes from the case itself, or from the one BN the test launches
COVERED = ({("EPI_BIAS_ACT", c[0]) for c in BIAS_ACT_CASES} | {("EPI_RES", c[0]) for c in RES_CASES}
           | {("EPI_SCALE_RELUMASK", c[0]) for c in SCALE_RELUMASK_CASES} | {("EPI_GATE_BWD", c[0]) for c in GATE_BWD_CASES}
           | {("EPI_DX", c[0]) for c in DX_CASES} | {("EPI_GATE", GATE_BN) for _ in GATE_CASES} | {("EPI_TOUT", TOUT_BN) for _ in TOUT_CASES}
           | {("EPI_CE", CE_BN) for _ in CE_CASES} | {("EPI_MOL", MOL_BN) for _ in MOL_CASES} | {("EPI_LSTM", LSTM_BN) for _ in LSTM_CASES})


def test_every_kernel_instantiation_has_a_case():
    src = open(os.path.join(ROOT, "tacotron-2_b200", "csrc", "t2_gemm.cu")).read()
    table = set((e, int(n)) for e, n in re.findall(r"^\s*T2_CASE\((EPI_\w+),\s*(\d+)\)", src, re.M))
    assert len(table) >= 15
    assert table <= COVERED, sorted(table - COVERED)
