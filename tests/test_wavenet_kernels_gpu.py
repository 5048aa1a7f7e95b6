"""The small kernels of the WaveNet engine (tacotron-2_b200/csrc/t2_wavenet.cu), one launch at a time through t2_dbg_wn_kernel, against
float64 references computed from the exact inputs the kernels read: bf16 inputs stay bf16, fixed-point inputs are exact integers, dropout
masks come from the host copy of the hash in mask_hash.py.

Bounds (u = 2^-24, BF = 2^-8 the unit roundoff of bf16 (8 significant bits), FX = 2^-40 the fixed-point resolution):
  first_conv            one fp32 add (or product + add for scalar input) then one bf16 rounding: BF |ref| + 2u (|x w| + |b|). Split rows:
                        hi = bf16(v), lo = bf16(v - hi), so |hi + lo - v| <= BF |v - hi| <= BF^2 |v| and |hi + lo - ref| <= 2^-16 |ref|
                        + 2u (|x w| + |b|). The dropout copy keeps
                        exactly the elements the hash keeps (bit for bit, moved by seed + *step) at BF |ref / (1 - p)| + 3u |ref| / (1 - p).
  first_conv_bwd        one-hot: with bf16 gradients of magnitude in [2^-30, 1] every addend is an exact multiple of FX, so the total is
                        the exact sum, rounded once to fp32 by the finalisation: equal to float32(float64 sum), bit for bit, and the same
                        in two launches. Scalar input: each block adds <= 64 products in fp32 (64 u sum |x dx|), its total is rounded to FX
                        (FX / 2 per block), the finalisation rounds once more (u |ref|).
  colsum                each of the 96 blocks adds ceil(rows / 96) bf16 values in fp32 ((ceil(rows / 96) + 1) u sum |x|), the product with
                        sc = scale / max(scalar, 1e-20) (itself one rounding) adds 2u, the fixed-point rounding FX / 2 per block, the
                        finalisation u |ref|. A zero scalar puts every non-zero column beyond the fixed-point range: NaN. dst2 == dst.
  derived_bias          bias_g: one fp32 add (u |ref|). bias_skip: L sequential products + adds: 2 L u sum_l |scale_l b_l|.
  skip_bias, fx_final.  a fixed-point total converted to fp32 (u), then one product or add (u): 2u (|ref| + |addend|). Zero totals leave
                        fx_finalize's element untouched (bit for bit); a poisoned total gives NaN.
  cl_to_chw             a copy: exact.
  gin_bias              Gi sequential fp32 products + adds onto b_gin, then one add onto the shared bias: (Gi + 2) u (|b_gin| + sum |W e|)
                        + u |ref|. An id outside [0, NS) gives NaN for the item; no ids, or the on flag 0, gives the shared bias exactly.
  gin_wgrad             integer totals exact as int64 (kFxPoison for a poisoned / out-of-range addend); dW_gin: B sequential fp32
                        products + adds of exact fixed-point values: (B + 1) u sum_b |e S| (+ u for the conversion of each S).
  gin_demb              per thread ceil(L G / 256) products + adds, an 8-level tree, then one add per item: (L G / 256 + B + 10) u sum |W S|.
                        A speaker row no item uses gets exactly 0 (its gradient), with spk[0] = 0 nothing is written.
Every check records its worst err / bound through parity_util.record. Outputs start as NaN (or a sentinel where the kernel adds or
must not write), and padding past the written region must keep it."""
import ctypes
import math

import numpy as np
import pytest
import torch

import mask_hash as mh
from parity_util import record
from t2_import import t2

pytestmark = pytest.mark.gpu
L = t2.lib
DEV = "cuda"
F64 = torch.float64
NAN = float("nan")
U = 2.0 ** -24
BF = 2.0 ** -8
FX = 2.0 ** -40
POISON = -(1 << 63)
IDS = dict(FIRST_CONV=10, FIRST_CONV_BWD=11, COLSUM=12, DERIVED_BIAS=13, SKIP_BIAS=14, FX_FINALIZE=15, CL_TO_CHW=16, GIN_BIAS=17,
           SET_SPEAKERS=18, GIN_WGRAD=19, GIN_DEMB=20)


def launch(kernel, p=(), i=(), f=(), seed=0, step=None):
    lib = L.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    c = L.DbgKernel()
    c.kernel = IDS[kernel]
    for k, v in enumerate(p):
        c.p[k] = None if v is None else (v if isinstance(v, int) else v.data_ptr())
    for k, v in enumerate(i):
        c.i[k] = int(v)
    for k, v in enumerate(f):
        c.f[k] = float(v)
    c.seed = seed
    c.step = None if step is None else step.data_ptr()
    L.check(lib.t2_dbg_wn_kernel(ctypes.byref(c), L.stream_ptr()))
    torch.cuda.synchronize()


def check(name, got, ref, bound, **info):
    err = (got.to(F64) - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=float("inf")).max().item() if err.numel() else 0.0
    record(name, worst_err_over_bound=ratio, **info)
    assert ratio <= 1.0, "%s: worst err / bound %.3g" % (name, ratio)


def all_nan(name, t):
    assert t.numel() == 0 or torch.isnan(t.float()).all().item(), "%s: written outside its bounds" % name


def nan_buf(shape, dtype=torch.float32):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


def bf16_grads(shape, gen, lo=-30):
    """bf16 values of magnitude in [2^lo, 1) with random signs: every one an exact multiple of 2^-40 when lo >= -32"""
    e = torch.randint(lo, 0, shape, generator=gen).double()
    m = 1 + torch.randint(0, 128, shape, generator=gen).double() / 128
    s = torch.where(torch.rand(shape, generator=gen) < 0.5, -1.0, 1.0).double()
    return (s * m * 2.0 ** e).to(torch.bfloat16).to(DEV)


def fx_value(a):
    """int64 tensor of fixed-point totals -> float64 values (NaN where out of range / poisoned)"""
    v = a.to(F64) * FX
    return torch.where((a > -(1 << 62)) & (a < (1 << 62)), v, torch.full_like(v, NAN))


# ------------------------------------------------------------------------------------------------------------------------------
# first (embedding) conv
# ------------------------------------------------------------------------------------------------------------------------------
FC_CASES = [(128, 1, 0, 0, 0.0), (128, 37, 0, 0, 0.05), (256, 197, 0, 0, 0.05), (256, 197, 1, 0, 0.05), (128, 64, 1, 0, 0.0),
            (128, 197, 0, 1, 0.0), (256, 37, 1, 1, 0.0)]


@pytest.mark.parametrize("R,npos,scalar,split,p", FC_CASES)
def test_first_conv(R, npos, scalar, split, p):
    g = torch.Generator().manual_seed(R + npos + 7 * scalar + 3 * split)
    Q = 1 if scalar else 256
    W = torch.randn(Q, R, generator=g).to(DEV)
    b = (torch.randn(R, generator=g) * 0.1).to(DEV)
    if scalar:
        xin = (torch.rand(npos, generator=g) * 2 - 1).to(DEV)
        prod = xin.to(F64)[:, None] * W.to(F64)
    else:
        xin = torch.randint(0, Q, (npos,), generator=g, dtype=torch.int32).to(DEV)
        prod = W.to(F64)[xin.long()]
    ref = prod + b.to(F64)
    rnd = 2 * U * (prod.abs() + b.to(F64).abs())
    width = 2 * R if split else R
    x = nan_buf((npos + 3, width), torch.bfloat16)
    xd = nan_buf((npos + 3, R), torch.bfloat16) if p > 0 else None
    step = torch.tensor([5], dtype=torch.int64, device=DEV)
    seed = 1234
    launch("FIRST_CONV", [xin, W, b, x, xd], [npos, R, scalar, split], [p], seed=seed, step=step)
    tag = "first_conv_R%d_n%d_s%d_split%d_p%g" % (R, npos, scalar, split, p)
    all_nan(tag + "_pad", x[npos:])
    if split:
        hi, lo = x[:npos, :R].to(F64), x[:npos, R:].to(F64)
        check(tag + "_hi", hi, ref, BF * ref.abs() + rnd)
        check(tag + "_hi_plus_lo", hi + lo, ref, 2.0 ** -16 * ref.abs() + rnd)
        return
    check(tag, x[:npos], ref, BF * ref.abs() + rnd)
    if xd is None:
        return
    all_nan(tag + "_xd_pad", xd[npos:])
    for st in (5, 6):
        if st == 6:
            step.fill_(6)
            xd.fill_(NAN)
            launch("FIRST_CONV", [xin, W, b, x, xd], [npos, R, scalar, split], [p], seed=seed, step=step)
        hs = mh.hash_seed((seed + st) & (2 ** 64 - 1), 0)
        keep = torch.from_numpy(mh.hash_keep16(hs, np.arange(npos * R, dtype=np.uint64), mh.keep_threshold16(p))).view(npos, R).to(DEV)
        kinv = 1.0 / float(np.float32(1) - np.float32(p))
        kinv = float(np.float32(kinv))
        got = xd[:npos].to(F64)
        assert torch.equal(got == 0, ~keep), "%s: dropout mask differs from the hash at step %d" % (tag, st)
        check(tag + "_xd_step%d" % st, got, torch.where(keep, ref * kinv, torch.zeros_like(ref)),
              BF * (ref * kinv).abs() + 3 * U * ref.abs() * kinv + rnd * kinv)
        if st == 5:
            mask5 = keep
    assert not torch.equal(mask5, keep), "seed + *step does not move the dropout mask"


@pytest.mark.parametrize("R,npos,scalar,same", [(128, 37, 0, 0), (128, 37, 0, 1), (256, 197, 0, 0), (256, 197, 0, 1), (128, 128, 0, 0),
                                                (256, 1, 0, 0), (128, 197, 1, 0), (256, 37, 1, 0), (128, 128, 1, 0)])
def test_first_conv_bwd(R, npos, scalar, same):
    g = torch.Generator().manual_seed(R * 3 + npos + same)
    Q = 1 if scalar else 256
    dx0 = bf16_grads((npos, R), g)
    if scalar:
        xin = (torch.rand(npos, generator=g) * 2 - 1).to(DEV)
        terms = xin.to(F64)[:, None] * dx0.to(F64)
        ref = terms.sum(0, keepdim=True)
        nblk = (npos + 63) // 64
        bound = 64 * U * terms.abs().sum(0, keepdim=True) + nblk * FX / 2 + U * ref.abs()
        used = torch.ones(1, dtype=torch.bool, device=DEV)
    else:
        idx = torch.full((npos,), 77, dtype=torch.int32) if same else torch.randint(0, 200, (npos,), generator=g, dtype=torch.int32)
        xin = idx.to(DEV)
        ref = torch.zeros(Q, R, dtype=F64, device=DEV).index_add_(0, xin.long(), dx0.to(F64))
        used = torch.zeros(Q, dtype=torch.bool, device=DEV)
        used[xin.long()] = True
    tag = "first_conv_bwd_R%d_n%d_s%d_same%d" % (R, npos, scalar, same)
    outs = []
    for _ in range(2):
        acc = torch.zeros(Q * R, dtype=torch.int64, device=DEV)
        dW = torch.where(used[:, None], torch.zeros(Q, R, device=DEV), torch.full((Q, R), NAN, device=DEV)).contiguous()
        launch("FIRST_CONV_BWD", [xin, dx0, acc, dW], [npos, R, scalar, Q])
        outs.append(dW.clone())
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), tag + ": two launches differ"
    dW = outs[0]
    all_nan(tag + "_unused_rows", dW[~used])
    if scalar:
        check(tag, dW, ref, bound)
    else:
        exact = ref[used].float()
        assert torch.equal(dW[used].view(torch.int32), exact.view(torch.int32)), tag + ": not the exact sum rounded once"
        record(tag, worst_err_over_bound=0.0, bit_exact=1)


# ------------------------------------------------------------------------------------------------------------------------------
# column sums of the bias gradients
# ------------------------------------------------------------------------------------------------------------------------------
def colsum_setup(jobs_spec, gen):
    """jobs_spec: [(rows, C, ld, scale, div_scalar, dup)] -> ws bf16 buffer, jobs int64 [n][7], scales fp32 [n], per-job (src, dst, dst2)"""
    srcs, off = [], 0
    for rows, C, ld, *_ in jobs_spec:
        srcs.append((off, rows, C, ld))
        off += rows * ld * 2
        off += (-off) % 16
    ws = torch.full((off // 2,), NAN, dtype=torch.bfloat16, device=DEV)
    jobs, scales, views, dst = [], [], [], 8
    for (so, rows, C, ld), (_, _, _, scale, div, dup) in zip(srcs, jobs_spec):
        m = ws[so // 2: so // 2 + rows * ld].view(rows, ld)
        m[:, :C] = (torch.randn(rows, C, generator=gen) * 0.5).to(torch.bfloat16).to(DEV)
        d2 = dst + C + 6 if dup else -1
        jobs.append([so, rows, C, ld, dst, d2, div])
        scales.append(scale)
        views.append((m[:, :C], dst, d2))
        dst = (d2 if dup else dst) + C + 10
    return ws, torch.tensor(jobs, dtype=torch.int64), torch.tensor(scales, dtype=torch.float32), views, dst


@pytest.mark.parametrize("case", ["small_rows", "many_rows", "mixed"])
def test_colsum(case):
    gen = torch.Generator().manual_seed(len(case))
    spec = {"small_rows": [(200, 80, 96, 1.0, -1, True), (1, 2, 2, 2.0, -1, False)],
            "many_rows": [(5000, 256, 264, 0.5, 1, False), (15360, 30, 32, 1.0, 2, True)],
            "mixed": [(383, 256, 256, 1.0, 1, True), (385, 128, 136, 0.25, -1, False), (96 * 4, 80, 82, 3.0, 2, True)]}[case]
    ws, jobs, scales, views, n_acc = colsum_setup(spec, gen)
    scal = torch.tensor([NAN, 37.5, 3.0], dtype=torch.float32, device=DEV)
    acc = torch.zeros(n_acc, dtype=torch.int64, device=DEV)
    grads = nan_buf((n_acc,))
    for _, d, d2 in views:
        C = _.shape[1]
        grads[d:d + C] = 0
        if d2 >= 0:
            grads[d2:d2 + C] = 0
    table = torch.empty(64 * len(spec), dtype=torch.uint8, device=DEV)
    launch("COLSUM", [ws, acc, grads, scal, table, jobs.data_ptr(), scales.data_ptr()], [len(spec), n_acc, ws.numel() * 2, 3])
    touched = torch.zeros(n_acc, dtype=torch.bool, device=DEV)
    for k, ((m, d, d2), (rows, C, ld, scale, div, dup)) in enumerate(zip(views, spec)):
        x = m.to(F64)
        sc = float(np.float32(scale) / np.float32(max(scal[div].item(), 1e-20))) if div >= 0 else scale
        ref = x.sum(0) * sc
        per = -(-rows // 96)
        bound = ((per + 1) * U * x.abs().sum(0) + 2 * U * x.abs().sum(0)) * abs(sc) + 96 * FX / 2 + U * ref.abs()
        check("colsum_%s_job%d_rows%d_C%d" % (case, k, rows, C), grads[d:d + C], ref, bound)
        touched[d:d + C] = True
        if d2 >= 0:
            assert torch.equal(grads[d:d + C].view(torch.int32), grads[d2:d2 + C].view(torch.int32)), "dst2 differs from dst"
            touched[d2:d2 + C] = True
    all_nan("colsum_%s_untouched" % case, grads[~touched])


def test_colsum_zero_scalar_is_nan():
    """scale / max(0, 1e-20) puts every non-zero column sum beyond the fixed-point range: NaN, not a finite value; an all-zero column
    stays 0"""
    gen = torch.Generator().manual_seed(3)
    spec = [(300, 64, 64, 1.0, 0, True)]
    ws, jobs, scales, views, n_acc = colsum_setup(spec, gen)
    m, d, d2 = views[0]
    m[:, 5] = 0
    scal = torch.zeros(1, dtype=torch.float32, device=DEV)
    acc = torch.zeros(n_acc, dtype=torch.int64, device=DEV)
    grads = torch.zeros(n_acc, device=DEV)
    table = torch.empty(64, dtype=torch.uint8, device=DEV)
    launch("COLSUM", [ws, acc, grads, scal, table, jobs.data_ptr(), scales.data_ptr()], [1, n_acc, ws.numel() * 2, 1])
    for base in (d, d2):
        col = grads[base:base + 64]
        assert col[5].item() == 0.0
        assert torch.isnan(torch.cat([col[:5], col[6:]])).all()
    record("colsum_zero_scalar", worst_err_over_bound=0.0)


# ------------------------------------------------------------------------------------------------------------------------------
# derived biases, skip-bias gradient, fixed-point finalisation, transpose
# ------------------------------------------------------------------------------------------------------------------------------
def offs_table(Lr, G, S, no_cin=()):
    """a flat parameter buffer (NaN between the tensors) and its [3L] table: per layer b_dil [G], b_cin [G] (or -1), b_skip [S]"""
    offs, pos = [], 4
    for l in range(Lr):
        o = [pos, -1, 0]
        pos += G + 4
        if l not in no_cin:
            o[1] = pos
            pos += G + 4
        o[2] = pos
        pos += S + 4
        offs += o
    return offs, pos


@pytest.mark.parametrize("Lr,G,S", [(1, 256, 256), (3, 512, 256), (1, 128, 256), (24, 512, 256)])
def test_derived_bias(Lr, G, S):
    gen = torch.Generator().manual_seed(Lr * G + S)
    offs, n = offs_table(Lr, G, S, no_cin=(1,))
    params = nan_buf((n,))
    for l in range(Lr):
        for k, w in ((0, G), (1, G), (2, S)):
            if offs[3 * l + k] >= 0:
                params[offs[3 * l + k]:offs[3 * l + k] + w] = torch.randn(w, generator=gen).to(DEV)
    scales = (torch.rand(Lr, generator=gen) + 0.5).to(DEV)
    d_offs = torch.tensor(offs, dtype=torch.int64, device=DEV)
    bias_g, bias_s = nan_buf((Lr * G + 40,)), nan_buf((S + 40,))
    launch("DERIVED_BIAS", [params, bias_g, bias_s, d_offs, scales], [Lr, G, S])
    P = params.to(F64)
    ref_g = torch.stack([P[offs[3 * l]:offs[3 * l] + G] + (P[offs[3 * l + 1]:offs[3 * l + 1] + G] if offs[3 * l + 1] >= 0 else 0)
                         for l in range(Lr)]).reshape(-1)
    terms = torch.stack([scales[l].double() * P[offs[3 * l + 2]:offs[3 * l + 2] + S] for l in range(Lr)])
    tag = "derived_bias_L%d_G%d_S%d" % (Lr, G, S)
    check(tag + "_gate", bias_g[:Lr * G], ref_g, U * ref_g.abs())
    check(tag + "_skip", bias_s[:S], terms.sum(0), 2 * Lr * U * terms.abs().sum(0))
    all_nan(tag + "_pad", torch.cat([bias_g[Lr * G:], bias_s[S:]]))


def fx_ints(shape, gen, scale=1.0):
    return torch.round(torch.randn(shape, generator=gen, dtype=F64) * scale / FX).to(torch.int64)


@pytest.mark.parametrize("Lr,S", [(1, 256), (24, 256), (30, 128)])
def test_skip_bias(Lr, S):
    gen = torch.Generator().manual_seed(Lr + S)
    skipsum = fx_ints((S,), gen, 3.0)
    skipsum[7] = POISON
    skipsum[8] = 1 << 62            # out of range
    skipsum[9] = 0
    skipsum = skipsum.to(DEV)
    offs, n = offs_table(Lr, 4, S)
    grads = nan_buf((n,))
    scales = (torch.rand(Lr, generator=gen) + 0.5).to(DEV)
    launch("SKIP_BIAS", [skipsum, grads, torch.tensor(offs, dtype=torch.int64, device=DEV), scales], [Lr, S])
    val = fx_value(skipsum)
    written = torch.zeros(n, dtype=torch.bool, device=DEV)
    tag = "skip_bias_L%d_S%d" % (Lr, S)
    for l in range(Lr):
        o = offs[3 * l + 2]
        got, ref = grads[o:o + S], scales[l].double() * val
        fin = torch.isfinite(ref)
        assert torch.isnan(got[~fin]).all() and got[9].item() == 0.0
        check(tag + "_l%d" % l, got[fin], ref[fin], 2 * U * ref[fin].abs() + 1e-300)
        written[o:o + S] = True
    all_nan(tag + "_rest", grads[~written])


def test_fx_finalize():
    gen = torch.Generator().manual_seed(9)
    n = 70001
    acc = fx_ints((n,), gen, 2.0)
    acc[::5] = 0
    acc[3] = POISON
    acc[4] = -(1 << 62)
    acc = acc.to(DEV)
    g0 = torch.randn(n, generator=gen).to(DEV)
    grads = g0.clone()
    launch("FX_FINALIZE", [acc, grads], [n])
    val = fx_value(acc)
    zero = acc == 0
    assert torch.equal(grads[zero].view(torch.int32), g0[zero].view(torch.int32)), "a zero total changed its element"
    assert torch.isnan(grads[3]) and torch.isnan(grads[4])
    ok = ~zero & torch.isfinite(val)
    ref = g0.double()[ok] + val[ok]
    check("fx_finalize", grads[ok], ref, U * (g0.double()[ok].abs() + val[ok].abs()) + U * ref.abs())


@pytest.mark.parametrize("B,T,C", [(2, 45, 80), (1, 33, 31), (3, 64, 96), (2, 7700, 80)])
def test_cl_to_chw(B, T, C):
    gen = torch.Generator().manual_seed(B + T + C)
    x = torch.randn(B, T, C, generator=gen).to(DEV)
    out = nan_buf((B * C * T + 77,))
    launch("CL_TO_CHW", [x, out], [B, T, C])
    assert torch.equal(out[:B * C * T].view(B, C, T), x.transpose(1, 2)), "transpose differs"
    all_nan("cl_to_chw_pad", out[B * C * T:])
    record("cl_to_chw_B%d_T%d_C%d" % (B, T, C), worst_err_over_bound=0.0)


# ------------------------------------------------------------------------------------------------------------------------------
# global (speaker) conditioning
# ------------------------------------------------------------------------------------------------------------------------------
class Gin:
    """a flat parameter buffer with W_gin [Gi][G] and b_gin [G] per layer (stride p_stride, NaN between) and gc_embedding [NS][Gi]"""
    def __init__(self, Lr, G, Gi, NS, gen):
        self.Lr, self.G, self.Gi, self.NS = Lr, G, Gi, NS
        self.p_k, self.p_b, self.p_stride = 8, 8 + Gi * G + 4, Gi * G + G + 16
        self.p_emb = self.p_k + Lr * self.p_stride + 4
        self.n = self.p_emb + NS * Gi + 8
        self.params = nan_buf((self.n,))
        for l in range(Lr):
            self.W(l)[:] = (torch.randn(Gi, G, generator=gen) * 0.3).to(DEV)
            self.b(l)[:] = (torch.randn(G, generator=gen) * 0.1).to(DEV)
        self.emb()[:] = torch.randn(NS, Gi, generator=gen).to(DEV)

    def W(self, l, t=None):
        t = self.params if t is None else t
        return t[self.p_k + l * self.p_stride:self.p_k + l * self.p_stride + self.Gi * self.G].view(self.Gi, self.G)

    def b(self, l, t=None):
        t = self.params if t is None else t
        return t[self.p_b + l * self.p_stride:self.p_b + l * self.p_stride + self.G]

    def emb(self, t=None):
        t = self.params if t is None else t
        return t[self.p_emb:self.p_emb + self.NS * self.Gi].view(self.NS, self.Gi)

    def offs(self):
        return [self.p_k, self.p_b, self.p_stride, self.p_emb]


@pytest.mark.parametrize("mode", ["ids", "off_flag", "no_ids"])
def test_gin_bias(mode):
    gen = torch.Generator().manual_seed(len(mode))
    Lr, B, G, Gi, NS = 3, 5, 64, 16, 6
    gp = Gin(Lr, G, Gi, NS, gen)
    bias_ld, out_l, out_b = G + 8, B * G + 16, G
    bias = (torch.randn(Lr * bias_ld, generator=gen)).to(DEV)
    ids = torch.tensor([1, 3, 1, NS, 0], dtype=torch.int32, device=DEV)     # item 3: an id outside [0, NS)
    on = torch.tensor([0 if mode == "off_flag" else 1], dtype=torch.int32, device=DEV)
    out = nan_buf((Lr * out_l + 8,))
    launch("GIN_BIAS", [gp.params, bias, on, ids if mode != "no_ids" else None, out],
           [Lr, B, G, Gi, NS, bias_ld, out_l, out_b] + gp.offs())
    written = torch.zeros_like(out, dtype=torch.bool)
    worst = 0.0
    for l in range(Lr):
        sb = bias[l * bias_ld:l * bias_ld + G].double()
        for b in range(B):
            o = l * out_l + b * out_b
            got = out[o:o + G]
            written[o:o + G] = True
            if mode != "ids":
                assert torch.equal(got, bias[l * bias_ld:l * bias_ld + G]), "no speaker term must give the shared bias exactly"
                continue
            if ids[b] >= NS:
                assert torch.isnan(got).all()
                continue
            e = gp.emb()[ids[b].item()].double()
            prod = gp.W(l).double() * e[:, None]
            s = gp.b(l).double() + prod.sum(0)
            ref = sb + s
            bound = (Gi + 2) * U * (gp.b(l).double().abs() + prod.abs().sum(0)) + U * ref.abs()
            worst = max(worst, ((got.double() - ref).abs() / bound).max().item())
    record("gin_bias_%s" % mode, worst_err_over_bound=worst)
    assert worst <= 1.0
    all_nan("gin_bias_%s_pad" % mode, out[~written])


def test_set_speakers():
    B = 37
    ids = torch.arange(B, dtype=torch.int32, device=DEV) * 3 - 4
    spk = torch.full((1 + B + 5,), -7, dtype=torch.int32, device=DEV)
    launch("SET_SPEAKERS", [spk, ids], [B])
    assert spk[0].item() == 1 and torch.equal(spk[1:1 + B], ids) and (spk[1 + B:] == -7).all()
    spk.fill_(-7)
    launch("SET_SPEAKERS", [spk, None], [B])
    assert spk[0].item() == 0 and (spk[1:] == -7).all()
    record("set_speakers", worst_err_over_bound=0.0)


def gin_grad_setup(Lr, B, G, Gi, NS, ids, on, gen, poison=False):
    gp = Gin(Lr, G, Gi, NS, gen)
    S = fx_ints((Lr, B, G), gen, 0.5)
    if poison:
        S[1, 2, 3] = POISON
        S[0, 1, 5] = 1 << 62
    spk = torch.tensor([on] + ids, dtype=torch.int32, device=DEV)
    # the bias tables index the same flat layout: b_dil / b_cin offsets, b_cin absent in layer 1
    offs = []
    base = gp.n
    for l in range(Lr):
        offs += [base, base + G + 4 if l != 1 else -1, 0]
        base += 2 * G + 12
    n = base
    return gp, S.to(DEV), spk, torch.tensor(offs, dtype=torch.int64, device=DEV), n


@pytest.mark.parametrize("on,poison", [(1, False), (1, True), (0, False)])
def test_gin_wgrad(on, poison):
    gen = torch.Generator().manual_seed(on + 2 * poison)
    Lr, B, G, Gi, NS = 3, 5, 96, 16, 6
    ids = [1, 3, 1, NS + 2, 0] if poison else [1, 3, 1, 2, 0]   # poison: an id outside [0, NS) too
    gp, S, spk, offs, n = gin_grad_setup(Lr, B, G, Gi, NS, ids, on, gen, poison)
    SENT = 12345
    gfx = torch.full((n,), SENT, dtype=torch.int64, device=DEV)
    grads = torch.full((n,), 7.0, device=DEV)
    params = torch.cat([gp.params, torch.zeros(n - gp.n, device=DEV)])
    launch("GIN_WGRAD", [params, spk, S, gfx, grads, offs], [Lr, B, G, Gi, NS] + gp.offs())
    Sc = S.cpu()
    expect = torch.full((n,), SENT, dtype=torch.int64)
    ofs = offs.cpu().tolist()
    for l in range(Lr):
        for g_ in range(G):
            tot, bad = 0, False
            for b in range(B):
                s = int(Sc[l, b, g_])
                if not (-(1 << 62) < s < (1 << 62)):
                    bad = True
                tot += s
            t = POISON if bad or not (-(1 << 62) < tot < (1 << 62)) else tot
            expect[ofs[3 * l] + g_] = t
            if ofs[3 * l + 1] >= 0:
                expect[ofs[3 * l + 1] + g_] = t
            if on:
                expect[gp.p_b + l * gp.p_stride + g_] = t
    assert torch.equal(gfx.cpu(), expect), "integer totals differ"
    tag = "gin_wgrad_on%d_poison%d" % (on, poison)
    if not on:
        assert (grads == 7.0).all(), "no speaker term: W_gin must get no gradient"
        record(tag, worst_err_over_bound=0.0)
        return
    worst = 0.0
    Sv = fx_value(S)
    for l in range(Lr):
        E = torch.stack([gp.emb()[i].double() if 0 <= i < NS else torch.full((Gi,), NAN, dtype=F64, device=DEV) for i in ids])  # [B][Gi]
        terms = E[:, :, None] * Sv[l][:, None, :]                                  # [B][Gi][G]
        ref = terms.sum(0)
        got = gp.W(l, grads).double()
        fin = torch.isfinite(ref)
        assert torch.isnan(got[~fin]).all()
        bound = (B + 2) * U * terms.abs().sum(0)
        worst = max(worst, ((got[fin] - ref[fin]).abs() / bound[fin]).nan_to_num(nan=math.inf).max().item() if fin.any() else 0.0)
    record(tag, worst_err_over_bound=worst)
    assert worst <= 1.0
    mask = torch.ones(n, dtype=torch.bool, device=DEV)
    for l in range(Lr):
        mask[gp.p_k + l * gp.p_stride:gp.p_k + l * gp.p_stride + Gi * G] = False
    assert (grads[mask] == 7.0).all(), "gin_wgrad wrote outside dW_gin"


@pytest.mark.parametrize("on", [1, 0])
def test_gin_demb(on):
    gen = torch.Generator().manual_seed(40 + on)
    Lr, B, G, Gi, NS = 4, 6, 512, 16, 7
    ids = [1, 3, 1, 1, 0, 3]             # speakers 2, 4, 5, 6 unused
    gp, S, spk, offs, n = gin_grad_setup(Lr, B, G, Gi, NS, ids, on, gen)
    params = torch.cat([gp.params, torch.zeros(n - gp.n, device=DEV)])
    gfx = torch.zeros(n, dtype=torch.int64, device=DEV)
    grads = torch.full((n,), -3.5, device=DEV)
    launch("GIN_DEMB", [params, spk, S, gfx, grads, offs], [Lr, B, G, Gi, NS] + gp.offs())
    de = gp.emb(grads)
    tag = "gin_demb_on%d" % on
    if not on:
        assert (grads == -3.5).all()
        record(tag, worst_err_over_bound=0.0)
        return
    Sv = fx_value(S)
    worst = 0.0
    for s in range(NS):
        items = [b for b in range(B) if ids[b] == s]
        if not items:
            assert torch.equal(de[s], torch.zeros_like(de[s])), "unused speaker row %d is not exactly 0" % s
            continue
        terms = torch.stack([torch.einsum("lkg,lg->k", torch.stack([gp.W(l).double() for l in range(Lr)]), Sv[:, b]) for b in items])
        absum = sum(torch.einsum("lkg,lg->k", torch.stack([gp.W(l).double().abs() for l in range(Lr)]), Sv[:, b].abs()) for b in items)
        ref = terms.sum(0)
        bound = (Lr * G / 256 + B + 10) * U * absum
        worst = max(worst, ((de[s].double() - ref).abs() / bound).max().item())
    record(tag, worst_err_over_bound=worst)
    assert worst <= 1.0
    mask = torch.ones(n, dtype=torch.bool, device=DEV)
    mask[gp.p_emb:gp.p_emb + NS * Gi] = False
    assert (grads[mask] == -3.5).all(), "gin_demb wrote outside the embedding gradient"
