"""The fp32-class mode (t2_taco_config_t.split_bf16) one launch at a time: the split-operand GEMM contractions, their epilogues, the
split attention step and the split row writers of the Tacotron engine (tacotron-2_b200/csrc/t2_tacotron.cu, t2_gemm.cu / .cuh), through
t2_dbg_taco_kernel (CONV_GEMM, LSTM_STEP, ATT_FWD with its split flag, ROWS), against float64 references computed from the exact
values hi + lo of every split input.

A split operand carries v as hi = bf16(v), lo = bf16(v - hi), so |lo| <= 2^-8 |hi|, and every contraction adds hi.hi + lo.hi + hi.lo
in fp32. The dropped lo.lo product is <= 2^-16 |a| |w| per term; losing hi.lo or lo.hi costs up to 2^-8 of it. Per-element bounds
(u = 2^-24, |A|.|W| the same contraction on absolute values):
  contraction            (2^-16 + 2^-26 K) |A|.|W| + 2^-23 |ref| + 1e-7 over K = 3 Cp per tap: the lo.lo term, then the fp32
                         accumulator of the tensor cores, which rounds toward zero once per 16-wide k-step (K / 16 roundings of up
                         to 2^-23, all of one sign for the coherent inputs below; the bound takes twice that), one rounding for the
                         bias add
  split storage          hi + lo of an fp32 value v is within 2^-17 |v| of it; the bound takes 2^-16 |v|. A written pair is also
                         checked bit for bit: hi == bf16_rn(v), lo == bf16_rn(v - hi) for the fp32 v the same launch stores
  tanh / sigmoid         tanhf_ / sigmoidf_ (ex2.approx + rcp.approx): 4e-7 absolute, then first-order propagation through the cell
  query (attention)      2 (2 D / 32 + 8) u |h|.(|Wq_hi| + |Wq_lo|): two products per K element per lane, then 5 shuffle levels
  location term          3xTF32 (big = tf32(x), small = tf32(x - big); small.big + big.small + big.big): the dropped small.small and
                         the remainders are <= 4 * 2^-22 of |cum| |U| per product, and 3 (KA + 1) products accumulate in fp32:
                         (2^-20 + 6 (KA + 1) u) P with P = sum_k |cum| |U| + |u0|, from the UNROUNDED cum and U. A single TF32
                         product rounds each operand by up to 2^-11, 2^5 above that budget.
  energies / alignments  as tests/test_taco_kernels_gpu.py, with the two terms above in place of the bf16-mode ones; the context has
                         no bf16 term (its pair is checked with the split-storage bound)
The inputs of the contraction cases have coherent signs and lo halves near 2^-8 |hi|, so that removing any one of the three products
moves the worst ratio far above 10 (a lost product adds ~2^-9 |A|.|W|, more than 20 times the bound at every K here). Every check records its worst err / bound
through parity_util.record. Outputs start as NaN; padding and rows past a length must still be NaN (or exactly 0 where a kernel writes
it), the stashes the split mode skips must stay NaN, and NaN in unread input channels shows they are not read."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import mask_hash as mh
from parity_util import record
from t2_import import t2

pytestmark = pytest.mark.gpu
L = t2.lib
DEV = "cuda"
F64 = torch.float64
NAN = float("nan")
U = 2.0 ** -24
TAN_ERR = 4e-7


def split_acc(K):
    """relative contraction bound of a split GEMM over K packed columns (3 per K element of the operands)"""
    return 2.0 ** -16 + 2.0 ** -26 * K
TACO = dict(ATT_FWD=1, CONV_GEMM=8, LSTM_STEP=9, ROWS=10)


# ------------------------------------------------------------------------------------------------------------------------------
# plumbing
# ------------------------------------------------------------------------------------------------------------------------------
def launch(kernel, p=(), i=(), f=(), seed=0, step=None, sync=True):
    lib = L.load()
    c = L.DbgKernel()
    c.kernel = TACO[kernel]
    for k, v in enumerate(p):
        c.p[k] = None if v is None else v.data_ptr()
    for k, v in enumerate(i):
        c.i[k] = int(v)
    for k, v in enumerate(f):
        c.f[k] = float(v)
    c.seed = seed
    c.step = None if step is None else step.data_ptr()
    L.check(lib.t2_dbg_taco_kernel(ctypes.byref(c), L.stream_ptr()))
    if sync:
        torch.cuda.synchronize()


def check(name, got, ref, bound, **info):
    err = (got.to(F64) - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=float("inf")).max().item() if err.numel() else 0.0
    record(name, worst_err_over_bound=ratio, **info)
    assert ratio <= 1.0, "%s: worst err / bound %.3g" % (name, ratio)


def all_nan(name, t):
    assert t.numel() == 0 or torch.isnan(t.float()).all().item(), "%s: written outside its bounds" % name


def nan_buf(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


def split(v):
    """(hi, lo) of an fp32 tensor: hi = bf16_rn(v), lo = bf16_rn(v - hi)"""
    v = v.float()
    hi = v.bfloat16()
    return hi, (v - hi.float()).bfloat16()


def pair(hi, lo):
    return hi.to(F64) + lo.to(F64)


def assert_split_exact(name, hi, lo, v):
    """hi == bf16_rn(v) and lo == bf16_rn(v - hi), bit for bit, for the fp32 values v"""
    eh, el = split(v)
    assert torch.equal(hi.view(torch.int16), eh.view(torch.int16)), name + ": hi is not bf16_rn(v)"
    assert torch.equal(lo.view(torch.int16), el.view(torch.int16)), name + ": lo is not bf16_rn(v - hi)"


def near_max_lo(shape, gen, scale=1.0, signed=False):
    """exact split pairs whose lo halves sit near their largest size: hi a random bf16, lo = 0.45..0.49 of hi's ulp with hi's sign
    (coherent signs when not signed: every value positive)"""
    hi = (torch.rand(shape, generator=gen) * 0.9 + 0.1) * scale
    if signed:
        hi = hi * torch.where(torch.rand(shape, generator=gen) < 0.5, -1.0, 1.0)
    hi = hi.bfloat16()
    ulp = torch.exp2(torch.floor(torch.log2(hi.float().abs())) - 7)
    lo = (hi.float().sign() * ulp * (0.45 + 0.04 * torch.rand(shape, generator=gen))).bfloat16()
    return hi, lo


def seed_offset(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# a. split conv / projection GEMMs through launch_bias_act(.split = 1)
# ------------------------------------------------------------------------------------------------------------------------------
def conv_inputs(B, T, C, N, ntaps, gen, signed=False):
    """activation rows [hi(Cp) | lo(Cp)] (zero channels C..Cp-1 in both halves, as f32_to_bf16_kernel<true> writes them) and packed
    weights [N][ntaps * 3 Cp] = [W_hi | W_hi | W_lo] per tap; returns the device buffers and the exact float64 operands"""
    Cp = (C + 63) // 64 * 64
    xh, xl = near_max_lo((B, T, C), gen, signed=signed)
    wh, wl = near_max_lo((N, ntaps, C), gen, scale=1.0 / (ntaps * C), signed=signed)
    a = torch.zeros(B, T, 2 * Cp, dtype=torch.bfloat16)
    a[..., :C], a[..., Cp:Cp + C] = xh, xl
    w = torch.zeros(N, ntaps, 3, Cp, dtype=torch.bfloat16)
    w[:, :, 0, :C], w[:, :, 1, :C], w[:, :, 2, :C] = wh, wh, wl
    return a.to(DEV), w.reshape(N, ntaps * 3 * Cp).contiguous().to(DEV), pair(xh, xl).to(DEV), pair(wh, wl).to(DEV)


def conv_ref(x, W, ntaps):
    """float64 'same' conv: out[b, t, n] = sum_j sum_c x[b, t + shift_j, c] W[n, j, c], shift_j = j - (ntaps - 1) // 2 (rows outside
    [0, T) of an item are zero); and the same contraction on |.|"""
    B, T, C = x.shape
    D = torch.zeros(B, T, W.shape[0], dtype=F64, device=DEV)
    Da = torch.zeros_like(D)
    for j in range(ntaps):
        sh = j - (ntaps - 1) // 2
        xs = torch.zeros_like(x)
        lo, hi = max(0, -sh), min(T, T - sh)
        if hi > lo:
            xs[:, lo:hi] = x[:, lo + sh:hi + sh]
        D += xs @ W[:, j].t()
        Da += xs.abs() @ W[:, j].abs().t()
    return D, Da


def act_ref(v, act):
    return v.relu() if act == 1 else torch.tanh(v) if act == 2 else v


CONV_CASES = [  # B, T, C, N, ntaps, BN, act, nvalid, ldo, outs ("b" split bf16 rows, "f" fp32, "bf" both), signed
    (2, 200, 80, 256, 1, 128, 1, 256, 256, "bf", False),      # C = 80: the zero channels 80..127 of hi and lo lie inside K
    (3, 77, 512, 512, 3, 256, 0, 512, 512, "bf", False),      # the encoder conv blocks
    (2, 131, 256, 256, 5, 128, 2, 256, 256, "b", True),
    (1, 33, 128, 128, 8, 128, 1, 128, 128, "bf", False),      # 16 segments: exactly kMaxSeg, as the CBHG bank
    (4, 129, 512, 81, 1, 128, 0, 81, 128, "f", False),        # the frame / stop projection: nvalid 81, ldo 128, fp32
    (2, 65, 256, 1024, 1, 256, 2, 1024, 1024, "bf", True),
    (1, 300, 80, 128, 3, 256, 0, 128, 128, "bf", False),
]


@pytest.mark.parametrize("B,T,C,N,ntaps,BN,act,nvalid,ldo,outs,signed", CONV_CASES)
def test_conv_gemm_split(B, T, C, N, ntaps, BN, act, nvalid, ldo, outs, signed):
    g = torch.Generator().manual_seed(B * 1000 + T + C + ntaps)
    Cp = (C + 63) // 64 * 64
    a, w, x, W = conv_inputs(B, T, C, N, ntaps, g, signed)
    bias = (torch.rand(N, generator=g) * 0.2 - 0.1).to(DEV)
    rows, slack = B * T, 3
    ob = nan_buf((rows + slack, 2 * ldo), torch.bfloat16) if "b" in outs else None
    of = nan_buf((rows + slack, ldo), torch.float32) if "f" in outs else None
    launch("CONV_GEMM", [a, w, bias, ob, of], [C, T, B, N, ntaps * 3 * Cp, ntaps, BN, act, ldo, nvalid, 0, 1, 0])
    D, Da = conv_ref(x, W[:nvalid], ntaps)
    pre = D + bias[:nvalid].to(F64)
    v = act_ref(pre, act).reshape(rows, nvalid)
    bound = (split_acc(3 * ntaps * Cp) * Da.reshape(rows, nvalid) + 2.0 ** -23 * v.abs() + 1e-7 + (TAN_ERR if act == 2 else 0))
    name = "conv_split_B%d_T%d_C%d_N%d_taps%d_BN%d_act%d_n%d_%s" % (B, T, C, N, ntaps, BN, act, nvalid, outs)
    if of is not None:
        check(name + "_f32", of[:rows, :nvalid], v, bound)
        all_nan(name + " f32 padding", of[:rows, nvalid:])
        all_nan(name + " f32 tail", of[rows:])
    if ob is not None:
        check(name + "_pair", pair(ob[:rows, :nvalid], ob[:rows, ldo:ldo + nvalid]), v, bound + 2.0 ** -16 * v.abs())
        if of is not None:
            assert_split_exact(name, ob[:rows, :nvalid], ob[:rows, ldo:ldo + nvalid], of[:rows, :nvalid])
        all_nan(name + " bf16 tail", ob[rows:])


# ------------------------------------------------------------------------------------------------------------------------------
# b. split EPI_BIAS_ACT with dropout: the bf16 path's mask, hash_row0
# ------------------------------------------------------------------------------------------------------------------------------
def dropout_launch(a, w, bias, C, T, Bn, N, ldo, pdrop, stream, seed, step, split_mode, row0, out_b=None, out_f=None):
    Cp = (C + 63) // 64 * 64
    launch("CONV_GEMM", [a, w, bias, out_b, out_f], [C, T, Bn, N, (3 if split_mode else 1) * Cp, 1, 128 if N % 256 else 256, 0, ldo, N,
                                                     stream, int(split_mode), row0], [pdrop], seed=seed, step=step)


DROP_CASES = [(80, 128, 3, 7, 0.5, False), (256, 256, 2, 33, 0.5, True), (256, 128, 32, 4, 0.1, True)]


@pytest.mark.parametrize("C,N,B,T,pdrop,use_off", DROP_CASES)
def test_split_bias_act_dropout_mask(C, N, B, T, pdrop, use_off):
    """The decoder prenet in time-major rows (T_out * B rows of one item): the split launch keeps exactly the elements the host hash
    keeps at index (hash_row0 + pos) * ldo + col (not at the split pitch 2 ldo), the same mask as the bf16-mode launch; one launch
    over T * B rows equals T launches over B rows with hash_row0 = t * B bit for bit, in both modes"""
    g = torch.Generator().manual_seed(C + N + B + T)
    Cp = (C + 63) // 64 * 64
    rows, ldo, stream, seed, off = T * B, N, 11, 4242, 77
    step = seed_offset(off) if use_off else None
    a, w, x, W = conv_inputs(1, rows, C, N, 1, g, signed=True)
    bias = (torch.rand(N, generator=g) * 0.2 - 0.1).to(DEV)
    # bf16-mode operands: the hi halves
    ab = a[..., :C].contiguous()
    wb = w.view(N, 3, Cp)[:, 0].contiguous()
    hs = mh.hash_seed(seed + (off if use_off else 0), stream)
    idx = np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(ldo) + np.arange(N, dtype=np.uint64)[None, :]
    keep = torch.from_numpy(mh.hash_uniform32(hs, idx) >= np.float32(pdrop)).to(DEV)
    kinv = float(np.float32(1) / (np.float32(1) - np.float32(pdrop)))
    name = "split_dropout_C%d_N%d_B%d_T%d_p%g_off%d" % (C, N, B, T, pdrop, use_off)
    outs = {}
    for sm in (True, False):
        full_b = nan_buf((rows, (2 if sm else 1) * ldo), torch.bfloat16)
        full_f = nan_buf((rows, ldo), torch.float32)
        if sm:
            dropout_launch(a, w, bias, C, rows, 1, N, ldo, pdrop, stream, seed, step, True, 0, full_b, full_f)
        else:
            dropout_launch(ab, wb, bias, C, rows, 1, N, ldo, pdrop, stream, seed, step, False, 0, full_b, full_f)
        step_b = nan_buf((rows, (2 if sm else 1) * ldo), torch.bfloat16)
        step_f = nan_buf((rows, ldo), torch.float32)
        for t in range(T):
            r = slice(t * B, (t + 1) * B)
            src = a[:, r] if sm else ab[:, r]
            dropout_launch(src, w if sm else wb, bias, C, B, 1, N, ldo, pdrop, stream, seed, step, sm, t * B, step_b[r], step_f[r])
        assert torch.equal(step_f, full_f) and torch.equal(step_b, full_b), \
            "%s: T launches with hash_row0 = t B differ from one launch (split %d)" % (name, sm)
        dropped = full_f == 0
        assert torch.equal(dropped, ~keep), "%s: the kept mask is not the host hash at (row0 + pos) ldo + col (split %d)" % (name, sm)
        outs[sm] = full_f
    D, Da = conv_ref(x, W, 1)
    v = (D[0] + bias.to(F64))
    v = torch.where(keep, v * kinv, torch.zeros_like(v))
    check(name + "_f32", outs[True], v, (split_acc(3 * Cp) * Da[0] + 2.0 ** -23 * v.abs() + 1e-7) * kinv)


# ------------------------------------------------------------------------------------------------------------------------------
# c. the split swapped LSTM step through lstm_step
# ------------------------------------------------------------------------------------------------------------------------------
def lstm_case(H, K, B, training, out_state, gen):
    # recurrent weights with coherent signs and near-maximal lo halves; rows permuted as the packing does (tile row p: gate p / 32,
    # unit 32 m_tile + p % 32)
    wh, wl = near_max_lo((4, H, K), gen, scale=2.0 / K)
    sh, sl = near_max_lo((B, K), gen)
    Wx = pair(wh, wl)                                                       # [4, H, K]
    perm = torch.tensor([(r % 128) // 32 * H + (r // 128) * 32 + r % 32 for r in range(4 * H)])
    wflat_h, wflat_l = wh.reshape(4 * H, K)[perm], wl.reshape(4 * H, K)[perm]
    wrec = torch.cat([wflat_h, wflat_h, wflat_l], 1).contiguous()          # [4H][W_hi | W_hi | W_lo]
    state = torch.cat([sh, sl, sh], 1).contiguous()                         # [B][hi | lo | hi]
    x = pair(sh, sl)
    kern = Wx.permute(2, 0, 1).reshape(K, 4 * H)                            # [K, 4H], column g H + u
    # pre cancels the (positive) contraction to O(1) pre-activations, so that the gates are far from saturation
    zc = x @ kern
    pre = (-zc + torch.randn(B, 4 * H, generator=gen, dtype=F64)).float()
    return wrec.to(DEV), state.to(DEV), x.to(DEV), kern.to(DEV), pre.to(DEV)


LSTM_CASES = [  # H, K, B, training, out_state
    (64, 64, 1, True, 0),
    (256, 256, 32, True, 1),        # encoder: K = H
    (256, 256, 33, False, 0),
    (1024, 1536, 33, True, 1),      # decoder cell 1 at the Cfg-3 widths: K = 2 H_enc + D
    (1024, 2048, 32, False, 0),     # decoder cell 2: K = 2 D
    (1024, 2048, 1, True, 1),
]


@pytest.mark.parametrize("H,K,B,training,out_state", LSTM_CASES)
def test_lstm_step_split(H, K, B, training, out_state):
    from oracle import tacotron as ot
    g = torch.Generator().manual_seed(H + K + B)
    wrec, state, x, kern, pre = lstm_case(H, K, B, training, out_state, g)
    ps = 4 * H + 8
    pre_b = torch.full((B, ps), NAN, device=DEV)
    pre_b[:, :4 * H] = pre
    bias = (torch.randn(4 * H, generator=g) * 0.5).to(DEV)
    c_prev = torch.randn(B, H, generator=g).to(DEV)
    hph, hpl = split(torch.randn(B, H, generator=g) * 0.5)
    ld_hp = 3 * K
    h_prev = nan_buf((B, ld_hp), torch.bfloat16)
    h_prev[:, :H], h_prev[:, K:K + H], h_prev[:, 2 * K:2 * K + H] = hph.to(DEV), hpl.to(DEV), hph.to(DEV)
    ld_hs, out_lo = 3 * K + 8, H + 64
    ld_ho = (3 if out_state else 2) * out_lo
    t, stream, z, seed, off = 5, 27, 0.1, 2024, 9
    lens = torch.tensor([(7 if b % 3 else 3) for b in range(B)], dtype=torch.int32, device=DEV)     # items 0, 3, ... have ended
    c_out = nan_buf((B + 1, H), torch.float32)
    h_state = nan_buf((B + 1, ld_hs), torch.bfloat16)
    h_out = nan_buf((B + 1, ld_ho), torch.bfloat16)
    gst, tst = nan_buf((B + 1, 4 * H), torch.bfloat16), nan_buf((B + 1, H), torch.bfloat16)
    launch("LSTM_STEP", [wrec, state, pre_b, bias, c_prev, c_out, h_prev, h_state, h_out, gst, tst, lens],
           [H, K, B, ps, ld_hp, ld_hs, ld_ho, t, stream, out_lo, out_state, int(training), 1], [z], seed=seed, step=seed_offset(off))
    zz = x @ kern + pre.to(F64) + bias.to(F64)
    dz = split_acc(3 * K) * (x.abs() @ kern.abs()) + 4 * U * (zz.abs() + pre.abs().to(F64) + bias.abs().to(F64)) + 1e-7
    cp, hp = c_prev.to(F64), pair(hph, hpl).to(DEV)
    cn, hn = ot.lstm_cell(x, cp, torch.zeros(B, 0, dtype=F64, device=DEV), kern, pre.to(F64) + bias.to(F64))
    gi, gj = torch.sigmoid(zz[:, :H]), torch.tanh(zz[:, H:2 * H])
    gf, go = torch.sigmoid(zz[:, 2 * H:3 * H] + 1), torch.sigmoid(zz[:, 3 * H:])
    dgi, dgj = gi * (1 - gi) * dz[:, :H] + TAN_ERR, (1 - gj * gj) * dz[:, H:2 * H] + TAN_ERR
    dgf, dgo = gf * (1 - gf) * dz[:, 2 * H:3 * H] + TAN_ERR, go * (1 - go) * dz[:, 3 * H:] + TAN_ERR
    dcn = cp.abs() * dgf + gj.abs() * dgi + gi * dgj + 4 * U * (gf * cp.abs() + (gi * gj).abs())
    tc = torch.tanh(cn)
    dhn = tc.abs() * dgo + go * ((1 - tc * tc) * dcn + TAN_ERR) + 2 * U * hn.abs()
    if training:
        idx = (np.uint64(t) * np.uint64(B) + np.arange(B, dtype=np.uint64)[:, None]) * np.uint64(H) + np.arange(H, dtype=np.uint64)[None, :]
        mc = torch.from_numpy(mh.hash_uniform32(mh.hash_seed(seed + off, stream * 2), idx) >= np.float32(z)).to(DEV).to(F64)
        mhm = torch.from_numpy(mh.hash_uniform32(mh.hash_seed(seed + off, stream * 2 + 1), idx) >= np.float32(z)).to(DEV).to(F64)
        cs, hs = ot.zoneout(cp, cn, z, True, mc), ot.zoneout(hp, hn, z, True, mhm)
        dcs, dhs = dcn * mc, dhn * mhm
    else:
        cs, hs = ot.zoneout(cp, cn, z, False), ot.zoneout(hp, hn, z, False)
        dcs, dhs = (1 - z) * dcn + 4 * U * (cs.abs() + cp.abs()), (1 - z) * dhn + 4 * U * (hs.abs() + hp.abs())
    live = (t < lens)[:, None]
    name = "lstm_split_H%d_K%d_B%d_train%d_os%d" % (H, K, B, training, out_state)
    check(name + "_c", c_out[:B], torch.where(live, cs, cp), torch.where(live, dcs, torch.zeros_like(dcs)) + 1e-30)
    hs_ref = torch.where(live, hs, hp)
    check(name + "_hstate", pair(h_state[:B, :H], h_state[:B, K:K + H]), hs_ref,
          torch.where(live, dhs, torch.zeros_like(dhs)) + 2.0 ** -16 * hs_ref.abs() + 1e-30)
    ho_ref = torch.where(live, hn, torch.zeros_like(hn))
    check(name + "_hout", pair(h_out[:B, :H], h_out[:B, out_lo:out_lo + H]), ho_ref,
          torch.where(live, dhn, torch.zeros_like(dhn)) + 2.0 ** -16 * ho_ref.abs() + 1e-30)
    # ended items: c and h_state carried unchanged (the same pair), h_out exactly 0 in every half
    # (the carried pair is re-split from the fp32 value hi + lo, which is exact: the same value, the canonical pair of it)
    dead = ~live[:, 0]
    assert torch.equal(c_out[:B][dead], c_prev[dead])
    assert_split_exact(name + " carried h_state", h_state[:B, :H][dead], h_state[:B, K:K + H][dead], (hph.float() + hpl.float()).to(DEV)[dead])
    halves = [h_out[:B, :H], h_out[:B, out_lo:out_lo + H]] + ([h_out[:B, 2 * out_lo:2 * out_lo + H]] if out_state else [])
    assert all(bool((hh[dead] == 0).all()) for hh in halves), "h_out of an ended item must be exactly 0"
    # state rows: the second hi copy is the first, bit for bit; h_out gets one only as a state row (out_state)
    assert torch.equal(h_state[:B, 2 * K:2 * K + H].view(torch.int16), h_state[:B, :H].view(torch.int16))
    if out_state:
        assert torch.equal(h_out[:B, 2 * out_lo:2 * out_lo + H].view(torch.int16), h_out[:B, :H].view(torch.int16))
        all_nan(name + " h_out padding", torch.cat([h_out[:, out_lo + H:2 * out_lo].flatten(), h_out[:, 2 * out_lo + H:].flatten()]))
    else:
        all_nan(name + " h_out past the pair", h_out[:, out_lo + H:])
    all_nan(name + " stashes (split mode writes none)", torch.cat([gst.flatten(), tst.flatten()]))
    all_nan(name + " padding", torch.cat([c_out[B:].flatten(), h_state[:, H:K].flatten(), h_state[:, K + H:2 * K].flatten(),
                                           h_state[:, 2 * K + H:].flatten(), h_state[B:].flatten(), h_out[B:].flatten(), h_out[:, H:out_lo].flatten()]))


# ------------------------------------------------------------------------------------------------------------------------------
# d. att_fwd_kernel<*, *, true>
# ------------------------------------------------------------------------------------------------------------------------------
def tf32_far(x, gen):
    """fp32 values whose TF32 rounding error is near its largest and of one sign: tf32(x) + 0.45..0.49 of its ulp"""
    b = x.float().contiguous().view(torch.int32) & ~0x1FFF
    base = b.view(torch.float32)
    ulp = torch.exp2(torch.floor(torch.log2(base.abs())) - 10)
    return (base + base.sign() * ulp * (0.45 + 0.04 * torch.rand(x.shape, generator=gen))).float()


def att_split_reference(h, Wq, Ub, KA, v, keys, vals, lens, cum, masked, D):
    """float64 alignments / context of one split step (h, Wq exact hi + lo; Ub the kernel's fp32 filter bank, UNROUNDED; cum fp32)"""
    N, Ti, A = keys.shape
    half = KA // 2
    ev = torch.arange(Ti, device=DEV)[None, :] < (lens[:, None] if masked else torch.full_like(lens, Ti)[:, None])
    q, qabs = h @ Wq.t(), h.abs() @ Wq.abs().t()
    Ud = Ub.to(F64)
    win = Fn.pad(cum.to(F64), (half, half)).unfold(1, KA, 1)
    pl = win @ Ud[:KA] + Ud[KA]
    P = win.abs() @ Ud[:KA].abs() + Ud[KA].abs()
    ky = torch.where(ev[..., None], keys.to(F64), torch.zeros((), dtype=F64, device=DEV))
    arg = ky + q[:, None, :] + pl
    d_arg = (2.0 ** -20 + 6 * (KA + 1) * U) * P + 2 * (2 * D / 32 + 8) * U * qabs[:, None, :] + 2 * U * arg.abs()
    t = torch.tanh(arg)
    v64 = v.to(F64)
    e = t @ v64
    d_e = ((1 - t * t) * d_arg) @ v64.abs() + TAN_ERR * v64.abs().sum() + 2 * (18 + A / 64) * U * (t.abs() @ v64.abs())
    e = torch.where(ev, e, torch.full_like(e, -math.inf))
    alpha = torch.softmax(e, dim=1)
    emax = torch.where(ev, d_e, torch.zeros_like(d_e)).amax(1, keepdim=True)
    rng = e.amax(1, keepdim=True) - torch.where(ev, e, torch.full_like(e, math.inf)).amin(1, keepdim=True)
    d_alpha = alpha * (2 * emax + 2.0 ** -20 * (1 + rng) + 2 * Ti * U + 4 * U)
    live = torch.arange(Ti, device=DEV)[None, :] < lens[:, None]
    vv = torch.where(live[..., None], vals, torch.zeros((), dtype=F64, device=DEV))
    ctx = torch.einsum("nj,njc->nc", alpha, vv)
    d_ctx = 1.01 * (torch.einsum("nj,njc->nc", d_alpha, vv.abs()) + 4 * Ti * U * torch.einsum("nj,njc->nc", alpha, vv.abs()))
    return alpha, d_alpha, ctx, d_ctx, ev


ATT_CASES = [  # B, Ti, A, KA, F, D, C2  (the shapes of tests/test_taco_kernels_gpu.py::ATT_CASES that the split mode runs)
    (3, 1, 128, 31, 32, 1024, 512), (4, 17, 128, 31, 32, 1024, 512), (32, 160, 128, 31, 32, 1024, 512), (3, 336, 128, 31, 32, 1024, 512),
    (3, 17, 64, 31, 32, 256, 256), (4, 160, 128, 31, 32, 1024, 1024), (1, 160, 64, 1, 1, 256, 256),
]
FLAGS = [(0, 0), (0, 1), (1, 0), (1, 1)]


@pytest.mark.parametrize("unmasked,noncum", FLAGS)
@pytest.mark.parametrize("B,Ti,A,KA,F,D,C2", ATT_CASES)
def test_att_fwd_split(B, Ti, A, KA, F, D, C2, unmasked, noncum):
    g = torch.Generator().manual_seed(B * 1000 + Ti + C2 + KA + 10 * unmasked + 20 * noncum)
    lens = torch.tensor([min(o, Ti) for o in [[1, 16 * (Ti // 32) + 1, max(Ti - 1, 1), Ti][b % 4] for b in range(B)]], dtype=torch.int32)
    lo_h2, lo_a, lo_b = D + 16, C2 + 8, C2 + 24
    ld_h2, ld_a, ld_b = lo_h2 + D + 8, 2 * lo_a + C2 + 8, lo_b + C2 + 8
    hh, hl = near_max_lo((B, D), g)
    h2 = torch.full((B, ld_h2), NAN).bfloat16()
    h2[:, :D], h2[:, lo_h2:lo_h2 + D] = hh, hl
    wh, wl = near_max_lo((A, D), g, scale=2.0 / D)
    WqT = torch.cat([wh, wl], 1).contiguous()
    # query source, query weights and values with coherent signs and near-maximal lo halves; a location branch with coherent signs (U >= 0) over a cum whose TF32 roundings are near-maximal and of one sign, and an attention
    # bias that brings the energies back to O(1)
    K = torch.rand(KA, F, generator=g) * 0.5
    bK = torch.rand(F, generator=g) * 0.1
    Wl = torch.rand(F, A, generator=g) / F
    cum = tf32_far(0.05 + torch.rand(B, Ti, generator=g) * 1.5, g)
    Uh = K.double() @ Wl.double()
    ba = (-(Uh.sum(0) * 0.8 + bK.double() @ Wl.double()) + torch.randn(A, generator=g, dtype=F64) * 0.1).float()
    v = torch.rand(A, generator=g) / math.sqrt(A) * 2
    keys = torch.randn(B, Ti, A, generator=g) * 0.5
    vh, vl = near_max_lo((B, Ti, C2), g)
    values = torch.cat([vh, vl], 2).contiguous()
    for b in range(B):
        keys[b, lens[b]:] = 0 if unmasked else NAN
        values[b, lens[b]:] = 0 if unmasked else NAN
    h2, WqT, K, bK, Wl, ba, v, keys, values, lens, cum = [x.to(DEV) for x in (h2, WqT, K, bK, Wl, ba, v, keys, values, lens, cum)]
    Ub = nan_buf(((KA + 1) * A,), torch.float32)
    cum_in = cum.clone()
    alpha = nan_buf((B, Ti), torch.float32)
    ctx_a, ctx_b = nan_buf((B, ld_a), torch.bfloat16), nan_buf((B, ld_b), torch.bfloat16)
    launch("ATT_FWD", [h2, WqT, K, bK, Wl, ba, Ub, v, keys, values, lens, cum, alpha, ctx_a, ctx_b],
           [B, Ti, D, A, KA, F, C2, ld_h2, ld_a, ld_b, unmasked, noncum, 1, lo_h2, lo_a, lo_b])
    tag = "att_fwd_split_um%d_nc%d_B%d_Ti%d_A%d_KA%d_D%d_C2%d" % (unmasked, noncum, B, Ti, A, KA, D, C2)
    h = pair(h2[:, :D], h2[:, lo_h2:lo_h2 + D])
    Wq = pair(WqT[:, :D], WqT[:, D:])
    vals = pair(values[..., :C2], values[..., C2:])
    ref_a, d_a, ref_c, d_c, ev = att_split_reference(h, Wq, Ub.view(KA + 1, A), KA, v, keys, vals, lens, cum_in, not unmasked, D)
    check(tag + "_alpha", torch.where(ev, alpha, torch.zeros_like(alpha)), ref_a, d_a + 1e-30)
    if not unmasked:
        assert bool((alpha[~ev] == 0).all()), "masked: alpha past len must be exactly 0"
    assert torch.equal(cum, alpha if noncum else cum_in + alpha), "the state must come back as alpha or cum + alpha"
    cb = pair(ctx_b[:, :C2], ctx_b[:, lo_b:lo_b + C2])
    check(tag + "_ctx_b", cb, ref_c, d_c + 2.0 ** -16 * ref_c.abs() + 1e-30)
    assert torch.equal(ctx_a[:, :C2].view(torch.int16), ctx_b[:, :C2].view(torch.int16))
    assert torch.equal(ctx_a[:, lo_a:lo_a + C2].view(torch.int16), ctx_b[:, lo_b:lo_b + C2].view(torch.int16))
    assert torch.equal(ctx_a[:, 2 * lo_a:2 * lo_a + C2].view(torch.int16), ctx_a[:, :C2].view(torch.int16)), "ctx_a: second hi copy"
    all_nan(tag + " ctx_a pad", torch.cat([ctx_a[:, C2:lo_a].flatten(), ctx_a[:, lo_a + C2:2 * lo_a].flatten(), ctx_a[:, 2 * lo_a + C2:].flatten()]))
    all_nan(tag + " ctx_b pad", torch.cat([ctx_b[:, C2:lo_b].flatten(), ctx_b[:, lo_b + C2:].flatten()]))


# ------------------------------------------------------------------------------------------------------------------------------
# e. the split row writers, bit for bit against the value the bf16 mode rounds
# ------------------------------------------------------------------------------------------------------------------------------
def rows(which, split_mode, p, i, f=(), seed=0, step=None):
    launch("ROWS", p, [which, split_mode] + list(i), f, seed=seed, step=step)


def test_embed_fwd_split():
    g = torch.Generator().manual_seed(1)
    NS, E, npos = 70, 512, 333
    table = (torch.randn(NS, E, generator=g) * 0.3).to(DEV)
    idx = torch.randint(0, NS, (npos,), generator=g, dtype=torch.int32).to(DEV)
    out = nan_buf((npos + 1, 2 * E), torch.bfloat16)
    ref = nan_buf((npos + 1, E), torch.bfloat16)
    rows(0, 1, [idx, table, out], [npos, E])
    rows(0, 0, [idx, table, ref], [npos, E])
    v = table[idx.long()]
    assert_split_exact("embed", out[:npos, :E], out[:npos, E:], v)
    assert torch.equal(out[:npos, :E].view(torch.int16), ref[:npos].view(torch.int16)), "hi must be what the bf16 mode writes"
    all_nan("embed tail", torch.cat([out[npos:].flatten(), ref[npos:].flatten()]))


def test_decin_split():
    g = torch.Generator().manual_seed(2)
    B, To, M = 3, 21, 80
    Cp = (M + 63) // 64 * 64
    tgt = (torch.randn(B, To, M, generator=g) * 2).to(DEV)
    out = nan_buf((To * B + 1, 2 * Cp), torch.bfloat16)
    ref = nan_buf((To * B, M), torch.bfloat16)
    rows(1, 1, [tgt, out], [B, To, M])
    rows(1, 0, [tgt, ref], [B, To, M])
    v = torch.cat([torch.zeros(1, B, M, device=DEV), tgt.transpose(0, 1)[:-1]]).reshape(To * B, M)   # row t b: target[b][t - 1]
    assert_split_exact("decin", out[:To * B, :M], out[:To * B, Cp:Cp + M], v)
    assert torch.equal(out[:To * B, :M].view(torch.int16), ref.view(torch.int16))
    # [hi(M) | pad | lo(M) | pad] at pitch 2 Cp: the padding is the engine's zero-initialised workspace and is never written
    all_nan("decin padding", torch.cat([out[:, M:Cp].flatten(), out[:, Cp + M:].flatten(), out[To * B:].flatten()]))


@pytest.mark.parametrize("clip,with_tgt", [(1, True), (0, False)])
def test_dec_finish_split(clip, with_tgt):
    g = torch.Generator().manual_seed(3 + clip)
    B, To, M = 3, 19, 80
    Cp = (M + 63) // 64 * 64
    projo = torch.full((To, B, 128), NAN)
    projo[..., :M + 1] = torch.randn(To, B, M + 1, generator=g) * 3
    projo = projo.to(DEV)
    tgt = torch.randn(B, To, M, generator=g).to(DEV) if with_tgt else None
    stop_t = (torch.rand(B, To, generator=g) < 0.2).float().to(DEV) if with_tgt else None
    lo_c, hi_c = -4.1, 4.0
    outs = {}
    for sm in (1, 0):
        dec_bm = nan_buf((B * To + 1, 2 * Cp if sm else M), torch.bfloat16)
        dec_f, stop = nan_buf((B, To, M), torch.float32), nan_buf((B, To), torch.float32)
        scal = torch.zeros(5, device=DEV)
        rows(2, sm, [projo, tgt, stop_t, dec_bm, dec_f, stop, scal, None], [B, To, M, clip], [lo_c, hi_c, 1.0])
        outs[sm] = (dec_bm, dec_f, stop, scal)
    (sb, sf, ss, sc), (bb, bf, bs, bc) = outs[1], outs[0]
    assert torch.equal(sf, bf) and torch.equal(ss, bs), "the fp32 outputs must not depend on the mode"
    assert torch.allclose(sc, bc, rtol=1e-6, atol=0), "the loss sums must not depend on the mode"
    v = projo[..., :M].transpose(0, 1).reshape(B * To, M)
    v = v.clamp(lo_c, hi_c) if clip else v
    assert torch.equal(sf.view(B * To, M), v)
    assert_split_exact("dec_finish", sb[:B * To, :M], sb[:B * To, Cp:Cp + M], v)
    assert torch.equal(sb[:B * To, :M].view(torch.int16), bb[:B * To].view(torch.int16))
    all_nan("dec_finish padding", torch.cat([sb[:, M:Cp].flatten(), sb[:, Cp + M:].flatten(), sb[B * To:].flatten()]))


@pytest.mark.parametrize("ratio", [None, 0.0, 1.0, 0.5])
def test_proj_bias_feedback_split(ratio):
    """the next decoder input row, from the predicted frame or (teacher-forcing ratio < 1) the target frame the draw picks"""
    g = torch.Generator().manual_seed(4)
    B, M, To, t, seed, off = 5, 80, 9, 3, 99, 4
    Cp = (M + 63) // 64 * 64
    p0 = torch.full((B, 128), NAN)
    p0[:, :M + 1] = torch.randn(B, M + 1, generator=g) * 2
    fb, sb = (torch.randn(M, generator=g) * 0.1).to(DEV), (torch.randn(1, generator=g)).to(DEV)
    tgt = torch.randn(B, To, M, generator=g).to(DEV) if ratio is not None else None
    res = {}
    for sm in (1, 0):
        p = p0.clone().to(DEV)
        nxt = nan_buf((B, 2 * Cp if sm else M), torch.bfloat16)
        choice = torch.full((To,), -1, dtype=torch.int32, device=DEV) if ratio is not None else None
        rows(3, sm, [p, fb, sb, nxt, tgt, choice], [B, M, To, t], [ratio or 0.0], seed=seed, step=seed_offset(off))
        res[sm] = (p, nxt, choice)
    (sp, sn, sch), (bp, bn, bch) = res[1], res[0]
    pv = p0.to(DEV)[:, :M + 1] + torch.cat([fb, sb])
    assert torch.equal(sp[:, :M + 1], pv) and torch.equal(bp[:, :M + 1], pv)
    all_nan("projection padding", sp[:, M + 1:])
    forced = False
    if ratio is not None:
        forced = bool(mh.hash_uniform32(mh.hash_seed(seed + off, 40), np.array([t], dtype=np.uint64))[0] < np.float32(ratio))
        assert int(sch[t]) == int(forced) and int(bch[t]) == int(forced)
    x = tgt[:, t] if forced else pv[:, :M]
    assert_split_exact("feedback", sn[:, :M], sn[:, Cp:Cp + M], x)
    assert torch.equal(sn[:, :M].view(torch.int16), bn.view(torch.int16))
    all_nan("feedback padding", torch.cat([sn[:, M:Cp].flatten(), sn[:, Cp + M:].flatten()]))


@pytest.mark.parametrize("C,Cp", [(80, 128), (128, 128), (1025, 1088)])
def test_f32_to_bf16_split(C, Cp):
    g = torch.Generator().manual_seed(C)
    R = 77
    x = (torch.randn(R, C, generator=g) * 3).to(DEV)
    out = nan_buf((R + 1, 2 * Cp), torch.bfloat16)
    ref = nan_buf((R * C + 1,), torch.bfloat16)
    rows(4, 1, [x, out], [R, C, Cp])
    rows(4, 0, [x, ref], [R, C, C])
    assert_split_exact("f32_to_bf16", out[:R, :C], out[:R, Cp:Cp + C], x)
    assert torch.equal(out[:R, :C].view(torch.int16), ref[:R * C].view(R, C).view(torch.int16))
    assert bool((out[:R, C:Cp] == 0).all()) and bool((out[:R, Cp + C:] == 0).all()), "channels C..Cp-1 must be exactly zero"
    all_nan("f32_to_bf16 tail", torch.cat([out[R:].flatten(), ref[R * C:]]))
