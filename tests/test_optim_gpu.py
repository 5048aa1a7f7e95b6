"""t2_adam_step (tacotron-2_b200/csrc/t2_optim.cu: sumsq_kernel, norms_kernel, adam_kernel), one call at a time against a float64
restatement of tf.train.AdamOptimizer with tf.clip_by_norm + tf.clip_by_value per tensor (WaveNet, wavenet.py:586-613, with the EMA) or
tf.clip_by_global_norm (Tacotron, tacotron.py:429-437). The reference starts from the kernel's own fp32 state (p, m, v, ema) before the
call, and the hyperparameters are the fp32 values the kernel receives, so 1 - beta and 1 - decay are exact in both. Over several steps
the reference never carries its own state forward: rounding differences cannot build up.

Bounds (u = 2^-24):
  clip factor   the kernel's squared norms are fp32 sums of positive terms: each square carries 2u (grad_scale product, square), then
                16 sequential adds per thread, a 5-level butterfly, 8 per-block adds, ceil(chunks / 32) + 5 levels over the chunk partials
                and, for the global norm, ceil(n_tensors / 32) + 5 more: depth D, relative error <= (D + 2) u. sqrt halves it; the
                division and the product with grad_scale add 2u, the product with the gradient u:  e_g = (D / 2 + 5) u relative on every
                clipped gradient (the clamp of clip_by_value is 1-Lipschitz). Where the clip is inactive the factor is exactly 1.
  m             (1 - b1) |g| e_g + 3u (b1 |m| + (1 - b1) |g|)                     (two products and one add, each rounded)
  v             (1 - b2) g^2 (2 e_g + e_g^2) + 4u (b2 v + (1 - b2) g^2)
  p             lr_t (|dm| + |m' / (sqrt v' + eps)| |d sqrt|) / (sqrt v' + eps) + 6u lr_t |m' / (sqrt v' + eps)| + 2u |p'|, with
                |d sqrt| = min(sqrt |dv|, |dv| / (2 sqrt v')) + 2u (sqrt v' + eps)   (lr_t itself is one rounding of the float64 value)
  ema           3u (1 - decay) |ema - p| + 2u |ema'|, from the kernel's own p'
Every bound is applied elementwise with a factor 2 of margin; non-finite entries must be non-finite in the same places. Each check
records its worst err / bound through parity_util.record.

Also checked: the same call on copies of the same state gives bit-identical p, m, v and ema while clips are active (the invariant that
keeps data-parallel replicas identical), and t2_launch_count() moves by the kernels actually launched: adam only without a norm clip,
sumsq + norms + adam with one."""
import ctypes
import math

import pytest
import torch

from parity_util import record
from t2_import import t2

pytestmark = pytest.mark.gpu
L = t2.lib
DEV = "cuda"
F64 = torch.float64
U = 2.0 ** -24
CHUNK = 4096


def f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------------------------
# tensor tables: lists of element counts (multiples of 4, as the engines lay them out)
# ------------------------------------------------------------------------------------------------------------------------------
def wavenet_table():
    from paper_hparams import hparams
    tensors, n = t2.wavenet.param_table(t2.wavenet.make_config(hparams, 2, 7700))
    offs = [t[1] for t in tensors] + [n]
    return [b - a for a, b in zip(offs, offs[1:])]


def tacotron_cbhg_table():
    from hparams import hparams
    hp = hparams.copy()
    hp.parse("predict_linear=True")
    T = t2.tacotron
    lib = L.load()
    cfg = T.make_config(hp, 2, 40, 80)
    n, pb, wb, nt = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    L.check(lib.t2_taco_sizes(ctypes.byref(cfg), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(nt)))
    tensors = L.param_table(lib.t2_taco_param_info, cfg, nt.value)
    cb = T.make_cbhg_config(hp, 2, 80, cfg.reg_weight)
    cn, cnt = ctypes.c_longlong(), ctypes.c_int()
    L.check(lib.t2_cbhg_sizes(ctypes.byref(cb), ctypes.byref(cn), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(cnt)))
    tensors += L.param_table(lib.t2_cbhg_param_info, cb, cnt.value, base=n.value)
    offs = [t[1] for t in tensors] + [n.value + cn.value]
    return [b - a for a, b in zip(offs, offs[1:])]


def synthetic_table(tail):
    """a tensor starting off a chunk boundary and spanning dozens of chunks, hundreds of 4-element tensors inside one chunk, empty
    tensors (first, between, and next to a chunk boundary), and a last tensor that ends `tail` elements past a multiple of 4096"""
    sizes = [0, 1000, 0, 37 * CHUNK + 1236]
    sizes += [4] * 300 + [0, 0] + [4] * 100
    sizes += [0, 4 * 513, 0]
    n = sum(sizes)
    sizes.append((-n) % CHUNK + CHUNK + tail)
    sizes.append(0)
    return sizes


TABLES = {"wavenet_paper": wavenet_table, "tacotron_cbhg": tacotron_cbhg_table,
          "synthetic_4096p4": lambda: synthetic_table(4), "synthetic_1024p4": lambda: synthetic_table(1024 + 4)}


# ------------------------------------------------------------------------------------------------------------------------------
# state, call, reference
# ------------------------------------------------------------------------------------------------------------------------------
class State:
    def __init__(self, sizes, seed, gnorms=None, ema=True):
        g = torch.Generator().manual_seed(seed)
        self.sizes = sizes
        self.offs = [0]
        for s in sizes:
            self.offs.append(self.offs[-1] + s)
        n = self.offs[-1]
        assert n % 4 == 0
        self.n = n
        self.p = (torch.randn(n, generator=g) * 0.1).to(DEV)
        self.m = (torch.randn(n, generator=g) * 1e-3).to(DEV)
        self.v = (torch.rand(n, generator=g) * 1e-5 + self.m.cpu().double().pow(2).float() * 2).to(DEV)
        self.ema = (self.p.cpu() + torch.randn(n, generator=g) * 1e-3).to(DEV) if ema else None
        grad = torch.randn(n, generator=g)
        if gnorms is not None:   # per-tensor target norms (of grad * grad_scale), None keeps the random values
            for t, target in enumerate(gnorms):
                a, b = self.offs[t], self.offs[t + 1]
                if b > a and target is not None:
                    grad[a:b] *= target / grad[a:b].double().norm().item()
        self.g = grad.to(DEV)
        self.offsets = torch.tensor(self.offs, dtype=torch.int64, device=DEV)
        self.scratch = torch.full((L.adam_scratch_floats(len(sizes), n),), float("nan"), dtype=torch.float32, device=DEV)

    def copy(self):
        c = State.__new__(State)
        c.__dict__.update(self.__dict__)
        for k in ("p", "m", "v", "g", "scratch"):
            setattr(c, k, getattr(self, k).clone())
        c.ema = None if self.ema is None else self.ema.clone()
        return c


HP = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-6, ema_decay=0.9999)


def adam_call(s, step, gscale=1.0, max_norm=0.0, max_value=0.0, gclip=0.0, lr=HP["lr"]):
    lib = L.load()
    L.check(lib.t2_adam_step(
        L.ptr(s.p), L.ptr(s.g), L.ptr(s.m), L.ptr(s.v), L.ptr(s.ema), L.ptr(s.offsets), len(s.sizes), ctypes.c_longlong(s.n),
        ctypes.c_float(lr), ctypes.c_float(HP["b1"]), ctypes.c_float(HP["b2"]), ctypes.c_float(HP["eps"]), step, ctypes.c_float(gscale),
        ctypes.c_float(max_norm), ctypes.c_float(max_value), ctypes.c_float(gclip), ctypes.c_float(HP["ema_decay"]), L.ptr(s.scratch),
        L.stream_ptr()))
    torch.cuda.synchronize()


def nan_max(x, c):
    return torch.where(torch.isnan(x), x, torch.clamp(x, min=c))


def reference(s, step, gscale=1.0, max_norm=0.0, max_value=0.0, gclip=0.0, lr=HP["lr"]):
    """float64 step from the fp32 state in s; returns (dict of references, dict of bounds)"""
    b1, b2, eps, dec = (f32(HP[k]) for k in ("b1", "b2", "eps", "ema_decay"))
    lr = f32(lr)
    gs = f32(gscale)
    lr_t = lr * math.sqrt(1 - b2 ** step) / (1 - b1 ** step)
    g = s.g.to(F64) * gs
    p, m, v = s.p.to(F64), s.m.to(F64), s.v.to(F64)
    nt = len(s.sizes)
    nch = (s.n + CHUNK - 1) // CHUNK
    depth = 16 + 5 + 8 + math.ceil(nch / 32) + 5
    fac = torch.ones_like(g)
    if gclip > 0:
        depth += math.ceil(nt / 32) + 5
        gn = g.pow(2).sum().sqrt().reshape(1)
        fac[:] = (f32(gclip) / nan_max(gn, f32(gclip)))
    elif max_norm > 0:
        for t in range(nt):
            a, b = s.offs[t], s.offs[t + 1]
            if b > a:
                fac[a:b] = f32(max_norm) / nan_max(g[a:b].pow(2).sum().sqrt().reshape(1), f32(max_norm))
    eg = (depth / 2 + 5) * U
    clipped = (gclip > 0 or max_norm > 0)
    g = g * fac
    if max_value > 0:
        g = torch.clamp(g, -f32(max_value), f32(max_value))
    ag = g.abs()
    e_g = ag * eg if clipped else ag * U
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    dm = (1 - b1) * e_g + 3 * U * (b1 * m.abs() + (1 - b1) * ag)
    dv = (1 - b2) * (2 * ag * e_g + e_g * e_g) + 4 * U * (b2 * v + (1 - b2) * g * g)
    sq = v1.sqrt()
    den = sq + eps
    upd = m1 / den
    dsq = torch.minimum(dv.sqrt(), torch.where(sq > 0, dv / (2 * sq), torch.full_like(sq, math.inf))) + 2 * U * den
    p1 = p - lr_t * upd
    dp = lr_t * (dm + upd.abs() * dsq) / den + 6 * U * lr_t * upd.abs() + 2 * U * p1.abs()
    ref = {"m": (m1, dm), "v": (v1, dv), "p": (p1, dp)}
    return ref, fac, dec


def compare(tag, s_before, s_after, ref, dec):
    worst = {}
    for k, (r, bound) in ref.items():
        got = getattr(s_after, k).to(F64)
        nonfin = ~torch.isfinite(r)
        assert torch.equal(nonfin, ~torch.isfinite(got)), "%s %s: non-finite entries differ (%d vs %d)" % (
            tag, k, int(nonfin.sum()), int((~torch.isfinite(got)).sum()))
        fin = ~nonfin
        err = (got[fin] - r[fin]).abs()
        ratio = (err / (2 * bound[fin])).nan_to_num(nan=math.inf).max().item() if err.numel() else 0.0
        worst[k] = ratio
        assert ratio <= 1.0, "%s %s: worst err / bound %.3g" % (tag, k, ratio)
    if s_before.ema is not None:
        e0, p1 = s_before.ema.to(F64), s_after.p.to(F64)
        r = e0 - (1 - dec) * (e0 - p1)
        bound = 3 * U * (1 - dec) * (e0 - p1).abs() + 2 * U * r.abs()
        got = s_after.ema.to(F64)
        fin = torch.isfinite(r)
        assert torch.equal(fin, torch.isfinite(got)), "%s ema: non-finite entries differ" % tag
        err = (got[fin] - r[fin]).abs()
        ratio = (err / (2 * bound[fin])).nan_to_num(nan=math.inf).max().item() if err.numel() else 0.0
        worst["ema"] = ratio
        assert ratio <= 1.0, "%s ema: worst err / bound %.3g" % (tag, ratio)
    record(tag, **{"worst_err_over_bound_" + k: v for k, v in worst.items()},
           worst_err_over_bound=max(worst.values()))


def run_and_check(tag, s, step, **kw):
    before = s.copy()
    ref, fac, dec = reference(before, step, **kw)
    adam_call(s, step, **kw)
    compare(tag, before, s, ref, dec)
    return fac


# ------------------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------------------
def wavenet_norms(sizes, gscale):
    """per-tensor target norms of the scaled gradient: every third tensor far above 100, the rest below"""
    out = []
    for t, s in enumerate(sizes):
        out.append(None if s == 0 else (300.0 + t if t % 3 == 0 else 0.5 + t % 7))
    return [None if x is None else x / gscale for x in out]


@pytest.mark.parametrize("table", sorted(TABLES))
@pytest.mark.parametrize("gscale", [1.0, 0.5, 1.0 / 3.0])
def test_per_tensor_clip(table, gscale):
    """clip_by_norm(100) active on some tensors, inactive on others, exactly at the limit on one; clip_by_value(5) active; steps 1, 2 and
    1000 with the EMA"""
    sizes = TABLES[table]()
    s = State(sizes, seed=len(sizes), gnorms=wavenet_norms(sizes, gscale))
    # one tensor exactly at the limit: n equal values c with n c^2 = 100^2, exact in fp32 for n a power of 4 and grad_scale a power of 2
    at = next((t for t, n in enumerate(sizes) if n > 0 and 4 ** round(math.log(n, 4)) == n), None)
    exact = at is not None and gscale in (1.0, 0.5)
    if exact:
        s.g[s.offs[at]:s.offs[at + 1]] = 100.0 / math.sqrt(sizes[at]) / gscale
    small = next(t for t, n in enumerate(sizes) if n > 0 and t % 3 == 1)
    s.g[s.offs[small]] = 40.0 / gscale   # a value clip in a tensor the norm clip leaves alone (norm < 100)
    for step in (1, 2, 1000):
        fac = run_and_check("adam_clip_norm_value_%s_gs%.3g_step%d" % (table, gscale, step), s, step, gscale=gscale, max_norm=100.0,
                            max_value=5.0)
        if step == 1:
            assert (fac < 1).any() and (fac == 1).any()
            if exact:
                assert fac[s.offs[at]].item() == 1.0


@pytest.mark.parametrize("table", sorted(TABLES))
def test_no_clip_and_value_clip_only(table):
    sizes = TABLES[table]()
    s = State(sizes, seed=7, ema=False)
    s.g.mul_(10.0)
    run_and_check("adam_noclip_%s" % table, s, 1)
    run_and_check("adam_valueclip_%s" % table, s, 2, max_value=5.0, gscale=1.0 / 3.0)


@pytest.mark.parametrize("table", sorted(TABLES))
@pytest.mark.parametrize("active", [True, False])
def test_global_clip(table, active):
    """clip_by_global_norm(1.0) active (norm >> 1) and inactive (norm 0.5), no EMA, steps 1, 2, 1000, grad_scale 1 and 1/3"""
    sizes = TABLES[table]()
    s = State(sizes, seed=11, ema=False)
    s.g.mul_((30.0 if active else 0.5) / s.g.double().norm().item())
    for step, gs in ((1, 1.0), (2, 1.0 / 3.0), (1000, 0.5)):
        fac = run_and_check("adam_global_%s_%s_step%d" % (table, "active" if active else "inactive", step), s, step, gscale=gs, gclip=1.0)
        assert (fac < 1).all() if active else (fac == 1).all()


@pytest.mark.parametrize("mode", ["per_tensor", "global"])
def test_replicas_bit_identical(mode):
    """the same call on copies of the same state, repeated, gives bit-identical p, m, v, ema while clips are active: two data-parallel
    replicas that apply the same averaged gradient stay identical"""
    sizes = tacotron_cbhg_table() if mode == "global" else wavenet_table()
    base = State(sizes, seed=3, gnorms=wavenet_norms(sizes, 1.0), ema=mode != "global")
    kw = dict(gclip=1.0) if mode == "global" else dict(max_norm=100.0, max_value=5.0)
    reps = [base.copy() for _ in range(4)]
    for step in (1, 2, 3):
        for r in reps:
            adam_call(r, step, gscale=0.5, **kw)
        for r in reps[1:]:
            for k in ("p", "m", "v") + (("ema",) if base.ema is not None else ()):
                a, b = getattr(reps[0], k), getattr(r, k)
                assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "%s step %d: %s differs between replicas" % (mode, step, k)
    record("adam_replicas_%s" % mode, bit_identical=1)


@pytest.mark.parametrize("clip", ["per_tensor", "global"])
def test_non_finite_gradients(clip):
    """one NaN and one Inf element in different tensors: a NaN norm makes the whole tensor (per-tensor) or every tensor (global) NaN,
    an Inf norm scales the tensor's finite gradients to 0 and the Inf one to NaN, as tf.clip_by_norm / clip_by_global_norm do"""
    sizes = synthetic_table(4)
    s = State(sizes, seed=5, ema=clip == "per_tensor")
    i_nan = s.offs[3] + 17
    i_inf = s.offs[6] + 1
    s.g[i_nan] = float("nan")
    s.g[i_inf] = float("inf")
    kw = dict(gclip=1.0) if clip == "global" else dict(max_norm=100.0, max_value=5.0)
    before = s.copy()
    run_and_check("adam_nonfinite_%s" % clip, s, 2, **kw)
    if clip == "global":
        assert torch.isnan(s.p).all()
    else:
        assert torch.isnan(s.p[s.offs[3]:s.offs[4]]).all() and torch.isnan(s.m[s.offs[3]:s.offs[4]]).all()
        assert torch.isnan(s.p[i_inf]) and torch.isfinite(s.p[s.offs[6]:i_inf]).all()
        assert torch.equal(s.m[s.offs[6]:i_inf], (before.m[s.offs[6]:i_inf].double() * f32(HP["b1"])).float())
        assert torch.isfinite(s.p[:s.offs[3]]).all() and torch.isfinite(s.p[s.offs[7]:]).all()


@pytest.mark.parametrize("mode", ["none", "per_tensor", "global"])
def test_launch_count(mode):
    """t2_launch_count() moves by the kernels the call launches: adam alone without a norm clip, sumsq + norms + adam with one"""
    s = State(synthetic_table(4), seed=1)
    kw = {"none": dict(max_value=5.0), "per_tensor": dict(max_norm=100.0), "global": dict(gclip=1.0)}[mode]
    lib = L.load()
    lib.t2_launch_count.restype = ctypes.c_longlong
    n0 = lib.t2_launch_count()
    adam_call(s, 1, **kw)
    assert lib.t2_launch_count() - n0 == (1 if mode == "none" else 3)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        adam_call(s, 2, **kw)
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "_kernel" in e.name]
    assert len(names) == (1 if mode == "none" else 3), names
