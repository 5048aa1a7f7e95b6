"""Float64 reference of the CBHG bidirectional GRU kernels (gru_fwd_kernel / gru_bwd_kernel, t2_cbhg.cu) and of the GRU weight and
bias gradients the backward pass derives from their outputs, each with a per-element error bound of the CUDA path.

Layout (rows b T + t): XP [B, T, 6RU] = [fw gates 2RU | fw cand RU | bw gates 2RU | bw cand RU] (the input projections, without biases),
out [B, T, 2RU] = [h fw | h bw]. Direction d processes t = 0..T-1 (fw) or T-1..0 (bw) over the whole padded sequence, from a zero state.

Forward (tf.nn.rnn_cell.GRUCell, r applied BEFORE the candidate matmul):
  a = XP_g + bg + h Wg_h ; r, u = sigmoid(a) ; c = tanh(XP_c + bc + (r h) Wc_h) ; h' = u h + (1 - u) c
with the recurrent rows Wg_h / Wc_h rounded to bf16 (round to nearest even), as the kernel keeps them in shared memory; XP and the
biases are read in fp32, and the state is fp32. What remains between the kernel and this reference is fp32 rounding and the fast
intrinsics; the bound delta of every quantity is carried to first order (|J_t| delta_{t-1} plus local terms). Carried through the whole
recurrence in absolute values, |J_t| grows the bound by a factor of 2 to 6 per step at the production initialisation (about 1e12 after
37 steps), so the GPU tests re-anchor every step on the kernel's own bf16 output of the previous step (`anchor`): h_prev is then known
to 2^-8 relative, and each bound spans one step. The local terms:
  gate / candidate dots   130 u sum|terms| (u = 2^-24; 64 k-pairs, two roundings each, plus the XP + bias add)
  sigmoid (__expf)        g (1 - g) (|d a| + 2^-21 (1 + |a|)) + 2u g   (relative error of __expf, then the add and one IEEE division)
  tanhf                   (1 - c^2) |d pre| + 4u |c|   (2 ulp)
  r h                     |h| d r + r d h + u |r h|
  state update            |h - c| d u + u d h + (1 - u) d c + 8u (|u h| + |(1 - u) c|)   (8u per operation chain)
  bf16 stores             + 2^-8 (|x| + delta)   (out, r, u, c, rh; bf16 unit roundoff)
Backward (BPTT, gru_bwd_kernel) consumes exactly what the kernel reads: dout fp32, the bf16 `out` as h_prev (NOT the fp32 state), the
bf16 r / u / c stashes and the bf16 recurrent rows. Per processed step, in reverse:
  g = dh + dout ; dc_pre = g (1 - u)(1 - c^2) ; drh = dc_pre Wc_h^T ; dr_pre = drh h_prev r (1 - r) ; du_pre = g (h_prev - c) u (1 - u)
  dh_prev = g u + drh r + [dr_pre | du_pre] Wg_h^T
  bounds: 8u per operation chain on every elementwise result, 130 u sum|terms| for the 128-term dot, 260 u sum|terms| for the 256-term
  dot (+ the two carried terms), first-order carry of delta(dh) through the same linear map in absolute values, 2^-8 for the bf16 dXP.
  Carried through all steps this bound, like the forward's, grows without limit (past 1 after about ten steps). The GPU tests therefore
  re-anchor it on the kernel's own dXP (`anchor`): the kernel's fp32 g of a step is recovered from its bf16 dc_pre = g (1 - u)(1 - c^2)
  or du_pre = g (h_prev - c) u (1 - u) to 2^-8 relative wherever that coefficient is not exactly 0, and the next processed step is
  re-derived from it, so every bound spans one step.
Every bound carries a factor-2 margin over the first-order terms (as in tests/test_taco_kernels_gpu.py).
Weight / bias gradients, from given operands (bf16 tensors the wgrad GEMM reads):
  input rows      h_last^T dXP_d ; gates recurrent rows sum_t h_prev(t)^T [dr_pre | du_pre](t), h_prev = out shifted by -1 (fw) / +1 (bw)
                  within each item and zero at its first processed step ; candidate recurrent rows (r h)^T dc_pre ; biases colsum(dXP_d)
  bounds          wgrad: 2 (N/16 + 16) u (|A|^T |B|) + 2u |ref| + 1e-7 (1 + max|ref|) (fp32 accumulation of N = B T bf16 products per
                  output, one rounding per 16-position wgmma step, as tests/test_gemm_epilogues_gpu.py's wgrad check with N in place
                  of a few hundred); colsums: 2 (N/64 + 64) u sum|.| + 2u |ref| (64 blocks of sequential fp32 adds, then 64 atomics)."""
import torch

F64 = torch.float64
U = 2.0 ** -24
BF = 2.0 ** -8                 # bf16 unit roundoff (8 significant bits; half an ulp is 2^-8 |x| at the bottom of a binade)
EXP_REL = 2.0 ** -21
TINY = 1e-30
BIG = 1e30                     # carried BPTT bounds saturate here (a bound this large passes anything finite; inf * 0 would be NaN)
RU = 128


def bf16(x):
    """round to bf16 (nearest even) and back to float64"""
    return x.to(torch.float32).to(torch.bfloat16).to(F64)


def recurrent(W, HU):
    """bf16 recurrent rows [RU, 2RU] / [RU, RU] of the gates / candidate kernels of one direction (W: dict gk, gb, ck, cb)"""
    return bf16(W["gk"][HU:]), bf16(W["ck"][HU:])


def stored(x, d):
    """bound of a bf16 store of a value x computed with first-order error d, with the factor-2 margin"""
    return 2 * d * (1 + BF) + BF * x.abs() + TINY


def _order(T, d):
    return range(T) if d == 0 else range(T - 1, -1, -1)


def forward(XP, Ws, HU, anchor=None, h0=None, fault=None):
    """XP [B, T, 6RU]; Ws = [fw, bw] dicts of fp32 gk [HU+RU, 2RU], gb [2RU], ck [HU+RU, RU], cb [RU].
    anchor: None carries the float64 state through the recurrence (the exact GRU); a [B, T, 2RU] bf16 `out` of the kernel re-anchors
    every step on the kernel's own previous output (h_prev = anchor, |h_fp32 - h_prev| <= 2^-8 |h_prev| / (1 - 2^-8); zero at the
    item's first processed step), so that every bound spans one step. h0: optional [2][B, RU] initial states (zero by default).
    fault (sensitivity tests): 'swap_ru' | 'no_gate_bias' | 'carry_items'.
    Returns dict: out [B, T, 2RU] (float64 h) and out_b (its bound as a bf16 store); for each direction d lists r, u, c, rh and their
    store bounds r_b, u_b, c_b, rh_b ([B, T, RU] each)."""
    if fault == "carry_items":         # the state carried from item b into item b + 1: item b + 1 starts where item b ended
        clean = forward(XP, Ws, HU)
        last = [clean["out"][:, -1, :RU], clean["out"][:, 0, RU:]]
        h0 = [torch.cat([torch.zeros_like(s[:1]), s[:-1]]) for s in last]
        return forward(XP, Ws, HU, h0=h0)
    if anchor is not None:
        hp_all = [h_prev(anchor, d) for d in range(2)]
    B, T, _ = XP.shape
    dev = XP.device
    X = XP.to(F64)
    res = {"out": torch.zeros(B, T, 2 * RU, dtype=F64, device=dev), "out_b": torch.zeros(B, T, 2 * RU, dtype=F64, device=dev)}
    for k in ("r", "u", "c", "rh"):
        res[k] = [torch.zeros(B, T, RU, dtype=F64, device=dev) for _ in range(2)]
        res[k + "_b"] = [torch.zeros(B, T, RU, dtype=F64, device=dev) for _ in range(2)]
    for d in range(2):
        W = Ws[d]
        Wg, Wc = recurrent(W, HU)
        Wga, Wca = Wg.abs(), Wc.abs()
        bg = W["gb"].to(dev, F64) if fault != "no_gate_bias" else torch.zeros(2 * RU, dtype=F64, device=dev)
        bc = W["cb"].to(dev, F64)
        h = torch.zeros(B, RU, dtype=F64, device=dev) if h0 is None else h0[d].to(dev, F64).clone()
        dh = torch.zeros_like(h)
        for t in _order(T, d):
            if anchor is not None:
                h = hp_all[d][:, t]
                dh = h.abs() * (BF / (1 - BF))
            xg, xc = X[:, t, d * 3 * RU:d * 3 * RU + 2 * RU], X[:, t, d * 3 * RU + 2 * RU:(d + 1) * 3 * RU]
            a = xg + bg + h @ Wg
            da = 130 * U * (xg.abs() + bg.abs() + h.abs() @ Wga) + dh @ Wga
            g = torch.sigmoid(a)
            dg = g * (1 - g) * (da + EXP_REL * (1 + a.abs())) + 2 * U * g
            if fault == "swap_ru":
                r, u, dr, du = g[:, RU:], g[:, :RU], dg[:, RU:], dg[:, :RU]
            else:
                r, u, dr, du = g[:, :RU], g[:, RU:], dg[:, :RU], dg[:, RU:]
            rh = r * h
            drh = h.abs() * dr + r * dh + U * rh.abs()
            pc = xc + bc + rh @ Wc
            dpc = 130 * U * (xc.abs() + bc.abs() + rh.abs() @ Wca) + drh @ Wca
            c = torch.tanh(pc)
            dc = (1 - c * c) * dpc + 4 * U * c.abs()
            hn = u * h + (1 - u) * c
            dhn = (h - c).abs() * du + u * dh + (1 - u) * dc + 8 * U * ((u * h).abs() + ((1 - u) * c).abs())
            res["out"][:, t, d * RU:(d + 1) * RU] = hn
            res["out_b"][:, t, d * RU:(d + 1) * RU] = stored(hn, dhn)
            for k, v, e in (("r", r, dr), ("u", u, du), ("c", c, dc), ("rh", rh, drh)):
                res[k][d][:, t] = v
                res[k + "_b"][d][:, t] = stored(v, e)
            h, dh = hn, dhn
    return res


def h_prev(out, d, fault=None):
    """h_prev of every step of direction d from out [B, T, 2RU]: the output of the previously processed step of the same item, zero at the
    item's first processed step. fault: 'shift_flip' (the other direction's shift) | 'boundary' (the shift runs across item boundaries)
    | 'bw_off' (bw: one step further)."""
    B, T, _ = out.shape
    o = out[..., d * RU:(d + 1) * RU].to(F64)
    sh = -1 if d == 0 else 1
    if fault == "shift_flip":
        sh = -sh
    if fault == "bw_off" and d == 1:
        sh = 2
    if fault == "boundary":
        flat = o.reshape(B * T, RU)
        z = torch.zeros(abs(sh), RU, dtype=F64, device=o.device)
        flat = torch.cat([z, flat[:-1]]) if sh < 0 else torch.cat([flat[1:], z])
        return flat.reshape(B, T, RU)
    hp = torch.zeros_like(o)
    if sh < 0:
        hp[:, -sh:] = o[:, :T + sh]
    else:
        hp[:, :T - sh] = o[:, sh:]
    return hp


def _anchor_g(g, dg, A, coef, anchor_ok):
    """the kernel's fp32 g recovered from one of its bf16 pre-activation gradients A = bf16(g coef (1 + 8u)), where coef (from the bf16
    stashes) is not 0: relative error 2^-8 / (1 - 2^-8) + 16u whatever the size of coef (+ the bf16 subnormal spacing / |coef|).
    Elementwise, the estimate with the smaller bound wins."""
    nz = coef != 0
    safe = torch.where(nz, coef, torch.ones_like(coef))
    ge = A / safe
    de = (BF / (1 - BF) + 16 * U) * ge.abs() * 1.01 + 1e-37 / safe.abs()
    use = nz & anchor_ok & (de < dg)
    return torch.where(use, ge, g), torch.where(use, de, dg)


def bptt(dout, out, r, u, c, Ws, HU, fault=None, anchor=None):
    """dXP [B, T, 6RU] and its per-element bound (bf16 store). dout [B, T, 2RU] fp32; out [B, T, 2RU] (what the kernel reads as h_prev);
    r, u, c: [2] lists of [B, T, RU] stashes; Ws as in forward. fault: 'bw_off' (h_prev one step off in bw) | 'no_drh_r' (drh r dropped
    from dh_prev).
    anchor: None carries the float64 dh (and its bound) through every step. A [B, T, 6RU] bf16 dXP of the kernel re-anchors it: after
    the outputs of a step are formed from the carried g = dh + dout, g is replaced, element by element, by the kernel's own g of that
    step recovered from its dc_pre (coefficient (1 - u)(1 - c^2)) or du_pre ((h_prev - c) u (1 - u)) wherever that bound is smaller, and
    dh of the next processed step is propagated from it. Every step's outputs are then checked one step away from the kernel's own
    previous step, as the forward is (the step's own outputs are never used to form its reference)."""
    B, T, _ = dout.shape
    dev = dout.device
    G = dout.to(F64)
    dXP = torch.zeros(B, T, 6 * RU, dtype=F64, device=dev)
    bnd = torch.zeros_like(dXP)
    for d in range(2):
        Wg, Wc = recurrent(Ws[d], HU)
        Wga, Wca = Wg.abs(), Wc.abs()
        HP = h_prev(out, d, "bw_off" if fault == "bw_off" else None)
        dh = torch.zeros(B, RU, dtype=F64, device=dev)
        ddh = torch.zeros_like(dh)
        o = d * 3 * RU

        def step(g, dg, uv, rv, cv, hp):
            dcp = g * (1 - uv) * (1 - cv * cv)
            ddcp = (1 - uv) * (1 - cv * cv) * dg + 8 * U * dcp.abs()
            drh = dcp @ Wc.t()
            ddrh = 130 * U * (dcp.abs() @ Wca.t()) + ddcp @ Wca.t()
            drp = drh * hp * rv * (1 - rv)
            ddrp = (hp * rv * (1 - rv)).abs() * ddrh + 8 * U * drp.abs()
            dup = g * (hp - cv) * uv * (1 - uv)
            ddup = ((hp - cv) * uv * (1 - uv)).abs() * dg + 8 * U * dup.abs()
            dgp, ddgp = torch.cat([drp, dup], 1), torch.cat([ddrp, ddup], 1)
            carried = g * uv + (drh * rv if fault != "no_drh_r" else 0)
            dh_new = carried + dgp @ Wg.t()
            ddh_new = (uv * dg + rv * ddrh + ddgp @ Wga.t() + 8 * U * ((g * uv).abs() + (drh * rv).abs())
                       + 260 * U * ((g * uv).abs() + (drh * rv).abs() + dgp.abs() @ Wga.t())).clamp(max=BIG)
            return (drp, dup, dcp), (ddrp, ddup, ddcp), dh_new, ddh_new

        for t in reversed(list(_order(T, d))):
            rv, uv, cv, hp = r[d][:, t].to(F64), u[d][:, t].to(F64), c[d][:, t].to(F64), HP[:, t]
            g = dh + G[:, t, d * RU:(d + 1) * RU]
            dg = ddh + U * g.abs()
            vals, bnds, dh, ddh = step(g, dg, uv, rv, cv, hp)
            for k in range(3):
                dXP[:, t, o + k * RU:o + (k + 1) * RU] = vals[k]
                bnd[:, t, o + k * RU:o + (k + 1) * RU] = stored(vals[k], bnds[k])
            if anchor is not None:
                A = anchor[:, t, o:o + 3 * RU].to(F64)
                ok = torch.isfinite(A).all(1, keepdim=True)
                g, dg = _anchor_g(g, dg, A[:, 2 * RU:], (1 - uv) * (1 - cv * cv), ok)
                g, dg = _anchor_g(g, dg, A[:, RU:2 * RU], (hp - cv) * uv * (1 - uv), ok)
                _, _, dh, ddh = step(g, dg, uv, rv, cv, hp)
    return dXP, bnd


def _wg(A, Bm):
    """A [B, T, m], Bm [B, T, n] -> (A^T Bm over all positions, the wgrad bound)"""
    a, b = A.reshape(-1, A.shape[-1]).to(F64), Bm.reshape(-1, Bm.shape[-1]).to(F64)
    N = a.shape[0]
    ref = a.t() @ b
    return ref, 2 * (N / 16 + 16) * U * (a.abs().t() @ b.abs()) + 2 * U * ref.abs() + 1e-7 * (1 + ref.abs().max().item())


def _colsum(X):
    x = X.reshape(-1, X.shape[-1]).to(F64)
    N = x.shape[0]
    ref = x.sum(0)
    return ref, 2 * (N / 64 + 64) * U * x.abs().sum(0) + 2 * U * ref.abs() + TINY


def weight_grads(h_last, dXP, out, rh, HU, fault=None):
    """{(d, block): (ref, bound)} for block in gk_in [HU, 2RU], gk_rec [RU, 2RU], ck_in [HU, RU], ck_rec [RU, RU], gb [2RU], cb [RU].
    h_last [B, T, HU], dXP [B, T, 6RU], out [B, T, 2RU], rh [2] x [B, T, RU]. fault: 'shift_flip' | 'boundary' (h_prev of the gates
    recurrent rows)."""
    res = {}
    for d in range(2):
        o = d * 3 * RU
        dg, dc = dXP[..., o:o + 2 * RU], dXP[..., o + 2 * RU:o + 3 * RU]
        res[(d, "gk_in")] = _wg(h_last, dg)
        res[(d, "ck_in")] = _wg(h_last, dc)
        res[(d, "gk_rec")] = _wg(h_prev(out, d, fault), dg)
        res[(d, "ck_rec")] = _wg(rh[d], dc)
        res[(d, "gb")] = _colsum(dg)
        res[(d, "cb")] = _colsum(dc)
    return res
