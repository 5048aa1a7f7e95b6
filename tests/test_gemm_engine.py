"""wgmma GEMM engine vs a float64 reference of the same contraction (bf16-rounded inputs). fp32 outputs must stay within the fp32
accumulation bound 2^-20 (|A|.|W|)[elem] + 2^-23 |ref| (one more rounding for the bias add / scale) + 1e-7; bf16 outputs add 2^-8 |ref|."""
import ctypes

import pytest
import torch

from parity_util import record
from t2_import import t2

pytestmark = pytest.mark.gpu
L = t2.lib


def _conv_ref(a, w, shifts, bias, relu):
    # a [B,T,C] fp32 (bf16 values), w [N, S*Kp]
    B, T, C = a.shape
    Kp = (C + 63) // 64 * 64
    out = torch.zeros(B, T, w.shape[0], device=a.device, dtype=a.dtype)
    for s, sh in enumerate(shifts):
        sh_a = torch.zeros_like(a)
        if sh < 0:
            if -sh < T:
                sh_a[:, -sh:, :] = a[:, :T + sh, :]
        elif sh > 0:
            if sh < T:
                sh_a[:, :T - sh, :] = a[:, sh:, :]
        else:
            sh_a = a
        out += sh_a @ w[:, s * Kp:s * Kp + C].t()
    if bias is not None:
        out += bias
    if relu:
        out = out.relu()
    return out


@pytest.mark.parametrize("B,T,C,N,BN,shifts", [
    (1, 128, 64, 128, 128, [0]),
    (2, 256, 256, 256, 256, [0]),
    (2, 384, 256, 512, 256, [-8, -4, 0]),
    (2, 200, 80, 128, 128, [0]),          # ragged T (tail tile) and C not a multiple of 64
    (1, 1000, 128, 256, 128, [-64, -32, 0]),
    (2, 640, 512, 256, 256, [64, 32, 0]),  # anti-causal taps (backward data gradient)
])
def test_conv_gemm(B, T, C, N, BN, shifts):
    lib = L.load()
    torch.manual_seed(0)
    dev = "cuda"
    a = (torch.randn(B, T, C, device=dev) * 0.5).bfloat16()
    Kp = (C + 63) // 64 * 64
    w = torch.zeros(N, len(shifts) * Kp, device=dev)
    for s in range(len(shifts)):
        w[:, s * Kp:s * Kp + C] = torch.randn(N, C, device=dev) / C ** 0.5
    w = w.bfloat16()
    bias = torch.randn(N, device=dev)
    out_f = torch.full((B, T, N), float("nan"), device=dev)
    out_b = torch.zeros(B, T, N, device=dev, dtype=torch.bfloat16)
    sh = (ctypes.c_int * len(shifts))(*shifts)
    L.check(lib.t2_dbg_conv_gemm(L.ptr(a), B, T, C, C, sh, len(shifts), L.ptr(w), N, BN, L.ptr(bias), 1,
                                 L.ptr(out_b), L.ptr(out_f), L.stream_ptr()))
    torch.cuda.synchronize()
    ref = _conv_ref(a.double(), w.double(), shifts, bias.double(), True)
    absref = _conv_ref(a.double().abs(), w.double().abs(), shifts, None, False)
    bound = 2.0 ** -20 * absref + 2.0 ** -23 * ref.abs() + 1e-7
    ratio = ((out_f.double() - ref).abs() / bound).max().item()
    ratio_b = ((out_b.double() - ref).abs() / (bound + 2.0 ** -8 * ref.abs())).max().item()
    record("conv_gemm_B%d_T%d_C%d_N%d_BN%d" % (B, T, C, N, BN), worst_err_over_bound=ratio, worst_err_over_bound_bf16=ratio_b)
    assert ratio <= 1.0, "fp32 output: worst err / bound %g" % ratio
    assert ratio_b <= 1.0, "bf16 output: worst err / bound %g" % ratio_b


@pytest.mark.parametrize("B,T,Ca,Cb,shift", [
    (1, 64, 128, 128, 0),
    (2, 256, 256, 512, 0),
    (2, 300, 80, 256, 0),     # ragged T, Ca not a multiple of 64
    (2, 512, 256, 256, -16),
    (1, 128, 128, 192, 0),    # 3 column blocks of 64
    (2, 200, 64, 320, 3),     # one full 256-wide tile + a 64-wide remainder
    (1, 64, 128, 64, 0),
])
def test_wgrad(B, T, Ca, Cb, shift):
    lib = L.load()
    torch.manual_seed(1)
    dev = "cuda"
    a = (torch.randn(B, T, Ca, device=dev) * 0.5).bfloat16()
    g = (torch.randn(B, T, Cb, device=dev) * 0.5).bfloat16()
    out = torch.full((Ca, Cb), float("nan"), device=dev)
    L.check(lib.t2_dbg_wgrad(L.ptr(a), Ca, L.ptr(g), Cb, B, T, shift, ctypes.c_float(0.5), L.ptr(out),
                             L.stream_ptr()))
    torch.cuda.synchronize()
    af = a.double()
    sa = torch.zeros_like(af)
    if shift < 0:
        sa[:, -shift:, :] = af[:, :T + shift, :]
    elif shift > 0:
        sa[:, :T - shift, :] = af[:, shift:, :]
    else:
        sa = af
    ref = 0.5 * torch.einsum("btm,btn->mn", sa, g.double())
    absref = 0.5 * torch.einsum("btm,btn->mn", sa.abs(), g.double().abs())
    ratio = ((out.double() - ref).abs() / (2.0 ** -20 * absref + 2.0 ** -23 * ref.abs() + 1e-7)).max().item()
    record("wgrad_B%d_T%d_Ca%d_Cb%d_shift%d" % (B, T, Ca, Cb, shift), worst_err_over_bound=ratio)
    assert ratio <= 1.0, "wgrad: worst err / bound %g" % ratio
