"""Float64 reference of the Fast-WaveNet AR synthesis kernel (wn_ar_kernel, t2_wavenet.cu) under teacher forcing at any dilated-convolution
kernel_size, and a mirror of the host's launch plan (t2_wn_ar_generate) with the kernel_size-dependent stage-1 width and ring depth.

As in wavenet_ar_reference.py (which covers kernel_size 3 with speaker conditioning): the parallel forward on the fed inputs in float64,
channels-last, with every weight rounded to bf16 exactly where ar_pack_kernel stores bf16 (dilated-conv, cin-conv, out-conv and
final-conv kernels, and the skip-conv kernel after the fp32 multiplication by its legacy skip scale); input_convolution, the biases,
the activations and the ring stay unrounded. Tap j of the dilated convolution reads x(t - (k - 1 - j) d). The conditioning is given as
the kernel sees it (`c_up`, [B, T, cin])."""
import math

import torch

from oracle import wavenet as ow
from wavenet_ar_reference import MAX_ITEMS, SMEM_LIMIT, skip_scales

SQRT_HALF = math.sqrt(0.5)


def reference_raw(inputs, c_up, params, hp, bf16=True):
    """inputs: [B, T] fed input of every step (scalar samples, or class indices for mulaw-quantize); c_up: [B, T, cin] conditioning.
    Returns the raw network outputs [B, T, out] in float64 on inputs' device. bf16=False skips the bf16 rounding."""
    f64 = torch.float64
    dev = inputs.device
    P = lambda n: params[n].to(dev, f64)
    rw = (lambda w: w.to(dev, torch.float32).to(torch.bfloat16).to(f64)) if bf16 else (lambda w: w.to(dev, f64))
    B, T = inputs.shape
    R, G, L, k = hp.residual_channels, hp.gate_channels, hp.layers, hp.kernel_size
    Gh = G // 2
    k_in = P("input_convolution/kernel")[0]
    h = k_in[inputs.long()] if ow.is_mulaw_quantize(hp.input_type) else inputs.to(f64).unsqueeze(-1) * k_in[0]
    h = h + P("input_convolution/bias")                            # [B, T, R]
    c = c_up.to(dev, f64)
    scales = skip_scales(hp)
    skip = torch.zeros(B, T, hp.skip_out_channels, dtype=f64, device=dev)
    skip_bias = torch.zeros(hp.skip_out_channels, dtype=f64, device=dev)
    for l in range(L):
        p = "ResidualConv1DGLU_%d/" % l
        d = ow.dilation_of(hp, l)
        wd = rw(params[p + "residual_block_causal_conv/kernel"])   # [k, R, G]
        assert wd.shape[0] == k
        gate = c @ rw(params[p + "residual_block_cin_conv/kernel"][0])
        for j in range(k):
            sh = (k - 1 - j) * d
            if sh >= T:
                continue
            hs = torch.cat([torch.zeros(B, sh, R, dtype=f64, device=dev), h[:, :T - sh]], dim=1) if sh else h
            gate = gate + hs @ wd[j]
        gate = gate + P(p + "residual_block_causal_conv/bias") + P(p + "residual_block_cin_conv/bias")
        z = torch.tanh(gate[..., :Gh]) * torch.sigmoid(gate[..., Gh:])
        o = z @ rw(params[p + "residual_block_out_conv/kernel"][0]) + P(p + "residual_block_out_conv/bias")
        h = (o + h) * SQRT_HALF if hp.residual_legacy else o + h
        ws = params[p + "residual_block_skip_conv/kernel"][0]
        ws = rw(ws.float() * torch.tensor(scales[l], dtype=torch.float32)) if bf16 else ws.to(dev, f64) * scales[l]
        skip = skip + z @ ws
        skip_bias = skip_bias + scales[l] * P(p + "residual_block_skip_conv/bias")
    y = torch.relu(skip + skip_bias)
    y = torch.relu(y @ rw(params["final_convolution_1/kernel"][0]) + P("final_convolution_1/bias"))
    return y @ rw(params["final_convolution_2/kernel"][0]) + P("final_convolution_2/bias")


def launch_plan(hp, B, cs, sms):
    """The host's launch choices in t2_wn_ar_generate for B items at cluster size cs on a device with `sms` SMs: clusters, items per
    cluster (ipc), the kernel's items-per-pass instantiation NI, whether each CTA's weight slice is prefetched into shared memory, the
    stage-1 width K1 = k R + cin, and the deepest ring (a power of two >= (k - 1) d + 1 slots)."""
    n_fit = sms // cs
    n = max(1, min(n_fit, B))
    ipc = -(-B // n)
    while ipc > MAX_ITEMS:
        n += 1
        ipc = -(-B // n)
    n = -(-B // ipc)
    ni = 1 if ipc <= 1 else (2 if ipc <= 2 else MAX_ITEMS)
    R, G, S, C, L, k = hp.residual_channels, hp.gate_channels, hp.skip_out_channels, hp.cin_channels, hp.layers, hp.kernel_size
    Gh = G // 2
    ZC, RC, SC, OC, K1 = Gh // cs, R // cs, S // cs, -(-hp.out_channels // cs), k * R + C
    per_rank_layer = 2 * ZC * K1 + (RC + SC) * Gh
    ld1 = (K1 + 3) & ~3
    locw = max(2 * ZC, RC + SC)
    smem = 4 * (ni * (ld1 + Gh + R + ZC + RC + locw + SC + S + cs * OC + ((C + 3) & ~3) + 1) + L * (2 * ZC + RC)
                + ((2 * L + 1 + 3) & ~3)) + 64
    wslots = 2 * per_rank_layer * 2 + 64
    prefetch = per_rank_layer % 8 == 0 and smem + wslots <= SMEM_LIMIT
    ring_slots = max(1 << ((k - 1) * ow.dilation_of(hp, l)).bit_length() for l in range(L))
    return dict(CS=cs, B=B, clusters=n, ipc=ipc, NI=ni, prefetch=bool(prefetch), K1=K1, ring_slots=ring_slots)
