"""Float64 reference of the Fast-WaveNet AR synthesis kernel (wn_ar_kernel, t2_wavenet.cu) under teacher forcing, and a mirror of the
host's launch plan (t2_wn_ar_generate).

Under teacher forcing the network's raw outputs are a function of the fed inputs alone, so the incremental pass equals the parallel
forward on the same input sequence (oracle.wavenet.step; tests/test_oracle_wavenet.py). `reference_raw` restates that forward in
float64, channels-last, with every weight rounded to bf16 exactly where ar_pack_kernel stores bf16:
  - the dilated-conv and cin-conv kernels, the out-conv kernel, and the final_convolution_1 / 2 kernels;
  - the skip-conv kernel AFTER the fp32 multiplication by the layer's legacy skip scale (the kernel folds the scale into it).
Everything the kernel keeps in fp32 stays unrounded here: input_convolution, every bias (the gate bias is b_dil + b_cin, plus the
speaker term), the activations and the ring. What is left between the two is fp32 accumulation order and the fast tanh / sigmoid.
The conditioning must be given as the kernel sees it (`c_up`, [B, T, cin]); NearestNeighbor with bf16-representable frames makes it
exact on both sides."""
import math

import torch

from oracle import wavenet as ow

SQRT_HALF = math.sqrt(0.5)
SMEM_LIMIT = 232448 - 1024                      # shared memory per CTA the host lets the kernel use (t2_wn_ar_generate)
MAX_ITEMS = 4                                   # kArMaxItems


def skip_scales(hp):
    """per-layer factor of the skip output when the legacy skip sum is folded out: (skips + s) * sqrt(1/2) per layer after the first"""
    L = hp.layers
    return [SQRT_HALF ** ((L - 1 if l == 0 else L - l) if hp.legacy else 0) for l in range(L)]


def reference_raw(inputs, c_up, params, hp, speakers=None, bf16=True):
    """inputs: [B, T] fed input of every step (scalar samples, or class indices for mulaw-quantize); c_up: [B, T, cin] conditioning;
    speakers: [B] ids (gin_channels > 0) or None. Returns the raw network outputs [B, T, out] in float64 on inputs' device.
    bf16=False skips the bf16 rounding: the result is then oracle.wavenet.step with the skip scales folded, in float64."""
    f64 = torch.float64
    dev = inputs.device
    P = lambda n: params[n].to(dev, f64)
    if bf16:
        rw = lambda w: w.to(dev, torch.float32).to(torch.bfloat16).to(f64)
    else:
        rw = lambda w: w.to(dev, f64)
    B, T = inputs.shape
    R, G, L = hp.residual_channels, hp.gate_channels, hp.layers
    Gh = G // 2
    k_in = P("input_convolution/kernel")[0]                       # [cin_in, R]
    if ow.is_mulaw_quantize(hp.input_type):
        h = k_in[inputs.long()]                                    # one-hot input: a row lookup
    else:
        h = inputs.to(f64).unsqueeze(-1) * k_in[0]
    h = h + P("input_convolution/bias")                            # [B, T, R]
    c = c_up.to(dev, f64)
    if speakers is not None:
        from wavenet_gin_oracle import fold_speaker
        ids = [int(v) for v in torch.as_tensor(speakers).reshape(-1).tolist()]
        folded = {s: fold_speaker(params, hp, s) for s in set(ids)}
    scales = skip_scales(hp)
    skip = torch.zeros(B, T, hp.skip_out_channels, dtype=f64, device=dev)
    skip_bias = torch.zeros(hp.skip_out_channels, dtype=f64, device=dev)
    for l in range(L):
        p = "ResidualConv1DGLU_%d/" % l
        d = ow.dilation_of(hp, l)
        wd = rw(params[p + "residual_block_causal_conv/kernel"])   # [3, R, G]: tap j reads x(t - (2 - j) d)
        gate = c @ rw(params[p + "residual_block_cin_conv/kernel"][0])
        for j in range(3):
            sh = (2 - j) * d
            if sh >= T:
                continue
            hs = torch.cat([torch.zeros(B, sh, R, dtype=f64, device=dev), h[:, :T - sh]], dim=1) if sh else h
            gate = gate + hs @ wd[j]
        bias = P(p + "residual_block_causal_conv/bias") + P(p + "residual_block_cin_conv/bias")
        if speakers is not None:                                   # per-item gate bias with the item's speaker term folded in
            bias = torch.stack([folded[s][p + "residual_block_causal_conv/bias"].to(dev, f64) for s in ids])
            gate = gate + (bias + P(p + "residual_block_cin_conv/bias"))[:, None, :]
        else:
            gate = gate + bias
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


def launch_plan(hp, B, cs, sms, prefetch_env=True):
    """The host's launch choices in t2_wn_ar_generate for B items at cluster size cs on a device with `sms` SMs: clusters, items per
    cluster (ipc), the kernel instantiation NI (wn_ar_kernel<1|2|4>), whether the last cluster is partly filled, whether more clusters
    are launched than fit at once (waves), and whether each CTA's weight slice is prefetched into shared memory.
    prefetch_env=False mirrors T2_AR_PREFETCH=0."""
    n_fit = sms // cs
    n = max(1, min(n_fit, B))
    ipc = -(-B // n)
    while ipc > MAX_ITEMS:
        n += 1
        ipc = -(-B // n)
    n = -(-B // ipc)
    ni = 1 if ipc <= 1 else (2 if ipc <= 2 else MAX_ITEMS)
    R, G, S, C, L = hp.residual_channels, hp.gate_channels, hp.skip_out_channels, hp.cin_channels, hp.layers
    Gh = G // 2
    ZC, RC, SC, OC, K1 = Gh // cs, R // cs, S // cs, -(-hp.out_channels // cs), 3 * R + C
    per_rank_layer = 2 * ZC * K1 + (RC + SC) * Gh
    ld1 = (K1 + 3) & ~3
    locw = max(2 * ZC, RC + SC)
    smem = 4 * (ni * (ld1 + Gh + R + ZC + RC + locw + SC + S + cs * OC + ((C + 3) & ~3) + 1) + L * (2 * ZC + RC)
                + ((2 * L + 1 + 3) & ~3)) + 64
    wslots = 2 * per_rank_layer * 2 + 64
    prefetch = prefetch_env and per_rank_layer % 8 == 0 and smem + wslots <= SMEM_LIMIT
    max_slots = max(1 << (2 * ow.dilation_of(hp, l)).bit_length() for l in range(L))   # pow2 >= 2d + 1
    return dict(CS=cs, B=B, clusters=n, ipc=ipc, NI=ni, ragged=B % ipc != 0, waves=n > n_fit, prefetch=bool(prefetch),
                ring_slots=max_slots)


def batch_for_ipc(target, cs, sms):
    """a batch size whose launch plan at cluster size cs has `target` items per cluster; target > MAX_ITEMS asks for the smallest batch
    that needs more clusters than fit (waves). ipc 2 and 3 leave the last cluster partly filled, ipc 4 fills every cluster."""
    n_fit = sms // cs
    if target <= 1:
        return min(5, n_fit)
    if target > MAX_ITEMS:
        return MAX_ITEMS * n_fit + 1
    return target * n_fit - (target < MAX_ITEMS)
