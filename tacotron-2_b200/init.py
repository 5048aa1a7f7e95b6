"""Fresh-variable initialisers for the flat parameter buffers (what `tf.global_variables_initializer()` does for the
reference graphs): glorot-uniform kernels (TF1 `get_variable` / `tf.layers` default), zero biases, batch-norm
gamma = 1 / beta = 0 / moving_mean = 0 / moving_variance = 1, and the nearest-neighbour "checkerboard free" kernels of the
WaveNet conditioning upsamplers when `hparams.NN_init` (wavenet_vocoder/models/modules.py:642-654, :724-733, :761-770).
Host-side plumbing only; the values are uploaded once into the C-ABI's parameter buffer."""
import math

import torch


def _fans(shape):
    if len(shape) == 1:
        return shape[0], shape[0]
    if len(shape) == 2:
        return shape[0], shape[1]
    receptive = 1
    for d in shape[:-2]:
        receptive *= d
    return receptive * shape[-2], receptive * shape[-1]


def glorot_uniform(shape, gen):
    fan_in, fan_out = _fans(shape)
    limit = math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand(shape, generator=gen, dtype=torch.float32) * 2.0 - 1.0) * limit


def truncated_normal(shape, std, gen):
    """tf.truncated_normal_initializer: normal draws, redrawn while beyond two standard deviations"""
    x = torch.randn(shape, generator=gen, dtype=torch.float32)
    while True:
        bad = x.abs() > 2.0
        if not bad.any():
            return x * std
        x[bad] = torch.randn(int(bad.sum()), generator=gen, dtype=torch.float32)


def nn_upsample_kernel(shape, scale, n_layers, nn_scaler, subpixel):
    """shape: TF kernel shape [freq_kernel, time_kernel, 1, filters]. One centre tap (SubPixel, odd time kernel) or a row
    of 1/overlap taps (ConvTranspose2D) on the middle frequency row, scaled by NN_scaler ** (1 / n_layers)."""
    kh, kw = shape[0], shape[1]
    k = torch.zeros(kh, kw, dtype=torch.float32)
    overlap = max(kw // scale, 1)
    even = kw % 2 == 0
    if subpixel:
        cols = [kw // 2 - 1, kw // 2] if even else [kw // 2]
    else:
        cols = list(range(kw))
    for j in cols:
        k[kh // 2, j] = 1.0 / overlap if even else 1.0
    k = k * nn_scaler ** (1.0 / n_layers)
    return k[:, :, None, None].expand(*shape).contiguous()


def nn_convtranspose1d_kernel(shape, n_layers, nn_scaler):
    """ConvTranspose1D._init_kernel (modules.py:724-733): shape [1, s, C, C] ([kh, kw, out, in]); every tap is the identity over the
    channels, scaled by NN_scaler ** (1 / n_layers). (Kernel size equals the stride, so the reference's 1 / overlap factor is 1.)"""
    _, s, c_out, c_in = shape
    eye = torch.eye(c_out, c_in, dtype=torch.float32) * nn_scaler ** (1.0 / n_layers)
    return eye.expand(1, s, c_out, c_in).contiguous()


def wavenet_variables(hp, tensors, seed=None):
    """tensors: [(name, offset, shape)] from t2_wn_param_info. Returns {name: tensor}."""
    gen = torch.Generator().manual_seed(int(hp.wavenet_random_seed if seed is None else seed))
    out = {}
    n_up = len(hp.upsample_scales)
    for name, _, shape in tensors:
        if name.endswith("bias"):
            out[name] = torch.zeros(shape)
        elif name == "gc_embedding":                 # truncated normal, std 0.1 (modules.py:10-21)
            out[name] = truncated_normal(shape, 0.1, gen)
        elif name.startswith("local_conditioning_upsampling") and hp.NN_init:
            i = int(name.split("/")[0].rsplit("_", 1)[-1]) - 1
            if hp.upsample_type == "1D":
                out[name] = nn_convtranspose1d_kernel(shape, n_up, hp.NN_scaler)
            else:
                out[name] = nn_upsample_kernel(shape, hp.upsample_scales[i], n_up, hp.NN_scaler, hp.upsample_type == "SubPixel")
        else:
            out[name] = glorot_uniform(shape, gen)
    return out


def tacotron_variables(hp, tensors, seed=None):
    """tensors: [(name, offset, shape, trainable)] from t2_taco_param_info."""
    gen = torch.Generator().manual_seed(int(hp.tacotron_random_seed if seed is None else seed))
    out = {}
    for name, _, shape, _ in tensors:
        if name.endswith(("gamma", "moving_variance")):
            out[name] = torch.ones(shape)
        elif name.endswith("RNN/gates/bias"):
            out[name] = torch.ones(shape)            # tf.nn.rnn_cell.GRUCell: gate bias initialiser 1.0
        elif "/T/bias" in name:
            out[name] = -torch.ones(shape)           # HighwayNet transform gate, tacotron/models/modules.py:10
        elif name.endswith(("beta", "moving_mean", "bias")):
            out[name] = torch.zeros(shape)
        else:
            out[name] = glorot_uniform(shape, gen)
    return out
