"""Speaker-conditioned forms of the WaveNet oracle's training step and incremental pass, built from oracle/wavenet.py without changing it.

train_step_g: oracle.wavenet.step already takes the speaker ids `g` (wavenet.py:669-678, modules.py:503-508); this is train_step with
them passed through. incremental_g: the speaker term of a layer is constant along time, so item b's incremental pass is the plain
oracle.incremental of that one item with b_gin + W_gin^T gc_embedding[id_b] folded into the layer's causal-conv bias."""
import torch

from oracle import wavenet as ow


def train_step_g(params, x, c, y, lengths, hp, g=None, dropout_masks=None, c_is_upsampled=False):
    """oracle.wavenet.train_step with speaker ids g ([B, 1] ints or None). Returns (loss, grads, y_hat)."""
    ps = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    y_hat = ow.step(x, c, ps, hp, dropout_masks=dropout_masks, c_is_upsampled=c_is_upsampled, g=g)
    loss = ow.loss_fn(y_hat, y, lengths, hp)
    keys = list(ps)
    gr = torch.autograd.grad(loss, [ps[k] for k in keys], allow_unused=True)
    grads = {k: (d if d is not None else torch.zeros_like(ps[k])) for k, d in zip(keys, gr)}
    return loss.detach(), grads, y_hat.detach()


def fold_speaker(params, hp, sid):
    """params of the same network with speaker `sid`'s gin term folded into every layer's causal-conv bias"""
    out = dict(params)
    e = params["gc_embedding"][int(sid)]
    for l in range(hp.layers):
        p = "ResidualConv1DGLU_%d/" % l
        term = e @ params[p + "residual_block_gin_conv/kernel"][0] + params[p + "residual_block_gin_conv/bias"]
        out[p + "residual_block_causal_conv/bias"] = params[p + "residual_block_causal_conv/bias"] + term
    return out


def incremental_g(initial_input, c, params, hp, time_length, g, **kw):
    """oracle.wavenet.incremental with speaker ids g ([B] or [B, 1]): one item at a time; per-item keyword tensors (test_inputs,
    u_mix, u_logistic, u_cat, normal) are sliced along dim 0. Returns (outputs, raw outputs) stacked over items."""
    g = torch.as_tensor(g).reshape(-1)
    outs, raws = [], []
    for b in range(initial_input.shape[0]):
        kb = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in kw.items()}
        o, r = ow.incremental(initial_input[b:b + 1], None if c is None else c[b:b + 1], fold_speaker(params, hp, g[b]), hp,
                              time_length, **kb)
        outs.append(o)
        raws.append(r)
    return torch.cat(outs), torch.cat(raws)
