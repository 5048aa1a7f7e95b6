"""Generates tests/golden/reference_attention.npz by EXECUTING the reference's own Tacotron graph code on the TF-1 stand-in, as
make_reference_graph_vectors.py does, for the two attention-state flags the CUDA path implements:

  python tests/golden/make_reference_attention_vectors.py    # needs /root/reference; only the committed .npz travels

The widths, the batch (rows of unequal length) and the variables are those of reference_graph.npz, which is read, not rewritten.
Scenarios (every hparam not listed keeps the reference's default):
  train_nocum     is_training=True, cumulative_weights=False: outputs, the four loss terms and d loss / d variable for every
                  trainable variable (autograd through the executed reference graph)
  train_nomask_g  is_training=True, mask_encoder=False: the same
  eval_nocum / eval_nomask    is_evaluating=True under each flag: outputs and losses
  synth_nocum / synth_nomask  free running under each flag: outputs (max_iters or the stop rule ends the loop)
Dropout / zoneout masks are recorded in execution order and stored in the oracle's convention (keys "<tag>_mask_*")."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_reference_graph_vectors import REF, SMALL  # noqa: E402


def main():
    assert os.path.isdir(REF), "the reference tree is needed to (re)generate these fixtures"
    import tf_shim
    import tf_shim_graph as G
    G.install()
    sys.path.insert(0, REF)
    import hparams as ref_hparams_mod
    rhp = ref_hparams_mod.hparams
    from tacotron.models.tacotron import Tacotron

    for k, v in SMALL.items():
        setattr(rhp, k, v)
    R = np.load(os.path.join(HERE, "reference_graph.npz"))
    variables = {str(n): torch.from_numpy(R["var/" + str(n)]).clone() for n in R["var_names"] if "CBHG" not in str(n) and "cbhg" not in str(n)}
    inputs, in_len, tgt_len = (torch.from_numpy(R[k]) for k in ("inputs", "input_lengths", "targets_lengths"))
    mel, stop = torch.from_numpy(R["mel_targets"]), torch.from_numpy(R["stop_targets"])
    B, T_in = inputs.shape
    T_out = mel.shape[1]
    split_infos = np.array([[T_in, T_out * rhp.num_mels, T_out, T_out * rhp.num_freq]], dtype=np.int32)
    out = {}
    Tt = tf_shim.T
    rhp.predict_linear, rhp.mask_decoder = False, False

    def run(seed, **kw):
        G.reset(seed=seed, variables=variables)
        model = Tacotron(rhp)
        args = dict(mel_targets=Tt(mel.clone()), stop_token_targets=Tt(stop.clone()), targets_lengths=Tt(tgt_len.clone()),
                    split_infos=split_infos)
        args.update(kw)
        model.initialize(Tt(inputs.clone()), Tt(in_len.clone()), **{k: v for k, v in args.items() if v is not None})
        return model, list(G.S.drops)

    def save_masks(tag, drops, training, T_steps):
        """the recorded draws in execution order -> the oracle's masks (as make_reference_graph_vectors.py stores them)"""
        q = list(drops)
        H, D = rhp.encoder_lstm_units, rhp.decoder_lstm_units
        keep = 1.0 - rhp.tacotron_dropout_rate

        def pop(scope_part, kind, shape):
            scope, k, m = q.pop(0)
            assert scope_part in scope and k == kind and tuple(m.shape) == tuple(shape), (tag, scope, k, tuple(m.shape), scope_part, shape)
            return m
        if training:
            for i in range(rhp.enc_conv_num_layers):
                out["%s_mask_enc_drop_%d" % (tag, i)] = (pop("encoder_convolutions", "layers.dropout", (B, T_in, rhp.enc_conv_channels)) / keep).numpy()
            for d in ("fw", "bw"):
                c, h = torch.zeros(T_in, B, H), torch.zeros(T_in, B, H)
                for tau in range(T_in):
                    mc = pop("bidirectional_rnn/" + d, "nn.dropout", (B, H))
                    mh = pop("bidirectional_rnn/" + d, "nn.dropout", (B, H))
                    for b in range(B):
                        t = tau if d == "fw" else int(in_len[b]) - 1 - tau     # the backward pass runs per-length reversed
                        if 0 <= t < T_in and tau < int(in_len[b]):
                            c[t, b], h[t, b] = mc[b], mh[b]
                out["%s_mask_enc_zone_%s_c" % (tag, d)], out["%s_mask_enc_zone_%s_h" % (tag, d)] = c.numpy(), h.numpy()
        pre = [[], []]
        zone = {(l, s): [] for l in (1, 2) for s in "ch"}
        for _ in range(T_steps):
            for i, n in enumerate(rhp.prenet_layers):
                pre[i].append(pop("decoder_prenet", "layers.dropout", (B, n)) / keep)
            if training:
                for key in zone:
                    zone[key].append(pop("decoder_LSTM", "nn.dropout", (B, D)))
        for i in range(len(rhp.prenet_layers)):
            out["%s_mask_prenet_drop_%d" % (tag, i)] = torch.stack(pre[i], dim=1).numpy()
        if training:
            for (l, s), v in zone.items():
                out["%s_mask_dec_zone_%d_%s" % (tag, l, s)] = torch.stack(v).numpy()
            for i in range(rhp.postnet_num_layers):
                out["%s_mask_post_drop_%d" % (tag, i)] = (pop("postnet_convolutions", "layers.dropout",
                                                              (B, T_steps, rhp.postnet_channels)) / keep).numpy()
        assert not q, tag

    def save_outputs(tag, model):
        out[tag + "_decoder_output"] = model.tower_decoder_output[0].detach().numpy()
        out[tag + "_mel_outputs"] = model.tower_mel_outputs[0].detach().numpy()
        out[tag + "_alignments"] = model.tower_alignments[0].detach().numpy()                  # [B, T_in, T_out]
        out[tag + "_stop_token_prediction"] = model.tower_stop_token_prediction[0].detach().numpy()

    def save_losses(tag, model):
        model.add_loss()
        for k in ("before_loss", "after_loss", "stop_token_loss", "regularization_loss", "loss"):
            out["%s_%s" % (tag, k)] = np.asarray(float(getattr(model, k)), dtype=np.float64)

    flags = {"nocum": ("cumulative_weights", False), "nomask": ("mask_encoder", False)}
    for name, (flag, value) in flags.items():
        setattr(rhp, flag, value)
        tag = "train_nocum" if name == "nocum" else "train_nomask_g"
        model, drops = run(21 if name == "nocum" else 22, is_training=True, global_step=Tt(torch.tensor(0)))
        save_masks(tag, drops, True, T_out)
        save_outputs(tag, model)
        save_losses(tag, model)
        model.loss.backward()
        for k, v in G.S.vars.items():
            if v.requires_grad:
                out["%s_grad/%s" % (tag, k)] = (v.grad if v.grad is not None else torch.zeros_like(v)).detach().numpy()
        print("%s: loss %.6f" % (tag, float(model.loss)))
        model, drops = run(23, is_evaluating=True)
        save_masks("eval_" + name, drops, False, T_out)
        save_outputs("eval_" + name, model)
        save_losses("eval_" + name, model)
        model, drops = run(24, mel_targets=None, stop_token_targets=None, targets_lengths=None)
        steps = int(model.tower_mel_outputs[0].shape[1])
        save_masks("synth_" + name, drops, False, steps)
        save_outputs("synth_" + name, model)
        print("synth_%s: %d decoder steps" % (name, steps))
        setattr(rhp, flag, not value)

    path = os.path.join(HERE, "reference_attention.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d arrays, %.1f KB" % (path, len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
