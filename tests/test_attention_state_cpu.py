"""The attention-state flags mask_encoder=False and cumulative_weights=False without a GPU: the hparam checks, the config fields the
engine is built with, the ctypes mirror of t2_taco_config_t, the library's 0 / 1 check (it runs before any driver call; the null buffers
passed here are never touched) and the oracle against the executed reference graph under each flag (tests/golden/reference_attention.npz,
make_reference_attention_vectors.py), at the tolerances of tests/test_reference_graph.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

import t2_tf_bundle
from hparams import hparams
from oracle import tacotron as ot
from t2_import import t2

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TOL = 2e-5
FLAGS = {"nocum": dict(cumulative_weights=False), "nomask": dict(mask_encoder=False)}


def _hp(**kw):
    hp = hparams.copy()
    hp.set_hparam("predict_linear", False)
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return hp


@pytest.mark.parametrize("flags", [dict(mask_encoder=False), dict(cumulative_weights=False), dict(mask_encoder=False, cumulative_weights=False)])
def test_flags_are_accepted_and_reach_the_config(flags):
    hp = _hp(**flags)
    assert t2.tacotron.unsupported_hparams(hp) == []
    cfg = t2.tacotron.make_config(hp, 4, 40, 80)
    assert cfg.unmasked_encoder == int("mask_encoder" in flags)
    assert cfg.noncumulative_weights == int("cumulative_weights" in flags)


def test_default_config_keeps_the_masked_cumulative_attention():
    cfg = t2.tacotron.make_config(_hp(), 4, 40, 80)
    assert cfg.unmasked_encoder == 0 and cfg.noncumulative_weights == 0


@pytest.mark.parametrize("flag,value", [("smoothing", True), ("synthesis_constraint", True)])
def test_other_attention_variants_stay_rejected_with_one_reason(flag, value):
    hp = _hp(mask_encoder=False, cumulative_weights=False, **{flag: value})
    bad = t2.tacotron.unsupported_hparams(hp)
    assert len(bad) == 1 and bad[0].startswith(flag + "="), bad


def test_struct_mirror_has_the_flags_before_the_ratio():
    lib = t2.lib.load()
    lib.t2_struct_size.argtypes = [ctypes.c_char_p]
    C = t2.tacotron.TacoConfig
    assert lib.t2_struct_size(b"t2_taco_config_t") == ctypes.sizeof(C)
    assert C._fields_[-3:] == [("unmasked_encoder", ctypes.c_int), ("noncumulative_weights", ctypes.c_int),
                               ("teacher_forcing_ratio", ctypes.c_float)]
    assert C.teacher_forcing_ratio.offset + 4 == ctypes.sizeof(C)


@pytest.mark.parametrize("field,value", [("unmasked_encoder", 2), ("unmasked_encoder", -1), ("noncumulative_weights", 2),
                                         ("noncumulative_weights", -1)])
def test_library_rejects_flag_values_other_than_0_and_1_before_any_launch(field, value):
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    cfg = t2.tacotron.make_config(_hp(), 2, 40, 8)
    setattr(cfg, field, value)
    null = ctypes.c_void_p(0)
    n, pb, wb, nt = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    rcs = [lib.t2_taco_sizes(ctypes.byref(cfg), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(nt)),
           lib.t2_taco_forward(ctypes.byref(cfg), null, null, null, null, null, null, null, null, 1, ctypes.c_ulonglong(0), null, null),
           lib.t2_taco_forward(ctypes.byref(cfg), null, null, null, null, null, null, null, null, 0, ctypes.c_ulonglong(0), null, null),
           lib.t2_taco_backward(ctypes.byref(cfg), null, null, null, null, null, null, null, null, ctypes.c_ulonglong(0), null, null)]
    for rc in rcs:
        assert rc == -1, (field, value, rc, lib.t2_last_error())
        assert field.encode() in lib.t2_last_error()


def test_sizes_accept_every_flag_combination():
    lib = t2.lib.load()
    sizes = set()
    for um in (0, 1):
        for nc in (0, 1):
            cfg = t2.tacotron.make_config(_hp(), 2, 40, 8)
            cfg.unmasked_encoder, cfg.noncumulative_weights = um, nc
            n, pb, wb, nt = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
            assert lib.t2_taco_sizes(ctypes.byref(cfg), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(nt)) == 0
            sizes.add((n.value, pb.value, wb.value, nt.value))
    assert len(sizes) == 1          # the flags add no parameter and no workspace


@pytest.mark.parametrize("bad", [(2, 0), (0, 2)])
def test_att_fwd_hook_rejects_bad_flags_before_any_launch(bad):
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    c = t2.lib.DbgKernel()
    c.kernel = 1
    for k in range(15):
        c.p[k] = 16 * (k + 1)                    # never dereferenced: the check comes first
    for k, v in enumerate([2, 40, 256, 128, 31, 32, 512, 256, 512, 512, bad[0], bad[1]]):
        c.i[k] = v
    assert lib.t2_dbg_taco_kernel(ctypes.byref(c), None) == -1
    assert b"unmasked / noncumulative" in lib.t2_last_error()


def test_att_bwd_hook_checks_its_arguments_before_any_launch():
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    c = t2.lib.DbgKernel()
    c.kernel = 7
    for k in range(16):
        c.p[k] = 16 * (k + 1)
    good = [2, 40, 256, 128, 31, 512, 256, 768, 0, 0]
    for k, v in enumerate(good):
        c.i[k] = v
    c.i[8] = 3
    assert lib.t2_dbg_taco_kernel(ctypes.byref(c), None) == -1 and b"unmasked / noncumulative" in lib.t2_last_error()
    c.i[8] = 0
    c.p[8] = None                               # the cumulative state is required unless non-cumulative
    assert lib.t2_dbg_taco_kernel(ctypes.byref(c), None) == -1 and b"cumrun" in lib.t2_last_error()
    c.p[8] = 16 * 9
    c.i[1] = 400                                # T_in past the shared-memory limit of the backward
    assert lib.t2_dbg_taco_kernel(ctypes.byref(c), None) != 0 and b"shared memory" in lib.t2_last_error()
    c.i[1] = 40
    c.p[12] = None
    assert lib.t2_dbg_taco_kernel(ctypes.byref(c), None) == -1 and b"null pointer argument 12" in lib.t2_last_error()


# ---- the oracle against the executed reference ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def R():
    return np.load(os.path.join(GOLDEN, "reference_attention.npz"))


@pytest.fixture(scope="module")
def G():
    return np.load(os.path.join(GOLDEN, "reference_graph.npz"))


def _ref_hp(G, **kw):
    hp = hparams.copy()
    for k, v in zip(G["small_hparams_keys"], G["small_hparams_values"]):
        setattr(hp, str(k), eval(str(v)))
    hp.predict_linear, hp.mask_decoder = False, False
    for k, v in kw.items():
        setattr(hp, k, v)
    return hp


def _params(G):
    out = {}
    for name in G["var_names"]:
        eng = t2_tf_bundle.engine_name("Tacotron_model/" + str(name))
        if "CBHG" not in eng and "cbhg" not in eng:
            out[eng] = torch.from_numpy(G["var/" + str(name)]).clone()
    return out


def _inputs(G):
    return (torch.from_numpy(G["inputs"]).long(), torch.from_numpy(G["input_lengths"]).long(), torch.from_numpy(G["mel_targets"]),
            torch.from_numpy(G["stop_targets"]))


def _masks(R, tag, training, hp):
    m = {"prenet_drop": [torch.from_numpy(R["%s_mask_prenet_drop_%d" % (tag, i)]) for i in range(len(hp.prenet_layers))]}
    if training:
        for i in range(hp.enc_conv_num_layers):
            m[("enc_drop", i)] = torch.from_numpy(R["%s_mask_enc_drop_%d" % (tag, i)])
        for i in range(hp.postnet_num_layers):
            m[("post_drop", i)] = torch.from_numpy(R["%s_mask_post_drop_%d" % (tag, i)])
        ez, dz = {}, {}
        for d in ("fw", "bw"):
            for s in "ch":
                a = torch.from_numpy(R["%s_mask_enc_zone_%s_%s" % (tag, d, s)])
                for t in range(a.shape[0]):
                    ez[(d, s, t)] = a[t]
        for l in (1, 2):
            for s in "ch":
                a = torch.from_numpy(R["%s_mask_dec_zone_%d_%s" % (tag, l, s)])
                for t in range(a.shape[0]):
                    dz[(l, s, t)] = a[t]
        m["enc_zone"], m["dec_zone"] = ez, dz
    return m


def _close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() if a.size else 0.0
    assert err <= tol * max(1.0, np.abs(b).max()), err
    return err


def _check_outputs(R, tag, out, stop_is_logit):
    _close(out["decoder_output"].detach(), R[tag + "_decoder_output"])
    _close(out["mel_outputs"].detach(), R[tag + "_mel_outputs"])
    _close(out["alignments"].detach().transpose(1, 2), R[tag + "_alignments"])
    _close(out["stop_logits" if stop_is_logit else "stop_token_prediction"].detach(), R[tag + "_stop_token_prediction"])


def _check_losses(R, tag, parts):
    for k, ref in (("before", "before_loss"), ("after", "after_loss"), ("stop", "stop_token_loss"), ("reg", "regularization_loss")):
        v = float(R["%s_%s" % (tag, ref)])
        assert abs(float(parts[k].detach()) - v) <= 1e-5 * max(1e-3, abs(v)), (tag, k)


@pytest.mark.parametrize("tag,name", [("train_nocum", "nocum"), ("train_nomask_g", "nomask")])
def test_training_under_each_flag_matches_the_executed_reference(R, G, tag, name):
    """outputs, losses and d loss / d variable for every trainable variable, every dropout / zoneout mask injected"""
    hp = _ref_hp(G, **FLAGS[name])
    params = {k: v.requires_grad_(ot.is_trainable(k)) for k, v in _params(G).items()}
    ids, in_len, mel, stop = _inputs(G)
    out = ot.forward(params, ids, in_len, mel, hp, training=True, masks=_masks(R, tag, True, hp))
    _check_outputs(R, tag, out, True)
    total, parts = ot.loss_fn(out, mel, stop, params, hp)
    _check_losses(R, tag, parts)
    total.backward()
    floor = 1e-3 * max(np.abs(R[k]).max() for k in R.files if k.startswith(tag + "_grad/"))
    n = 0
    for name_tf in G["var_names"]:
        eng = t2_tf_bundle.engine_name("Tacotron_model/" + str(name_tf))
        key = "%s_grad/%s" % (tag, name_tf)
        if key not in R.files:
            continue
        g = params[eng].grad
        g = torch.zeros_like(params[eng]) if g is None else g
        ref = R[key]
        err = np.abs(g.numpy() - ref).max()
        assert err <= 2e-4 * max(np.abs(ref).max(), floor), (eng, err, np.abs(ref).max())
        n += 1
    assert n >= 30
    a = out["alignments"].detach()
    pad = torch.arange(a.shape[2])[None, :] >= in_len[:, None]
    if name == "nomask":
        assert float(a[1][:, pad[1]].min()) > 0                        # attention mass on the padding
    else:
        assert float(a[1][:, pad[1]].abs().max()) == 0


@pytest.mark.parametrize("name", ["nocum", "nomask"])
def test_evaluation_and_synthesis_under_each_flag_match_the_executed_reference(R, G, name):
    hp = _ref_hp(G, **FLAGS[name])
    params = _params(G)
    ids, in_len, mel, stop = _inputs(G)
    assert len(set(in_len.tolist())) > 1                                # rows of unequal length
    with torch.no_grad():
        out = ot.forward(params, ids, in_len, mel, hp, training=False, masks=_masks(R, "eval_" + name, False, hp))
        _check_outputs(R, "eval_" + name, out, True)
        _, parts = ot.loss_fn(out, mel, stop, params, hp)
        _check_losses(R, "eval_" + name, parts)
        tag = "synth_" + name
        pm = _masks(R, tag, False, hp)["prenet_drop"]
        steps = R[tag + "_mel_outputs"].shape[1]
        syn = ot.synthesize(params, ids, in_len, hp, prenet_masks=[[m[:, t] for m in pm] for t in range(steps)])
        _check_outputs(R, tag, syn, False)
