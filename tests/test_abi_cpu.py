"""CPU-side checks of the C-ABI: the in-tree library loads, exports every function include/t2b200.h declares, reports
errors through return codes (no GPU compute is launched here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "t2b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(t2_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from t2_import import t2
    lib = t2.lib.load()
    names = _declared()
    assert len(names) >= 30
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.t2_abi_version() == 3


def test_errors_are_return_codes_with_messages():
    from t2_import import t2
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    cfg = t2.wavenet.WnConfig()          # all zeros: invalid
    sz = t2.wavenet.WnSizes()
    rc = lib.t2_wn_sizes(ctypes.byref(cfg), ctypes.byref(sz))
    assert rc < 0 and len(lib.t2_last_error()) > 0
    with pytest.raises(t2.lib.T2Error):
        t2.lib.check(rc)


def test_layout_queries_match_the_oracle_parameter_tables():
    """host logic without a GPU: the C++ layout enumerates the same (name, shape) list as the oracle"""
    from hparams import hparams, paper_hparams
    from oracle import tacotron as ot
    from oracle import wavenet as ow
    from t2_import import t2
    lib = t2.lib.load()
    hp = paper_hparams()
    hp.parse("input_type=mulaw-quantize,quantize_channels=256,out_channels=256,upsample_type=SubPixel,upsample_scales=[11,25]")
    cfg = t2.wavenet.make_config(hp, 2, 275 * 4)
    sz = t2.wavenet.WnSizes()
    t2.lib.check(lib.t2_wn_sizes(ctypes.byref(cfg), ctypes.byref(sz)))
    name = ctypes.create_string_buffer(160)
    off, nd, shp = ctypes.c_longlong(), ctypes.c_int(), (ctypes.c_int * 4)()
    got = []
    for i in range(sz.n_tensors):
        t2.lib.check(lib.t2_wn_param_info(ctypes.byref(cfg), i, name, 160, ctypes.byref(off), ctypes.byref(nd), shp))
        got.append((name.value.decode(), tuple(shp[k] for k in range(nd.value))))
    assert got == [(k, tuple(v)) for k, v in ow.param_shapes(hp).items()]
    hp2 = hparams.copy()
    hp2.set_hparam("predict_linear", False)
    tc = t2.tacotron.make_config(hp2, 4, 40, 80)
    n, pb, wb, nt, tr = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int(), ctypes.c_int()
    t2.lib.check(lib.t2_taco_sizes(ctypes.byref(tc), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(nt)))
    got = []
    for i in range(nt.value):
        t2.lib.check(lib.t2_taco_param_info(ctypes.byref(tc), i, name, 160, ctypes.byref(off), ctypes.byref(nd), shp, ctypes.byref(tr)))
        got.append((name.value.decode(), tuple(shp[k] for k in range(nd.value)), bool(tr.value)))
    assert got == [(k, tuple(v), ot.is_trainable(k)) for k, v in ot.param_shapes(hp2).items()]
    hp3 = hparams.copy()
    hp3.set_hparam("predict_linear", True)
    cc = t2.tacotron.make_cbhg_config(hp3, 4, 80, 0.0)
    t2.lib.check(lib.t2_cbhg_sizes(ctypes.byref(cc), None, None, None, ctypes.byref(nt)))
    got = [(k, shape, trainable) for k, _, shape, trainable in t2.lib.param_table(lib.t2_cbhg_param_info, cc, nt.value)]
    cbhg = list(ot.param_shapes(hp3).items())[len(ot.param_shapes(hp2)):]
    assert len(cbhg) > 0 and got == [(k, tuple(v), ot.is_trainable(k)) for k, v in cbhg]


def test_product_path_has_no_oracle_import():
    """the shipped package must never route through the CPU oracle"""
    pkg = os.path.join(ROOT, "tacotron-2_b200")
    for f in os.listdir(pkg):
        if f.endswith(".py"):
            assert not re.search(r"^\s*(from|import)\s+oracle", open(os.path.join(pkg, f)).read(), re.M), f
    assert not re.search(r"^\s*(from|import)\s+oracle", open(os.path.join(ROOT, "datasets", "audio.py")).read(), re.M)


def test_product_initialiser_matches_reference_init_rules():
    """tacotron-2_b200/init.py (product side): same NN_init upsampling kernels as the oracle, glorot limits, unit batch-norm"""
    import math

    import torch
    from hparams import hparams, paper_hparams
    from oracle import tacotron as ot
    from oracle import wavenet as ow
    from t2_import import t2
    for hp in (paper_hparams(), hparams.copy()):
        tens = [(k, 0, tuple(v)) for k, v in ow.param_shapes(hp).items()]
        a, b = t2.init.wavenet_variables(hp, tens, 7), ow.init_params(hp, seed=7)
        for k in b:
            assert a[k].shape == b[k].shape
            if k.endswith("bias"):
                assert a[k].abs().max() == 0
            elif "upsampling" in k:
                assert torch.equal(a[k], b[k]), k
    k = "residual_block_causal_conv_ResidualConv1DGLU_3/kernel"
    kk = [n for n in a if n.endswith("kernel") and a[n].dim() == 3 and a[n].shape[0] == 3][0]
    kw, cin, cout = a[kk].shape
    lim = math.sqrt(6.0 / (kw * cin + kw * cout))
    assert a[kk].abs().max() <= lim and a[kk].abs().max() > 0.95 * lim
    hp = hparams.copy()
    hp.set_hparam("predict_linear", False)
    tens = [(n, 0, tuple(v), ot.is_trainable(n)) for n, v in ot.param_shapes(hp).items()]
    p = t2.init.tacotron_variables(hp, tens, 3)
    assert all((p[n] == 1).all() for n in p if n.endswith(("gamma", "moving_variance")))
    assert all((p[n] == 0).all() for n in p if n.endswith(("beta", "moving_mean", "bias")))
    e = p["inputs_embedding"]
    assert e.abs().max() <= math.sqrt(6.0 / sum(e.shape))


def test_reference_python_surface_validates_like_the_reference():
    """create_model / initialize argument checks fire before any GPU work (tacotron.py:41-54, wavenet models/__init__.py:6-9)"""
    import torch
    from hparams import hparams
    from tacotron.models import create_model as create_taco
    from wavenet_vocoder.models import create_model as create_wn
    from wavenet_vocoder import util
    with pytest.raises(Exception, match="Unknown model"):
        create_taco("Tacotron3", hparams)
    with pytest.raises(Exception, match="Unknow model"):
        hp = hparams.copy()
        hp.parse("input_type=raw,out_channels=30")
        create_wn("WaveRNN", hp)
    bad = hparams.copy()
    bad.parse("input_type=mulaw-quantize,quantize_channels=256,out_channels=30")
    with pytest.raises(RuntimeError):
        create_wn("WaveNet", bad)
    m = create_taco("Tacotron", hparams)
    ids, lens = torch.zeros(2, 5, dtype=torch.int32), torch.tensor([5, 4])
    mel, stop = torch.zeros(2, 7, hparams.num_mels), torch.zeros(2, 7)
    with pytest.raises(ValueError):
        m.initialize(ids, lens, stop_token_targets=stop)                    # stop targets without mel targets
    with pytest.raises(ValueError):
        m.initialize(ids, lens, mel_targets=mel)                            # mel targets without stop targets
    with pytest.raises(ValueError):
        m.initialize(ids, lens, mel, stop, is_training=True)                # predict_linear=True (default) without linear targets
    hp_mel = hparams.copy()
    hp_mel.set_hparam("predict_linear", False)
    with pytest.raises(RuntimeError):
        create_taco("Tacotron", hp_mel).initialize(ids, lens, mel, stop, is_training=True, is_evaluating=True)
    with pytest.raises(ValueError):
        m.initialize(ids, lens, mel, gta=True, linear_targets=mel)
    assert util.is_mulaw_quantize("mulaw-quantize") and util.is_scalar_input("raw") and not util.is_raw("mulaw")
    with pytest.raises(AssertionError):
        util.is_mulaw("pcm")
    mask = util.sequence_mask([3, 1], max_len=4, expand=False)
    assert mask.tolist() == [[1, 1, 1, 0], [1, 0, 0, 0]] and util.sequence_mask([2, 1]).shape == (2, 2, 1)


def test_ctypes_struct_mirrors_match_the_library():
    """every POD struct that crosses the C-ABI has the same size in the Python mirror (field order is checked by the GPU tests)"""
    import ctypes
    from t2_import import t2
    lib = t2.lib.load()
    lib.t2_struct_size.argtypes = [ctypes.c_char_p]
    pairs = {"t2_wn_config_t": t2.wavenet.WnConfig, "t2_wn_sizes_t": t2.wavenet.WnSizes, "t2_taco_config_t": t2.tacotron.TacoConfig,
             "t2_cbhg_config_t": t2.tacotron.CbhgConfig, "t2_audio_config_t": t2.audio.AudioConfig,
             "t2_dbg_act_t": t2.lib.DbgAct, "t2_dbg_gemm_t": t2.lib.DbgGemm, "t2_dbg_wgrad_tile_t": t2.lib.DbgWgradTile,
             "t2_dbg_kernel_t": t2.lib.DbgKernel}
    for name, mirror in pairs.items():
        assert lib.t2_struct_size(name.encode()) == ctypes.sizeof(mirror), name
    assert lib.t2_struct_size(b"nope") == -1


def test_split_k_rejects_non_atomic_output_modes():
    """Split-K makes several CTAs add partial sums into the same output elements, so every destination in use must take mode 2
    (atomic add). The check runs before any driver call. Nothing is launched: the rejected calls stop at the split-K check, and the
    calls that pass it have a null weight pointer, which the weight tensor-map encoding refuses before any launch (on a host without a
    driver the activation map encoding already fails). The fake pointers are never dereferenced."""
    from t2_import import t2
    lib = t2.lib.load()
    EPI_TOUT = 9
    fake = 1 << 20                                     # 16-byte aligned, never touched

    def call(ksplit, mode0, mode1, dst1=True, rows0=64, rows1=128, epi=EPI_TOUT, w=fake):
        c = t2.lib.DbgGemm()
        c.a[0] = t2.lib.DbgAct(fake, 512, 128, 1, 1, 512)
        c.na = 1
        c.seg[0] = t2.lib.DbgSeg(0, 0, 0, 8, 0, 1)
        c.nseg = 1
        c.w, c.wN, c.wK, c.wL = w, 32, 512, 1
        c.T, c.B, c.n_tiles, c.ksplit, c.epi, c.BN = 128, 1, 1, ksplit, epi, 32
        c.ptr[0], c.ptr[1] = fake, (fake if dst1 else None)
        c.i[0], c.i[1], c.i[2], c.i[3], c.i[4], c.i[5], c.i[6] = rows0, 32, mode0, rows1, 32, mode1, 32
        return lib.t2_dbg_act_gemm(ctypes.byref(c), None)

    for m0, m1 in [(0, 2), (1, 2), (2, 0), (2, 1), (0, 0), (1, 1)]:
        rc = call(4, m0, m1)
        assert rc == -1, (m0, m1, rc)
        assert b"split-K" in lib.t2_last_error(), lib.t2_last_error()
    # accepted by the split-K check (an unused destination's mode is not checked), then refused for the null weight pointer
    for kw in (dict(dst1=False), dict(rows1=64), {}):
        mode1 = 2 if not kw else 0
        rc = call(4, 2, mode1, w=None, **kw)
        assert rc != 0 and b"split-K" not in lib.t2_last_error(), (kw, rc, lib.t2_last_error())
    assert call(4, 2, 2, epi=2) == -1 and b"split-K" in lib.t2_last_error()           # split-K with a non-accumulating epilogue
    assert call(16, 2, 2) == -1 and b"split-K" in lib.t2_last_error()                  # fewer k-blocks (8) than slices


def test_act_gemm_rejects_bad_cluster_and_segments():
    """argument checks of the engine hook that need no device"""
    from t2_import import t2
    lib = t2.lib.load()
    fake = 1 << 20
    c = t2.lib.DbgGemm()
    c.a[0] = t2.lib.DbgAct(fake, 64, 128, 1, 1, 64)
    c.na, c.nseg = 1, 1
    c.seg[0] = t2.lib.DbgSeg(0, 0, 0, 1, 0, 1)
    c.w, c.wN, c.wK, c.wL = fake, 128, 64, 1
    c.T, c.B, c.n_tiles, c.epi, c.BN = 128, 1, 1, 2, 128
    c.cluster = 3
    assert lib.t2_dbg_act_gemm(ctypes.byref(c), None) == -1 and b"cluster" in lib.t2_last_error()
    c.cluster = 0
    c.seg[0] = t2.lib.DbgSeg(1, 0, 0, 1, 0, 1)                 # map 1 of 1
    assert lib.t2_dbg_act_gemm(ctypes.byref(c), None) == -1 and b"segment" in lib.t2_last_error()
    c.seg[0] = t2.lib.DbgSeg(0, 0, 0, 2, 0, 1)                 # 2 k-blocks, weight has 1
    assert lib.t2_dbg_act_gemm(ctypes.byref(c), None) == -1 and b"packed weight" in lib.t2_last_error()


def test_training_rejects_t_in_past_the_attention_backward_limit():
    """The attention backward keeps a [T_in + KA - 1][A + 8] fp32 tile in shared memory, which at attention_dim 128 / kernel 31 holds
    T_in <= 336 within the 232,448 B per-block limit. A training forward or backward past that returns T2_ERR_UNSUPPORTED_SHAPE with a
    message naming the limit, before any driver call: the null buffers here are never touched. Only refused shapes are passed, so
    nothing can be launched."""
    from hparams import hparams
    from t2_import import t2
    lib = t2.lib.load()
    hp = hparams.copy()
    hp.set_hparam("predict_linear", False)
    null = ctypes.c_void_p(0)
    for T_in in (337, 1024):
        cfg = t2.tacotron.make_config(hp, 2, T_in, 8)
        assert (cfg.attention_dim, cfg.attention_kernel) == (128, 31)
        rcs = [lib.t2_taco_forward(ctypes.byref(cfg), null, null, null, null, null, null, null, null, 1, ctypes.c_ulonglong(0), null, null),
               lib.t2_taco_backward(ctypes.byref(cfg), null, null, null, null, null, null, null, null, ctypes.c_ulonglong(0), null, null)]
        for rc in rcs:
            assert rc == -2, (T_in, rc, lib.t2_last_error())
            msg = lib.t2_last_error()
            assert b"T_in <= 336" in msg and b"232448" in msg, msg


def _taco_hook(kernel, p, i, f=()):
    from t2_import import t2
    lib = t2.lib.load()
    c = t2.lib.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = v
    for k, v in enumerate(i):
        c.i[k] = v
    for k, v in enumerate(f):
        c.f[k] = v
    return lib.t2_dbg_taco_kernel(ctypes.byref(c), None), lib.t2_last_error()


# the fp32-class (split-bf16) hooks of tests/test_split_operands_gpu.py: each call below breaks exactly one argument of an otherwise
# valid launch, and is refused before any driver call (the fake pointers are never dereferenced)
_FAKE = [16 * (k + 1) for k in range(16)]
CONV_GOOD = [128, 40, 2, 128, 3 * 3 * 128, 3, 128, 0, 128, 128, 0, 1, 0]   # C, T, Bn, N, wK, ntaps, BN, act, ldo, nvalid, stream, split, row0
LSTM_GOOD = [64, 64, 2, 256, 192, 192, 256, 0, 0, 128, 0, 1, 1]            # H, K, B, pre_stride, ld_hp, ld_hs, ld_ho, t, stream, out_lo,
                                                                           # out_state, training, split
ATT_GOOD = [2, 40, 256, 128, 31, 32, 512, 520, 1040 + 512, 1040, 0, 0, 1, 264, 520, 520]


@pytest.mark.parametrize("k,v,msg", [(5, 9, b"tap count"), (5, 0, b"tap count"), (11, 2, b"split flag"), (6, 64, b"bad shape"),
                                     (4, 3 * 3 * 128 - 8, b"bad shape"), (7, 3, b"bad shape"), (9, 129, b"bad shape"),
                                     (8, 120, b"bad shape"), (12, -1, b"bad shape")])
def test_conv_gemm_hook_rejects_bad_arguments(k, v, msg):
    """ntaps = 9 is 18 segments in split mode, more than kMaxSeg = 16"""
    i = list(CONV_GOOD)
    i[k] = v
    rc, err = _taco_hook(8, _FAKE[:5], i)
    assert rc == -1 and msg in err, err


def test_conv_gemm_hook_needs_an_output_and_nine_taps_are_fine_only_in_bf16_mode():
    i = list(CONV_GOOD)
    rc, err = _taco_hook(8, _FAKE[:3] + [0, 0], i)
    assert rc == -1 and b"bad pointers" in err
    i[5], i[4], i[11] = 9, 9 * 128, 0
    i[0] = 100                                    # bf16 mode: 9 segments pass the tap check; C % 8 != 0 is refused next
    rc, err = _taco_hook(8, _FAKE[:5], i)
    assert rc == -1 and b"bad shape" in err, err


@pytest.mark.parametrize("k,v,msg", [(12, 2, b"flags"), (11, 2, b"flags"), (10, 2, b"flags"), (0, 48, b"pitch"), (1, 96, b"pitch"),
                                     (4, 64 + 63, b"pitch"), (5, 128 + 63, b"pitch"), (9, 63, b"pitch"), (6, 128 + 63, b"pitch"),
                                     (3, 255, b"pitch"), (7, -1, b"flags")])
def test_lstm_step_hook_rejects_bad_arguments(k, v, msg):
    i = list(LSTM_GOOD)
    i[k] = v
    rc, err = _taco_hook(9, _FAKE[:12], i, [0.1])
    assert rc == -1 and msg in err, err


def test_lstm_step_hook_rejects_split_offsets_in_bf16_mode_and_a_bad_zoneout_rate():
    i = list(LSTM_GOOD)
    i[12] = 0                                     # bf16 mode with out_lo / out_state set
    rc, err = _taco_hook(9, _FAKE[:12], i, [0.1])
    assert rc == -1 and b"pitch" in err, err
    rc, err = _taco_hook(9, _FAKE[:12], LSTM_GOOD, [1.0])
    assert rc == -1 and b"flags" in err, err


@pytest.mark.parametrize("k,v", [(12, 2), (13, 255), (15, 511), (14, 511), (9, 1031), (7, 519)])
def test_att_fwd_hook_checks_the_split_offsets(k, v):
    i = list(ATT_GOOD)
    i[k] = v
    rc, err = _taco_hook(1, _FAKE[:15], i)
    assert rc == -1 and b"lo offsets" in err, err


def test_att_fwd_hook_rejects_lo_offsets_in_bf16_mode_and_rows_rejects_a_bad_writer():
    i = list(ATT_GOOD)
    i[12] = 0
    rc, err = _taco_hook(1, _FAKE[:15], i)
    assert rc == -1 and b"lo offsets" in err, err
    rc, err = _taco_hook(10, _FAKE[:8], [5, 1, 2, 8, 80])
    assert rc == -1 and b"bad writer" in err, err
    rc, err = _taco_hook(10, _FAKE[:8], [1, 1, 2, 8, 129])        # split decoder-input rows hold at most 128 mels per half
    assert rc == -1 and b"decin" in err, err


def _cbhg_hook(kernel, p, i, f=()):
    from t2_import import t2
    lib = t2.lib.load()
    c = t2.lib.DbgKernel()
    c.kernel = kernel
    for k, v in enumerate(p):
        c.p[k] = v
    for k, v in enumerate(i):
        c.i[k] = v
    for k, v in enumerate(f):
        c.f[k] = v
    return lib.t2_dbg_cbhg_kernel(ctypes.byref(c), None), lib.t2_last_error()


# the loss / parameter-table hooks of tests/test_taco_loss_kernels_gpu.py: one broken argument each, refused before any driver call
LOSS_GOOD = {0: [0, 2, 5, 80, 1], 1: [1, 2, 5, 80, 0], 2: [2, 2, 5, 80, 1], 3: [3, 2, 5, 80, 1, 0, 5], 4: [4, 10, 80], 5: [5, 100],
             6: [6, 10, 512], 7: [7, 2, 5, 512], 8: [8, 100, 80, 128, 256]}


@pytest.mark.parametrize("i,p_null,msg", [
    ([0, 2, 5, 128, 1], None, b"bad shape"), ([2, 2, 5, 80, 2], None, b"clip flag"), ([0, 0, 5, 80, 1], None, b"bad shape"),
    (LOSS_GOOD[0], 0, b"mel_finish: null"), (LOSS_GOOD[1], 0, b"loss_norm: null"), (LOSS_GOOD[2], 7, b"loss_seed: null"),
    ([3, 2, 5, 80, 1, 3, 3], None, b"step range"), ([3, 2, 5, 80, 1, 0, 6], None, b"step range"), (LOSS_GOOD[3], 8, b"choice is required"),
    ([4, 10, 128], None, b"proj_bias"), (LOSS_GOOD[4], 2, b"proj_bias"), ([5, 0], None, b"relu_drop_bwd"), ([6, 10, 0], None, b"embed_bwd"),
    (LOSS_GOOD[7], 1, b"mask_values"), ([8, 100, 80, 64, 256], None, b"bias_colsum"), ([8, 100, 80, 128, 64], None, b"bias_colsum"),
    ([9, 1, 1, 1, 1], None, b"selector")])
def test_loss_hook_rejects_bad_arguments(i, p_null, msg):
    p = list(_FAKE[:9])
    if p_null is not None:
        p[p_null] = 0
    rc, err = _taco_hook(11, p, i, [-4.1, 4.0, 1.0])
    assert rc == -1 and msg in err, err


def test_loss_hook_accepts_nothing_but_the_documented_rates_and_lengths():
    rc, err = _taco_hook(11, _FAKE[:3], [5, 100], [1.0])              # relu_drop_bwd: dropout rate 1 divides by 0
    assert rc == -1 and b"relu_drop_bwd" in err, err
    rc, err = _taco_hook(11, _FAKE[:3], [6, 0, 8])
    assert rc == -1 and b"embed_bwd" in err, err


PACK_GOOD = [0, 4096, 32, 32, 0, 64, 128, 0, 64, 1, 0, 32, 0]         # -, bytes, W, grid_x, src, K, N, dst, ld, transpose, col0, perm, part
PACK_SPLIT_GOOD = [1, 4096, 32, 32, 0, 64, 128, 0, 192, 0, 128, 64, 32]  # -, bytes, W, grid_x, src, K, N, dst, ld, col_hi, col_lo, slot, perm


@pytest.mark.parametrize("split,k,v,msg", [
    (0, 11, 16, b"gate permutation"), (0, 11, 64, b"gate permutation"), (0, 9, 0, b"gate permutation"), (0, 6, 129, b"gate permutation"),
    (0, 2, 64, b"bad arguments"), (0, 12, 1, b"bad arguments"), (0, 5, 0, b"bad arguments"), (0, 3, 0, b"bad arguments"),
    (0, 8, 63, b"leading dimension"), (0, 1, 47, b"job buffer"), (1, 12, 96, b"gate permutation"), (1, 2, 128, b"gate permutation"),
    (1, 8, 191, b"leading dimension"), (1, 1, 143, b"job buffer"), (1, 11, -1, b"bad arguments")])
def test_pack_hook_rejects_bad_jobs(split, k, v, msg):
    """a gate permutation must transpose, with N = gates * perm and perm % W == 0 (W = 32: 4 gates, W = 128: 2 halves); a PackJob is
    48 bytes, so one job needs 48 B of job buffer and a split triple 144 B"""
    i = list(PACK_SPLIT_GOOD if split else PACK_GOOD)
    i[k] = v
    rc, err = _taco_hook(12, _FAKE[:3], i, [1.0])
    assert rc == -1 and msg in err, err


def test_params_hook_rejects_null_pointers_and_empty_tables():
    rc, err = _taco_hook(12, [_FAKE[0], 0, _FAKE[2]], PACK_GOOD, [1.0])
    assert rc == -1 and b"pack: bad arguments" in err, err
    for which in (2, 3):
        rc, err = _taco_hook(12, _FAKE[:3], [which, 0], [1e-6])
        assert rc == -1 and b"reg" in err, err
        rc, err = _taco_hook(12, [_FAKE[0], 0, _FAKE[2]], [which, 4], [1e-6])
        assert rc == -1 and b"reg" in err, err
    rc, err = _taco_hook(12, _FAKE[:3], [4, 1])
    assert rc == -1 and b"selector" in err, err


LIN_GOOD = [2, 5, 1025, 1032, 185, 1]                                # B, T, NF, NFP, n_prio, clip


@pytest.mark.parametrize("k,v", [(3, 1024), (4, 0), (4, 1026), (5, 2), (0, 0), (1, 0), (2, 0)])
def test_linear_hook_rejects_bad_arguments(k, v):
    i = list(LIN_GOOD)
    i[k] = v
    rc, err = _cbhg_hook(9, _FAKE[:6], i, [-4.1, 4.0, 1e-6])
    assert rc == -1 and b"LINEAR" in err, err


def test_linear_and_add_hooks_reject_null_pointers_and_bad_selectors():
    for null in (0, 3):
        p = list(_FAKE[:6])
        p[null] = 0
        rc, err = _cbhg_hook(9, p, LIN_GOOD, [-4.1, 4.0, 1e-6])
        assert rc == -1 and b"LINEAR" in err, err
    rc, err = _cbhg_hook(10, _FAKE[:5], [2, 10])
    assert rc == -1 and b"selector" in err, err
    rc, err = _cbhg_hook(10, [0] + _FAKE[1:3], [0, 10])
    assert rc == -1 and b"add_k" in err, err
    rc, err = _cbhg_hook(10, _FAKE[:5], [1, 10, 129])
    assert rc == -1 and b"dmel_k" in err, err
    rc, err = _cbhg_hook(10, _FAKE[:4] + [0], [1, 10, 80])
    assert rc == -1 and b"dmel_k" in err, err
