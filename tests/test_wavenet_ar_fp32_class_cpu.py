"""Fast-WaveNet AR synthesis in the fp32-class mode (split_bf16 = 1), host side: the packed-weight and workspace sizes, the launch plan
with 4-byte weight slots, the synthesizer's precision argument, and argument checks that return before any launch. No device needed.

The fp32-class mode stores the synthesis weights as plain fp32 (4 bytes per weight, slice-major as in the bf16 mode) and reads the
conditioning in fp32 where it lies, so it needs no bf16 c_up block in the workspace. The bf16 mode's sizes are pinned to the values the
library reported before the fp32-class mode existed."""
import ctypes

import pytest

from hparams import hparams
from paper_hparams import hparams as paper_hparams
from t2_import import t2
from wavenet_ar_kernel_size_reference import launch_plan as ks_launch_plan
from wavenet_ar_reference import SMEM_LIMIT
from wavenet_ar_reference import launch_plan as bf16_launch_plan

WN = t2.wavenet
INVALID_ARG, UNSUPPORTED_SHAPE = -1, -2
B, T = 2, 2750                       # T a multiple of the hop size (275) of both configurations

# (packed_bytes, workspace_bytes) of t2_wn_ar_sizes in the bf16 mode at B 2, T 2750
BF16_SIZES = {
    "default-gin0-cs1": (6127112, 11091200), "default-gin0-cs8": (6128672, 11091200), "default-gin0-cs16": (6130752, 11091200),
    "default-gin16-cs1": (6127112, 11132160), "default-gin16-cs8": (6128672, 11132160), "default-gin16-cs16": (6130752, 11132160),
    "paper-gin0-cs1": (27354232, 4896768), "paper-gin0-cs8": (27355264, 4896768), "paper-gin0-cs16": (27355264, 4896768),
    "paper-gin16-cs1": (27354232, 4995072), "paper-gin16-cs8": (27355264, 4995072), "paper-gin16-cs16": (27355264, 4995072),
    "ks2-gin0-cs1": (4816392, 6900992), "ks2-gin0-cs8": (4817952, 6900992), "ks2-gin0-cs16": (4820032, 6900992),
    "ks2-gin16-cs1": (4816392, 6941952), "ks2-gin16-cs8": (4817952, 6941952), "ks2-gin16-cs16": (4820032, 6941952),
    "ks4-gin0-cs1": (7437832, 11091200), "ks4-gin0-cs8": (7439392, 11091200), "ks4-gin0-cs16": (7441472, 11091200),
    "ks4-gin16-cs1": (7437832, 11132160), "ks4-gin16-cs8": (7439392, 11132160), "ks4-gin16-cs16": (7441472, 11132160),
}


def _hp(name, gin=0):
    hp = (paper_hparams if name == "paper" else hparams).copy()
    if name in ("ks2", "ks4"):
        hp.set_hparam("kernel_size", int(name[2]))
    if gin:
        hp.parse("gin_channels=%d,n_speakers=4" % gin)
    return hp


def _sizes(cfg, cs):
    pb, wb = ctypes.c_longlong(), ctypes.c_longlong()
    t2.lib.check(t2.lib.load().t2_wn_ar_sizes(ctypes.byref(cfg), cs, ctypes.byref(pb), ctypes.byref(wb)))
    return pb.value, wb.value


def _align(n):
    return -(-n // 256) * 256


def n_weights(hp, cs):
    """synthesis weights of ar_pack_kernel: per (layer, rank) slice 2 ZC rows of K1 = k R + cin, then RC + SC rows of Gh; the two
    head blocks"""
    R, Gh, S, C, L = hp.residual_channels, hp.gate_channels // 2, hp.skip_out_channels, hp.cin_channels, hp.layers
    K1 = hp.kernel_size * R + C
    per_rank_layer = 2 * (Gh // cs) * K1 + (R // cs + S // cs) * Gh
    return per_rank_layer * cs * L + S * S + cs * -(-hp.out_channels // cs) * S, per_rank_layer


def launch_plan_fp32(hp, B, cs, sms, prefetch_env=True):
    """t2_wn_ar_generate's launch choices in the fp32-class mode: as in the bf16 mode (wavenet_ar_kernel_size_reference.launch_plan)
    except that each per-layer weight slot holds 4-byte weights, so the double-buffered shared-memory prefetch needs twice the room.
    prefetch_env=False mirrors T2_AR_PREFETCH=0."""
    plan = ks_launch_plan(hp, B, cs, sms)
    R, G, S, C, L = hp.residual_channels, hp.gate_channels, hp.skip_out_channels, hp.cin_channels, hp.layers
    Gh = G // 2
    ZC, RC, SC, OC, K1, ni = Gh // cs, R // cs, S // cs, -(-hp.out_channels // cs), plan["K1"], plan["NI"]
    _, per_rank_layer = n_weights(hp, cs)
    ld1 = (K1 + 3) & ~3
    locw = max(2 * ZC, RC + SC)
    smem = 4 * (ni * (ld1 + Gh + R + ZC + RC + locw + SC + S + cs * OC + ((C + 3) & ~3) + 1) + L * (2 * ZC + RC)
                + ((2 * L + 1 + 3) & ~3)) + 64
    wslots = 2 * per_rank_layer * 4 + 64
    plan["prefetch"] = bool(prefetch_env and (per_rank_layer * 4) % 16 == 0 and smem + wslots <= SMEM_LIMIT)
    plan["slice_bytes"] = per_rank_layer * 4
    return plan


_CASES = sorted(BF16_SIZES)


@pytest.mark.parametrize("case", _CASES)
def test_bf16_sizes_are_unchanged(case):
    name, gin, cs = case.split("-")
    cfg = WN.make_config(_hp(name, int(gin[3:])), B, T, False, 0.0)
    assert _sizes(cfg, int(cs[2:])) == BF16_SIZES[case]


@pytest.mark.parametrize("case", _CASES)
def test_split_weight_block_is_four_bytes_per_weight(case):
    """the same weights and fp32 bias block as the bf16 mode, 4 bytes per weight instead of 2; the workspace drops the bf16 c_up"""
    name, gin, cs = case.split("-")
    hp, cs = _hp(name, int(gin[3:])), int(cs[2:])
    nw, _ = n_weights(hp, cs)
    pb16, wb16 = BF16_SIZES[case]
    bias = pb16 - _align(2 * nw)
    assert bias == 4 * (hp.layers * (hp.gate_channels + hp.residual_channels) + 2 * hp.skip_out_channels
                        + cs * -(-hp.out_channels // cs))
    pb, wb = _sizes(WN.make_config(hp, B, T, False, 0.0, precision="fp32-class"), cs)
    assert pb == _align(4 * nw) + bias
    assert wb == wb16 - _align(B * T * hp.cin_channels * 2)


def test_launch_plan_prefetch_decision():
    """two fp32 slots of the default widths' slice (R 128 / G 256 / S 128: 37 KB at cluster size 16) fit next to the activations;
    the paper widths' (R 256 / G 512 / S 256: 141 KB at cluster size 16) do not, though two bf16 slots of them do"""
    sms = 132
    for name, cs, want in (("default", 16, True), ("default", 8, True), ("paper", 16, False), ("paper", 8, False),
                           ("ks4", 16, True)):
        hp = _hp(name)
        plan = launch_plan_fp32(hp, 20, cs, sms)
        print("plan %s cs %d: fp32 slice %d bytes, prefetch %s (bf16: %s)" % (
            name, cs, plan["slice_bytes"], plan["prefetch"], bf16_launch_plan(hp, 20, cs, sms)["prefetch"]))
        assert plan["prefetch"] == want, (name, cs, plan)
        assert not launch_plan_fp32(hp, 20, cs, sms, prefetch_env=False)["prefetch"]
    assert bf16_launch_plan(_hp("paper"), 20, 16, sms)["prefetch"]


@pytest.mark.parametrize("precision", ["fp32", "fp64", "FP32-CLASS", None])
def test_synthesizer_rejects_an_unknown_precision(precision):
    with pytest.raises(t2.lib.T2Error, match="precision must be 'bf16' or 'fp32-class'"):
        WN.WaveNetSynthesizer(_hp("default"), 2, 2750, cluster_size=8, precision=precision)


def _split_cfg(**kw):
    hp = hparams.copy()
    hp.parse("layers=6,stacks=2,upsample_type=NearestNeighbor")
    for k, v in kw.items():
        hp.set_hparam(k, v)
    return WN.make_config(hp, 2, 64, False, 0.0, precision="fp32-class")


def _generate(lib, cfg, cs, bufs=None):
    p = bufs or [None] * 6
    return lib.t2_wn_ar_generate(ctypes.byref(cfg), cs, p[0], p[1], p[2], p[3], p[4], None, None, None, ctypes.c_ulonglong(0),
                                 p[5], None, None)


def test_malformed_split_calls_fail_before_any_launch():
    lib = t2.lib.load()
    lib.t2_last_error.restype = ctypes.c_char_p
    n0 = lib.t2_launch_count()
    fake = ctypes.c_void_p(1 << 20)                   # never dereferenced: every call below returns before touching a buffer
    good = _split_cfg()
    pb, wb = ctypes.c_longlong(), ctypes.c_longlong()
    for cs in (3, 0, 32):
        assert lib.t2_wn_ar_sizes(ctypes.byref(good), cs, ctypes.byref(pb), ctypes.byref(wb)) == INVALID_ARG
        assert lib.t2_wn_ar_pack(ctypes.byref(good), cs, fake, fake, fake, None) == INVALID_ARG
        assert _generate(lib, good, cs, [fake] * 6) == INVALID_ARG
    dropout = _split_cfg()
    dropout.dropout = 0.05                            # the fp32-class mode has no dropout
    assert lib.t2_wn_ar_sizes(ctypes.byref(dropout), 8, ctypes.byref(pb), ctypes.byref(wb)) == INVALID_ARG
    assert lib.t2_wn_ar_pack(ctypes.byref(dropout), 8, fake, fake, fake, None) == INVALID_ARG
    assert _generate(lib, dropout, 8, [fake] * 6) == INVALID_ARG
    # null buffers
    assert lib.t2_wn_ar_pack(ctypes.byref(good), 8, None, None, None, None) == INVALID_ARG
    for i in range(6):
        bufs = [fake] * 6
        bufs[i] = None
        assert _generate(lib, good, 8, bufs) == INVALID_ARG, i
    # shapes the AR kernel cannot run
    no_cin = _split_cfg(cin_channels=0)
    assert _generate(lib, no_cin, 8, [fake] * 6) == UNSUPPORTED_SHAPE
    wide_r = _split_cfg(residual_channels=256, gate_channels=512, skip_out_channels=128)
    assert lib.t2_wn_ar_sizes(ctypes.byref(wide_r), 8, ctypes.byref(pb), ctypes.byref(wb)) == UNSUPPORTED_SHAPE
    assert _generate(lib, wide_r, 8, [fake] * 6) == UNSUPPORTED_SHAPE
    assert lib.t2_wn_ar_set_speakers(ctypes.byref(good), 8, fake, fake, fake, None, None) == INVALID_ARG   # no gin_channels
    assert len(lib.t2_last_error()) > 0
    assert lib.t2_launch_count() == n0
