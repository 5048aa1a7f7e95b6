"""CPU: every split-bf16 (fp32-class) code path of the CUDA sources has a per-launch test against a float64 reference. A split path is
a __global__ kernel templated on kSplit, a __global__ kernel with an `int split` argument, or a GEMM-engine epilogue that branches on
its split flag e.i[11]. SPLIT_COVERAGE maps each one to `file::test`; the test fails when a split path appears without an entry, or
when an entry names a test that does not exist."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tacotron-2_b200", "csrc")
_SPLIT = "test_split_operands_gpu.py::"
_GEMM = "test_gemm_epilogues_gpu.py::"
_TACO = "test_taco_kernels_gpu.py::"
_CBHG = "test_cbhg_fp32_class_gpu.py::"

SPLIT_COVERAGE = {
    # kernels templated on kSplit
    "att_fwd_kernel": _SPLIT + "test_att_fwd_split",
    "f32_to_bf16_kernel": _SPLIT + "test_f32_to_bf16_split",
    "maxpool_fwd_k": _CBHG + "test_split_maxpool_is_exact",
    "highway_fwd_k": _CBHG + "test_split_highway",
    "gru_fwd_kernel": _CBHG + "test_split_gru_fwd",
    # kernels with an `int split` argument
    "embed_fwd_kernel": _SPLIT + "test_embed_fwd_split",
    "decin_kernel": _SPLIT + "test_decin_split",
    "dec_finish_kernel": _SPLIT + "test_dec_finish_split",
    "proj_bias_feedback_kernel": _SPLIT + "test_proj_bias_feedback_split",
    "bn_apply_kernel": _TACO + "test_taco_bn_fwd",
    "first_conv_kernel": "test_wavenet_kernels_gpu.py::test_first_conv",
    "up1d_fwd_kernel": "test_wavenet_upsample_gpu.py::test_1d_split_rows",
    "upsample_fwd_kernel": "test_wavenet_upsample_gpu.py::test_1d_split_rows",
    # epilogues branching on e.i[11]; EPI_BIAS_ACT and EPI_LSTM through the production helpers launch_bias_act / lstm_step
    "EPI_GATE": _GEMM + "test_gate",
    "EPI_RES": _GEMM + "test_res",
    "EPI_BIAS_ACT": _SPLIT + "test_conv_gemm_split",
    "EPI_LSTM": _SPLIT + "test_lstm_step_split",
}


def split_paths():
    paths = set()
    for f in sorted(os.listdir(CSRC)):
        if not f.endswith((".cu", ".cuh")):
            continue
        src = open(os.path.join(CSRC, f)).read()
        for m in re.finditer(r"template\s*<([^>]*)>\s*__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src):
            if re.search(r"\bbool\s+kSplit\b", m.group(1)):
                paths.add(m.group(2))
        for m in re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(([^)]*)\)", src):
            if re.search(r"\bint\s+split\b", m.group(2)):
                paths.add(m.group(1))
        starts = [(m.start(), m.group(1)) for m in re.finditer(r"struct\s+Epilogue<(EPI_\w+)\s*,[^>]*>\s*\{", src)]
        for k, (s, name) in enumerate(starts):
            body = src[s:starts[k + 1][0] if k + 1 < len(starts) else len(src)]
            if "e.i[11]" in body:
                paths.add(name)
    return paths


def test_every_split_path_has_a_per_launch_test():
    paths = split_paths()
    assert {"att_fwd_kernel", "decin_kernel", "EPI_LSTM", "EPI_BIAS_ACT"} <= paths, paths      # the scan itself still finds them
    missing = sorted(paths - set(SPLIT_COVERAGE))
    assert not missing, "split code paths without a per-launch test: %s" % missing
    stale = sorted(set(SPLIT_COVERAGE) - paths)
    assert not stale, "entries for split paths that no longer exist: %s" % stale
    for path, t in SPLIT_COVERAGE.items():
        f, name = t.split("::")
        assert re.search(r"^def %s\(" % name, open(os.path.join(ROOT, "tests", f)).read(), re.M), (path, t)
