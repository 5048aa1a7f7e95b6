"""Every __global__ kernel of the library (tacotron-2_b200/csrc/*.cu, *.cuh) is either launched by a per-kernel test that compares it with
a float64 reference (COVERAGE), or named in EXEMPT with the existing end-to-end or per-call test that covers it. The Tacotron, CBHG,
parameter-table and batch-norm kernels keep their map in tests/test_taco_kernels_gpu.py (COVERAGE / EXEMPT there, checked by its own CPU
test); this test adds the rest of the library and fails for a kernel added anywhere without an entry."""
import os
import re

import test_taco_kernels_gpu as taco

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tacotron-2_b200", "csrc")

_WK = "test_wavenet_kernels_gpu.py::"
_AK = "test_audio_kernels_gpu.py::"
_AUDIO = "test_audio_gpu.py::"
COVERAGE = {
    "first_conv_kernel": _WK + "test_first_conv", "first_conv_bwd_kernel": _WK + "test_first_conv_bwd", "colsum_kernel": _WK + "test_colsum",
    "derived_bias_kernel": _WK + "test_derived_bias", "skip_bias_kernel": _WK + "test_skip_bias", "fx_finalize_kernel": _WK + "test_fx_finalize",
    "cl_to_chw_kernel": _WK + "test_cl_to_chw", "gin_bias_kernel": _WK + "test_gin_bias", "set_speakers_kernel": _WK + "test_set_speakers",
    "gin_wgrad_kernel": _WK + "test_gin_wgrad", "gin_demb_kernel": _WK + "test_gin_demb",
    "sumsq_kernel": "test_optim_gpu.py::test_per_tensor_clip", "norms_kernel": "test_optim_gpu.py::test_global_clip",
    "adam_kernel": "test_optim_gpu.py::test_per_tensor_clip",
    "fx_colsum_kernel": "test_gemm_epilogues_gpu.py::test_fx_colsum_exact_for_representable_addends",
    "rng_uniform_kernel": "test_gemm_epilogues_gpu.py::test_host_hash_matches_device",
    "upsample_fwd_kernel": "test_wavenet_upsample_gpu.py::test_kernel_sweep",
    "upsample_bwd_param_kernel": "test_wavenet_upsample_gpu.py::test_kernel_sweep",
    "upsample_bwd_input_kernel": "test_wavenet_upsample_gpu.py::test_kernel_sweep",
    "up1d_fwd_kernel": "test_wavenet_upsample_gpu.py::test_kernel_sweep", "up1d_bwd_input_kernel": "test_wavenet_upsample_gpu.py::test_kernel_sweep",
    "up1d_bwd_param_kernel": "test_wavenet_upsample_gpu.py::test_kernel_sweep",
    "stft_mel_kernel_v2": _AK + "test_stft_mel_raw_db", "gl_init_phase_kernel": _AK + "test_gl_init_phase", "gl_istft_kernel": _AK + "test_gl_istft",
    "gl_ola_kernel": _AK + "test_gl_ola", "gl_stft_kernel": _AK + "test_gl_stft", "preemphasis_kernel": _AK + "test_preemphasis_restarts_every_row",
    "mulaw_quantize_kernel": _AUDIO + "test_mulaw_quantize_bit_exact", "mulaw_kernel": _AUDIO + "test_mulaw_quantize_bit_exact",
    "inv_mulaw_quantize_kernel": _AUDIO + "test_inv_mulaw_roundtrip_bit_exact",
    "inv_mulaw_kernel": "test_reference_pinned.py::test_cuda_mulaw_matches_reference_tensor_path",
}
EXEMPT = {
    "act_gemm_kernel": "test_gemm_epilogues_gpu.py::test_bias_act", "wgrad_gemm_kernel": "test_gemm_epilogues_gpu.py::test_wgrad_tiles",
    "wn_chain_kernel": "test_wavenet_persistent_gpu.py::test_persistent_chain_matches_per_layer_launches_bit_for_bit",
    "ar_pack_kernel": "test_wavenet_ar_gpu.py::test_ar_teacher_forced_mulaw", "wn_ar_kernel": "test_wavenet_ar_gpu.py::test_ar_teacher_forced_mulaw",
}


def kernels():
    """{kernel name: source file} of every __global__ function in the library"""
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh")):
            src = open(os.path.join(CSRC, f)).read()
            for n in re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src):
                out[n] = f
    return out


def test_every_kernel_of_the_library_is_covered():
    names = kernels()
    assert len(names) == 76, "kernel count changed to %d: map the new kernels and update this count" % len(names)
    maps = [COVERAGE, EXEMPT, taco.COVERAGE, taco.EXEMPT]
    for a in range(len(maps)):
        for b in range(a + 1, len(maps)):
            assert not set(maps[a]) & set(maps[b]), "a kernel is mapped twice: %s" % sorted(set(maps[a]) & set(maps[b]))
    missing = sorted(n for n in names if not any(n in m for m in maps))
    assert not missing, "kernels without a test: %s" % missing
    stale = sorted(n for m in (COVERAGE, EXEMPT) for n in m if n not in names)
    assert not stale, "entries for kernels that no longer exist: %s" % stale
    for k, t in list(COVERAGE.items()) + list(EXEMPT.items()):
        f, name = t.split("::")
        assert re.search(r"^def %s\(" % name, open(os.path.join(ROOT, "tests", f)).read(), re.M), (k, t)
