"""Generates tests/golden/reference_wavenet_kernel_size.npz by EXECUTING the reference's WaveNet graph code (`WaveNet.initialize` in
its training, evaluation and synthesis branches, `step`, `incremental`, `add_loss`) at dilated-convolution kernel_size 2 and 4, with
the machinery of make_reference_wavenet_graph_vectors.py (same TF-1 stand-in, SMALL widths, inputs and recorded draws).

  python tests/golden/make_reference_wavenet_kernel_size_vectors.py        # needs /root/reference; only the committed .npz travels

Scenarios, each at kernel_size 2 and 4 (tag suffix _k2 / _k4):
  ce_subpixel   input_type mulaw-quantize (256 classes), SubPixel conditioning upsampling, masked cross entropy
  mol_2d        input_type raw, 2-component mixture-of-logistics head, ConvTranspose2D upsampling
  gauss_nn      input_type raw, single-Gaussian head, NearestNeighbor upsampling
The arrays are those of reference_wavenet_graph.npz under the tags above (shared: c, input_lengths, small_hparams_*)."""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_reference_wavenet_graph_vectors as M  # noqa: E402

KERNEL_SIZES = (2, 4)
TAGS = ("ce_subpixel", "mol_2d", "gauss_nn")      # the scenario names the generator runs its evaluation and synthesis branches for


def main():
    base = dict(M.SCENARIOS)
    out = {}
    for k in KERNEL_SIZES:
        M.SCENARIOS = {tag: dict(base[tag], kernel_size=k) for tag in TAGS}
        with tempfile.TemporaryDirectory() as tmp:
            M.HERE = tmp                              # where main() writes its archive (tf_shim is already importable from HERE)
            M.main()
            with np.load(os.path.join(tmp, "reference_wavenet_graph.npz")) as R:
                for name in R.files:
                    tag = next((t for t in TAGS if name.startswith(t + "_")), None)
                    key = name if tag is None else "%s_k%d%s" % (tag, k, name[len(tag):])
                    assert tag is not None or key not in out or np.array_equal(out[key], R[name]), key
                    out[key] = R[name]
    path = os.path.join(HERE, "reference_wavenet_kernel_size.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d arrays, %.1f KB" % (path, len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
