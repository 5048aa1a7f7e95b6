#!/bin/bash
# Regenerates every reference-executed fixture under tests/golden/ (needs /root/reference) and reports which files changed.
# The generators are deterministic: a second run must leave `git status tests/golden` clean.
set -e
cd "$(dirname "$0")/.."
for g in make_reference_vectors make_reference_text make_reference_graph_vectors make_reference_attention_vectors make_reference_wavenet_graph_vectors \
         make_reference_wavenet_kernel_size_vectors; do
  echo "== tests/golden/$g.py"
  python tests/golden/$g.py 2>&1 | grep -E "^wrote|^train:|arrays" | tail -2
done
git status --short tests/golden
