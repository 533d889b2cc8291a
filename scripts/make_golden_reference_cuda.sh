#!/bin/sh
# Records the reference CUDA outputs the GPU parity tests compare against (tests/reference_cuda.py) into DIR; copy the .npz files from
# there into tests/golden/.  Needs a GPU and oracle/_ref built (python oracle/build_ref.py, which needs the reference's sources).
set -e
[ -n "$1" ] || { echo "usage: $0 DIR" >&2; exit 2; }
cd "$(dirname "$0")/.."
BF_RECORD_REFERENCE_CUDA="$(realpath -m "$1")" python -m pytest -q -m gpu -p no:cacheprovider tests/test_tsdf_vs_reference_gpu.py tests/test_solver_vs_reference_gpu.py
