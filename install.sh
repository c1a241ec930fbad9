#!/usr/bin/env bash
# Build the sm_90a kernel library in-tree and install the package in editable mode.
#   ./install.sh            nvcc build + pip install -e . (no dependency resolution: use requirements.txt for that)
#   ./install.sh --deps     also install requirements.txt first
set -euo pipefail
cd "$(dirname "$0")"
if [[ "${1:-}" == "--deps" ]]; then
  python -m pip install -r requirements.txt
fi
python -m gllm_b200.build
GLLM_B200_SKIP_BUILD=1 python -m pip install --no-build-isolation --no-deps -e .
python -c "import gllm_b200; print('gllm_b200', gllm_b200.__file__)"
