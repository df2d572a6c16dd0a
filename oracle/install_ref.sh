#!/usr/bin/env bash
# Install the UNMODIFIED reference (yang-song/score_sde_pytorch) under oracle/_ref so that
# `bench.py --impl reference` can time the reference's own CPU path on the host cores of the benchmark machine.
#
# The reference is a flat directory of Python modules with no setup.py / pyproject.toml, so
# `pip install --target` has nothing to build; the install is a plain copy of its sources.  oracle/_ref is
# git-ignored: no reference source enters the history.  Usage: oracle/install_ref.sh REFERENCE_CHECKOUT
#
# The reference's `op/` package JIT-compiles two CUDA extensions at import (op/upfirdn2d.py:10-16,
# op/fused_act.py:11-17); they are built here once into oracle/_ref/_ext (TORCH_EXTENSIONS_DIR) so the benchmark
# machine only has to re-link/verify them.  On CPU tensors the reference never calls them (op/upfirdn2d.py:146-149).
set -euo pipefail
REPO="$(cd "$(dirname "$0")/.." && pwd)"
SRC="${1:?usage: install_ref.sh REFERENCE_CHECKOUT}"
DST="$REPO/oracle/_ref"
if [ ! -d "$SRC" ]; then echo "install_ref: $SRC not found (nothing to do)"; exit 0; fi
mkdir -p "$DST"
# sources only: no notebooks / images / VCS data
( cd "$SRC" && tar --exclude=.git --exclude=assets --exclude='*.ipynb' -cf - . ) | ( cd "$DST" && tar -xf - )
echo "install_ref: copied $(find "$DST" -name '*.py' | wc -l) python files to $DST"
# pre-build the JIT extensions for sm_90 (no GPU needed)
export TORCH_EXTENSIONS_DIR="$REPO/oracle/_ref/_ext" TORCH_CUDA_ARCH_LIST="9.0"
python - <<'EOF'
import os, sys, types, time
repo = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(os.environ['TORCH_EXTENSIONS_DIR']))))
sys.path.insert(0, repo)
import bench
t0 = time.time()
bench.import_reference()
print(f'install_ref: reference imports (extensions built/cached in {time.time() - t0:.0f} s)')
EOF
