#!/usr/bin/env bash
# Install the UNMODIFIED reference (ShuhongChen/panic3d-anime-reconstruction) into baseline/_ref.
#
# The reference is not a pip package (no setup.py / pyproject), so "install" = a verbatim copy of its code
# directories.  baseline/_ref is git-ignored (reference sources never enter this repository's history) but NOT
# gpurun-ignored, so it travels to the GPU box, where /root/reference does not exist.  Used by
#   * bench.py --impl reference / cpu_baseline   (kind "reference": the imported reference renderer timed on CPU)
#   * bench_ref_gpu.py                           (the reference's own GPU path - eager PyTorch + its JIT CUDA plugins -
#                                                 timed beside ours on the same GPU; config-3 G.f sweep)
# Run in the build container:  bash baseline/install_ref.sh
set -euo pipefail
SRC=${1:-/root/reference}
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
DST="$HERE/_ref"
[ -d "$SRC/_train/eg3dc/src/training" ] || { echo "no reference tree at $SRC" >&2; exit 1; }
rm -rf "$DST"
mkdir -p "$DST"
for d in _train _databacks _util _scripts; do
    cp -r "$SRC/$d" "$DST/$d"
done
find "$DST" -name '__pycache__' -type d -prune -exec rm -rf {} +
( cd "$SRC" && find _train _databacks _util _scripts -type f -name '*.py' -o -name '*.cu' -o -name '*.cpp' -o -name '*.h' | sort | xargs sha1sum ) > "$DST/MANIFEST.sha1"
echo "installed $(find "$DST" -type f | wc -l) files ($(du -sh "$DST" | cut -f1)) into $DST"
# pre-build the reference's CUDA plugins for sm_90 (cross-compiles without a GPU); bench_config3.py / bench_ops.py point
# TORCH_EXTENSIONS_DIR at this directory on the GPU box
python "$HERE/prebuild_ref_plugins.py" "$DST" "$DST/_torch_ext" 2>&1 | grep -v "No CUDA runtime" || true
