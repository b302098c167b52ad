#!/usr/bin/env bash
# TEST / BASELINE INFRASTRUCTURE ONLY.  Stages the UNMODIFIED Python sources of the reference that sit either side of the
# rasterizer (its autograd wrapper, gaussian_renderer.render/integrate, the loss / depth / SH helpers, the appearance network,
# utils/tetmesh.py, train.py, extract_mesh.py and dtu_eval/eval.py as text, eval_tnt/*.py) into baseline/_ref/gof_ref_py/ -- git-ignored, but shipped to the
# GPU box -- so that tests and `bench.py --impl reference` can run the reference's OWN code there (/root/reference does not
# exist on the GPU box).  Nothing under gaussian-opacity-fields_b200/ reads this directory.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${GOF_REFERENCE_ROOT:-/root/reference}"
OUT="$HERE/_ref/gof_ref_py"
if [ ! -d "$REF" ]; then
  echo "[stage_ref] $REF not present (GPU box?) - keeping staged files in $OUT"; exit 0
fi
mkdir -p "$OUT/diff_gaussian_rasterization" "$OUT/gaussian_renderer" "$OUT/utils" "$OUT/scene" "$OUT/text"
cp "$REF/submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py" "$OUT/diff_gaussian_rasterization/__init__.py"
cp "$REF/gaussian_renderer/__init__.py" "$OUT/gaussian_renderer/__init__.py"
for f in sh_utils loss_utils depth_utils general_utils graphics_utils tetmesh; do cp "$REF/utils/$f.py" "$OUT/utils/$f.py"; done
cp "$REF/scene/appearance_network.py" "$OUT/scene/appearance_network.py"
# whole scripts / classes that cannot be imported here (plyfile, simple_knn, open3d ... are absent): kept as text, tests
# extract single functions from them with `ast`
cp "$REF/train.py" "$OUT/text/train.py"
cp "$REF/extract_mesh.py" "$OUT/text/extract_mesh.py"
cp "$REF/scene/gaussian_model.py" "$OUT/text/gaussian_model.py"
cp "$REF/scene/cameras.py" "$OUT/text/cameras.py"
cp "$REF/dtu_eval/eval.py" "$OUT/text/dtu_eval.py"
# eval_tnt/run.py and the modules it imports, run by tests/_tnt_scenes.py with stub open3d / trimesh / matplotlib modules
mkdir -p "$OUT/eval_tnt"
for f in run config registration evaluation trajectory_io util plot; do cp "$REF/eval_tnt/$f.py" "$OUT/eval_tnt/$f.py"; done
echo "[stage_ref] staged reference Python into $OUT"
