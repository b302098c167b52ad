#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY.  Builds the UNMODIFIED reference simple-knn extension
# (<original project>/submodules/simple-knn: spatial.cu, simple_knn.cu, ext.cpp) for sm_90a straight from the sources
# where they lie (no copy into this repo; its setup.py is NOT run).
# Output: oracle/_ref/simple_knn_ref_C*.so -- a pybind module exposing the reference's distCUDA2 (ext.cpp).
# oracle/_ref/ is git-ignored.  Used only by tests/golden/make_golden_knn.py (the stored reference outputs) and
# tools/knn_bench.py.  The product path never loads it.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${GOF_REFERENCE_ROOT:-/root/reference}/submodules/simple-knn"
OUT="$HERE/_ref"
if [ ! -d "$REF" ]; then
  echo "[build_ref_knn] $REF not present - keeping prebuilt files in $OUT"; exit 0
fi
mkdir -p "$OUT/obj_knn"
PY="${PYTHON:-python}"
NAME=simple_knn_ref_C
EXT_SUFFIX="$($PY -c 'import sysconfig;print(sysconfig.get_config_var("EXT_SUFFIX"))')"
TARGET="$OUT/${NAME}${EXT_SUFFIX}"
if [ -f "$TARGET" ] && [ "${FORCE:-0}" != "1" ]; then echo "[build_ref_knn] up to date: $TARGET"; exit 0; fi
INCS="$($PY - <<'PY'
import sysconfig
from torch.utils.cpp_extension import include_paths
print(" ".join("-I"+p for p in include_paths("cuda")), "-I"+sysconfig.get_paths()["include"])
PY
)"
TORCH_LIB="$($PY -c 'import torch,os;print(os.path.join(os.path.dirname(torch.__file__),"lib"))')"
ABI="$($PY -c 'import torch;print(int(torch._C._GLIBCXX_USE_CXX11_ABI))')"
COMMON="-std=c++17 -O3 -DTORCH_EXTENSION_NAME=$NAME -DTORCH_API_INCLUDE_EXTENSION_H -D_GLIBCXX_USE_CXX11_ABI=$ABI $INCS -I$REF"
# setup.py passes no nvcc flags; '-include cfloat' supplies FLT_MAX (simple_knn.cu:154), which CUDA 12.9's headers no
# longer pull in; nvcc's default -fmad=true is kept (it defines the reference's FP results: FMUL, FFMA, FFMA)
NVCC="nvcc -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -Xcompiler -fno-gnu-unique -include cfloat -w $COMMON"
pids=()
for f in spatial.cu simple_knn.cu; do
  o="$OUT/obj_knn/$(basename "${f%.cu}").o"
  ( [ -f "$o" ] || $NVCC -c "$REF/$f" -o "$o" ) &
  pids+=($!)
done
( [ -f "$OUT/obj_knn/ext.o" ] || g++ -fPIC -w $COMMON -c "$REF/ext.cpp" -o "$OUT/obj_knn/ext.o" ) &
pids+=($!)
for p in "${pids[@]}"; do wait "$p"; done
g++ -shared -o "$TARGET" "$OUT"/obj_knn/*.o -L"$TORCH_LIB" -Wl,-rpath,"$TORCH_LIB" -lc10 -ltorch_cpu -ltorch -ltorch_python -lc10_cuda -ltorch_cuda -L/usr/local/cuda/lib64 -lcudart
echo "[build_ref_knn] built $TARGET"
