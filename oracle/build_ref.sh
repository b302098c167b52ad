#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY.  Builds the UNMODIFIED reference rasterizer
# (<original project>/submodules/diff-gaussian-rasterization) for sm_90a straight from the
# sources where they lie (no copy into this repo; the reference's own setup.py/CMake is NOT run).
# Output: oracle/_ref/gof_ref_C*.so  -- a pybind module exposing the reference's four `_C`
# entry points (ext.cpp:16-19).  oracle/_ref/ is git-ignored.
# It is used only by tests/golden/make_golden*.py (the stored reference outputs) and
# bench.py --impl reference.  The product path never loads it.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${GOF_REFERENCE_ROOT:-/root/reference}/submodules/diff-gaussian-rasterization"
OUT="$HERE/_ref"
if [ ! -d "$REF" ]; then
  echo "[build_ref] $REF not present - keeping prebuilt files in $OUT"; exit 0
fi
mkdir -p "$OUT/obj"
PY="${PYTHON:-python}"
NAME=gof_ref_C
EXT_SUFFIX="$($PY -c 'import sysconfig;print(sysconfig.get_config_var("EXT_SUFFIX"))')"
TARGET="$OUT/${NAME}${EXT_SUFFIX}"
if [ -f "$TARGET" ] && [ "${FORCE:-0}" != "1" ]; then echo "[build_ref] up to date: $TARGET"; exit 0; fi
INCS="$($PY - <<'PY'
import sysconfig
from torch.utils.cpp_extension import include_paths
print(" ".join("-I"+p for p in include_paths("cuda")), "-I"+sysconfig.get_paths()["include"])
PY
)"
TORCH_LIB="$($PY -c 'import torch,os;print(os.path.join(os.path.dirname(torch.__file__),"lib"))')"
ABI="$($PY -c 'import torch;print(int(torch._C._GLIBCXX_USE_CXX11_ABI))')"
COMMON="-std=c++17 -O3 -DTORCH_EXTENSION_NAME=$NAME -DTORCH_API_INCLUDE_EXTENSION_H -D_GLIBCXX_USE_CXX11_ABI=$ABI $INCS -I$REF -I$REF/third_party/glm"
# reference flags (setup.py:29): -Xcompiler -fno-gnu-unique; '-include cstdint' is needed by gcc 13
# for rasterizer_impl.h (std::uintptr_t); nvcc default -fmad=true kept (it defines the reference's FP results)
NVCC="nvcc -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -Xcompiler -fno-gnu-unique -include cstdint --expt-relaxed-constexpr -w $COMMON"
pids=()
for f in cuda_rasterizer/rasterizer_impl.cu cuda_rasterizer/forward.cu cuda_rasterizer/backward.cu rasterize_points.cu; do
  o="$OUT/obj/$(basename "${f%.cu}").o"
  ( [ -f "$o" ] || $NVCC -c "$REF/$f" -o "$o" ) &
  pids+=($!)
done
( [ -f "$OUT/obj/ext.o" ] || g++ -fPIC -w $COMMON -c "$REF/ext.cpp" -o "$OUT/obj/ext.o" ) &
pids+=($!)
for p in "${pids[@]}"; do wait "$p"; done
g++ -shared -o "$TARGET" "$OUT"/obj/*.o -L"$TORCH_LIB" -Wl,-rpath,"$TORCH_LIB" -lc10 -ltorch_cpu -ltorch -ltorch_python -lc10_cuda -ltorch_cuda -L/usr/local/cuda/lib64 -lcudart
echo "[build_ref] built $TARGET"
