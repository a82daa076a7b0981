#!/usr/bin/env bash
# Test infrastructure only -- builds the UNMODIFIED reference (src-d/kmcuda) for sm_90 from the
# sources (KMCUDA_REFERENCE_SRC, default /root/reference/src) into oracle/_ref/libKMCUDA.so.
# Nothing from the reference tree is copied into this repository; oracle/_ref/ is git-ignored
# The recipe follows SURVEY.md section 8c:
# direct nvcc/g++ commands, not the reference's (obsolete) CMake build.
set -euo pipefail
REF=${KMCUDA_REFERENCE_SRC:-/root/reference/src}
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/_ref"
if [ ! -d "$REF" ]; then
  echo "build_ref: $REF not present -- keeping prebuilt $OUT" >&2
  exit 0
fi
mkdir -p "$OUT/obj"
if [ -f "$OUT/libKMCUDA.so" ] && [ "$OUT/libKMCUDA.so" -nt "$REF/kmeans.cu" ] && [ "$OUT/libKMCUDA.so" -nt "$HERE/build_ref.sh" ]; then
  echo "build_ref: $OUT/libKMCUDA.so up to date"; exit 0
fi
PYINC=$(python3 -c 'import sysconfig;print(sysconfig.get_paths()["include"])')
NPINC=$(python3 -c 'import numpy;print(numpy.get_include())')
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
for f in kmeans knn transpose; do
  "$NVCC" -std=c++14 -arch sm_90 -DCUDA_ARCH=90 -D_FORCE_INLINES -O3 -w \
      -Xcompiler -fPIC -c "$REF/$f.cu" -o "$OUT/obj/$f.o" &
done
g++ -std=c++11 -O2 -fPIC -fopenmp -w -DCUDA_ARCH=90 -I/usr/local/cuda/include \
    -c "$REF/kmcuda.cc" -o "$OUT/obj/kmcuda.o" &
g++ -std=c++11 -O2 -fPIC -w -DCUDA_ARCH=90 -I/usr/local/cuda/include -I"$PYINC" -I"$NPINC" \
    -c "$REF/python.cc" -o "$OUT/obj/python.o" &
wait
"$NVCC" -shared -o "$OUT/libKMCUDA.so" "$OUT"/obj/*.o -lcurand -lgomp
echo "build_ref: built $OUT/libKMCUDA.so"
