#!/bin/bash
# Kernel-tuning aid: build alternative compilations of the engine library into build/variants/ (see sw_variant_bench.py).
#   tools/build_variants.sh name1:"-DFOO=1 -DBAR=2" name2:"..." ...
set -e
cd "$(dirname "$0")/.."
mkdir -p build/variants
for v in "$@"; do
  name=${v%%:*}; flags=${v#*:}
  ( /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC $flags -Xptxas -v \
      -shared -o build/variants/lib_$name.so vartrix_b200/csrc/vtx_api.cu -ldl 2> build/variants/$name.log \
      || { echo "BUILD FAILED: $name"; tail -5 build/variants/$name.log; } ) &
  while [ "$(jobs -r | wc -l)" -ge 6 ]; do sleep 1; done
done
wait
for v in "$@"; do name=${v%%:*}; echo "== $name: $(grep -A2 'Function properties for _ZN3vtx13vtx_k_sw_fold' build/variants/$name.log | grep -E 'spill|registers' | tr -s ' ' | tr '\n' ' ')"; done
