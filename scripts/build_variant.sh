#!/bin/bash
# build_variant.sh NAME "-DKNOB=..." : same sources, other tuning knobs -> experiments/_variants/libb200q_NAME.so (select with B200Q_LIB_PATH)
set -e
cd "$(dirname "$0")/.."
name=$1; shift
out=experiments/_variants; mkdir -p $out/obj_$name
for f in b200q_decode_i0 b200q_decode_i1 b200q_decode_i2 b200q_decode_i3 b200q_decode b200q_gemm b200q_reduce b200q_api b200q_wire; do
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr "$@" \
     -c ik_llama_cpp_b200/csrc/$f.cu -o $out/obj_$name/$f.o 2>/dev/null &
done
wait
/usr/local/cuda/bin/nvcc -shared -o $out/libb200q_$name.so $out/obj_$name/*.o -cudart static -Xlinker --no-undefined 2>/dev/null
rm -rf $out/obj_$name
echo $out/libb200q_$name.so
