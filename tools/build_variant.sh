#!/bin/bash
# Build an A/B variant of libgsb200 with extra -D flags: tools/build_variant.sh <name> "<flags>"  ->  3dgs.cpp_b200/libgsb200v_<name>.so
# (run it with GSB200_LIB=... or tools/run_ab.sh libgsb200v_<name>.so; variants are git-ignored)
set -e
name=$1; flags=$2
cd "$(dirname "$0")/../3dgs.cpp_b200"
mkdir -p /tmp/gsb_var_$name
objs=""
for f in csrc/*.cu; do
  o=/tmp/gsb_var_$name/$(basename $f .cu).o
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -fmad=false -Xcompiler -fPIC,-Wall -I../include -Icsrc $flags -Xptxas -v -c $f -o $o 2> $o.log &
  objs="$objs $o"
done
wait
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o libgsb200v_$name.so $objs -cudart static
grep -h -A2 "k_blend\|k_onesweep\|k_project\|k_emit\|k_sort_hist" /tmp/gsb_var_$name/*.log | grep -E "Used" | sort | uniq -c | head -20
