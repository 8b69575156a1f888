#!/bin/bash
# usage: tools/build_variant.sh <name> [extra nvcc flags...]  -> variants/lib_<name>.so
# Another build of the product library for same-box A/B runs (tools/ab_probe.py --lib name=variants/lib_<name>.so).
set -e
name=$1; shift
root=$(cd "$(dirname "$0")/.." && pwd)
out=$root/variants/build_$name
mkdir -p $out
objs=""
for f in api pipeline transfer preprocess integrate regularize knn; do
  nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -ftz=true -fmad=false -prec-div=true -prec-sqrt=true \
       -Xcompiler -fPIC "$@" -c $root/surfelmeshing_b200/csrc/$f.cu -o $out/$f.o &
  objs="$objs $out/$f.o"
done
wait
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o $root/variants/lib_$name.so $objs
rm -rf $out
echo $root/variants/lib_$name.so
