#!/bin/bash
# Builds experiment variants of libdaachorse_b200.so (sm_90a) next to the default one (tools/alt/lib_<name>.so;
# *.so is git-ignored) and prints the command that A/B-tests them against the default build in ONE run on one
# GPU -- different machines differ by a few per cent, so variants are only comparable within a run.
#   tools/ab_variants.sh l2hint "-DDACH_L2HINT"   q14 "-DDACH_LANE_Q=14"
set -e
cd "$(dirname "$0")/../daachorse_b200/csrc"
make -s >/dev/null
mkdir -p ../../tools/alt
names=()
while [ $# -ge 2 ]; do
  name=$1; flags=$2; shift 2
  /usr/local/cuda/bin/nvcc $flags -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC \
      -c dev_scan.cu -o /tmp/dev_scan_$name.o
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../tools/alt/lib_$name.so \
      build/host_build.o build/host_wire.o build/dev_image.o build/capi.o /tmp/dev_scan_$name.o -Xlinker --no-undefined
  names+=($name)
  echo "built tools/alt/lib_$name.so ($flags)"
done
echo
echo "for v in default ${names[*]}; do L=; [ \$v != default ] && L=\$PWD/tools/alt/lib_\$v.so; DACH_LIB=\$L python bench.py --steps 5 --warmup 3 --no-cpu --no-e2e 2>/dev/null | python -c \"import json,sys; d=json.loads(sys.stdin.read()); print(\\\"\$v\\\", d[\\\"value\\\"], d[\\\"roofline\\\"][\\\"achieved\\\"])\"; done"
