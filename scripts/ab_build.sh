#!/bin/bash
# A/B tooling for kernel experiments: build one library per set of extra nvcc flags into scripts/variants/ (git-ignored,
# travels with gpurun), then compare them on the SAME box in alternating runs:
#
#   scripts/ab_build.sh base="" unroll2="-DMAPDN_SWEEP_UNROLL=2"
#   gpurun --timeout 600 -- 'scripts/ab_run.sh 3 base unroll2'
#
# Box-to-box variation is 1-2 %, so numbers from different gpurun calls are not comparable at that level.
set -e
cd "$(dirname "$0")/.."
mkdir -p scripts/variants
for spec in "$@"; do
  name="${spec%%=*}"; flags="${spec#*=}"
  echo "building scripts/variants/$name.so with: $flags"
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --shared -Xcompiler -fPIC \
       --expt-relaxed-constexpr $flags -o scripts/variants/$name.so mapdn_b200/csrc/mapdn_b200.cu &
done
wait
ls -la scripts/variants
