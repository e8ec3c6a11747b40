#!/bin/bash
# Builds scripts/variants/<name>.so from an OLDER commit's kernel sources, patched to the current C-ABI (reset gained a
# `converged_dev` argument in ABI 2; the old kernel ignores it), so that scripts/ab_run.sh can compare it with the
# in-tree library in alternating runs on ONE box:   scripts/ab_build_ref.sh r01 e79f6c5 ["-DMAPDN_EXP_..."]
set -e
cd "$(dirname "$0")/.."
name=$1; rev=$2; flags=$3
tmp=$(mktemp -d /tmp/mapdn_ref.XXXX)
git archive "$rev" include mapdn_b200/csrc | tar -x -C "$tmp"
sed -i 's/#define MAPDN_ABI_VERSION 1/#define MAPDN_ABI_VERSION 2/' "$tmp/include/mapdn_b200.h"
python - "$tmp" <<'PY'
import sys, re
t = sys.argv[1]
for f in ("include/mapdn_b200.h", "mapdn_b200/csrc/mapdn_b200.cu"):
    s = open(f"{t}/{f}").read()
    s, n = re.subn(r"(mapdn_status mapdn_reset\(.*?)(void\* stream\))", r"\1uint8_t* converged_dev, \2", s, count=1, flags=re.S)
    assert n == 1, (f, n)
    open(f"{t}/{f}", "w").write(s)
PY
mkdir -p scripts/variants
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --shared -Xcompiler -fPIC --expt-relaxed-constexpr \
     $flags -o scripts/variants/$name.so "$tmp/mapdn_b200/csrc/mapdn_b200.cu"
rm -rf "$tmp"
ls -la scripts/variants/$name.so
