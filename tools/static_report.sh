#!/bin/bash
# Static (no-GPU) evidence: per-kernel registers / spills / shared memory from ptxas, and the SASS
# mnemonics that show which hardware paths the kernels use (TMA bulk copy = UBLKCP, mbarrier = SYNCS, 128-bit
# global loads, L2 cache-hint loads).  Usage: tools/static_report.sh > static_resources.txt
set -e
cd "$(dirname "$0")/../rocksplicator_b200/csrc"
ARCH="-gencode arch=compute_90a,code=sm_90a"
TMP=$(mktemp -d -p .)
trap 'rm -rf "$TMP"' EXIT
echo "# nvcc $ARCH -O3 -std=c++17 -lineinfo -Xptxas -v   ($(nvcc --version | grep release | sed 's/.*release //'))"
for f in k_apply k_read k_compact; do
  echo "## $f.cu"
  nvcc $ARCH -O3 -std=c++17 -lineinfo -Xptxas -v -c $f.cu -o $TMP/$f.o 2>&1 | c++filt |
    awk '/Compiling entry function/ {name=$0; sub(/.*function .(void )?/, "", name); sub(/\(.*/, "", name)}
         /spill stores/ {spill=$0; sub(/^ +/, "", spill)}
         /Used [0-9]+ registers/ {u=$0; sub(/.*Used/, "Used", u); printf "%-28s %s | %s\n", name, u, spill}'
  echo "### SASS mnemonics ($f.o)"
  cuobjdump -sass $TMP/$f.o | grep -oE "\b(UBLKCP[.A-Z0-9_]*|SYNCS[.A-Z0-9_]*|LDG\.E\.128[.A-Z0-9_]*|LDG\.E\.64[.A-Z0-9_]*|STG\.E\.128[.A-Z0-9_]*|ATOMG[.A-Z0-9_]*|ATOM[.A-Z0-9_]*|SHFL[.A-Z0-9_]*|VOTE[.A-Z0-9_]*|MATCH[.A-Z0-9_]*|LDS[.A-Z0-9_]*|STS[.A-Z0-9_]*)" |
    sort | uniq -c | sort -rn | head -24
done
