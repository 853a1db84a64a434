#!/bin/bash
# Binary evidence for the shipped library (no GPU needed): per-kernel resource usage and SASS opcode histograms.
#   bash scripts/sass_report.sh [tag]    -> profiles/<tag>_res_usage.txt, profiles/<tag>_sass_histogram.txt
# nvdisasm on the extracted cubins (cuobjdump -sass leaves out the bodies of __noinline__ device functions, which is where the wavefront
# routines live).
set -eu
TAG=${1:-r02}
LIB=$(pwd)/avian_b200/lib/libavian_b200.so
OUT=$(pwd)/profiles
mkdir -p $OUT
cuobjdump -res-usage $LIB 2>/dev/null | grep -A1 "Function" | grep -v "^--" | paste - - | sed 's/^ *Function //' | c++filt | sort > $OUT/${TAG}_res_usage.txt
TMP=$(mktemp -d); cd $TMP
cuobjdump -xelf all $LIB >/dev/null 2>&1
hist() { grep -E "^\s+/\*[0-9a-f]{4,}\*/" | sed -E 's/^\s+\/\*[0-9a-f]+\*\/\s+(@!?U?P[0-9T]+ )?//' | awk '{print $1}' | sed 's/;$//' | sort | uniq -c | sort -rn | awk '{printf "%8d %s\n", $1, $2}'; }
{
  echo "# SASS opcode histograms of avian_b200/lib/libavian_b200.so (nvdisasm -c of every cubin in the fat binary).  Opcodes to look for:"
  echo "#   LDG.E.STRONG.GPU + CCTL.IVALL                          ld.acquire.gpu polls of the wavefront event counters (no membar after a poll)"
  echo "#   MEMBAR.ALL.GPU                                         fence.acq_rel.gpu before a wavefront item stores its counters"
  echo "#   MEMBAR.SC.GPU                                          __threadfence() (grid barriers); none in the wavefront routines"
  echo "#   LDL / STL                                              local memory (spills); none in the f32 wavefront routines"
  echo "#   LDGSTS.E.BYPASS.128                                    cp.async staging of the constraint rows into shared memory"
  for f in solver_host broadphase contacts narrow aabb; do
    echo "== $f.cu: memory / synchronisation opcodes"
    nvdisasm -c $f.sm_90a.cubin 2>/dev/null | hist | grep -E "LDG|STG|LDGSTS|MEMBAR|CCTL|LDS|STS|ATOM|RED|BAR|ERRBAR|LDL|STL|UBLKCP|UTMA|SYNCS|MATCH|VOTE|SHFL" || true
  done
  echo "== solver_host.cu: all opcodes, top 60"
  nvdisasm -c solver_host.sm_90a.cubin 2>/dev/null | hist | head -60
} > $OUT/${TAG}_sass_histogram.txt
cd /; rm -rf $TMP
grep -E "MEMBAR|LDL|STL" $OUT/${TAG}_sass_histogram.txt || true
