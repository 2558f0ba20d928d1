#!/bin/bash
# Build kernel variants of the library into build/variants/ (shipped to the GPU box, git-ignored), one per NAME=FLAGS pair:
#   tools/sweep_variants.sh base="" fence="-DKT_WAIT_MODE=0" slots16="-DKT_SLOT_CAP=16"
# then on the GPU:  tools/sweep_run.sh [bench args]     (every variant on the same box, back to back, twice)
# Switches (kt_kernels.cuh): KT_WAIT_MODE, KT_SLOT_CAP, KT_TILE_RECONCILE, KT_HEAVY_PODS, KT_STAGE_CHUNK, KT_EVAL_PAIR, KT_DECIDE_UNROLLED,
# KT_SCATTER_WORDS, KT_BULK_ROWS, KT_SMEM_ADD32, KT_QUAD_FENCE, KT_QUAD_DRYRUN; (kt_engine.cu): KT_WIDE_TILES, KT_PASS_PDL.
set -e
cd "$(dirname "$0")/.."
mkdir -p build/variants
for v in "$@"; do
  name=${v%%=*}
  flags=${v#*=}
  out=$PWD/build/variants/libkt_$name.so
  make -s -C kube_throttler_b200/csrc -B OUT=$out NVCCFLAGS_EXTRA="$flags" > /dev/null 2>&1
  echo "built $out  [$flags]"
done
