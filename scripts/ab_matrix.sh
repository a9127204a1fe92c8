#!/bin/bash
# A/B of the library's switches on 480x854 inference (+ the fwd+bwd graph), one process per switch, both orders.
# Usage on a GPU box:  bash scripts/ab_matrix.sh > ab_matrix.txt 2>&1   (about 15 s per line pair)
cd "$(dirname "$0")/.."
export OSVOS_ENV_RELOAD=1
for sw in OSVOS_FUSE_STAGE1 OSVOS_CONV_N256 OSVOS_FOLD_SIDE OSVOS_HALO_LEAN; do
  echo "== $sw = 1 / 0"
  timeout 200 python scripts/ab_env.py $sw 1 0 --train || echo "FAILED: $sw"
done
for hw in "240 427" "720 1280" "1080 1920"; do
  echo "== OSVOS_FUSE_STAGE1 at $hw"
  timeout 200 python scripts/ab_env.py OSVOS_FUSE_STAGE1 1 0 $hw || echo "FAILED"
done
