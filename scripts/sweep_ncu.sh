#!/bin/bash
# BASELINE.json configs[4] with counters: one eager forward per resolution under ncu (per-launch duration, tensor-pipe
# activity, DRAM bytes), condensed by scripts/sweep_table.py.  Usage on a GPU box: bash scripts/sweep_ncu.sh [tag]
cd "$(dirname "$0")/.."
tag=${1:-sweep}
out=${OSVOS_RESULTS:-results}   # output directory (git-ignored)
mkdir -p "$out"
M=gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active,dram__bytes_read.sum,dram__bytes_write.sum,launch__grid_size
for hw in "240 427" "480 854" "720 1280" "1080 1920"; do
  set -- $hw
  timeout 300 ncu --metrics $M --clock-control none -k regex:"conv|side|tail|stage1" -c 40 --csv --log-file $out/${tag}_sweep_launches_$1x$2.csv \
      python scripts/one_forward.py $1 $2 > $out/${tag}_sweep_$1x$2.log 2>&1
done
python scripts/sweep_table.py $out/${tag}_sweep_launches_ > $out/${tag}_sweep_counters.txt
timeout 600 python scripts/sweep.py exact > $out/${tag}_resolution_sweep_exact.txt 2>&1
cat $out/${tag}_sweep_counters.txt $out/${tag}_resolution_sweep_exact.txt
