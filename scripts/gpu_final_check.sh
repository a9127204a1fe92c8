#!/bin/bash
# Final single-GPU validation of a commit: smoke(), the full GPU suite, the bench lines (inference / fwd+bwd / reference arm),
# launch lists of one forward and one training step.  Usage on a GPU box: bash scripts/gpu_final_check.sh [tag]
cd "$(dirname "$0")/.."
tag=${1:-final}
out=${OSVOS_RESULTS:-results}   # output directory (git-ignored)
mkdir -p "$out"
( timeout 600 python -c "import __graft_entry__ as g; g.smoke()" ) > $out/${tag}_smoke.txt 2>&1
( timeout 1800 python -m pytest tests -m gpu -q -p no:cacheprovider 2>&1 | tail -15 ) > $out/${tag}_pytest.txt
( timeout 600 python bench.py --steps 20 --warmup 5 ) > $out/${tag}_bench.json 2>$out/${tag}_bench.err
( timeout 600 python bench.py ) > $out/${tag}_bench_default_flags.json 2>/dev/null
( timeout 300 python bench.py --impl reference --steps 20 --warmup 5 ) > $out/${tag}_bench_reference.json 2>/dev/null
( timeout 300 python bench.py --steps 20 --warmup 5 --workload train480 --skip cpu_baseline ) > $out/${tag}_bench_train480.json 2>/dev/null
M=gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active,dram__bytes_read.sum,dram__bytes_write.sum,launch__grid_size
( timeout 300 ncu --metrics $M --clock-control none -k regex:"conv|side|tail|stage1" -c 40 --csv --log-file $out/${tag}_launches_infer480.csv python scripts/one_forward.py ) > $out/${tag}_ncu.log 2>&1
( timeout 400 ncu --metrics $M --clock-control none -k regex:"conv|side|tail|wgrad|unpool|stage1" -c 120 --csv --log-file $out/${tag}_launches_train480.csv python scripts/one_train_step.py ) > $out/${tag}_ncu_train.log 2>&1
tail -4 $out/${tag}_smoke.txt; tail -3 $out/${tag}_pytest.txt; head -c 300 $out/${tag}_bench.json; echo; head -c 300 $out/${tag}_bench_default_flags.json; echo; head -c 300 $out/${tag}_bench_reference.json; echo; head -c 300 $out/${tag}_bench_train480.json
