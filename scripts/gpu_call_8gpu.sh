#!/bin/bash
# 8-GPU evidence: bench.py under torchrun at N = 8 and N = 4 (dp = parent training, batch 12 per GPU, one
# NCCL allreduce per step; headline = inference replicas)
cd "$(dirname "$0")/.."
out=${OSVOS_RESULTS:-results}   # output directory (git-ignored)
mkdir -p "$out"
tag=${1:-c10}
nvidia-smi -L > $out/${tag}_gpus.txt
( NCCL_DEBUG=INFO NCCL_DEBUG_SUBSYS=INIT timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29541 bench.py --gpus 8 --steps 20 --warmup 5 --skip gpu_reference,cpu_baseline,e2e_extra ) > $out/${tag}_bench_8gpu.json 2>$out/${tag}_bench_8gpu.err
( CUDA_VISIBLE_DEVICES=0,1,2,3 timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 --master-port 29542 bench.py --gpus 4 --steps 20 --warmup 5 --skip gpu_reference,cpu_baseline,e2e_extra,parity,roofline ) > $out/${tag}_bench_4gpu.json 2>$out/${tag}_bench_4gpu.err
grep -i "nvls" $out/${tag}_bench_8gpu.err | head -4
python - <<PY
import json
for n in (8, 4):
    try:
        d = json.load(open("$out/${tag}_bench_%dgpu.json" % n))
        dp = d["dp"]
        print(n, "value", d["value"], "dp", {k: dp.get(k) for k in ("fps", "fps_per_gpu", "ms_per_step", "allreduce_ms", "allreduce_in_step_ms")}, "parity", (dp.get("parity") or {}).get("worst_rel_err"))
    except Exception as e:
        print(n, "failed", e)
PY
tail -c 300 $out/${tag}_bench_8gpu.err | tail -3
