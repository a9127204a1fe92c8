#!/bin/bash
# 2-GPU validation: data-parallel parity test, bench.py under torchrun, the reference arm under
# torchrun, and the train_parent.py entry point
cd "$(dirname "$0")/.."
out=${OSVOS_RESULTS:-results}   # output directory (git-ignored)
mkdir -p "$out"
tag=${1:-c8}
nvidia-smi -L > $out/${tag}_gpus.txt
( timeout 600 python -m pytest tests/test_gpu_dp.py -m gpu -q -s -p no:cacheprovider 2>&1 | tail -15 ) > $out/${tag}_dp_test.txt
( timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 bench.py --gpus 2 --steps 20 --warmup 5 ) > $out/${tag}_bench_2gpu.json 2>$out/${tag}_bench_2gpu.err
( timeout 300 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29534 bench.py --impl reference --gpus 2 --steps 3 --warmup 1 ) > $out/${tag}_bench_ref_2gpu.json 2>$out/${tag}_bench_ref_2gpu.err
( OSVOS_SAVE_ROOT=/tmp/osvos_models timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29535 train_parent.py --synthetic --epochs 3 --iters-per-epoch 12 --n-ave-grad 2 --batch 2 --height 240 --width 427 --lr 1e-10 ) > $out/${tag}_train_parent_2gpu.txt 2>&1
( OSVOS_SAVE_ROOT=/tmp/osvos_models timeout 600 python train_online.py --synthetic --iters 200 --height 240 --width 427 --no-save ) > $out/${tag}_train_online.txt 2>&1
tail -3 $out/${tag}_dp_test.txt; tail -c 1200 $out/${tag}_bench_2gpu.json; echo; tail -c 400 $out/${tag}_bench_2gpu.err; tail -6 $out/${tag}_train_parent_2gpu.txt; tail -8 $out/${tag}_train_online.txt
