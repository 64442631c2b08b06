#!/bin/bash
# Multi-GPU sweep (run on a box with up to 8 GPUs: bash tools/multigpu_r2.sh): config-5 score sweep, ECAPA
# data-parallel training step and the extraction bench at 1 / 2 / 4 / 8 GPUs.  Writes one JSON line per run into gpurun_out/.
set -u
mkdir -p gpurun_out
NG=$(python -c "import torch; print(torch.cuda.device_count())")
out_s=gpurun_out/score_sweep_r2.jsonl; out_t=gpurun_out/train_scale_r2.jsonl; out_b=gpurun_out/bench_scale_r2.jsonl
: > $out_s; : > $out_t; : > $out_b
port=29600
for n in 1 2 4 8; do
  [ "$n" -gt "$NG" ] && break
  port=$((port+1))
  if [ "$n" -eq 1 ]; then run="python"; else run="python -m torch.distributed.run --nnodes=1 --nproc-per-node $n --master-addr 127.0.0.1 --master-port $port"; fi
  $run tools/score_sweep.py 2>gpurun_out/score_sweep_n$n.err | grep '^{' >> $out_s
  $run tools/train_bench.py --steps 20 2>gpurun_out/train_bench_n$n.err | grep '^{' >> $out_t
  $run bench.py --gpus $n --steps 50 --warmup 5 --no-cpu-baseline 2>gpurun_out/bench_n$n.err | grep '^{' >> $out_b
done
wc -l $out_s $out_t $out_b
