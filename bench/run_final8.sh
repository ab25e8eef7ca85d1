#!/bin/bash
# 8-GPU evidence the driver's scaling run does not produce: the ResNet-18 / ResNet-50 encrypted-FedAvg stage
# (pipelined, with the SM partition) with per-chunk timelines.
N=8
mkdir -p gpurun_out
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
B="--gpus $N --steps 3 --warmup 3 --local-epochs 1 --steps-per-epoch 5 --val-steps 1 --no-own-baseline --skip-e2e"
HEFL_TIMELINE=gpurun_out/fedavg_timeline_8gpu_default.json timeout 300 $TR --master-port 29721 bench.py --model resnet18 --he-preset n8192_l4 $B > gpurun_out/bench_resnet18_8gpu.json 2> gpurun_out/r18_8.err
HEFL_TIMELINE=gpurun_out/fedavg_timeline_8gpu_resnet50.json timeout 300 $TR --master-port 29723 bench.py --model resnet50 --he-preset n16384_l4 --dtype fp8 $B > gpurun_out/bench_resnet50_fp8_8gpu.json 2> gpurun_out/r50_8.err
for f in bench_resnet18_8gpu bench_resnet50_fp8_8gpu; do python -c "
import json
try:
    d=json.load(open('gpurun_out/$f.json')); print('$f', round(d['ms_per_step'],2), d['stage_ms_last_round'], d.get('allreduce_checked'))
except Exception as e: print('$f failed', e)"; done
tail -3 gpurun_out/r18_8.err
