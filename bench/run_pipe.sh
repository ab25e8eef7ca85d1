#!/bin/bash
# ResNet-18 FedAvg stage with its per-chunk timeline: bash bench/run_pipe.sh <N> (results under $OUT, default bench_out)
N=${1:-2}
OUT=${OUT:-bench_out}
mkdir -p $OUT
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
ARGS="bench.py --gpus $N --steps 3 --warmup 3 --model resnet18 --he-preset n8192_l4 --local-epochs 1 --steps-per-epoch 5 --val-steps 1 --no-own-baseline --skip-e2e"
HEFL_TIMELINE=$OUT/fedavg_timeline_${N}gpu.json timeout 300 $TR --master-port 29711 $ARGS > $OUT/pipe_${N}.json 2> $OUT/pipe_${N}.err
python - <<PY
import json
try:
    d=json.load(open("$OUT/pipe_${N}.json")); print(d["stage_ms_last_round"], "ms/round", round(d["ms_per_step"],2))
except Exception as e:
    print("failed", e); print(open("$OUT/pipe_${N}.err").read()[-1500:])
PY
