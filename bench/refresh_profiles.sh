#!/bin/bash
# Regenerates every single-GPU artefact (run from the repository root on the GPU machine);
# then:
#   python bench/make_profiles.py && python bench/roofline.py && python bench/make_sass.py
# (multi-GPU artefacts: bash bench/run_mgpu.sh N and bash bench/run_pipe.sh N under gpurun --gpus N).
set -u
mkdir -p gpurun_out
rm -f gpurun_out/*.ncu-rep
T="timeout 280"
$T python bench/nn_micro.py      > gpurun_out/nn_micro.log 2>&1
$T python bench/he_micro.py      > gpurun_out/he_micro_v2.log 2>&1
HEFL_HE_V1=1 $T python bench/he_micro.py > gpurun_out/he_micro_v1.log 2>&1
$T python bench/resnet_micro.py  > gpurun_out/resnet_micro.log 2>&1
$T python bench/tcconv_micro.py  > gpurun_out/tcconv_micro.log 2>&1
NCU="ncu --set full --clock-control none --import-source on -f"
$T $NCU -c 1 -k regex:tap_gemm_kernel -o gpurun_out/prof_fwd0_v4 python bench/scratch/one_step.py 3 > /dev/null 2>&1
$T $NCU -c 1 -k regex:wgrad0_gather   -o gpurun_out/prof_gather python bench/scratch/one_step.py 3 > /dev/null 2>&1
$T $NCU -c 1 -k regex:head_cluster    -o gpurun_out/prof_head_cluster python bench/scratch/one_step.py 3 > /dev/null 2>&1
$T $NCU -c 1 -k regex:wgrad_kernel --launch-skip 4 -o gpurun_out/prof_wgrad1 python bench/scratch/one_step.py 3 > /dev/null 2>&1
$T $NCU -c 4 -s 4 -k 'regex:encrypt2_kernel|ntt2_kernel|decrypt2_kernel' -o gpurun_out/prof_he2_n8192 python bench/he_prof.py n8192_l4 600 > /dev/null 2>&1
$T $NCU -c 3 -s 6 -k 'regex:kmajor_gemm_kernel|wgrad_mn_kernel' -o gpurun_out/prof_tcconv_3x3_c128 python bench/tcconv_one.py > /dev/null 2>&1
$T $NCU -c 1 -s 1 -k 'regex:mx_gemm_kernel' -o gpurun_out/prof_mx_gemm python bench/tcconv_one.py > /dev/null 2>&1
$T ncu --metrics gpu__time_duration.sum --clock-control none --launch-skip 75 -c 45 --csv \
   --log-file gpurun_out/launches_v6.csv python bench/scratch/one_step.py 4 > /dev/null 2>&1
$T ncu --metrics gpu__time_duration.sum --clock-control none --csv \
   --log-file gpurun_out/launches_resnet18_tc.csv python bench/resnet_step.py resnet18 tc 3 > /dev/null 2>&1
timeout 600 python bench.py --steps 5 --warmup 3 > gpurun_out/bench_1gpu.json 2> gpurun_out/bench_1gpu.err
B="--steps 3 --warmup 3 --local-epochs 1 --steps-per-epoch 5 --val-steps 1 --no-own-baseline"
$T python bench.py --model resnet18 --he-preset n8192_l4 $B > gpurun_out/bench_resnet18_bf16.json 2> gpurun_out/bench_resnet18.err
$T python bench.py --model resnet50 --he-preset n16384_l4 $B > gpurun_out/bench_resnet50_bf16.json 2> gpurun_out/bench_resnet50.err
$T python bench.py --model resnet50 --he-preset n16384_l4 --dtype fp8 $B > gpurun_out/bench_resnet50_fp8.json 2> gpurun_out/bench_resnet50_fp8.err
$T python bench.py --model resnet18 --he-preset n8192_l4 --nn-backend cudnn $B > gpurun_out/bench_resnet18_cudnn.json 2> /dev/null
cut -c1-300 gpurun_out/bench_1gpu.json; for f in resnet18_bf16 resnet50_bf16 resnet50_fp8 resnet18_cudnn; do python -c "
import json; d=json.load(open('gpurun_out/bench_$f.json')); print('$f', round(d['ms_per_step'],2), d['config']['nn_backend'], d['stage_ms_last_round'])"; done
