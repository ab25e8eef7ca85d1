#!/bin/bash
# compute-sanitizer passes on small shapes (SURVEY.md §5.2). Run on the GPU box:
#   gpurun -- bash bench/sanitize.sh
# Cross-GPU races are outside what racecheck can see; the flag protocol of the fused all-reduce is
# covered by the multi-rank stress tests instead (tests/mp_allreduce_worker.py).
set -u
mkdir -p gpurun_out
CS=/usr/local/cuda/bin/compute-sanitizer
run() { # name tool pytest-args...
  local name=$1 tool=$2; shift 2
  timeout 280 $CS --tool $tool --error-exitcode 9 --print-limit 5 python -m pytest "$@" -x -q -m gpu > gpurun_out/sanitize_$name.log 2>&1
  echo "$name ($tool): rc=$? $(grep -E 'ERROR SUMMARY|passed|failed' gpurun_out/sanitize_$name.log | tr '\n' ' ')"
}
if [ "${1:-all}" != "new" ]; then
run he_memcheck memcheck tests/test_gpu_he.py -k "ntt_gpu_matches_cpu and 10 or pointwise or local_sum or protocol_single_gpu"
run he_racecheck racecheck tests/test_gpu_he.py -k "ntt_gpu_matches_cpu and 12 or coeff_packing"
run he_synccheck synccheck tests/test_gpu_he.py -k "fedavg_end_to_end or encrypt_decrypt_gpu_bit_exact and 4096"
run conv_memcheck memcheck tests/test_gpu_conv.py -k "unpool or preprocess or (fwd_pool and 20) or (wgrad and 20) or (dgrad and 14)"
fi
# kernels added later: gather wgrad (66-pixel case), dense head (cluster kernel with DSMEM, and the 4-kernel
# fallback), s-packed first layer (70-pixel case), BatchNorm / avg-pool / fp8 quantise
if [ "${1:-all}" = "new" ] || [ "${1:-all}" = "all" ]; then
run new_memcheck memcheck tests/test_gpu_conv.py -k "(gather and 66) or (head and 8-2-True) or (spack and 70)"
run new_racecheck racecheck tests/test_gpu_conv.py -k "(gather and 66) or (head and 8-2-True-512)"
run resnet_memcheck memcheck tests/test_gpu_resnet.py -k "(bn_act and shape2) or avgpool or fp8_conv1x1"
fi
