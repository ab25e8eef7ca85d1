#!/bin/sh
# builds the stand-alone microbenchmarks next to their sources (binaries are git-ignored)
cd "$(dirname "$0")" && for f in *.cu; do nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o "${f%.cu}.bin" "$f"; done
