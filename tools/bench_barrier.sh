#!/bin/sh
# Build and run the grid-barrier microbenchmark (tools/bench_barrier.cu) on the local GPU.
set -e
cd "$(dirname "$0")/.."
mkdir -p tools/_build
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -ccbin /usr/bin/g++ -o tools/_build/bench_barrier tools/bench_barrier.cu
exec tools/_build/bench_barrier
