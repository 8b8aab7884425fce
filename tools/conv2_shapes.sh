#!/bin/sh
# Builds tools/conv2_shapes.cu into a temporary directory and runs it on GPU 0, after the card's name, power limit and
# clocks. Arguments go to the probe (batches per warpgroup, default 4000).
set -e
here=$(cd "$(dirname "$0")" && pwd)
nvcc=${NVCC:-$(command -v nvcc || echo "${CUDA_HOME:-/usr/local/cuda}/bin/nvcc")}
tmp=$(mktemp -d)
trap 'rm -rf "$tmp"' EXIT
"$nvcc" -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I"$here/../gpd_b200/csrc" -o "$tmp/conv2_shapes" \
  "$here/conv2_shapes.cu"
nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv
"$tmp/conv2_shapes" "$@"
