#!/bin/bash
# build_variant.sh <name> [extra nvcc flags...]: developer A/B builds of the CUDA library into dvo_slam_b200/variants/
set -e
name=$1; shift
mkdir -p dvo_slam_b200/variants
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr \
  "$@" -shared -o dvo_slam_b200/variants/$name.so dvo_slam_b200/csrc/pyramid.cu dvo_slam_b200/csrc/tracker.cu dvo_slam_b200/csrc/capi.cu dvo_slam_b200/csrc/sharded.cu 2>&1 | grep -E "error|warning: v" || true
ls -la dvo_slam_b200/variants/$name.so
