#!/bin/bash
# build_variant.sh <name> [extra nvcc flags...]: developer A/B builds of the CUDA library into dvo_slam_b200/variants/, from
# the sources that __graft_entry__.build() compiles
set -e
name=$1; shift
mkdir -p dvo_slam_b200/variants
srcs=$(python3 -c "import __graft_entry__ as g; print(' '.join('dvo_slam_b200/csrc/' + s for s in g.SOURCES))")
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr \
  "$@" -shared -o dvo_slam_b200/variants/$name.so $srcs 2>&1 | grep -E "error|warning: v" || true
ls -la dvo_slam_b200/variants/$name.so
