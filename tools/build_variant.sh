#!/bin/bash
# build an A/B variant of the engine: tools/build_variant.sh <name> [-DFLAG=VAL ...]  ->  hdl_graph_slam_b200/_lib/alt/libb200reg_<name>.so
set -e
cd "$(dirname "$0")/.."
name=$1; shift
mkdir -p hdl_graph_slam_b200/_lib/alt
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared -ccbin /usr/bin/g++ "$@" \
  -o hdl_graph_slam_b200/_lib/alt/libb200reg_$name.so hdl_graph_slam_b200/csrc/api.cu -lnccl
echo built $name
