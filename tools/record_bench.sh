#!/bin/bash
# Records behind BASELINE.md §3: the GPU's identity and power limit, the whole test suite, smoke(), and bench.py lines of every
# workload (the 16-CTA-cluster A/B pairs as well).  Run from the repository root on the GPU:
#   bash tools/record_bench.sh OUT_DIR [all|tests|bench]
set -u
O=${1:?output directory}
PART=${2:-all}
mkdir -p "$O"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm,memory.total,driver_version --format=csv > "$O/gpu.csv"
python -c "import __graft_entry__ as g; g.build()" > "$O/build.log" 2>&1 || { tail -20 "$O/build.log"; exit 1; }
if [ "$PART" != "bench" ]; then
  timeout 1500 python -m pytest tests -q -p no:cacheprovider -rs > "$O/pytest.txt" 2>&1; echo "pytest exit $?" >> "$O/pytest.txt"
  timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$O/smoke.txt" 2>&1; echo "smoke exit $?" >> "$O/smoke.txt"
fi
[ "$PART" = "tests" ] && exit 0
run() {  # run NAME [ENV=VALUE ...] -- bench.py arguments: the JSON line goes to NAME.json
  local name=$1; shift
  local envs=()
  while [ "$1" != "--" ]; do envs+=("$1"); shift; done; shift
  timeout 900 env "${envs[@]}" python bench.py "$@" > "$O/$name.json" 2> "$O/$name.err" || tail -5 "$O/$name.err"
}
run gicp_odometry_1 -- --gpus 1 --steps 200 --warmup 5 --dump-outputs "$O/outputs_gicp_odometry_1"
run gicp_odometry_2 -- --gpus 1 --steps 200 --warmup 5 --cpu-sample 0 --no-anchor --dump-outputs "$O/outputs_gicp_odometry_2"
run gicp_odometry_cluster8 B2R_NO_CLUSTER16=1 -- --gpus 1 --steps 200 --warmup 5 --cpu-sample 0 --no-anchor
run ndt_odometry_1 -- --workload ndt_odometry_hdl32e_128k --steps 50 --warmup 5 --cpu-sample 2 --no-anchor
run ndt_odometry_2 -- --workload ndt_odometry_hdl32e_128k --steps 50 --warmup 5 --cpu-sample 0 --no-anchor
run ndt_odometry_cluster8 B2R_NO_CLUSTER16=1 -- --workload ndt_odometry_hdl32e_128k --steps 50 --warmup 5 --cpu-sample 0 --no-anchor
run voxelgrid_1 -- --workload voxelgrid --steps 200 --warmup 5 --dump-outputs "$O/outputs_voxelgrid"
run voxelgrid_2 -- --workload voxelgrid --steps 200 --warmup 5
run voxelgrid_cluster8 B2R_NO_CLUSTER16=1 -- --workload voxelgrid --steps 200 --warmup 5
run loop_batch -- --workload loop_batch --dump-outputs "$O/outputs_loop_batch"
run kitti_pipeline -- --workload kitti_pipeline --steps 100 --warmup 5 --dump-outputs "$O/outputs_kitti_pipeline"
run kitti_pipeline_cluster8 B2R_NO_CLUSTER16=1 -- --workload kitti_pipeline --steps 100 --warmup 5 --cpu-sample 0
