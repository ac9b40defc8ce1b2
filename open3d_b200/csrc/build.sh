#!/bin/bash
# Builds libo3db200.so (sm_90a only) in-tree next to the python package.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libo3db200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
ARCH=(-gencode arch=compute_90a,code=sm_90a)
FLAGS=("${ARCH[@]}" -lineinfo -O3 -std=c++17
       -Xcompiler -fPIC,-ffp-contract=off,-Wall,-Wno-unused-function
       --expt-relaxed-constexpr ${O3DB_NVCC_EXTRA:-})
cd "${HERE}"
OBJS=()
PIDS=()
for f in common icp tsdf comm pointcloud raycast odometry extract projection knn smooth dbscan fps segment boundary remove fpfh ransac fgr; do
  EXTRA=()
  # ransac.cu and fgr.cu state one evaluation order for their f64 arithmetic: every op rounded, no FMA
  # (DESIGN.md §4.25, §4.26)
  [[ "${f}" == ransac || "${f}" == fgr ]] && EXTRA=(-fmad=false)
  "${NVCC}" "${FLAGS[@]}" "${EXTRA[@]}" -c "${f}.cu" -o "${f}.o" &
  PIDS+=($!)
  OBJS+=("${f}.o")
done
for p in "${PIDS[@]}"; do wait "$p"; done
"${NVCC}" "${ARCH[@]}" -shared -o "${OUT}" "${OBJS[@]}" -ldl
rm -f "${OBJS[@]}"
echo "built ${OUT}"
