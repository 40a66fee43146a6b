#!/usr/bin/env bash
# Builds graphcast_b200/libgraphcast_b200.so for the H100 (sm_90a), in the source tree.
set -euo pipefail
here="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
out="${here}/../libgraphcast_b200.so"
nvcc -std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a \
  -DGCB_BOUNDED_WAIT ${GCB_EXTRA_NVCC_FLAGS:-} \
  -Xcompiler -fPIC -shared \
  -o "${out}" "${here}/api.cu" -lcudart
echo "built ${out}"
