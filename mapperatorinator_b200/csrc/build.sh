#!/usr/bin/env bash
# Builds libmapperatorinator_b200.so in-tree for sm_90a (H100; cross-compiles without a GPU).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libmapperatorinator_b200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr -Xcompiler -fPIC -Xcompiler -O3)
if [[ "${MB200_PTXAS_V:-0}" == "1" ]]; then FLAGS+=(-Xptxas -v); fi
mkdir -p "${HERE}/build"
pids=()
for f in c_abi gemm gemm_tc norm attention attention_tc mel audio decode beam decode_mega decode_mega2 engine_model engine_dit slider score; do
  ( "${NVCC}" "${FLAGS[@]}" -c "${HERE}/${f}.cu" -o "${HERE}/build/${f}.o" ) &
  pids+=($!)
done
for p in "${pids[@]}"; do wait "$p"; done
"${NVCC}" -shared -o "${OUT}" "${HERE}"/build/*.o -lcudart
echo "built ${OUT}"
