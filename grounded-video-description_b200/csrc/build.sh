#!/bin/bash
# Builds libgvd_b200.so (sm_90a) next to the package; invoked by __graft_entry__.build().
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libgvd_b200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden
       --expt-relaxed-constexpr -Xptxas -v ${NVCC_EXTRA:-})
mkdir -p "${HERE}/build"
objs=()
for src in gvd_gemm gvd_wgmma gvd_attn gvd_rowops gvd_decode gvd_beam gvd_losses gvd_skinny gvd_train gvd_tfm gvd_tfm_train gvd_api; do
  obj="${HERE}/build/${src}.o"
  if [[ ! -f "$obj" || "${HERE}/${src}.cu" -nt "$obj" || "${HERE}/gvd_common.cuh" -nt "$obj" || "${HERE}/gvd_kernels.cuh" -nt "$obj" || "${HERE}/gvd_gemm.cuh" -nt "$obj" || "${HERE}/gvd_wgmma.cuh" -nt "$obj" || "${HERE}/../../include/gvd_b200.h" -nt "$obj" ]]; then
    "$NVCC" "${FLAGS[@]}" -c "${HERE}/${src}.cu" -o "$obj" 2> "${HERE}/build/${src}.ptxas.log" || { cat "${HERE}/build/${src}.ptxas.log"; exit 1; }
  fi
  objs+=("$obj")
done
"$NVCC" -shared -o "$OUT" "${objs[@]}"
echo "built $OUT"
