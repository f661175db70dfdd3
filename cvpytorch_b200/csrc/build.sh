#!/usr/bin/env bash
# Builds libcvb200.so (sm_90a only: H100) next to the Python package.  Usage: build.sh [diag] [extra nvcc flags]
#   build.sh diag ...  builds libcvb200_diag.so instead: same sources with -DCVB_DIAG=1 (per-role cycle counters + CVB_DBG switches of the
#   conv kernel; used by tools/conv_pipeline_profile.py and tools/head_profile.py through CVB_DIAG_LIB=1, never by the product path)
# The translation units compile in parallel into a temporary directory; only the library lands in the tree.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/../libcvb200.so"
EXTRA=()
if [[ "${1:-}" == "diag" ]]; then
  shift
  OUT="$HERE/../libcvb200_diag.so"
  EXTRA=(-DCVB_DIAG=1)
fi
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-O3 -I"$HERE/../../include")
TMP="$(mktemp -d)"
trap 'rm -rf "$TMP"' EXIT
pids=()
for src in api conv_tc aux_kernels nms train_kernels yolox_loss yolov5_loss fcos_loss ema sgd coco_eval seg_eval; do
  FILE_FLAGS=()
  # the losses, the EMA and SGD follow the reference's fp32 operation order, and the COCO evaluation pycocotools' float64 one: no contracted
  # multiply-adds
  [[ "$src" == yolox_loss || "$src" == yolov5_loss || "$src" == fcos_loss || "$src" == ema || "$src" == sgd || "$src" == coco_eval ]] && FILE_FLAGS=(--fmad=false)
  "$NVCC" "${FLAGS[@]}" "${FILE_FLAGS[@]}" "${EXTRA[@]}" "$@" -c "$HERE/$src.cu" -o "$TMP/$src.o" &
  pids+=($!)
done
for p in "${pids[@]}"; do wait "$p"; done
"$NVCC" -gencode arch=compute_90a,code=sm_90a --shared -o "$TMP/lib.so" "$TMP"/*.o -lcudart
mv -f "$TMP/lib.so" "$OUT"
echo "built $OUT"
