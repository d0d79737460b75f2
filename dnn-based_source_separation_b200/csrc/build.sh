#!/bin/bash
# Builds libctn_b200.so in-tree for sm_90a (H100).  Usage: csrc/build.sh [extra nvcc flags]
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OUT="$HERE/../libctn_b200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
mkdir -p "$HERE/build"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -I"$ROOT/include" -I"$HERE" "$@")
pids=()
for f in ctn_api ctn_encdec ctn_norm ctn_loss ctn_tcn_simt ctn_wgmma ctn_train ctn_wgrad_wgmma ctn_causal ctn_causal_train ctn_dprnn ctn_optim ctn_conv ctn_lstm ctn_dptnet ctn_sepformer ctn_tasnet ctn_galr ctn_pitx ctn_online ctn_ola ctn_bss ctn_bss_images ctn_probe; do
  if [ ! -f "$HERE/build/$f.o" ] || [ "$HERE/$f.cu" -nt "$HERE/build/$f.o" ] || [ "$HERE/ctn_common.cuh" -nt "$HERE/build/$f.o" ] \
     || [ "$HERE/ctn_internal.h" -nt "$HERE/build/$f.o" ] || [ "$ROOT/include/ctn_b200.h" -nt "$HERE/build/$f.o" ] || [ "$ROOT/include/ctn_b200_probe.h" -nt "$HERE/build/$f.o" ] \
     || [ "$HERE/ctn_wgmma_ptx.cuh" -nt "$HERE/build/$f.o" ] || [ "$HERE/ctn_sisdr_grad.cuh" -nt "$HERE/build/$f.o" ] \
     || [ "$HERE/ctn_dw_math.cuh" -nt "$HERE/build/$f.o" ] || [ "$HERE/build.sh" -nt "$HERE/build/$f.o" ]; then
    "$NVCC" "${FLAGS[@]}" -c "$HERE/$f.cu" -o "$HERE/build/$f.o" &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [ -n "$p" ] && wait "$p"; done
"$NVCC" -shared -gencode arch=compute_90a,code=sm_90a -o "$OUT" "$HERE"/build/ctn_api.o "$HERE"/build/ctn_encdec.o "$HERE"/build/ctn_norm.o \
  "$HERE"/build/ctn_loss.o "$HERE"/build/ctn_tcn_simt.o "$HERE"/build/ctn_wgmma.o "$HERE"/build/ctn_train.o "$HERE"/build/ctn_wgrad_wgmma.o "$HERE"/build/ctn_causal.o "$HERE"/build/ctn_causal_train.o "$HERE"/build/ctn_dprnn.o "$HERE"/build/ctn_optim.o "$HERE"/build/ctn_conv.o "$HERE"/build/ctn_lstm.o "$HERE"/build/ctn_dptnet.o "$HERE"/build/ctn_sepformer.o "$HERE"/build/ctn_tasnet.o "$HERE"/build/ctn_galr.o "$HERE"/build/ctn_pitx.o "$HERE"/build/ctn_online.o "$HERE"/build/ctn_ola.o "$HERE"/build/ctn_bss.o "$HERE"/build/ctn_bss_images.o "$HERE"/build/ctn_probe.o -lcudart
echo "built $OUT"
