#!/bin/bash
# Builds libi3d_b200.so (sm_90a only, H100) in-tree: intrinsic3d_b200/libi3d_b200.so
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../libi3d_b200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
"$NVCC" -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 \
    -Xcompiler -fPIC,-O3 -ccbin /usr/bin/g++ -shared $EXTRA_NVCC_FLAGS \
    -o "$OUT" "$HERE/i3d_engine.cu" "$HERE/i3d_fusion.cu" "$HERE/i3d_frames.cu" "$HERE/i3d_mesh.cu" "$HERE/i3d_render.cu" "$HERE/i3d_texture.cu" "$HERE/i3d_distance.cu" "$HERE/i3d_grid_from_mesh.cu" "$HERE/i3d_raster.cu"
echo "built $OUT"
