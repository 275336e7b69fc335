#!/bin/bash
# Build libssn_b200.so in-tree for sm_90a (H100); the .so and the objects under build/ are git-ignored.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall -I../../include"
mkdir -p build
pids=()
for f in engine simt_conv simt_glue heads classifier umma_conv umma_wgrad s2d_glue glue_vec tc_glue detect detection_ap classification_ap video_agg proposals proposal_lists proposal_ar bn_train frames jpeg inception_v3 train_loop optical_flow jpeg_encode jpeg_roundtrip frame_resize; do
  if [ ! -f build/$f.o ] || [ $f.cu -nt build/$f.o ] || [ common.cuh -nt build/$f.o ] || [ graph.cuh -nt build/$f.o ] || [ umma_conv.cuh -nt build/$f.o ] || [ umma_dev.cuh -nt build/$f.o ] || [ rank_key.cuh -nt build/$f.o ] || [ interp_ap.cuh -nt build/$f.o ] || [ jpeg_common.cuh -nt build/$f.o ] || [ jpeg_block.cuh -nt build/$f.o ] || [ ../../include/ssnb.h -nt build/$f.o ] || [ build.sh -nt build/$f.o ]; then
    $NVCC $FLAGS ${PTXAS_V:+-Xptxas -v} -c $f.cu -o build/$f.o &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
$NVCC $ARCH -shared -o ../ssn_b200/libssn_b200.so build/engine.o build/simt_conv.o build/simt_glue.o build/heads.o build/classifier.o build/umma_conv.o build/umma_wgrad.o build/s2d_glue.o build/glue_vec.o build/tc_glue.o build/detect.o build/detection_ap.o build/classification_ap.o build/video_agg.o build/proposals.o build/proposal_lists.o build/proposal_ar.o build/bn_train.o build/frames.o build/jpeg.o build/inception_v3.o build/train_loop.o build/optical_flow.o build/jpeg_encode.o build/jpeg_roundtrip.o build/frame_resize.o -lcudart_static -ldl -lpthread -lrt
echo "built ../ssn_b200/libssn_b200.so"
