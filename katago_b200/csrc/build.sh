#!/bin/bash
# Builds libkgb200.so in-tree for sm_90a (cross-compiles without a GPU).  Invoked by __graft_entry__.build().
set -e
cd "$(dirname "$0")"
OUT=../libkgb200.so
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -Xcompiler -Wall"
# nothing to do when the library was built from exactly these sources (content hash; the object directory does not travel to
# the GPU box and file times may not survive the copy)
SRCHASH=$(cat *.cu *.cuh *.cpp *.h ../../include/*.h build.sh | sha256sum | cut -d' ' -f1)
if [ -f $OUT ] && [ -f $OUT.srchash ] && [ "$(cat $OUT.srchash)" = "$SRCHASH" ] && [ -z "${KGB_FORCE_BUILD}" ]; then
  echo "up to date $(readlink -f $OUT)"
  exit 0
fi
mkdir -p ../_build
for f in kgb_conv_wg.cu kgb_kernels.cu kgb_api.cu kgb_selfplay.cu; do
  o=../_build/${f%.cu}.o
  if [ ! -f $o ] || [ $f -nt $o ] || [ kgb_conv.cuh -nt $o ] || [ kgb_wgmma.cuh -nt $o ] || [ kgb_kernels.cuh -nt $o ] || [ kgb_model.h -nt $o ] || [ kgb_board.cuh -nt $o ] || [ kgb_ladder.cuh -nt $o ] || [ kgb_history.cuh -nt $o ] || [ kgb_devrand.cuh -nt $o ] || [ kgb_scorevalue.h -nt $o ] || [ kgb_handle.h -nt $o ] || [ kgb_rand.h -nt $o ] || [ ../../include/kgb200.h -nt $o ]; then
    X=""
    # the search arithmetic follows the reference's doubles operation by operation: no FMA contraction there
    if [ $f = kgb_selfplay.cu ]; then X="-fmad=false"; fi
    rm -f $o
    $NVCC $FLAGS $X ${EXTRA_NVCC_FLAGS} -c $f -o $o &
  fi
done
for f in kgb_model.cpp kgb_rand.cpp kgb_scorevalue.cpp; do
  o=../_build/${f%.cpp}.o
  if [ ! -f $o ] || [ $f -nt $o ] || [ kgb_model.h -nt $o ] || [ kgb_rand.h -nt $o ] || [ kgb_scorevalue.h -nt $o ]; then
    rm -f $o
    g++ -O2 -std=c++17 -fPIC -fvisibility=hidden -Wall -c $f -o $o &
  fi
done
wait
# a failed compile leaves no object behind (removed above), so the link below fails too instead of reusing a stale one
for o in kgb_conv_wg kgb_kernels kgb_api kgb_selfplay kgb_model kgb_rand kgb_scorevalue; do
  [ -f ../_build/$o.o ] || { echo "build failed: $o" >&2; exit 1; }
done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o $OUT ../_build/kgb_conv_wg.o ../_build/kgb_kernels.o ../_build/kgb_api.o ../_build/kgb_selfplay.o ../_build/kgb_model.o ../_build/kgb_rand.o ../_build/kgb_scorevalue.o -lz -ldl -cudart shared
echo $SRCHASH > $OUT.srchash
echo "built $(readlink -f $OUT)"
