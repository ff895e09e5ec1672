#!/bin/bash
# A/B helper for kernel experiments: builds one library per set of extra nvcc flags into tools/ab/ (git-ignored),
# then prints the command that runs the parity tests once and the kernel-only bench for every variant, to be run on the GPU machine.
#   tools/ab_variants.sh base "" t256 "-DTW_NOISE2_THREADS=256 -DTW_NOISE2_MIN_BLOCKS=3" lut2 "-DTW_SIMPLEX_LUT=2 -DTW_NOISE2_THREADS=256 -DTW_NOISE2_MIN_BLOCKS=5"
# Knobs that exist today: TW_SIMPLEX_LUT (0 no table, 1 gradient, 2 + first hash, 3 + second hash folded = shipped), TW_NOISE2_MIN_BLOCKS,
# TW_NOISE2_THREADS, TW_NOISE2_BLOCK_CELLS, TW_NOISE2_PERSISTENT, TW_DWARP_WIN_OCTAVES, TW_DWARP_WIN_THREADS, TW_DWARP_WARP_MARGIN (tw_heightgen.cu); run-time: TW_NOISE_SCALAR=1 (scalar kernel), TW_EROSION_LANES, TW_PIPE_CHUNKS.
set -e
cd "$(dirname "$0")/.."
mkdir -p tools/ab
names=()
while [ $# -ge 2 ]; do
  name=$1; flags=$2; shift 2
  echo "== building $name: $flags"
  TW_EXTRA_NVCC_FLAGS="$flags" TW_BUILD_LIB="$PWD/tools/ab/lib_$name.so" TW_BUILD_OBJDIR="$PWD/tools/ab/obj_$name" python 3dworld_b200/build.py --force > /dev/null
  rm -rf "tools/ab/obj_$name"
  names+=("$name")
done
echo "run on the GPU machine:"
echo "bash -c 'cp 3dworld_b200/lib3dworld_b200.so /tmp/lib_shipped.so; for v in ${names[*]}; do cp tools/ab/lib_\$v.so 3dworld_b200/lib3dworld_b200.so; echo == \$v; python -m pytest tests/test_gpu_heightgen.py -x -q | tail -1; python bench.py --kernel-only --steps 10 --warmup 3 | cut -c1-160; done'"
