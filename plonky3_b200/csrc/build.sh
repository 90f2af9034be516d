#!/bin/bash
# Builds libp3gpu.so for sm_90a (H100) in-tree (plonky3_b200/libp3gpu.so).  Usage: build.sh [extra nvcc flags]
set -e
cd "$(dirname "$0")"
OUT=${P3GPU_OUT:-../libp3gpu.so}
OBJ=${P3GPU_OBJ:-../../build/obj}
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -ccbin /usr/bin/g++ $*"
mkdir -p $OBJ
pids=()
for f in ntt hash fri open peer air air_program air_check keccak_air blake3_air sha256_air poseidon1_air challenger query capi; do
  $NVCC $FLAGS -c $f.cu -o $OBJ/$f.o &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC $ARCH -shared -ccbin /usr/bin/g++ -o $OUT $OBJ/{ntt,hash,fri,open,peer,air,air_program,air_check,keccak_air,blake3_air,sha256_air,poseidon1_air,challenger,query,capi}.o
echo "built $(realpath $OUT)"
