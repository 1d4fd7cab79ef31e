#!/bin/bash
# Build an A/B variant of the Kuka kernels: scripts/build_variant.sh <name> <extra nvcc flags...>  ->  csrc/libsrl_variant_<name>.so
# (selected at run time with SRL_SIM_CUDA_LIB=<path>; variants are git-ignored build products that travel to the GPU box)
set -e
cd "$(dirname "$0")/../robotics-rl-srl_b200/csrc"
name=$1; shift
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
$NVCC -O3 -std=c++17 -lineinfo $ARCH -Xcompiler -fPIC -cudart static --prec-div=false --prec-sqrt=false -Xptxas -v "$@" -c kuka_kernels.cu -o variant_$name.o 2> variant_$name.ptxas.log
$NVCC $ARCH -shared -cudart static -o libsrl_variant_$name.so srl_sim_abi.o mobile_kernels.o variant_$name.o distractor_kernels.o policy_kernels.o ppo2_kernels.o render_kernels.o
grep -A2 "ILb0ELb0ELb0" variant_$name.ptxas.log | grep -E "stack|registers" || true
