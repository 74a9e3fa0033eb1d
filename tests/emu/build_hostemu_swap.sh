#!/bin/bash
# Host-emulated tl/nvl plugin with the in-place alltoall(v) swap kernel (tests/emu/nvl_emu_launch_swap.cpp) into build-emu/lib/ucc_swap,
# next to the libcudart_emu.so of tests/emu/build_hostemu.sh.  Reuses that script's objects of the plugin's host code: run it first.
# Use with UCC_MODULE_DIR=$PWD/build-emu/lib/ucc_swap and libucc.so from ucc_b200/lib.
set -e
cd "$(dirname "$0")/../.."
OUT=build-emu/lib; MOD=$OUT/ucc_swap; OBJ=build-emu/obj
for f in tl_nvl.c tl_nvl_coll.c tl_nvl_team.c tl_nvl_direct.c tl_nvl_memh.c ucc_cuda_util.c; do [ -f $OBJ/$f.o ]; done
[ -f $OUT/ucc/libucc_mc_cuda.so ]
mkdir -p $MOD
CUDA_INC=/usr/local/cuda/include
CF="-O0 $EMU_EXTRA -fPIC -D_GNU_SOURCE -Iinclude -Isrc -I$CUDA_INC -Wall -Wno-unused-parameter -Wno-unused-function"
${EMU_CXX:-g++} $CF -std=c++17 -pthread -Isrc/components/tl/nvl/kernels -Itests/emu -c tests/emu/nvl_emu_launch_swap.cpp -o $OBJ/nvl_emu_launch_swap.o
${EMU_CXX:-g++} $EMU_EXTRA -shared -o $MOD/libucc_tl_nvl.so $OBJ/tl_nvl.c.o $OBJ/tl_nvl_coll.c.o $OBJ/tl_nvl_team.c.o $OBJ/tl_nvl_direct.c.o $OBJ/tl_nvl_memh.c.o $OBJ/ucc_cuda_util.c.o $OBJ/nvl_emu_launch_swap.o \
    -Lucc_b200/lib -lucc -L$OUT -lcudart_emu -Wl,-rpath,'$ORIGIN/..' -Wl,-rpath,$PWD/ucc_b200/lib -lpthread -ldl
cp $OUT/ucc/libucc_mc_cuda.so $MOD/
echo "HOSTEMU_SWAP_BUILD_OK $MOD"
