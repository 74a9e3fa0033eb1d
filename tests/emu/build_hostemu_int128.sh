#!/bin/bash
# Host-emulated tl/nvl plugin with INT128 / UINT128 in its datatype table: build-emu/lib/ucc_int128/{libucc_tl_nvl.so,libucc_mc_cuda.so}.
# Links tests/emu/nvl_emu_launch_int128.cpp with the host objects build_hostemu.sh left in build-emu/obj (run that first).
# Use with UCC_MODULE_DIR=$PWD/build-emu/lib/ucc_int128 and libucc.so from ucc_b200/lib.
set -e
cd "$(dirname "$0")/../.."
OUT=build-emu/lib; MOD=$OUT/ucc_int128; OBJ=build-emu/obj
mkdir -p $MOD
CUDA_INC=/usr/local/cuda/include
CF="-O0 $EMU_EXTRA -fPIC -D_GNU_SOURCE -Iinclude -Isrc -I$CUDA_INC -Wall -Wno-unused-parameter -Wno-unused-function"
${EMU_CXX:-g++} $CF -std=c++17 -pthread -Isrc/components/tl/nvl/kernels -Itests/emu -c tests/emu/nvl_emu_launch_int128.cpp -o $OBJ/nvl_emu_launch_int128.o
${EMU_CXX:-g++} $EMU_EXTRA -shared -o $MOD/libucc_tl_nvl.so $OBJ/tl_nvl.c.o $OBJ/tl_nvl_coll.c.o $OBJ/tl_nvl_team.c.o $OBJ/tl_nvl_direct.c.o $OBJ/tl_nvl_memh.c.o $OBJ/ucc_cuda_util.c.o $OBJ/nvl_emu_launch_int128.o \
    -Lucc_b200/lib -lucc -L$OUT -lcudart_emu -Wl,-rpath,'$ORIGIN/..' -Wl,-rpath,$PWD/ucc_b200/lib -lpthread -ldl
cp $OUT/ucc/libucc_mc_cuda.so $MOD/
echo "HOSTEMU_INT128_BUILD_OK $MOD"
