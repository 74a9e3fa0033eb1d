// The tl/nvl kernel sources compiled as plain C++ (NVL_HOST_EMU): every CUDA thread is an OS thread, a CTA's threads meet at a
// pthread barrier, every "GPU" is a heap in this address space and the NVSwitch multicast window is a fake address range (g_emu).
// Defines g_emu: include it in exactly one translation unit of a program (the emulated plugin's launchers, or one driver).
#pragma once
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <vector>
#include <pthread.h>
#include <cuda_runtime_api.h>
#include <vector_types.h>
#include <vector_functions.h>
#define NVL_HOST_EMU 1
#ifndef __launch_bounds__
#define __launch_bounds__(...)
#endif
struct emu_dim3 { unsigned x, y, z; };
static thread_local emu_dim3 threadIdx, blockIdx, blockDim, gridDim;
static thread_local pthread_barrier_t *emu_cta_barrier;
static inline void __syncthreads() { pthread_barrier_wait(emu_cta_barrier); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline unsigned atomicAdd(unsigned *p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_ACQ_REL); }

#include "nvl_reduce_impl.cuh"
nvl_emu_world g_emu;   /* filled by the drivers; the emulated plugin leaves it empty: its teams never get an mc_heap */
#include "nvl_kernels.cu"
#include "nvl_pipe.cu"
#include "nvl_symm.cu"
#include "nvl_push.cu"
#include "nvl_oneshot_rs.cu"
#include "nvl_p2p.cu"
#include "nvl_swap.cu"
