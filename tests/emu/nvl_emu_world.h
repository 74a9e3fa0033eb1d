// Harness of the kernel drivers (nvl_emu*.cpp): N emulated GPUs' heaps in one address space, and a launch that runs a grid on every
// rank at once, one OS thread per CUDA thread.
#pragma once
#include "nvl_emu_prelude.h"

#define CHECK(c) do { if (!(c)) { printf("EMU FAIL line %d: %s\n", __LINE__, #c); exit(1); } } while (0)

struct World {
    int N; size_t data_size, user_size, heap_size;
    std::vector<char *> heaps; uint32_t host_err = 0;
    World(int n, size_t data, size_t user) : N(n), data_size(data), user_size(user)
    {
        heap_size = NVL_DATA_OFFSET + data + user;
        for (int p = 0; p < n; p++) { char *h = (char *)calloc(1, heap_size + 64); CHECK(h); heaps.push_back((char *)(((uintptr_t)h + 63) & ~(uintptr_t)63)); }
        g_emu.n = n; g_emu.heap_size = heap_size; g_emu.mc_base = (char *)(uintptr_t)0x500000000000ull;
        for (int p = 0; p < n; p++) g_emu.heaps[p] = heaps[p];
    }
    nvl_team_dev_t team(int r, bool nvls) const
    {
        nvl_team_dev_t t; memset(&t, 0, sizeof(t));
        t.rank = r; t.size = N; for (int p = 0; p < N; p++) t.heap[p] = heaps[p];
        t.mc_heap = nvls ? g_emu.mc_base : nullptr; t.data_size = data_size; t.timeout_ns = 60ull * 1000000000ull; t.host_err = const_cast<uint32_t *>(&host_err);
        return t;
    }
    char *user(int r) const { return heaps[r] + NVL_DATA_OFFSET + data_size; }
};

// run fn(rank) as a grid of nb x nt threads on every rank concurrently
template <typename F> static void launch_all(int N, int nb, int nt, F fn)
{
    std::vector<pthread_barrier_t> bars((size_t)N * nb);
    for (auto &b : bars) pthread_barrier_init(&b, nullptr, (unsigned)nt);
    std::vector<std::thread> th;
    th.reserve((size_t)N * nb * nt);
    for (int r = 0; r < N; r++) for (int b = 0; b < nb; b++) for (int t = 0; t < nt; t++)
        th.emplace_back([=, &bars]() {
            threadIdx = {(unsigned)t, 0, 0}; blockIdx = {(unsigned)b, 0, 0}; blockDim = {(unsigned)nt, 1, 1}; gridDim = {(unsigned)nb, 1, 1};
            emu_cta_barrier = &bars[(size_t)r * nb + b];
            fn(r);
        });
    for (auto &x : th) x.join();
    for (auto &b : bars) pthread_barrier_destroy(&b);
}
