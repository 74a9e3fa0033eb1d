// Host emulation of tl/nvl collective kernels on the real datatypes (the emulation itself: nvl_emu_prelude.h).  Exercises the
// kernels' indexing / phase / flag logic without a GPU (the staged kernel, validated on real GPUs, is run too as a control).
#include <cmath>
#include "nvl_emu_world.h"

template <typename T> static T val(int r, size_t i) { return (T)((i * 7 + (size_t)r * 13) % 23); }

template <typename T> static void check_allreduce(const char *name, const std::vector<T *> &dst, int N, size_t count, int op)
{
    for (int r = 0; r < N; r++) for (size_t i = 0; i < count; i++) {
        double e = 0; for (int p = 0; p < N; p++) { double v = (double)val<T>(p, i); e = p == 0 ? v : (op == NVL_OP_MAX ? std::max(e, v) : e + v); }
        if (op == NVL_OP_AVG) e /= N;
        if (std::fabs((double)dst[r][i] - e) > 1e-3 * std::max(1.0, std::fabs(e))) { printf("EMU FAIL %s: rank %d elem %zu got %g expected %g\n", name, r, i, (double)dst[r][i], e); exit(1); }
    }
}

// allreduce through `kernel` (staged / pipe): plain tensors outside the heaps
template <typename T, typename K> static void run_allreduce(const char *name, World &w, K kernel, size_t count, int op, bool nvls, bool inplace, int nb, int nt, int repeats, size_t misalign = 0)
{
    const int N = w.N;
    std::vector<std::vector<T>> sb(N, std::vector<T>(count + 64)), db(N, std::vector<T>(count + 64, (T)-1));
    std::vector<T *> src(N), dst(N);
    for (int r = 0; r < N; r++) { src[r] = sb[r].data() + 16 + misalign; dst[r] = inplace ? src[r] : db[r].data() + 16 + misalign; }
    for (int it = 0; it < repeats; it++) {
        for (int r = 0; r < N; r++) for (size_t i = 0; i < count; i++) src[r][i] = val<T>(r, i);
        for (int r = 0; r < N; r++) { sb[r][15 + misalign] = (T)99; if (!inplace) { db[r][15 + misalign] = (T)77; db[r][16 + misalign + count] = (T)77; } }
        launch_all(N, nb, nt, [&](int r) {
            nvl_red_args_t a; memset(&a, 0, sizeof(a));
            a.team = w.team(r, nvls); a.src = src[r]; a.dst = dst[r]; a.count = count; a.op = op; a.kind = NVL_RED_ALLREDUCE; a.use_nvls = nvls;
            kernel(a);
        });
        CHECK(w.host_err == 0);
        check_allreduce<T>(name, dst, N, count, op);
        if (!inplace) for (int r = 0; r < N; r++) CHECK(db[r][15 + misalign] == (T)77 && db[r][16 + misalign + count] == (T)77); /* nothing written outside dst */
    }
    printf("  ok %-40s count %zu N %d grid %dx%d%s%s x%d\n", name, count, N, nb, nt, inplace ? " inplace" : "", misalign ? " unaligned" : "", repeats);
}

// zero-copy two-shot (direct) kernel: every rank reads the peers' src and writes the peers' dst in place
template <int NP, int U> static void run_direct(World &w, size_t count, int op, bool inplace, int nb, int nt)
{
    const int N = w.N;
    std::vector<std::vector<float>> sb(N, std::vector<float>(count + 64)), db(N, std::vector<float>(count + 64, -1.f));
    std::vector<float *> src(N), dst(N);
    for (int r = 0; r < N; r++) { src[r] = sb[r].data() + 16; dst[r] = inplace ? src[r] : db[r].data() + 16; for (size_t i = 0; i < count; i++) src[r][i] = val<float>(r, i); if (!inplace) { db[r][15] = 77.f; db[r][16 + count] = 77.f; } }
    launch_all(N, nb, nt, [&](int r) {
        nvl_red_args_t a; memset(&a, 0, sizeof(a));
        a.team = w.team(r, false); a.src = src[r]; a.dst = dst[r]; a.count = count; a.op = op; a.kind = NVL_RED_ALLREDUCE; a.direct = NVL_DIRECT_FULL;
        for (int p = 0; p < N; p++) { a.d.src[p] = (const char *)src[p]; a.d.dst[p] = (char *)dst[p]; }
        nvl_reduce_direct_kernel<float>(a);
    });
    CHECK(w.host_err == 0);
    check_allreduce<float>("direct", dst, N, count, op);
    if (!inplace) for (int r = 0; r < N; r++) CHECK(db[r][15] == 77.f && db[r][16 + count] == 77.f);
    printf("  ok %-40s count %zu N %d grid %dx%d%s\n", "direct (zero-copy two-shot, control)", count, N, nb, nt, inplace ? " inplace" : "");
}

template <typename T> static void run_symm(World &w, size_t count, int op, bool inplace, int nb, int nt)
{
    const int N = w.N;
    std::vector<T *> src(N), dst(N);
    const size_t bytes = ((count * sizeof(T) + 255) / 256) * 256;
    CHECK(2 * bytes + 256 <= w.user_size);
    for (int r = 0; r < N; r++) { src[r] = (T *)w.user(r); dst[r] = inplace ? src[r] : (T *)(w.user(r) + bytes); memset(w.user(r), 0x5a, 2 * bytes + 256); for (size_t i = 0; i < count; i++) src[r][i] = val<T>(r, i); }
    launch_all(N, nb, nt, [&](int r) {
        nvl_red_args_t a; memset(&a, 0, sizeof(a));
        a.team = w.team(r, true); a.src = src[r]; a.dst = dst[r]; a.count = count; a.op = op; a.kind = NVL_RED_ALLREDUCE; a.use_nvls = 1;
        a.d.src[0] = (const char *)src[r]; a.d.dst[0] = (char *)dst[r];
        nvl_allreduce_symm_kernel<T>(a);
    });
    CHECK(w.host_err == 0);
    check_allreduce<T>("symm allreduce", dst, N, count, op);
    for (int r = 0; r < N; r++) { const unsigned char *g = (const unsigned char *)(dst[r] + count); for (size_t i = 0; i < 64; i++) CHECK(g[i] == 0x5a || (char *)g + i >= w.user(r) + 2 * bytes + 256); }
    printf("  ok %-40s count %zu N %d grid %dx%d%s\n", "symm allreduce", count, N, nb, nt, inplace ? " inplace" : "");
}

static void run_symm_rs(World &w, size_t blk, int nb, int nt)
{
    const int N = w.N; const size_t count = blk * N;
    std::vector<std::vector<float>> out(N, std::vector<float>(blk + 8, -1.f));
    for (int r = 0; r < N; r++) { float *s = (float *)w.user(r); for (size_t i = 0; i < count; i++) s[i] = val<float>(r, i); }
    launch_all(N, nb, nt, [&](int r) {
        nvl_red_args_t a; memset(&a, 0, sizeof(a));
        a.team = w.team(r, true); a.src = w.user(r); a.dst = out[r].data() + 1 /* unaligned destination */; a.count = count; a.op = NVL_OP_SUM; a.kind = NVL_RED_REDUCE_SCATTER; a.use_nvls = 1;
        for (int p = 0; p < N; p++) { a.rs_offset[p] = (size_t)p * blk; a.rs_count[p] = blk; }
        a.d.src[0] = w.user(r);
        nvl_allreduce_symm_kernel<float>(a);
    });
    for (int r = 0; r < N; r++) { for (size_t i = 0; i < blk; i++) { float e = 0; for (int p = 0; p < N; p++) e += val<float>(p, (size_t)r * blk + i); CHECK(out[r][1 + i] == e); } CHECK(out[r][0] == -1.f && out[r][1 + blk] == -1.f); }
    printf("  ok %-40s blk %zu N %d grid %dx%d\n", "symm reduce_scatter", blk, N, nb, nt);
}

static void run_symm_ag(World &w, size_t blk_bytes, bool inplace, int nb, int nt)
{
    const int N = w.N;
    std::vector<std::vector<unsigned char>> mine(N, std::vector<unsigned char>(blk_bytes + 32));
    for (int r = 0; r < N; r++) { memset(w.user(r), 0x11, blk_bytes * N + 64); for (size_t i = 0; i < blk_bytes; i++) mine[r][16 + i] = (unsigned char)(r * 31 + i); if (inplace) memcpy(w.user(r) + r * blk_bytes, mine[r].data() + 16, blk_bytes); }
    launch_all(N, nb, nt, [&](int r) {
        nvl_xchg_args_t a; memset(&a, 0, sizeof(a));
        a.team = w.team(r, true); a.dst = w.user(r); a.src = inplace ? (const void *)(w.user(r) + r * blk_bytes) : (const void *)(mine[r].data() + 16); a.src_bytes = blk_bytes; a.push_off = (size_t)r * blk_bytes;
        nvl_allgather_symm_kernel(a);
    });
    for (int r = 0; r < N; r++) { for (int p = 0; p < N; p++) for (size_t i = 0; i < blk_bytes; i++) CHECK((unsigned char)w.user(r)[p * blk_bytes + i] == (unsigned char)(p * 31 + i)); for (int i = 0; i < 64; i++) CHECK(w.user(r)[blk_bytes * N + i] == 0x11); }
    printf("  ok %-40s blk %zu B N %d grid %dx%d%s\n", "symm allgather", blk_bytes, N, nb, nt, inplace ? " inplace" : "");
}

// exchange kernel (pull / NVLS push / ring), arguments built the way tl_nvl_coll.c:xchg_init* builds them
enum { XCHG_AG_PULL, XCHG_A2A_PULL, XCHG_AG_MC, XCHG_AG_RING };
static unsigned char pat(int from, int to, size_t i) { return (unsigned char)(from * 37 + to * 11 + i * 3 + 1); }
static void run_xchg(World &w, int mode, size_t blk, int nb, int nt, size_t misalign = 0)
{
    const int N = w.N; const bool a2a = mode == XCHG_A2A_PULL;
    const size_t ablk = (blk + 15) / 16 * 16;
    std::vector<std::vector<unsigned char>> sb(N, std::vector<unsigned char>((a2a ? blk * N : blk) + 64)), db(N, std::vector<unsigned char>(blk * N + 64, 0xee));
    for (int r = 0; r < N; r++) for (int to = 0; to < (a2a ? N : 1); to++) for (size_t i = 0; i < blk; i++) sb[r][16 + misalign + to * blk + i] = pat(r, a2a ? to : 0, i);
    for (int rep = 0; rep < 2; rep++) {
        for (int r = 0; r < N; r++) memset(db[r].data(), 0xee, db[r].size());
        launch_all(N, nb, nt, [&](int r) {
            nvl_xchg_args_t a; memset(&a, 0, sizeof(a));
            a.team = w.team(r, mode == XCHG_AG_MC); a.src = sb[r].data() + 16 + misalign; a.dst = db[r].data() + 16 + misalign;
            a.src_bytes = a2a ? blk * N : blk;
            for (int p = 0; p < N; p++) {
                a.pull_bytes[p] = blk; a.dst_off[p] = (size_t)p * blk;
                a.pull_off[p] = a2a ? (size_t)r * blk : ((mode == XCHG_AG_MC || mode == XCHG_AG_RING) ? (size_t)p * ablk : 0);
            }
            a.self_off = a2a ? (size_t)r * blk : 0;
            if (mode == XCHG_AG_MC) { a.use_mc = 1; a.push_off = (size_t)r * ablk; }
            if (mode == XCHG_AG_RING) { a.ring = 1; a.ring_pos = r; for (int q = 0; q < N; q++) a.ring_order[q] = q; }
            nvl_exchange_kernel(a);
        });
        CHECK(w.host_err == 0);
        for (int r = 0; r < N; r++) {
            for (int p = 0; p < N; p++) for (size_t i = 0; i < blk; i++)
                if (db[r][16 + misalign + p * blk + i] != pat(p, a2a ? r : 0, i)) { printf("EMU FAIL xchg mode %d: rank %d block %d byte %zu\n", mode, r, p, i); exit(1); }
            CHECK(db[r][15 + misalign] == 0xee && db[r][16 + misalign + blk * N] == 0xee);
        }
    }
    static const char *names[] = {"exchange allgather pull (control)", "exchange alltoall pull (control)", "exchange allgather nvls push (control)", "exchange allgather ring (control)"};
    printf("  ok %-40s blk %zu B N %d grid %dx%d%s\n", names[mode], blk, N, nb, nt, misalign ? " unaligned" : "");
}

// zero-copy push exchange: allgather (same block to everybody) and alltoall (block p to member p)
static void run_push(World &w, bool a2a, size_t blk, int nb, int nt, size_t misalign = 0, bool inplace_ag = false)
{
    const int N = w.N;
    std::vector<std::vector<unsigned char>> sb(N, std::vector<unsigned char>((a2a ? blk * N : blk) + 64)), db(N, std::vector<unsigned char>(blk * N + 64, 0xee));
    for (int rep = 0; rep < 2; rep++) {
        for (int r = 0; r < N; r++) {
            memset(db[r].data(), 0xee, db[r].size());
            for (int to = 0; to < (a2a ? N : 1); to++) for (size_t i = 0; i < blk; i++) {
                unsigned char v = pat(r, a2a ? to : 0, i);
                if (inplace_ag) db[r][16 + misalign + r * blk + i] = v; else sb[r][16 + misalign + to * blk + i] = v;
            }
        }
        launch_all(N, nb, nt, [&](int r) {
            nvl_push_args_t a; memset(&a, 0, sizeof(a));
            a.team = w.team(r, false);
            a.src = inplace_ag ? (const void *)(db[r].data() + 16 + misalign + r * blk) : (const void *)(sb[r].data() + 16 + misalign);
            for (int p = 0; p < N; p++) { a.send_off[p] = a2a ? (size_t)p * blk : 0; a.send_bytes[p] = blk; a.land_off[p] = (size_t)r * blk; a.dst_of[p] = (char *)db[p].data() + 16 + misalign; }
            nvl_exchange_push_kernel(a);
        });
        CHECK(w.host_err == 0);
        for (int r = 0; r < N; r++) {
            for (int p = 0; p < N; p++) for (size_t i = 0; i < blk; i++)
                if (db[r][16 + misalign + p * blk + i] != pat(p, a2a ? r : 0, i)) { printf("EMU FAIL push: rank %d block %d byte %zu\n", r, p, i); exit(1); }
            CHECK(db[r][15 + misalign] == 0xee && db[r][16 + misalign + blk * N] == 0xee);
        }
    }
    printf("  ok %-40s blk %zu B N %d grid %dx%d%s%s\n", a2a ? "push alltoall" : "push allgather", blk, N, nb, nt, misalign ? " unaligned" : "", inplace_ag ? " inplace" : "");
}

// one-shot reduce_scatter(v); interleaved with one-shot allreduces, which share the slot parity / sequence counters
static void run_oneshot_rs(World &w, const std::vector<size_t> &counts, int op, bool inplace, int nb, int nt, size_t misalign = 0)
{
    const int N = w.N;
    std::vector<size_t> off(N); size_t total = 0;
    for (int p = 0; p < N; p++) { off[p] = total; total += counts[p]; }
    std::vector<std::vector<float>> sb(N, std::vector<float>(total + 64)), db(N, std::vector<float>(total + 64, -7.f));
    for (int rep = 0; rep < 3; rep++) {
        for (int r = 0; r < N; r++) { for (size_t i = 0; i < total; i++) sb[r][16 + misalign + i] = val<float>(r, i + rep); std::fill(db[r].begin(), db[r].end(), -7.f); }
        launch_all(N, nb, nt, [&](int r) {
            nvl_red_args_t a; memset(&a, 0, sizeof(a));
            a.team = w.team(r, false); a.src = sb[r].data() + 16 + misalign; a.count = total; a.op = op; a.kind = NVL_RED_REDUCE_SCATTER;
            a.dst = inplace ? (void *)(sb[r].data() + 16 + misalign + off[r]) : (void *)(db[r].data() + 16 + misalign);
            for (int p = 0; p < N; p++) { a.rs_offset[p] = off[p]; a.rs_count[p] = counts[p]; }
            nvl_reduce_scatter_oneshot_kernel<float>(a);
        });
        CHECK(w.host_err == 0);
        for (int r = 0; r < N; r++) {
            const float *out = inplace ? sb[r].data() + 16 + misalign + off[r] : db[r].data() + 16 + misalign;
            for (size_t i = 0; i < counts[r]; i++) {
                double e = 0; for (int p = 0; p < N; p++) { double v = val<float>(p, off[r] + i + rep); e = p == 0 ? v : (op == NVL_OP_MAX ? std::max(e, v) : e + v); }
                if (op == NVL_OP_AVG) e /= N;
                if (std::fabs(out[i] - e) > 1e-3 * std::max(1.0, std::fabs(e))) { printf("EMU FAIL oneshot rs: rank %d elem %zu got %g expected %g\n", r, i, out[i], e); exit(1); }
            }
            if (!inplace) CHECK(db[r][15 + misalign] == -7.f && db[r][16 + misalign + counts[r]] == -7.f);
        }
        if (rep == 0)   // a one-shot allreduce in between: same parity protocol
            run_allreduce<float>("oneshot allreduce (interleaved)", w, [](nvl_red_args_t a) { nvl_allreduce_oneshot_kernel<float>(a); }, 515, NVL_OP_SUM, false, false, nb, nt, 1);
    }
    printf("  ok %-40s total %zu N %d grid %dx%d%s%s\n", "oneshot reduce_scatter(v)", total, N, nb, nt, inplace ? " inplace" : "", misalign ? " unaligned" : "");
}

// alltoallv push with a skewed (MoE-like) traffic matrix: landing offsets are looked up in the receiver's published table
static void run_push_a2av(World &w, int nb, int nt)
{
    const int N = w.N;
    std::vector<std::vector<size_t>> m(N, std::vector<size_t>(N));           // m[s][d] bytes from s to d; rank 0 is the hot expert
    for (int s = 0; s < N; s++) for (int d = 0; d < N; d++) m[s][d] = d == 0 ? 3000 + 17 * s : (s == d ? 0 : 40 + 4 * ((s + d) % 3));
    std::vector<std::vector<unsigned char>> sb(N), db(N);
    std::vector<std::vector<size_t>> sd(N, std::vector<size_t>(N)), rd(N, std::vector<size_t>(N));
    for (int r = 0; r < N; r++) {
        size_t so = 0, ro = 0;
        for (int p = 0; p < N; p++) { sd[r][p] = so; so += m[r][p] + 5; rd[r][p] = ro; ro += m[p][r] + 3; }   // gaps between blocks
        sb[r].assign(so + 64, 0); db[r].assign(ro + 64, 0xee);
        for (int p = 0; p < N; p++) for (size_t i = 0; i < m[r][p]; i++) sb[r][16 + sd[r][p] + i] = pat(r, p, i);
    }
    for (int rep = 0; rep < 2; rep++) {
        for (int r = 0; r < N; r++) std::fill(db[r].begin(), db[r].end(), 0xee);
        launch_all(N, nb, nt, [&](int r) {
            nvl_push_args_t a; memset(&a, 0, sizeof(a));
            a.team = w.team(r, false); a.src = sb[r].data() + 16; a.lookup = 1;
            for (int p = 0; p < N; p++) { a.send_off[p] = sd[r][p]; a.send_bytes[p] = m[r][p]; a.recv_off[p] = rd[r][p]; a.land_off[p] = rd[r][r]; a.dst_of[p] = (char *)db[p].data() + 16; }
            nvl_exchange_push_kernel(a);
        });
        CHECK(w.host_err == 0);
        for (int r = 0; r < N; r++) for (int p = 0; p < N; p++) {
            for (size_t i = 0; i < m[p][r]; i++) if (db[r][16 + rd[r][p] + i] != pat(p, r, i)) { printf("EMU FAIL push a2av: rank %d from %d byte %zu\n", r, p, i); exit(1); }
            for (size_t i = 0; i < 3; i++) CHECK(db[r][16 + rd[r][p] + m[p][r] + i] == 0xee);   // the gap behind every block is untouched
        }
    }
    printf("  ok %-40s N %d grid %dx%d (hot receiver)\n", "push alltoallv", N, nb, nt);
}

int main(int argc, char **argv)
{
    const std::string what = argc > 1 ? argv[1] : "all";
    for (int N : {2, 3}) {
        // small data region so that a few thousand elements already need many rounds / chunks
        World w(N, 48 * 1024, 1 << 20);
        // std::vector data is only 8/16-byte aligned from malloc; +16 elements keeps float vectors 16-byte aligned relative to the base,
        // so force alignment by construction below: vectors of 4-byte types start 64 bytes into a malloc block (16-byte aligned on glibc)
        if (what == "all" || what == "staged") {
            run_allreduce<float>("staged p2p (control)", w, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<float>(a); }, 9001, NVL_OP_SUM, false, false, 2, 64, 2);
            run_allreduce<float>("staged nvls (control)", w, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<float>(a); }, 9001, NVL_OP_SUM, true, false, 2, 64, 2);
            run_allreduce<float>("oneshot (control)", w, [](nvl_red_args_t a) { nvl_allreduce_oneshot_kernel<float>(a); }, 3001, NVL_OP_SUM, false, false, 2, 64, 3);
            run_allreduce<float>("steps ring (control)", w, [](nvl_red_args_t a) { a.sched = 1; nvl_reduce_steps_kernel<float>(a); }, 3001, NVL_OP_SUM, false, false, 2, 64, 2);
            if (N == 2) run_allreduce<float>("steps rhd (control)", w, [](nvl_red_args_t a) { a.sched = 2; nvl_reduce_steps_kernel<float>(a); }, 3001, NVL_OP_AVG, false, true, 2, 64, 2);
            if (N == 2) { run_direct<2, 4>(w, 9001, NVL_OP_SUM, false, 2, 64); run_direct<2, 4>(w, 777, NVL_OP_MAX, true, 3, 32); }
            else { run_direct<4, 2>(w, 9001, NVL_OP_SUM, false, 2, 64); run_direct<4, 2>(w, 777, NVL_OP_MAX, true, 3, 32); }
        }
        if (what == "all" || what == "xchg") {
            for (int mode : {XCHG_AG_PULL, XCHG_A2A_PULL, XCHG_AG_MC, XCHG_AG_RING}) {
                run_xchg(w, mode, 4096, 2, 64);
                run_xchg(w, mode, 1003, 3, 32);                 // ragged block size
                if (mode != XCHG_AG_MC) run_xchg(w, mode, 2000, 2, 64, 3);   // unaligned user buffers
            }
        }
        if (what == "all" || what == "push") {
            for (bool a2a : {false, true}) { run_push(w, a2a, 4096, 2, 64); run_push(w, a2a, 1003, 3, 32); run_push(w, a2a, 2002, 2, 64, 2); run_push(w, a2a, 777, 2, 64, 3); }
            run_push(w, false, 4096, 2, 64, 0, true);
            run_push_a2av(w, 2, 64); run_push_a2av(w, 3, 32);
        }
        if (what == "all" || what == "oneshot_rs") {
            run_oneshot_rs(w, std::vector<size_t>(N, 1000), NVL_OP_SUM, false, 2, 64);
            run_oneshot_rs(w, std::vector<size_t>(N, 1003), NVL_OP_AVG, true, 2, 64);
            { std::vector<size_t> c(N); for (int p = 0; p < N; p++) c[p] = 5 + 701 * (size_t)p; run_oneshot_rs(w, c, NVL_OP_MAX, false, 2, 64, 1); }   // reduce_scatterv, unaligned
            { std::vector<size_t> c(N, 0); c[N - 1] = 64; run_oneshot_rs(w, c, NVL_OP_SUM, false, 2, 32); }                                                // empty blocks
        }
        if (what == "all" || what == "pipe") {
            auto pipe_f = [](nvl_red_args_t a) { nvl_allreduce_nvls_pipe_kernel<float>(a); };
            auto pipe_i = [](nvl_red_args_t a) { nvl_allreduce_nvls_pipe_kernel<int32_t>(a); };
            run_allreduce<float>("nvls_pipe f32 sum", w, pipe_f, 9001, NVL_OP_SUM, true, false, 2, 128, 3);           // ~6 chunks, ragged tail, 3 launches (epochs)
            run_allreduce<float>("nvls_pipe f32 sum 1 chunk", w, pipe_f, 700, NVL_OP_SUM, true, false, 3, 128, 2);
            run_allreduce<float>("nvls_pipe f32 sum 2 chunks", w, pipe_f, 2 * N * 1020, NVL_OP_SUM, true, false, 2, 128, 1);
            run_allreduce<float>("nvls_pipe f32 avg inplace", w, pipe_f, 12345, NVL_OP_AVG, true, true, 2, 128, 2);
            run_allreduce<float>("nvls_pipe f32 sum unaligned", w, pipe_f, 5003, NVL_OP_SUM, true, false, 2, 128, 1, 1);
            run_allreduce<int32_t>("nvls_pipe i32 max", w, pipe_i, 4097, NVL_OP_MAX, true, false, 1, 256, 1);
            run_allreduce<float>("nvls_pipe tiny", w, pipe_f, 3, NVL_OP_SUM, true, false, 2, 128, 2);
        }
        if (what == "all" || what == "symm") {
            run_symm<float>(w, 9001, NVL_OP_SUM, false, 2, 64);
            run_symm<float>(w, 9001, NVL_OP_AVG, true, 3, 64);
            run_symm<float>(w, 5, NVL_OP_SUM, true, 2, 64);
            run_symm<int32_t>(w, 4099, NVL_OP_MAX, false, 1, 128);
            run_symm_rs(w, 1028, 2, 64);
            run_symm_rs(w, 4, 3, 32);
            run_symm_ag(w, 4096 + 16, false, 2, 64);
            run_symm_ag(w, 1008, true, 2, 64);
        }
    }
    if (what == "soak2") {   // two full rounds + a short RAGGED last round, 2 ranks (the geometry of the GPU regression test)
        World w(2, 1 << 20, 0);
        run_allreduce<float>("staged p2p ragged short last round", w, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<float>(a); }, 576722, NVL_OP_SUM, false, false, 2, 64, 30);
    }
    if (what == "soak") {   // the geometry of the full-stack emulation (tests/hostemu_worker.py): 4 ranks, 1 MB data region, 4 rounds, many launches
        World w(4, 1 << 20, 0);
        run_allreduce<float>("staged p2p multi-round soak", w, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<float>(a); }, 900000, NVL_OP_SUM, false, false, 2, 64, 25);
        run_allreduce<float>("staged nvls multi-round soak", w, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<float>(a); }, 900000, NVL_OP_SUM, true, false, 2, 64, 25);
        run_allreduce<float>("nvls_pipe multi-chunk soak", w, [](nvl_red_args_t a) { nvl_allreduce_nvls_pipe_kernel<float>(a); }, 900000, NVL_OP_SUM, true, false, 2, 128, 25);
    }
    printf("NVL_EMU_OK\n");
    return 0;
}
