// Host emulation of the tl/nvl reduction kernels on complex float / double (nvl_c64 / nvl_c128): every algorithm that reduces
// complex data (one-shot, staged P2P and NVLS, zero-copy, ring, rhd, one-shot reduce_scatter(v), nvls_pipe, symmetric memory) at
// every team-size class.  Inputs are Gaussian integers with components in {-2..2}: their sums and products over up to 8 ranks are
// exact in float whatever the order, so SUM / PROD are compared bit for bit; AVG is exact for power-of-two teams.
#include <cmath>
#include <complex>
#include "nvl_emu_world.h"

template <typename R> static nvl_complex<R> cval(int r, size_t i)
{ return {(R)((int)((i * 7 + (size_t)r * 13) % 5) - 2), (R)((int)((i * 3 + (size_t)r * 11 + 1) % 5) - 2)}; }

// reference in complex128
template <typename R> static std::complex<double> cref(int N, size_t i, int op)
{
    std::complex<double> e;
    for (int p = 0; p < N; p++) {
        const nvl_complex<R> v = cval<R>(p, i);
        const std::complex<double> x(v.re, v.im);
        e = p == 0 ? x : (op == NVL_OP_PROD ? e * x : e + x);
    }
    return op == NVL_OP_AVG ? e / (double)N : e;
}

template <typename R> static void check_elem(const char *name, nvl_complex<R> got, int N, size_t i, int op, int rank)
{
    const std::complex<double> e = cref<R>(N, i, op);
    const bool exact = op != NVL_OP_AVG || (N & (N - 1)) == 0;
    const double tol = exact ? 0.0 : 1e-6 * std::max(1.0, std::abs(e));
    if (std::fabs(got.re - e.real()) > tol || std::fabs(got.im - e.imag()) > tol) {
        printf("EMU FAIL %s: rank %d elem %zu got (%g, %g) expected (%g, %g)\n", name, rank, i, (double)got.re, (double)got.im, e.real(), e.imag());
        exit(1);
    }
}

static const char *op_name(int op) { return op == NVL_OP_SUM ? "sum" : (op == NVL_OP_PROD ? "prod" : "avg"); }

// allreduce through `kernel`; the zero-copy pointer tables are always filled (only the direct kernel reads them)
template <typename R, typename K> static void run_c_allreduce(const char *name, World &w, K kernel, size_t count, int op, bool nvls, bool inplace, int nb, int nt, int repeats, size_t misalign = 0)
{
    typedef nvl_complex<R> C;
    const int N = w.N;
    const C guard = {(R)-7, (R)-7};
    std::vector<std::vector<C>> sb(N, std::vector<C>(count + 64)), db(N, std::vector<C>(count + 64, guard));
    std::vector<C *> src(N), dst(N);
    for (int r = 0; r < N; r++) { src[r] = sb[r].data() + 16 + misalign; dst[r] = inplace ? src[r] : db[r].data() + 16 + misalign; }
    for (int it = 0; it < repeats; it++) {
        for (int r = 0; r < N; r++) { for (size_t i = 0; i < count; i++) src[r][i] = cval<R>(r, i); if (!inplace) { dst[r][-1] = guard; dst[r][count] = guard; } }
        launch_all(N, nb, nt, [&](int r) {
            nvl_red_args_t a; memset(&a, 0, sizeof(a));
            a.team = w.team(r, nvls); a.src = src[r]; a.dst = dst[r]; a.count = count; a.op = op; a.kind = NVL_RED_ALLREDUCE; a.use_nvls = nvls;
            for (int p = 0; p < N; p++) { a.d.src[p] = (const char *)src[p]; a.d.dst[p] = (char *)dst[p]; }
            kernel(a);
        });
        CHECK(w.host_err == 0);
        for (int r = 0; r < N; r++) for (size_t i = 0; i < count; i++) check_elem<R>(name, dst[r][i], N, i, op, r);
        if (!inplace) for (int r = 0; r < N; r++) CHECK(!memcmp(&dst[r][-1], &guard, sizeof(C)) && !memcmp(&dst[r][count], &guard, sizeof(C)));
    }
    printf("  ok %-34s c%-3zu %-4s count %zu N %d grid %dx%d%s%s x%d\n", name, 8 * sizeof(C), op_name(op), count, N, nb, nt, inplace ? " inplace" : "", misalign ? " unaligned" : "", repeats);
}

// one-shot reduce_scatter(v)
template <typename R> static void run_c_oneshot_rs(World &w, const std::vector<size_t> &counts, int op, bool inplace, int nb, int nt, size_t misalign = 0)
{
    typedef nvl_complex<R> C;
    const int N = w.N;
    const C guard = {(R)-7, (R)-7};
    std::vector<size_t> off(N); size_t total = 0;
    for (int p = 0; p < N; p++) { off[p] = total; total += counts[p]; }
    std::vector<std::vector<C>> sb(N, std::vector<C>(total + 64)), db(N, std::vector<C>(total + 64, guard));
    for (int r = 0; r < N; r++) for (size_t i = 0; i < total; i++) sb[r][16 + misalign + i] = cval<R>(r, i);
    launch_all(N, nb, nt, [&](int r) {
        nvl_red_args_t a; memset(&a, 0, sizeof(a));
        a.team = w.team(r, false); a.src = sb[r].data() + 16 + misalign; a.count = total; a.op = op; a.kind = NVL_RED_REDUCE_SCATTER;
        a.dst = inplace ? (void *)(sb[r].data() + 16 + misalign + off[r]) : (void *)(db[r].data() + 16 + misalign);
        for (int p = 0; p < N; p++) { a.rs_offset[p] = off[p]; a.rs_count[p] = counts[p]; }
        nvl_reduce_scatter_oneshot_kernel<C>(a);
    });
    CHECK(w.host_err == 0);
    for (int r = 0; r < N; r++) {
        const C *out = inplace ? sb[r].data() + 16 + misalign + off[r] : db[r].data() + 16 + misalign;
        for (size_t i = 0; i < counts[r]; i++) check_elem<R>("oneshot reduce_scatter(v)", out[i], N, off[r] + i, op, r);
        if (!inplace) CHECK(!memcmp(&db[r][15 + misalign], &guard, sizeof(C)) && !memcmp(&db[r][16 + misalign + counts[r]], &guard, sizeof(C)));
    }
    printf("  ok %-34s c%-3zu %-4s total %zu N %d grid %dx%d%s%s\n", "oneshot reduce_scatter(v)", 8 * sizeof(C), op_name(op), total, N, nb, nt, inplace ? " inplace" : "", misalign ? " unaligned" : "");
}

// in-place / out-of-place NVLS allreduce on symmetric user memory (c64 only: no in-switch path for double)
static void run_c_symm(World &w, size_t count, int op, bool inplace, int nb, int nt)
{
    const int N = w.N;
    const size_t bytes = ((count * sizeof(nvl_c64) + 255) / 256) * 256;
    CHECK(2 * bytes + 256 <= w.user_size);
    std::vector<nvl_c64 *> src(N), dst(N);
    for (int r = 0; r < N; r++) {
        src[r] = (nvl_c64 *)w.user(r); dst[r] = inplace ? src[r] : (nvl_c64 *)(w.user(r) + bytes);
        memset(w.user(r), 0x5a, 2 * bytes + 256);
        for (size_t i = 0; i < count; i++) src[r][i] = cval<float>(r, i);
    }
    launch_all(N, nb, nt, [&](int r) {
        nvl_red_args_t a; memset(&a, 0, sizeof(a));
        a.team = w.team(r, true); a.src = src[r]; a.dst = dst[r]; a.count = count; a.op = op; a.kind = NVL_RED_ALLREDUCE; a.use_nvls = 1;
        a.d.src[0] = (const char *)src[r]; a.d.dst[0] = (char *)dst[r];
        nvl_allreduce_symm_kernel<nvl_c64>(a);
    });
    CHECK(w.host_err == 0);
    for (int r = 0; r < N; r++) {
        for (size_t i = 0; i < count; i++) check_elem<float>("symm allreduce", dst[r][i], N, i, op, r);
        const unsigned char *g = (const unsigned char *)(dst[r] + count);
        for (size_t i = 0; i < 64; i++) CHECK(g[i] == 0x5a || (char *)g + i >= w.user(r) + 2 * bytes + 256);
    }
    printf("  ok %-34s c64  %-4s count %zu N %d grid %dx%d%s\n", "symm allreduce", op_name(op), count, N, nb, nt, inplace ? " inplace" : "");
}

// c64 SUM reinterprets the same bytes as a float vector: the complex kernel must give the float kernel's bits
template <typename K64, typename K32> static void run_c64_bits_vs_f32(const char *name, World &w, K64 k64, K32 k32, size_t count, bool nvls, int nb, int nt)
{
    const int N = w.N;
    std::vector<std::vector<nvl_c64>> src(N, std::vector<nvl_c64>(count)), out64(N, std::vector<nvl_c64>(count));
    std::vector<std::vector<float>> out32(N, std::vector<float>(2 * count));
    for (int r = 0; r < N; r++) for (size_t i = 0; i < count; i++) src[r][i] = {0.1f * (float)((i * 7 + r * 13) % 23) + 1.f / 3.f, -0.3f * (float)((i * 5 + r) % 17) + 1.f / 7.f};
    for (int pass = 0; pass < 2; pass++) {
        launch_all(N, nb, nt, [&](int r) {
            nvl_red_args_t a; memset(&a, 0, sizeof(a));
            a.team = w.team(r, nvls); a.src = src[r].data(); a.op = NVL_OP_SUM; a.kind = NVL_RED_ALLREDUCE; a.use_nvls = nvls;
            if (pass == 0) { a.dst = out64[r].data(); a.count = count; k64(a); }
            else { a.dst = out32[r].data(); a.count = 2 * count; k32(a); }
        });
        CHECK(w.host_err == 0);
    }
    for (int r = 0; r < N; r++) CHECK(!memcmp(out64[r].data(), out32[r].data(), count * sizeof(nvl_c64)));
    printf("  ok %-34s c64  sum  count %zu N %d: same bits as the f32 kernel\n", name, count, N);
}

template <typename R> static void complex_suite(World &w)
{
    typedef nvl_complex<R> C;
    const int N = w.N;
    const bool pow2 = (N & (N - 1)) == 0;
    auto oneshot = [](nvl_red_args_t a) { nvl_allreduce_oneshot_kernel<C>(a); };
    auto staged = [](nvl_red_args_t a) { nvl_reduce_staged_kernel<C>(a); };
    auto direct = [](nvl_red_args_t a) { a.direct = NVL_DIRECT_FULL; nvl_reduce_direct_kernel<C>(a); };
    auto ring = [](nvl_red_args_t a) { a.sched = 1; nvl_reduce_steps_kernel<C>(a); };
    auto rhd = [](nvl_red_args_t a) { a.sched = 2; nvl_reduce_steps_kernel<C>(a); };
    for (int op : {NVL_OP_SUM, NVL_OP_AVG, NVL_OP_PROD}) {
        run_c_allreduce<R>("direct (zero-copy two-shot)", w, direct, 1001, op, false, false, 2, 32, 1);   // odd count: ragged tail of the last slice
        if (N > 4) continue;   // eight members: the direct kernel's largest size class only
        run_c_allreduce<R>("oneshot", w, oneshot, 1001, op, false, false, 2, 64, 2);
        run_c_allreduce<R>("staged p2p multi-round", w, staged, 9001, op, false, false, 2, 64, 2);
        run_c_allreduce<R>("ring", w, ring, 1001, op, false, true, 2, 64, 1);
        if (pow2) run_c_allreduce<R>("rhd", w, rhd, 1001, op, false, false, 2, 64, 1);
        run_c_oneshot_rs<R>(w, std::vector<size_t>(N, 1000), op, false, 2, 64);
        { std::vector<size_t> c(N); for (int p = 0; p < N; p++) c[p] = 5 + 701 * (size_t)p; run_c_oneshot_rs<R>(w, c, op, true, 2, 64); }   // ragged blocks, in place
    }
    // blocks that are not 16-byte aligned (an odd complex-float offset): the guarded element path everywhere
    if (sizeof(R) == 4 && N <= 3) {
        run_c_allreduce<R>("staged p2p unaligned", w, staged, 3001, NVL_OP_PROD, false, false, 2, 64, 1, 1);
        run_c_allreduce<R>("oneshot unaligned", w, oneshot, 777, NVL_OP_SUM, false, false, 3, 32, 1, 1);
        { std::vector<size_t> c(N); for (int p = 0; p < N; p++) c[p] = 3 + 2 * (size_t)p; run_c_oneshot_rs<R>(w, c, NVL_OP_AVG, false, 2, 32, 1); }
    }
}

int main()
{
    for (int N : {2, 3, 4, 8}) {
        World w(N, 48 * 1024, 1 << 20);   // small data region: a few thousand elements already take several rounds / chunks
        complex_suite<float>(w);
        complex_suite<double>(w);
        if (N > 3) continue;
        // in-switch paths, complex float SUM / AVG only
        auto nvls = [](nvl_red_args_t a) { nvl_reduce_staged_kernel<nvl_c64>(a); };
        auto pipe = [](nvl_red_args_t a) { nvl_allreduce_nvls_pipe_kernel<nvl_c64>(a); };
        for (int op : {NVL_OP_SUM, NVL_OP_AVG}) {
            run_c_allreduce<float>("staged nvls multi-round", w, nvls, 9001, op, true, false, 2, 64, 2);
            run_c_allreduce<float>("nvls_pipe", w, pipe, 9001, op, true, op == NVL_OP_AVG, 2, 128, 2);
            run_c_symm(w, 4097, op, op == NVL_OP_AVG, 2, 64);
        }
        run_c_allreduce<float>("nvls_pipe unaligned", w, pipe, 3001, NVL_OP_SUM, true, false, 2, 128, 1, 1);
        // same bits as the f32 kernels on the same bytes (count a multiple of 2N: both types cut the vector into the same slices)
        const size_t cnt = 2 * (size_t)N * 700;
        run_c64_bits_vs_f32("oneshot", w, [](nvl_red_args_t a) { nvl_allreduce_oneshot_kernel<nvl_c64>(a); }, [](nvl_red_args_t a) { nvl_allreduce_oneshot_kernel<float>(a); }, cnt, false, 2, 64);
        run_c64_bits_vs_f32("staged p2p", w, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<nvl_c64>(a); }, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<float>(a); }, cnt, false, 2, 64);
        run_c64_bits_vs_f32("staged nvls", w, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<nvl_c64>(a); }, [](nvl_red_args_t a) { nvl_reduce_staged_kernel<float>(a); }, cnt, true, 2, 64);
    }
    printf("NVL_EMU_OK\n");
    return 0;
}
