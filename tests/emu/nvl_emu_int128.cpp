// Host emulation of the tl/nvl reduction kernels on 128-bit integers (nvl_i128 / nvl_u128): one-shot, staged two-shot over several
// heap rounds, zero-copy, ring, rhd and one-shot reduce_scatter(v), every operator, teams of 2, 3 and 4, buffers aligned and 8 bytes
// off 16-byte alignment (the guarded element path).  Inputs mix small values, the limits, low words of all ones or zero under a
// non-zero high word, and random values; the reference wraps mod 2^128 on the host, so every result is compared bit for bit.
#include "nvl_emu_world.h"

static uint64_t mix(uint64_t x)
{ x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }

template <typename T> static T val(int r, size_t i)
{
    const uint64_t h = mix(i * 1000003u + (uint64_t)r * 7919u + 1);
    switch (i % 4) {
    case 0: return (T)((int)((i * 7 + (size_t)r * 13) % 9) - 4);
    case 1: { const nvl_u128 lim[] = {0, ~(nvl_u128)0, (nvl_u128)1 << 127, ((nvl_u128)1 << 127) - 1, 1, (nvl_u128)5 << 64 | ~0ull};
              return (T)lim[(i / 4 + (size_t)r) % 6]; }
    case 2: return (T)((nvl_u128)(h | 1) << 64 | ((h >> 7) & 1 ? ~0ull : 0));   // carries and borrows between the 64-bit halves
    default: return (T)((nvl_u128)h << 64 | mix(h));
    }
}

template <typename T> static T ref(int N, size_t i, int op)
{
    T a = val<T>(0, i);
    for (int p = 1; p < N; p++) {
        const T x = val<T>(p, i);
        switch (op) {
        case NVL_OP_SUM: case NVL_OP_AVG: a = (T)((nvl_u128)a + (nvl_u128)x); break;
        case NVL_OP_PROD: a = (T)((nvl_u128)a * (nvl_u128)x); break;
        case NVL_OP_MAX: a = a > x ? a : x; break;
        case NVL_OP_MIN: a = a < x ? a : x; break;
        case NVL_OP_LAND: a = (T)(a && x); break;
        case NVL_OP_LOR: a = (T)(a || x); break;
        case NVL_OP_LXOR: a = (T)(!a != !x); break;
        case NVL_OP_BAND: a &= x; break;
        case NVL_OP_BOR: a |= x; break;
        default: a ^= x; break;
        }
    }
    return op == NVL_OP_AVG ? (T)(a / (T)N) : a;    // truncating division of the wrapped sum
}

template <typename T> static void check_elem(const char *name, const char *p, int N, size_t i, int op, int rank)
{
    T got; memcpy(&got, p, sizeof(T));
    const T e = ref<T>(N, i, op);
    if (got != e) {
        printf("EMU FAIL %s: %s op %d N %d rank %d elem %zu got %016llx%016llx expected %016llx%016llx\n", name, (T)-1 > 0 ? "u128" : "i128", op, N, rank, i,
               (unsigned long long)((nvl_u128)got >> 64), (unsigned long long)got, (unsigned long long)((nvl_u128)e >> 64), (unsigned long long)e);
        exit(1);
    }
}

static const unsigned char GUARD = 0xa5;

// allreduce through `kernel` on buffers `mis` bytes past a 16-byte boundary; the zero-copy pointer tables are always filled
template <typename T, typename K> static void run_allreduce(const char *name, World &w, K kernel, size_t count, int op, bool inplace, size_t mis, int nb, int nt)
{
    const int N = w.N;
    const size_t bytes = count * 16;
    std::vector<std::vector<nvl_u128>> sb(N, std::vector<nvl_u128>(count + 8)), db(N, std::vector<nvl_u128>(count + 8));
    std::vector<char *> src(N), dst(N);
    for (int r = 0; r < N; r++) {
        src[r] = (char *)sb[r].data() + 64 + mis; dst[r] = inplace ? src[r] : (char *)db[r].data() + 64 + mis;
        memset(db[r].data(), GUARD, (count + 8) * 16);
        for (size_t i = 0; i < count; i++) { const T v = val<T>(r, i); memcpy(src[r] + i * 16, &v, 16); }
    }
    launch_all(N, nb, nt, [&](int r) {
        nvl_red_args_t a; memset(&a, 0, sizeof(a));
        a.team = w.team(r, false); a.src = src[r]; a.dst = dst[r]; a.count = count; a.op = op; a.kind = NVL_RED_ALLREDUCE;
        for (int p = 0; p < N; p++) { a.d.src[p] = src[p]; a.d.dst[p] = dst[p]; }
        kernel(a);
    });
    CHECK(w.host_err == 0);
    for (int r = 0; r < N; r++) {
        for (size_t i = 0; i < count; i++) check_elem<T>(name, dst[r] + i * 16, N, i, op, r);
        if (inplace) continue;
        for (size_t b = 0; b < 64 + mis; b++) CHECK((unsigned char)((char *)db[r].data())[b] == GUARD);
        for (size_t b = 64 + mis + bytes; b < (count + 8) * 16; b++) CHECK((unsigned char)((char *)db[r].data())[b] == GUARD);
        for (size_t i = 0; i < count; i++) { const T v = val<T>(r, i); CHECK(!memcmp(src[r] + i * 16, &v, 16)); }
    }
}

// one-shot reduce_scatter(v), ragged blocks
template <typename T> static void run_oneshot_rs(World &w, const std::vector<size_t> &counts, int op, bool inplace, size_t mis, int nb, int nt)
{
    const int N = w.N;
    std::vector<size_t> off(N); size_t total = 0;
    for (int p = 0; p < N; p++) { off[p] = total; total += counts[p]; }
    std::vector<std::vector<nvl_u128>> sb(N, std::vector<nvl_u128>(total + 8)), db(N, std::vector<nvl_u128>(total + 8));
    for (int r = 0; r < N; r++) {
        memset(db[r].data(), GUARD, (total + 8) * 16);
        for (size_t i = 0; i < total; i++) { const T v = val<T>(r, i); memcpy((char *)sb[r].data() + 64 + mis + i * 16, &v, 16); }
    }
    launch_all(N, nb, nt, [&](int r) {
        nvl_red_args_t a; memset(&a, 0, sizeof(a));
        a.team = w.team(r, false); a.src = (char *)sb[r].data() + 64 + mis; a.count = total; a.op = op; a.kind = NVL_RED_REDUCE_SCATTER;
        a.dst = inplace ? (char *)sb[r].data() + 64 + mis + off[r] * 16 : (char *)db[r].data() + 64 + mis;
        for (int p = 0; p < N; p++) { a.rs_offset[p] = off[p]; a.rs_count[p] = counts[p]; }
        nvl_reduce_scatter_oneshot_kernel<T>(a);
    });
    CHECK(w.host_err == 0);
    for (int r = 0; r < N; r++) {
        const char *out = inplace ? (char *)sb[r].data() + 64 + mis + off[r] * 16 : (char *)db[r].data() + 64 + mis;
        for (size_t i = 0; i < counts[r]; i++) check_elem<T>("oneshot reduce_scatter(v)", out + i * 16, N, off[r] + i, op, r);
        if (!inplace) for (size_t b = 64 + mis + counts[r] * 16; b < (total + 8) * 16; b++) CHECK((unsigned char)((char *)db[r].data())[b] == GUARD);
    }
}

template <typename T> static void int128_suite(World &w)
{
    const int N = w.N;
    auto oneshot = [](nvl_red_args_t a) { nvl_allreduce_oneshot_kernel<T>(a); };
    auto staged = [](nvl_red_args_t a) { nvl_reduce_staged_kernel<T>(a); };
    auto direct = [](nvl_red_args_t a) { a.direct = NVL_DIRECT_FULL; nvl_reduce_direct_kernel<T>(a); };
    auto ring = [](nvl_red_args_t a) { a.sched = 1; nvl_reduce_steps_kernel<T>(a); };
    auto rhd = [](nvl_red_args_t a) { a.sched = 2; nvl_reduce_steps_kernel<T>(a); };
    for (int op = 0; op < NVL_OP_LAST; op++) {
        run_allreduce<T>("direct (zero-copy two-shot)", w, direct, 203, op, false, 0, 2, 32);
        run_allreduce<T>("oneshot", w, oneshot, 203, op, op == NVL_OP_AVG, 0, 2, 32);
        run_allreduce<T>("ring", w, ring, 203, op, false, 0, 2, 32);
        if ((N & (N - 1)) == 0) run_allreduce<T>("rhd", w, rhd, 203, op, false, 0, 2, 32);
        { std::vector<size_t> c(N); for (int p = 0; p < N; p++) c[p] = 3 + 5 * (size_t)p; run_oneshot_rs<T>(w, c, op, op == NVL_OP_BXOR, 0, 2, 32); }
    }
    for (int op : {NVL_OP_SUM, NVL_OP_PROD, NVL_OP_MAX, NVL_OP_AVG}) {
        run_allreduce<T>("staged p2p multi-round", w, staged, 7001, op, false, 0, 2, 64);
        // 8 bytes off alignment: the guarded element path of every kernel that takes such buffers
        run_allreduce<T>("staged p2p unaligned", w, staged, 301, op, false, 8, 2, 32);
        run_allreduce<T>("oneshot unaligned", w, oneshot, 301, op, false, 8, 2, 32);
        run_allreduce<T>("ring unaligned", w, ring, 301, op, false, 8, 2, 32);
        { std::vector<size_t> c(N); for (int p = 0; p < N; p++) c[p] = 2 + 3 * (size_t)p; run_oneshot_rs<T>(w, c, op, false, 8, 2, 32); }
    }
    printf("  ok int128 / uint128 kernels N %d (%s)\n", N, (T)-1 > 0 ? "u128" : "i128");
}

int main()
{
    for (int N : {2, 3, 4}) {
        World w(N, 48 * 1024, 1 << 20);   // small data region: a few thousand elements already take several rounds
        int128_suite<nvl_i128>(w);
        int128_suite<nvl_u128>(w);
    }
    printf("NVL_EMU_OK\n");
    return 0;
}
