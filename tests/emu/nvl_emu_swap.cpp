// Host emulation of in-place alltoall(v) on tl/nvl: the pairwise swap kernel (kernels/nvl_swap.cu) and the heap-staged fallback
// (the pull kernel reading the peers' staged copies, run the way launch_swap in tl_nvl_coll.c runs it), team sizes 2, 3, 4 and 8.
// Every case is checked here; given a directory, the driver also writes each result there for the NumPy oracle of
// tests/test_nvl_swap.py.  Buffers start as init_byte(rank, offset) everywhere, gaps between the regions included.
#include "nvl_emu_world.h"

static unsigned char init_byte(int r, size_t i)
{
    const uint64_t x = (uint64_t)i * 0x9E3779B1ull + (uint64_t)r * 0x85EBCA77ull;
    return (unsigned char)((x ^ (x >> 15)) & 0xff);
}

struct Case {
    std::string name;
    int N;
    size_t bytes;                    // buffer bytes per rank
    std::vector<size_t> off, len;    // [r * N + p]: rank r's region for member p
    bool lookup;                     // alltoallv
};

static Case a2a_case(int N, size_t blk)
{
    Case c{"alltoall", N, blk * N, std::vector<size_t>((size_t)N * N), std::vector<size_t>((size_t)N * N, blk), false};
    for (int r = 0; r < N; r++) for (int p = 0; p < N; p++) c.off[r * N + p] = (size_t)p * blk;
    return c;
}

// symmetric skewed counts (rank 0 is hot), zero-length pairs, a gap in front of every region (1-7 bytes, or 16 with 16-byte
// aligned regions); mismatch: the pair (0, 1) disagrees on its length (a user error: only the common prefix may move)
static Case a2av_case(int N, bool aligned, bool mismatch)
{
    Case c{aligned ? "alltoallv aligned" : "alltoallv", N, 0, std::vector<size_t>((size_t)N * N), std::vector<size_t>((size_t)N * N), true};
    for (int r = 0; r < N; r++) for (int p = 0; p < N; p++) {
        const int lo = std::min(r, p), hi = std::max(r, p);
        size_t l = lo == 0 ? 5000 + 997 * (size_t)hi : 300 + 61 * (size_t)(lo * hi % 7);
        if (r != p && (lo + hi) % 4 == 3) l = 0;
        c.len[r * N + p] = r == p ? 100 + (size_t)r : l;
    }
    if (mismatch) { c.name += " mismatched pair"; c.len[0 * N + 1] = 5003; c.len[1 * N + 0] = 1234; }
    for (int r = 0; r < N; r++) {
        size_t o = 0;
        for (int p = 0; p < N; p++) { o += aligned ? 16 : (size_t)((r + 3 * p) % 7 + 1); c.off[r * N + p] = o; o += c.len[r * N + p]; if (aligned) o = (o + 15) & ~(size_t)15; }
        c.bytes = std::max(c.bytes, o + 9);
    }
    return c;
}

static int n_dumped = 0;

static void run_case(World &w, const Case &c, bool staged, int nb, int nt, const char *dir)
{
    const int N = c.N;
    std::vector<std::vector<unsigned char>> mem(N, std::vector<unsigned char>(c.bytes + 64));
    std::vector<unsigned char *> buf(N);
    for (int r = 0; r < N; r++) {
        buf[r] = (unsigned char *)(((uintptr_t)mem[r].data() + 31) & ~(uintptr_t)15);
        memset(mem[r].data(), 0xee, mem[r].size());
        for (size_t i = 0; i < c.bytes; i++) buf[r][i] = init_byte(r, i);
    }
    if (staged)   // launch_swap: the self-copy kernel into the staging area runs in each rank's stream ahead of the pull kernel
        for (int r = 0; r < N; r++) memcpy(w.heaps[r] + NVL_DATA_OFFSET + NVL_XCHG_TABLE_BYTES, buf[r], c.bytes);
    launch_all(N, nb, nt, [&](int r) {
        if (staged) {
            nvl_xchg_args_t x; memset(&x, 0, sizeof(x));
            x.team = w.team(r, false); x.src = buf[r]; x.dst = buf[r]; x.src_bytes = c.bytes; x.self_off = c.off[r * N + r];
            x.publish_table = c.lookup; x.direct = 1;
            for (int p = 0; p < N; p++) {
                x.stage_off[p] = c.off[r * N + p]; x.dst_off[p] = c.off[r * N + p]; x.pull_bytes[p] = c.len[r * N + p];
                x.pull_off[p] = c.lookup ? NVL_XCHG_LOOKUP : c.off[p * N + r];
                x.d.src[p] = w.heaps[p] + NVL_DATA_OFFSET + NVL_XCHG_TABLE_BYTES;
            }
            nvl_exchange_kernel(x);
        } else {
            nvl_swap_args_t a; memset(&a, 0, sizeof(a));
            a.team = w.team(r, false); a.buf = (char *)buf[r]; a.lookup = c.lookup;
            for (int p = 0; p < N; p++) { a.dst_of[p] = (char *)buf[p]; a.off[p] = c.off[r * N + p]; a.len[p] = c.len[r * N + p]; }
            nvl_exchange_swap_kernel(a);
        }
    });
    CHECK(w.host_err == 0);
    for (int r = 0; r < N; r++) {
        std::vector<unsigned char> exp(c.bytes);
        for (size_t i = 0; i < c.bytes; i++) exp[i] = init_byte(r, i);
        for (int p = 0; p < N; p++) {
            if (p == r) continue;
            const size_t L = std::min(c.len[r * N + p], c.len[p * N + r]);
            for (size_t i = 0; i < L; i++) exp[c.off[r * N + p] + i] = init_byte(p, c.off[p * N + r] + i);
        }
        for (size_t i = 0; i < c.bytes; i++)
            if (buf[r][i] != exp[i]) { printf("EMU FAIL %s%s N %d: rank %d byte %zu got %d expected %d\n", c.name.c_str(), staged ? " staged" : "", N, r, i, buf[r][i], exp[i]); exit(1); }
        for (size_t i = 0; i < 16; i++) CHECK(buf[r][-1 - (ptrdiff_t)i] == 0xee && buf[r][c.bytes + i] == 0xee);   // nothing outside the buffer
    }
    if (dir) {   // header (N, bytes, staged, lookup), off[N * N], len[N * N], then every rank's buffer
        char path[4096];
        snprintf(path, sizeof(path), "%s/case_%03d.bin", dir, n_dumped++);
        FILE *f = fopen(path, "wb");
        CHECK(f);
        const uint64_t hdr[4] = {(uint64_t)N, (uint64_t)c.bytes, (uint64_t)staged, (uint64_t)c.lookup};
        fwrite(hdr, sizeof(hdr), 1, f);
        for (size_t i = 0; i < c.off.size(); i++) { uint64_t v = c.off[i]; fwrite(&v, 8, 1, f); }
        for (size_t i = 0; i < c.len.size(); i++) { uint64_t v = c.len[i]; fwrite(&v, 8, 1, f); }
        for (int r = 0; r < N; r++) fwrite(buf[r], 1, c.bytes, f);
        fclose(f);
    }
    size_t blk = c.lookup ? 0 : c.len[0];
    printf("  ok %-40s %s N %d bytes %zu%s grid %dx%d\n", c.name.c_str(), staged ? "staged" : "swap  ", N, c.bytes, c.lookup ? "" : (" blk " + std::to_string(blk)).c_str(), nb, nt);
}

int main(int argc, char **argv)
{
    const char *dir = argc > 2 ? argv[2] : nullptr;
    for (int N : {2, 3, 4, 8}) {
        World w(N, 10 << 20, 0);
        for (bool staged : {false, true}) {
            for (size_t blk : {0, 1, 15, 16, 4097}) run_case(w, a2a_case(N, blk), staged, 2, 64, dir);
            run_case(w, a2a_case(N, 1000), staged, 3, 48, dir);   // a partial group of 32 threads in the grid
            run_case(w, a2a_case(N, N == 2 ? (4 << 20) : (N == 3 ? (3 << 20) + 5 : (N == 4 ? (2 << 20) + 1 : (1 << 20) + 3))), staged, 2, 64, dir);   // megabytes
            run_case(w, a2av_case(N, false, false), staged, 2, 64, dir);
            run_case(w, a2av_case(N, true, false), staged, 3, 32, dir);
            if (!staged) run_case(w, a2av_case(N, false, true), false, 2, 64, dir);   // the staged pull copies the receiver's length
        }
    }
    printf("NVL_EMU_OK\n");
    return 0;
}
