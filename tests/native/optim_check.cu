// Host-side check of the Adam step's tensor table (gsr_adam_plan / gsr_adam_find / gsr_adam_chunk in
// dreamscene_b200/csrc/common.cuh): every element of every tensor is covered by exactly one CTA, float4 runs only
// where all four arrays are 16-byte aligned, empty tensors take no CTA.  Built with nvcc and run on the CPU by
// tests/test_optim_cpu.py (no GPU needed).
#include <cstdio>
#include <vector>
#include "common.cuh"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++fails; } } while (0)

alignas(16) static float pool[4][1 << 16];

// One plan over `sizes` (offset = element offset of every array: 0 aligned, else an unaligned view).
static void check_plan(const std::vector<long long>& sizes, int offset) {
    std::vector<b200gsr_adam_tensor> t(sizes.size());
    long long at = offset;
    for (size_t i = 0; i < sizes.size(); ++i) {
        t[i] = b200gsr_adam_tensor{pool[0] + at, pool[1] + at, pool[2] + at, pool[3] + at, sizes[i],
                                   0.1f, 0.999f, 0.001f, 1e-15f, -0.01f, 0.03f};
        at += (sizes[i] + 3) / 4 * 4 + 4;                   // keep every tensor's alignment that of `offset`
    }
    GsrAdamTable tab;
    const long long blocks = gsr_adam_plan((int)t.size(), t.data(), &tab);
    long long want_blocks = 0;
    int nonempty = 0;
    for (long long n : sizes) { want_blocks += (n + GSR_ADAM_CHUNK - 1) / GSR_ADAM_CHUNK; nonempty += n > 0; }
    CHECK(blocks == want_blocks && tab.count == nonempty);
    std::vector<std::vector<int>> seen(tab.count);
    for (int k = 0; k < tab.count; ++k) {
        seen[k].assign((size_t)tab.e[k].n, 0);
        CHECK(tab.e[k].vec == (offset % 4 == 0));
    }
    for (long long b = 0; b < blocks; ++b) {
        const int k = gsr_adam_find(tab, b);
        CHECK(k >= 0 && k < tab.count);
        const GsrAdamEntry& e = tab.e[k];
        const GsrAdamChunk c = gsr_adam_chunk(e, b);
        CHECK(c.start >= 0 && c.start < c.end && c.end <= e.n && c.start <= c.vend && c.vend <= c.end);
        CHECK(c.start % 4 == 0 && (c.vend - c.start) % 4 == 0 && c.end - c.vend < (e.vec ? 4 : GSR_ADAM_CHUNK + 1));
        if (!e.vec) CHECK(c.vend == c.start);
        for (long long i = c.start; i < c.end; ++i) seen[k][(size_t)i]++;
    }
    for (int k = 0; k < tab.count; ++k)
        for (int s : seen[k]) CHECK(s == 1);
}

int main() {
    for (long long n : {0LL, 1LL, 3LL, 4LL, 5LL, 4095LL, 4096LL, 4097LL, 12289LL})
        for (int off : {0, 1, 2, 4}) check_plan({n}, off);
    for (int off : {0, 3}) {
        check_plan({0, 1, 3, 4, 5}, off);
        check_plan({5, 0, 0, 9000, 1, 4096, 0}, off);
        std::vector<long long> full(B200GSR_ADAM_MAX_TENSORS);
        for (int i = 0; i < B200GSR_ADAM_MAX_TENSORS; ++i) full[i] = (i * 517) % 1500;
        check_plan(full, off);
    }
    // the reference's 7 groups at P = 1.2M, M = 16 (background [3,1,1] last)
    {
        const long long P = 1200000;
        std::vector<b200gsr_adam_tensor> t(7);
        const long long ns[7] = {3 * P, 3 * P, 45 * P, P, 3 * P, 4 * P, 3};
        long long blocks = 0;
        for (int i = 0; i < 7; ++i) {
            t[i] = b200gsr_adam_tensor{pool[0], pool[1], pool[2], pool[3], ns[i], 0.1f, 0.999f, 0.001f, 1e-15f, -0.01f, 0.03f};
            blocks += (ns[i] + GSR_ADAM_CHUNK - 1) / GSR_ADAM_CHUNK;
        }
        GsrAdamTable tab;
        CHECK(gsr_adam_plan(7, t.data(), &tab) == blocks && tab.count == 7);
        CHECK(gsr_adam_find(tab, blocks - 1) == 6 && gsr_adam_find(tab, 0) == 0);
    }
    std::printf(fails ? "%d checks failed\n" : "adam table ok\n", fails);
    return fails ? 1 : 0;
}
