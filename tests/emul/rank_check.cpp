// rank_check.cpp -- TEST HARNESS (not shipped): plp_core.h's rank-sum rules on the CPU.  rank_from_hist against the pairwise
// definition on random histograms (whole, and split into runs with the ref entries below each run, as the warps of
// mpileup_rank.cuh split it), rank_depth_over at 2^21 - 1 against 2^21, and T at that boundary: one value shared by every
// entry gives the largest tie term, n^3 - n, which must come out exact.  Built and run by tests/test_ranksums.py, also under
// -fsanitize=address,undefined.  Prints "ok" and exits 0, or names the first failure and exits 1.
#include <stdio.h>
#include <stdint.h>
#include <vector>
#include "../../samtools_b200/csrc/plp_core.h"
using namespace plp;

static int fail(const char *what) { printf("FAIL %s\n", what); return 1; }

int main()
{
    uint32_t rng = 2463534242u;
    auto rnd = [&](uint32_t m) { rng ^= rng << 13; rng ^= rng >> 17; rng ^= rng << 5; return rng % m; };
    for (int it = 0; it < 2000; ++it) {
        const int nb = 1 + (int)rnd(it % 3 == 0 ? RS_POS_CAP : RS_QBINS);
        std::vector<uint32_t> ref((size_t)nb), alt((size_t)nb);
        const int fill = 1 + (int)rnd(40);
        for (int k = 0; k < fill; ++k) ++(rnd(2) ? ref : alt)[rnd((uint32_t)nb)];
        uint64_t u2 = 0, t = 0;
        rank_from_hist(ref.data(), alt.data(), nb, u2, t);
        uint64_t w2 = 0, wt = 0;
        for (int a = 0; a < nb; ++a) {
            for (int r = 0; r < nb; ++r) w2 += (uint64_t)alt[(size_t)a] * ref[(size_t)r] * (a > r ? 2 : a == r ? 1 : 0);
            const uint64_t n = (uint64_t)ref[(size_t)a] + alt[(size_t)a];
            wt += n * n * n - n;
        }
        if (u2 != w2 || t != wt) return fail("rank_from_hist against the pairwise definition");
        // the same histograms in runs of `per` bins, each started from the ref entries below it
        const int per = 1 + (int)rnd(8);
        uint64_t s2 = 0, st = 0, below = 0;
        for (int lo = 0; lo < nb; lo += per) {
            const int hi = lo + per < nb ? lo + per : nb;
            rank_from_hist(ref.data() + lo, alt.data() + lo, hi - lo, s2, st, below);
            for (int b = lo; b < hi; ++b) below += ref[(size_t)b];
        }
        if (s2 != w2 || st != wt) return fail("rank_from_hist in runs");
    }
    if (rank_depth_over(RS_MAX_DEPTH) || !rank_depth_over((uint64_t)RS_MAX_DEPTH + 1)) return fail("rank_depth_over at 2^21 - 1 / 2^21");
    if (RS_MAX_DEPTH != 2097151u) return fail("RS_MAX_DEPTH");
    {   // n = 2^21 - 1 entries of one value: T = n^3 - n below 2^63, U2 = n_ref n_alt (every pair tied)
        const uint64_t n = RS_MAX_DEPTH, nr = n / 2 + 1, na = n - nr;
        uint32_t r[1] = {(uint32_t)nr}, a[1] = {(uint32_t)na};
        uint64_t u2 = 0, t = 0;
        rank_from_hist(r, a, 1, u2, t);
        const unsigned __int128 want = (unsigned __int128)n * n * n - n;
        if (want > (unsigned __int128)INT64_MAX || t != (uint64_t)want || u2 != nr * na) return fail("T and U2 at n = 2^21 - 1");
        // the bound has a margin of one entry: 2^21 entries would still just fit, 2^21 + 1 would wrap
        const unsigned __int128 n1 = n + 1, n2 = n + 2;
        if (n1 * n1 * n1 - n1 > (unsigned __int128)INT64_MAX || n2 * n2 * n2 - n2 <= (unsigned __int128)INT64_MAX) return fail("the margin of the bound");
    }
    printf("ok\n");
    return 0;
}
