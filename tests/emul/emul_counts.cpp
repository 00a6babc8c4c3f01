// emul_counts.cpp -- DEBUG HARNESS, NOT PART OF THE PRODUCT: the emulation harness (emul_engine.cpp) plus the per-column
// counts of b200_mpileup_counts, stepped on the CPU through the same mp_entry_channel the CUDA kernel k_mp_counts
// (mpileup_cnt.cuh) calls.  Built by tests/test_counts.py together with the CLI, so that `counts` is checked without a GPU.
#include "emul_engine.cpp"

extern "C" int b200_mpileup_counts(b200_engine_t *e, int32_t min_baseQ, uint32_t *out, size_t cap, int64_t *n_cols)
{
    if (!e->staged) { e->err = "no staged batch"; return -1; }
    if (e->cf.mode != B200_MODE_MPILEUP) { e->err = "mpileup counts need a batch staged in B200_MODE_MPILEUP"; return -1; }
    View v; fill_view(e, v, nullptr, nullptr, 0, 0, 1);
    const int64_t n = v.ncols;
    *n_cols = n;
    if (!out) return 0;
    if (cap < (size_t)n) { e->err = "count buffer too small"; return -2; }
    std::fill(out, out + (size_t)v.n_files * CNT_PLANES * (size_t)n, 0u);
    for (int f = 0; f < v.n_files; ++f)
        for (int32_t c = 0; c < (int32_t)n; ++c) {   // the walk of one lane of k_mp_counts: the column's reads in file order
            uint32_t *o = out + (size_t)f * CNT_PLANES * (size_t)n + (size_t)c;
            const ReadRange rr = read_range(v, f, c >> 5);
            for (int32_t t = 0; t < rr.n; ++t) {
                const ReadDesc d = v.desc[range_at(rr, t)];
                if ((uint32_t)(c - d.rpos) >= (uint32_t)(d.rend - d.rpos)) continue;
                o[(size_t)CNT_NPLP * n]++;
                Ent en; resolve(v, d, c, en);
                if (ent_qual(v, d, en) < min_baseQ) continue;
                const int x = mp_entry_channel(v, d, v.cigar + d.cig_off, en, c);
                const int r = (d.fl & RD_REV) ? CNT_REV : 0;
                o[(size_t)(r + (x & 15)) * n]++;
                if (x & CNT_BIT_INS) o[(size_t)(r + CNT_INS_NEXT) * n]++;
                if (x & CNT_BIT_DEL) o[(size_t)(r + CNT_DEL_NEXT) * n]++;
            }
        }
    return 0;
}
