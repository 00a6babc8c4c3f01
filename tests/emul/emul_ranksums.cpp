// emul_ranksums.cpp -- DEBUG HARNESS, NOT PART OF THE PRODUCT: the emulation harness with the read-position sums
// (emul_psums.cpp) plus the rank sums of b200_mpileup_ranksums, stepped on the CPU through the same plp_core.h functions
// the CUDA kernels (mpileup_rank.cuh) call: ent_qual, mp_entry_rank (over mp_entry_channel, mp_entry_base, mp_entry_qs and
// qpos5_of), rank_from_hist and rank_depth_over.  Built by tests/test_ranksums.py together with the CLI, so that
// `counts --ranksums` is checked without a GPU, and built again there under the address and undefined-behaviour sanitizers.
#include "emul_psums.cpp"

extern "C" int b200_mpileup_ranksums(b200_engine_t *e, int32_t min_baseQ, int64_t *out, size_t cap, int64_t *n_cols)
{
    if (!e->staged) { e->err = "no staged batch"; return -1; }
    if (e->cf.mode != B200_MODE_MPILEUP) { e->err = "mpileup rank sums need a batch staged in B200_MODE_MPILEUP"; return -1; }
    View v; fill_view(e, v, nullptr, nullptr, 0, 0, 1);
    const int64_t n = v.ncols;
    *n_cols = n;
    if (!out) return 0;
    if (cap < (size_t)n) { e->err = "rank sum buffer too small"; return -2; }
    std::fill(out, out + (size_t)v.n_files * RS_PLANES * (size_t)n, 0);
    std::vector<uint32_t> h(2 * (size_t)RS_BINS);   // ref histogram, then alt
    bool deep = false;
    for (int f = 0; f < v.n_files; ++f)
        for (int32_t c = 0; c < (int32_t)n; ++c) {
            int64_t *o = out + (size_t)f * RS_PLANES * (size_t)n + (size_t)c;
            std::fill(h.begin(), h.end(), 0u);
            lane_walk(v, f, c, min_baseQ, [&](const ReadDesc &d, const Ent &en, int q) {
                const EntRank r = mp_entry_rank(v, d, en, c, q);
                if (r.cls == RS_NONE) return;
                uint32_t *hc = h.data() + (size_t)(r.cls - RS_REF) * RS_BINS;
                for (int k = 0; k < 3; ++k) {
                    if (r.bin[k] < k * RS_QBINS || r.bin[k] >= k * RS_QBINS + rs_nbins(k)) abort();   // each bin inside its value's range
                    ++hc[r.bin[k]];
                }
                ++o[(size_t)(RS_NREF + r.cls - RS_REF) * n];
            });
            const int64_t nr = o[(size_t)RS_NREF * n], na = o[(size_t)RS_NALT * n];
            deep |= rank_depth_over((uint64_t)(nr + na));
            if (nr == 0 || na == 0) continue;
            for (int var = 0; var < 3; ++var) {
                uint64_t u2 = 0, t = 0;
                rank_from_hist(h.data() + var * RS_QBINS, h.data() + RS_BINS + var * RS_QBINS, rs_nbins(var), u2, t);
                o[(size_t)(RS_U2 + 2 * var) * n] = (int64_t)u2;
                o[(size_t)(RS_U2 + 2 * var + 1) * n] = (int64_t)t;
            }
        }
    if (deep) { e->err = "a column has more than 2097151 reference and non-reference bases: its rank sums would not fit in 64 bits"; return -1; }
    return 0;
}
