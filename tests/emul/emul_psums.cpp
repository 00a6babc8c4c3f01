// emul_psums.cpp -- DEBUG HARNESS, NOT PART OF THE PRODUCT: the emulation harness with the quality sums (emul_qsums.cpp)
// plus the read-position sums of b200_mpileup_psums / b200_indel_psums, stepped on the CPU through the same plp_core.h
// functions the CUDA kernels (mpileup_cnt.cuh, mpileup_indel.cuh) call: ent_qual, mp_entry_channel, mp_entry_ps (over
// qpos5_of), ps_sq_over, mp_entry_indel, ins_symbols and indel_allele_equal.  Built by tests/test_psums.py together with
// the CLI, so that `counts --psums` and `indels --psums` are checked without a GPU.
#include "emul_qsums.cpp"

namespace {
// cell += x of a sum of squares; true where the sum would exceed INT64_MAX (the kernels' flag)
bool add_sq(int64_t &cell, uint64_t x)
{
    const uint64_t old = (uint64_t)cell;
    cell = (int64_t)(old + x);
    return ps_sq_over(old, x);
}
}  // namespace

extern "C" int b200_mpileup_psums(b200_engine_t *e, int32_t min_baseQ, int64_t *out, size_t cap, int64_t *n_cols)
{
    if (!e->staged) { e->err = "no staged batch"; return -1; }
    if (e->cf.mode != B200_MODE_MPILEUP) { e->err = "mpileup position sums need a batch staged in B200_MODE_MPILEUP"; return -1; }
    View v; fill_view(e, v, nullptr, nullptr, 0, 0, 1);
    const int64_t n = v.ncols;
    *n_cols = n;
    if (!out) return 0;
    if (cap < (size_t)n) { e->err = "position sum buffer too small"; return -2; }
    std::fill(out, out + (size_t)v.n_files * PS_PLANES * (size_t)n, 0);
    bool over = false;
    for (int f = 0; f < v.n_files; ++f)
        for (int32_t c = 0; c < (int32_t)n; ++c) {
            int64_t *o = out + (size_t)f * PS_PLANES * (size_t)n + (size_t)c;
            lane_walk(v, f, c, min_baseQ, [&](const ReadDesc &d, const Ent &en, int) {
                const EntPs x = mp_entry_ps(d, en);
                const int k = ((d.fl & RD_REV) ? PS_REV : 0) + (mp_entry_channel(v, d, v.cigar + d.cig_off, en, c) & 15);
                o[(size_t)k * n] += x.bp5;
                over |= add_sq(o[(size_t)(PS_SQ + k) * n], x.sq);
            });
        }
    if (over) { e->err = "a column's sum of squared read positions would exceed 2^63 - 1"; return -1; }
    return 0;
}

extern "C" int b200_indel_psums(b200_engine_t *e, b200_indel_psum_t *out, size_t cap_rows)
{
    auto it = g_tables.find(e);
    if (it == g_tables.end()) { e->err = "no indel table: call b200_mpileup_indels on the staged batch first"; return -1; }
    const IndelTable &t = it->second;
    if (out && cap_rows < t.rows.size()) { e->err = "position sum buffer too small"; return -2; }
    std::vector<b200_indel_psum_t> ps(t.rows.size());
    View v; fill_view(e, v, nullptr, nullptr, 0, 0, 1);
    const int32_t min_baseQ = g_ind_minq[e];
    bool over = false;
    // the events of every (column, file), in the table's order, each added to its allele's row
    size_t r0 = 0;
    for (int32_t c = 0; c < v.ncols; ++c)
        for (int f = 0; f < v.n_files; ++f) {
            size_t r1 = r0;
            while (r1 < t.rows.size() && t.rows[r1].col == c && t.rows[r1].file == f) ++r1;
            lane_walk(v, f, c, min_baseQ, [&](const ReadDesc &d, const Ent &en, int) {
                if ((d.fl & RD_SIMPLE) || !en.indel) return;
                const uint32_t *cg = v.cigar + d.cig_off;
                int del_len;
                const int ins = mp_entry_indel(d, cg, en, del_len);
                const EntPs x = mp_entry_ps(d, en);
                for (int k = 0; k < 2; ++k) {
                    if (k == 0 ? ins < 0 : del_len == 0) continue;
                    const int32_t len = k == 0 ? ins : -del_len;
                    std::string sym((size_t)(len > 0 ? len : 0), '?');
                    if (len > 0) ins_symbols(v, d, cg, en, false, '*', &sym[0]);
                    size_t r = r0;
                    while (r < r1 && !indel_allele_equal(len, sym.data(), t.rows[r].len, t.seq.data() + t.rows[r].seq_off)) ++r;
                    if (r == r1) abort();   // every event has its allele in the table
                    int64_t *o = &ps[r].bp5_fwd + ((d.fl & RD_REV) ? 1 : 0);
                    o[0] += x.bp5;
                    over |= add_sq(o[2], x.sq);
                }
            });
            r0 = r1;
        }
    if (over) { e->err = "an indel allele's sum of squared read positions would exceed 2^63 - 1"; return -1; }
    if (out && !ps.empty()) memcpy(out, ps.data(), ps.size() * sizeof(b200_indel_psum_t));
    return 0;
}
