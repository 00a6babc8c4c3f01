// emul_qsums.cpp -- DEBUG HARNESS, NOT PART OF THE PRODUCT: the emulation harness with the indel table (emul_indels.cpp)
// plus the per-column counts and the quality sums of b200_mpileup_qsums / b200_indel_qsums, stepped on the CPU through the
// same plp_core.h functions the CUDA kernels (mpileup_cnt.cuh, mpileup_indel.cuh) call: ent_qual, mp_entry_channel,
// mp_entry_qs, mp_entry_indel, ins_symbols and indel_allele_equal.  Built by tests/test_qsums.py together with the CLI, so
// that `counts --qsums` and `indels --qsums` are checked without a GPU.
#include <map>
// the allele sums take the -Q of the table's call: the harness's b200_mpileup_indels is wrapped to remember it
#define b200_mpileup_indels emul_mpileup_indels
#include "emul_indels.cpp"
#undef b200_mpileup_indels

namespace {
std::map<const b200_engine *, int32_t> g_ind_minq;

// one lane of mp_col_planes (mpileup_cnt.cuh): the reads over column c of file f in file order; add(d, e, q) for every entry
// that passes -Q.  Returns n_plp.
template <class Add>
uint32_t lane_walk(const View &v, int f, int32_t c, int32_t min_baseQ, Add add)
{
    uint32_t nplp = 0;
    const ReadRange rr = read_range(v, f, c >> 5);
    for (int32_t t = 0; t < rr.n; ++t) {
        const ReadDesc d = v.desc[range_at(rr, t)];
        if ((uint32_t)(c - d.rpos) >= (uint32_t)(d.rend - d.rpos)) continue;
        ++nplp;
        Ent en; resolve(v, d, c, en);
        const int q = ent_qual(v, d, en);
        if (q < min_baseQ) continue;
        add(d, en, q);
    }
    return nplp;
}

template <class Add, class Fin>
int col_planes(b200_engine_t *e, const char *what, int planes, uint32_t *out, size_t cap, int64_t *n_cols, int32_t min_baseQ, Add add, Fin fin)
{
    if (!e->staged) { e->err = "no staged batch"; return -1; }
    if (e->cf.mode != B200_MODE_MPILEUP) { e->err = std::string("mpileup ") + what + " need a batch staged in B200_MODE_MPILEUP"; return -1; }
    View v; fill_view(e, v, nullptr, nullptr, 0, 0, 1);
    const int64_t n = v.ncols;
    *n_cols = n;
    if (!out) return 0;
    if (cap < (size_t)n) { e->err = "buffer too small"; return -2; }
    std::fill(out, out + (size_t)v.n_files * (size_t)planes * (size_t)n, 0u);
    for (int f = 0; f < v.n_files; ++f)
        for (int32_t c = 0; c < (int32_t)n; ++c) {
            uint32_t *o = out + (size_t)f * (size_t)planes * (size_t)n + (size_t)c;
            const uint32_t nplp = lane_walk(v, f, c, min_baseQ, [&](const ReadDesc &d, const Ent &en, int q) { add(v, o, (size_t)n, d, en, c, q); });
            if (fin(o, (size_t)n, nplp) != 0) { e->err = "a column too deep for 32-bit sums"; return -1; }
        }
    return 0;
}
}  // namespace

extern "C" int b200_mpileup_counts(b200_engine_t *e, int32_t min_baseQ, uint32_t *out, size_t cap, int64_t *n_cols)
{
    return col_planes(e, "counts", CNT_PLANES, out, cap, n_cols, min_baseQ,
        [](const View &v, uint32_t *o, size_t n, const ReadDesc &d, const Ent &en, int32_t c, int) {
            const int x = mp_entry_channel(v, d, v.cigar + d.cig_off, en, c);
            const int r = (d.fl & RD_REV) ? CNT_REV : 0;
            o[(size_t)(r + (x & 15)) * n]++;
            if (x & CNT_BIT_INS) o[(size_t)(r + CNT_INS_NEXT) * n]++;
            if (x & CNT_BIT_DEL) o[(size_t)(r + CNT_DEL_NEXT) * n]++;
        },
        [](uint32_t *o, size_t n, uint32_t nplp) { o[(size_t)CNT_NPLP * n] = nplp; return 0; });
}

extern "C" int b200_mpileup_qsums(b200_engine_t *e, int32_t min_baseQ, uint32_t *out, size_t cap, int64_t *n_cols)
{
    return col_planes(e, "quality sums", QS_PLANES, out, cap, n_cols, min_baseQ,
        [](const View &v, uint32_t *o, size_t n, const ReadDesc &d, const Ent &en, int32_t c, int q) {
            const EntQs x = mp_entry_qs(q, d);
            const int k = ((d.fl & RD_REV) ? QS_REV : 0) + (mp_entry_channel(v, d, v.cigar + d.cig_off, en, c) & 15);
            o[(size_t)k * n] += x.bq;
            o[(size_t)(QS_MQ + k) * n] += x.mq;
            o[(size_t)(QS_MQ0 + k) * n] += x.mq0;
        },
        [](uint32_t *, size_t, uint32_t nplp) { return nplp > QS_MAX_DEPTH ? -1 : 0; });
}

extern "C" int b200_mpileup_indels(b200_engine_t *e, int32_t min_baseQ, int64_t *n_alleles, uint64_t *n_seq_bytes)
{
    g_ind_minq[e] = min_baseQ;
    return emul_mpileup_indels(e, min_baseQ, n_alleles, n_seq_bytes);
}

extern "C" int b200_indel_qsums(b200_engine_t *e, b200_indel_qsum_t *out, size_t cap_rows)
{
    auto it = g_tables.find(e);
    if (it == g_tables.end()) { e->err = "no indel table: call b200_mpileup_indels on the staged batch first"; return -1; }
    const IndelTable &t = it->second;
    if (out && cap_rows < t.rows.size()) { e->err = "quality sum buffer too small"; return -2; }
    std::vector<b200_indel_qsum_t> qs(t.rows.size());
    View v; fill_view(e, v, nullptr, nullptr, 0, 0, 1);
    const int32_t min_baseQ = g_ind_minq[e];
    // the events of every (column, file), in the table's order, each added to its allele's row
    size_t r0 = 0;
    for (int32_t c = 0; c < v.ncols; ++c)
        for (int f = 0; f < v.n_files; ++f) {
            size_t r1 = r0;
            while (r1 < t.rows.size() && t.rows[r1].col == c && t.rows[r1].file == f) ++r1;
            lane_walk(v, f, c, min_baseQ, [&](const ReadDesc &d, const Ent &en, int q) {
                if ((d.fl & RD_SIMPLE) || !en.indel) return;
                const uint32_t *cg = v.cigar + d.cig_off;
                int del_len;
                const int ins = mp_entry_indel(d, cg, en, del_len);
                const EntQs x = mp_entry_qs(q, d);
                for (int k = 0; k < 2; ++k) {
                    if (k == 0 ? ins < 0 : del_len == 0) continue;
                    const int32_t len = k == 0 ? ins : -del_len;
                    std::string sym((size_t)(len > 0 ? len : 0), '?');
                    if (len > 0) ins_symbols(v, d, cg, en, false, '*', &sym[0]);
                    size_t r = r0;
                    while (r < r1 && !indel_allele_equal(len, sym.data(), t.rows[r].len, t.seq.data() + t.rows[r].seq_off)) ++r;
                    if (r == r1) abort();   // every event has its allele in the table
                    uint32_t *o = reinterpret_cast<uint32_t *>(&qs[r]) + ((d.fl & RD_REV) ? 1 : 0);
                    o[0] += x.bq; o[2] += x.mq; o[4] += x.mq0;
                }
            });
            r0 = r1;
        }
    for (const b200_indel_t &a : t.rows)
        if (a.fwd > QS_MAX_DEPTH || a.rev > QS_MAX_DEPTH) { e->err = "an indel allele too deep for 32-bit sums"; return -1; }
    if (out && !qs.empty()) memcpy(out, qs.data(), qs.size() * sizeof(b200_indel_qsum_t));
    return 0;
}
