// emul_indels.cpp -- DEBUG HARNESS, NOT PART OF THE PRODUCT: the emulation harness (emul_engine.cpp) plus the indel allele
// table of b200_mpileup_indels / b200_fetch_indels, stepped on the CPU per column in file order through the same plp_core.h
// functions the CUDA kernels (mpileup_indel.cuh) call: mp_entry_indel, ins_symbols, indel_key and indel_allele_equal.
// Built by tests/test_indels.py together with the CLI, so that `indels` is checked without a GPU.
#include <map>
#include <utility>
// the table belongs to the staged batch: the harness's b200_stage is wrapped to drop it
#define b200_stage emul_stage_batch
#include "emul_engine.cpp"
#undef b200_stage

namespace {
struct IndelTable { std::vector<b200_indel_t> rows; std::string seq; };
std::map<const b200_engine *, IndelTable> g_tables;
}

extern "C" int b200_stage(b200_engine_t *e, const b200_batch_t *b, const b200_stage_conf_t *cf, b200_stage_stats_t *stats)
{
    g_tables.erase(e);
    return emul_stage_batch(e, b, cf, stats);
}

extern "C" int b200_mpileup_indels(b200_engine_t *e, int32_t min_baseQ, int64_t *n_alleles, uint64_t *n_seq_bytes)
{
    g_tables.erase(e);
    if (!e->staged) { e->err = "no staged batch"; return -1; }
    if (e->cf.mode != B200_MODE_MPILEUP) { e->err = "mpileup indels need a batch staged in B200_MODE_MPILEUP"; return -1; }
    const char *kb = getenv("B200_INDEL_KEY_BITS");
    const int bits = kb ? atoi(kb) : 64;
    const uint64_t mask = bits >= 64 ? ~0ull : bits <= 0 ? 0ull : (1ull << bits) - 1;
    View v; fill_view(e, v, nullptr, nullptr, 0, 0, 1);
    IndelTable t;
    for (int32_t c = 0; c < v.ncols; ++c)
        for (int f = 0; f < v.n_files; ++f) {
            // the alleles of (c, f) in first-appearance order; candidates by key, told apart by indel_allele_equal
            std::multimap<uint64_t, size_t> by_key;
            const ReadRange rr = read_range(v, f, c >> 5);
            for (int32_t k = 0; k < rr.n; ++k) {
                const int32_t i = range_at(rr, k);
                const ReadDesc d = v.desc[i];
                if ((d.fl & RD_SIMPLE) || (uint32_t)(c - d.rpos) >= (uint32_t)(d.rend - d.rpos)) continue;
                Ent en; resolve(v, d, c, en);
                if (!en.indel || ent_qual(v, d, en) < min_baseQ) continue;
                const uint32_t *cg = v.cigar + d.cig_off;
                int del_len;
                const int ins = mp_entry_indel(d, cg, en, del_len);
                for (int x = 0; x < 2; ++x) {
                    if (x == 0 ? ins < 0 : del_len == 0) continue;
                    const int32_t len = x == 0 ? ins : -del_len;
                    std::string sym((size_t)(len > 0 ? len : 0), '?');
                    if (len > 0) ins_symbols(v, d, cg, en, false, '*', &sym[0]);
                    const uint64_t key = indel_key(len, sym.data(), mask);
                    size_t hit = SIZE_MAX;
                    for (auto r = by_key.equal_range(key); r.first != r.second && hit == SIZE_MAX; ++r.first) {
                        const b200_indel_t &a = t.rows[r.first->second];
                        if (indel_allele_equal(len, sym.data(), a.len, t.seq.data() + a.seq_off)) hit = r.first->second;
                    }
                    if (hit == SIZE_MAX) {
                        hit = t.rows.size();
                        b200_indel_t a; memset(&a, 0, sizeof a);
                        a.col = c; a.file = f; a.len = len; a.seq_off = t.seq.size();
                        t.rows.push_back(a); t.seq += sym;
                        by_key.emplace(key, hit);
                    }
                    if (d.fl & RD_REV) t.rows[hit].rev++; else t.rows[hit].fwd++;
                }
            }
        }
    *n_alleles = (int64_t)t.rows.size(); *n_seq_bytes = t.seq.size();
    g_tables[e] = std::move(t);
    return 0;
}

extern "C" int b200_fetch_indels(b200_engine_t *e, b200_indel_t *alleles, size_t cap_alleles, char *seq, size_t cap_seq)
{
    auto it = g_tables.find(e);
    if (it == g_tables.end()) { e->err = "no indel table: call b200_mpileup_indels on the staged batch first"; return -1; }
    const IndelTable &t = it->second;
    if (alleles && cap_alleles < t.rows.size()) { e->err = "allele buffer too small"; return -2; }
    if (seq && cap_seq < t.seq.size()) { e->err = "symbol buffer too small"; return -2; }
    if (alleles && !t.rows.empty()) memcpy(alleles, t.rows.data(), t.rows.size() * sizeof(b200_indel_t));
    if (seq && !t.seq.empty()) memcpy(seq, t.seq.data(), t.seq.size());
    return 0;
}
