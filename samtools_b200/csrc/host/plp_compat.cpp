// plp_compat.cpp -- htslib-compatible pileup iterators (tier T1) on top of the CUDA engine.
// Interface and semantics: include/b200_htslib_compat.h (htslib sam.h bam_plp_* / bam_mplp_*;
// reference call sites bam_plbuf.c:40-66, bam_plcmd.c:581-607, coverage.c:572-589).
//
// One iterator = one engine handle.  Reads are pulled (or pushed) until a WINDOW is complete -- the reference sequence
// changes, the input ends, or the collected reads exceed a payload budget (B200_PLP_WINDOW_BYTES, default 256 MiB of
// bases) -- then packed into the SoA batch image and staged, and the device returns every (read, column) entry -- the
// bam_pileup1_t fields -- column-major; next()/auto() walk that table.  A window cut inside a reference sequence ends at
// the start of the read that triggered it: every read that starts before it is in hand, so all columns below the cut can be
// served; the reads reaching the cut stay (the halo: the -r rule of bam_plcmd.c:550-554, plus the reads ending right at the
// cut, which the max-depth rule still counts as buffered there) and are staged again with the next window, which reports
// only columns from the cut on and does not judge the halo reads' max-depth verdicts again (B200_RB_MAXDEPTH_*).  Host memory is bounded by the budget, and a push /
// next client sees columns long before the reference sequence ends.  With overlaps enabled the tweaked qualities are copied back into the
// iterator's read copies, which is what the caller sees through plp[i].b, as in htslib.
#include "../../../include/b200_htslib_compat.h"
#include "../../../include/b200_pileup.h"
#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

extern "C" {

bam1_t *bam_init1(void) { return (bam1_t *)calloc(1, sizeof(bam1_t)); }
void bam_destroy1(bam1_t *b) { if (b) { free(b->data); free(b); } }
bam1_t *bam_copy1(bam1_t *dst, const bam1_t *src)
{
    if (dst->m_data < (uint32_t)src->l_data) {
        uint8_t *d = (uint8_t *)realloc(dst->data, (size_t)src->l_data ? (size_t)src->l_data : 1);
        if (!d) return nullptr;
        dst->data = d; dst->m_data = (uint32_t)src->l_data;
    }
    if (src->l_data) memcpy(dst->data, src->data, (size_t)src->l_data);
    dst->core = src->core; dst->id = src->id; dst->l_data = src->l_data;
    return dst;
}

}  // extern "C"

namespace {

constexpr int64_t kPosMax = ((int64_t)INT32_MAX << 32) | UINT32_MAX;
constexpr int64_t kSlabCols = 1 << 20;

// one past the last reference position of a record (pos + reference length of its CIGAR; zero-length: pos)
int64_t read_end(const bam1_t *b)
{
    const uint32_t *cg = bam_get_cigar(b);
    int64_t e = b->core.pos;
    for (uint32_t k = 0; k < b->core.n_cigar; ++k) { const int op = cg[k] & 0xf; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) e += cg[k] >> 4; }
    return e;
}

uint32_t name_bit(const char *s)
{
    uint32_t h = (uint32_t)*s;
    if (h) for (++s; *s; ++s) h = (h << 5) - h + (uint32_t)*s;
    h += ~(h << 15); h ^= (h >> 10); h += (h << 3); h ^= (h >> 6); h += ~(h << 11); h ^= (h >> 16);
    return h & 1;
}

}  // namespace

struct b200_plp {
    bam_plp_auto_f func = nullptr; void *data = nullptr;
    b200_engine_t *eng = nullptr;
    int maxcnt = 8000; bool overlaps = false, eof = false, error = false;
    bam1_t *tmp = nullptr;                 // callback target
    std::vector<bam1_t *> accum;           // reads of the contig being collected
    std::vector<bam1_t *> batch;           // reads of the contig being served
    bam1_t *pending = nullptr;             // the read that completed the window: first read of the next contig, or of the next window
    bool cut = false;                      // pending continues the SAME reference sequence (window cut at its start)
    int64_t serve_beg = -1, serve_end = kPosMax;   // columns [serve_beg, serve_end) of the staged batch are handed out
    int64_t next_beg = -1;                 // where the next window of the current reference sequence starts (-1: at its first read)
    size_t accum_bytes = 0, budget = (size_t)256 << 20;
    std::vector<uint8_t> accum_done, batch_done;   // read's pair overlap was already tweaked in an earlier window (halo reads)
    std::vector<uint8_t> accum_md, batch_md;       // max-depth verdict of an earlier window (B200_RB_MAXDEPTH_*; halo reads)
    std::vector<bam_pileup_cd> accum_cd, batch_cd; bam_pileup_cd pending_cd;   // client data of the same reads
    bam_plp_cd_f construct = nullptr, destruct = nullptr;
    int last_tid = -1; hts_pos_t last_pos = -1;
    // served contig
    bool serving = false; int tid = -1; int64_t win_base = 0, n_cols = 0, col = 0, slab_beg = 0, slab_end = 0;
    std::vector<uint32_t> col_n; std::vector<b200_pileup1_t> ents; size_t ent_pos = 0;
    std::vector<bam_pileup1_t> plp;
    // packing scratch
    std::vector<int64_t> pos, mpos, isize, prev, file_start; std::vector<uint16_t> flag; std::vector<uint8_t> mapq, rbits, seq4, qual;
    std::vector<int32_t> l_qseq, mtid; std::vector<uint32_t> n_cigar, cigar; std::vector<uint64_t> cigar_off, qual_off;
};

static void free_reads(b200_plp *it, std::vector<bam1_t *> &v, std::vector<bam_pileup_cd> &cd)
{
    for (size_t i = 0; i < v.size(); ++i) {
        if (it->destruct) it->destruct(it->data, v[i], &cd[i]);
        bam_destroy1(v[i]);
    }
    v.clear(); cd.clear();
}
static void free_pending(b200_plp *it)
{
    if (!it->pending) return;
    if (it->destruct) it->destruct(it->data, it->pending, &it->pending_cd);
    bam_destroy1(it->pending); it->pending = nullptr;
}

static int stage_batch(b200_plp *it)
{
    const size_t n = it->batch.size();
    it->pos.clear(); it->mpos.clear(); it->isize.clear(); it->prev.clear(); it->flag.clear(); it->mapq.clear(); it->rbits.clear();
    it->seq4.clear(); it->qual.clear(); it->l_qseq.clear(); it->mtid.clear(); it->n_cigar.clear(); it->cigar.clear();
    it->cigar_off.clear(); it->qual_off.clear();
    std::unordered_map<std::string, int64_t> names;
    for (size_t i = 0; i < n; ++i) {
        const bam1_t *b = it->batch[i];
        const bam1_core_t &c = b->core;
        it->pos.push_back(c.pos); it->mpos.push_back(c.mpos); it->isize.push_back(c.isize); it->flag.push_back(c.flag);
        it->mapq.push_back(c.qual); it->l_qseq.push_back(c.l_qseq); it->mtid.push_back(c.mtid); it->n_cigar.push_back(c.n_cigar);
        it->cigar_off.push_back(it->cigar.size());
        const uint32_t *cg = bam_get_cigar(b);
        it->cigar.insert(it->cigar.end(), cg, cg + c.n_cigar);
        if (it->qual.size() & 1) it->qual.push_back(0);
        const uint64_t qo = it->qual.size();
        it->qual_off.push_back(qo);
        const uint8_t *q = bam_get_qual(b), *s = bam_get_seq(b);
        it->qual.insert(it->qual.end(), q, q + c.l_qseq);
        it->seq4.resize((qo + (uint64_t)c.l_qseq + 1) / 2 + 1, 0);
        for (int32_t k = 0; k < c.l_qseq; ++k) { const uint64_t m = qo + (uint64_t)k; it->seq4[m >> 1] |= (uint8_t)(bam_seqi(s, k) << ((~m & 1) << 2)); }
        uint8_t rb = 0; int64_t pv = -1;
        if (it->overlaps && !it->batch_done[i]) {   // a halo read whose pair was tweaked in an earlier window takes no part again
            const char *qn = bam_get_qname(b);
            auto f = names.find(qn);
            if (f != names.end()) { pv = f->second; f->second = (int64_t)i; } else names.emplace(qn, (int64_t)i);
            if (name_bit(qn)) rb |= B200_RB_NAME_ODD;
        }
        rb |= it->batch_md[i];
        it->prev.push_back(pv); it->rbits.push_back(rb);
    }
    if (it->seq4.size() * 2 < it->qual.size() + 2) it->seq4.resize((it->qual.size() + 2) / 2, 0);
    it->file_start = {0, (int64_t)n};
    b200_batch_t bt; memset(&bt, 0, sizeof bt);
    bt.n_files = 1; bt.n_reads = (int64_t)n; bt.file_start = it->file_start.data();
    bt.pos = it->pos.data(); bt.flag = it->flag.data(); bt.mapq = it->mapq.data(); bt.l_qseq = it->l_qseq.data(); bt.n_cigar = it->n_cigar.data();
    bt.cigar_off = it->cigar_off.data(); bt.qual_off = it->qual_off.data(); bt.mtid = it->mtid.data(); bt.mpos = it->mpos.data(); bt.isize = it->isize.data();
    bt.prev_same_name = it->prev.data(); bt.rbits = it->rbits.data();
    bt.cigar = it->cigar.data(); bt.n_cigar_total = it->cigar.size(); bt.seq4 = it->seq4.data(); bt.qual = it->qual.data(); bt.qual_bytes = it->qual.size();
    bt.tid = it->tid; bt.tid_len = 0; bt.tid_name = "";
    b200_stage_conf_t sc; memset(&sc, 0, sizeof sc);
    sc.mode = B200_MODE_MPILEUP; sc.overlaps = it->overlaps; sc.max_depth = it->maxcnt;
    // filters are the callback's business (bam_plp_push drops only unmapped reads)
    sc.beg = it->serve_beg >= 0 ? it->serve_beg : it->batch[0]->core.pos; sc.end = it->serve_end;
    b200_stage_stats_t st;
    if (b200_stage(it->eng, &bt, &sc, &st) != 0) { fprintf(stderr, "[b200 bam_plp] %s\n", b200_last_error(it->eng)); return -1; }
    it->win_base = sc.beg; it->n_cols = st.n_cols;
    if (it->overlaps) {   // hand the tweaked qualities to the caller-visible copies
        std::vector<uint8_t> q(it->qual.size() + 8);
        if (b200_fetch_qual(it->eng, q.data(), it->qual.size()) != 0) return -1;
        for (size_t i = 0; i < n; ++i) memcpy(bam_get_qual(it->batch[i]), q.data() + it->qual_off[i], (size_t)it->batch[i]->core.l_qseq);
        // both mates staged together -> their tweak has happened (and is now in the copies): not again in a later window
        for (size_t i = 0; i < n; ++i) if (it->prev[i] >= 0) { it->batch_done[i] = 1; it->batch_done[(size_t)it->prev[i]] = 1; }
    }
    if (it->serve_end < kPosMax && it->maxcnt > 0) {   // the halo reads take this window's max-depth verdicts to the next one
        std::vector<uint8_t> keep(n);
        if (b200_fetch_mapq_keep(it->eng, nullptr, keep.data(), n) != 0) return -1;
        for (size_t i = 0; i < n; ++i)
            if (const uint8_t b = B200_RB_MAXDEPTH_OF(keep[i])) it->batch_md[i] = b;
    }
    it->col = 0; it->slab_beg = it->slab_end = 0; it->ent_pos = 0;
    return 0;
}

static int load_slab(b200_plp *it)
{
    it->slab_beg = it->slab_end;
    it->slab_end = std::min(it->n_cols, it->slab_beg + kSlabCols);
    const int64_t nc = it->slab_end - it->slab_beg;
    it->col_n.assign((size_t)nc + 1, 0);
    if (it->ents.size() < (size_t)1 << 20) it->ents.resize((size_t)1 << 20);
    for (;;) {
        size_t ne = 0;
        int rc = b200_pileup_entries(it->eng, 0, it->win_base + it->slab_beg, it->win_base + it->slab_end, it->col_n.data(), it->ents.data(),
                                     it->ents.size(), &ne);
        if (rc == -2) { it->ents.resize(ne + 1024); continue; }
        if (rc != 0) { fprintf(stderr, "[b200 bam_plp] %s\n", b200_last_error(it->eng)); return -1; }
        break;
    }
    it->ent_pos = 0;
    return 0;
}

// next column with n_plp > 0 of the contig being served, or nullptr when it is exhausted
static const bam_pileup1_t *serve(b200_plp *it, int *_tid, hts_pos_t *_pos, int *_n)
{
    while (it->serving) {
        if (it->col >= it->n_cols) {
            it->serving = false;
            if (it->serve_end < kPosMax) {
                // window cut inside the reference sequence: reads reaching the cut go back to the front of the collection --
                // those ending right at it too, as the max-depth rule still counts them as buffered there
                std::vector<bam1_t *> keep; std::vector<bam_pileup_cd> keep_cd; std::vector<uint8_t> keep_done, keep_md; size_t bytes = 0;
                for (size_t i = 0; i < it->batch.size(); ++i) {
                    bam1_t *b = it->batch[i];
                    if (read_end(b) >= it->serve_end) {
                        keep.push_back(b); keep_cd.push_back(it->batch_cd[i]); keep_done.push_back(it->batch_done[i]); keep_md.push_back(it->batch_md[i]);
                        bytes += (size_t)b->core.l_qseq;
                    } else { if (it->destruct) it->destruct(it->data, b, &it->batch_cd[i]); bam_destroy1(b); }
                }
                it->batch.clear(); it->batch_cd.clear(); it->batch_done.clear(); it->batch_md.clear();
                keep.insert(keep.end(), it->accum.begin(), it->accum.end()); keep_cd.insert(keep_cd.end(), it->accum_cd.begin(), it->accum_cd.end());
                keep_done.insert(keep_done.end(), it->accum_done.begin(), it->accum_done.end());
                keep_md.insert(keep_md.end(), it->accum_md.begin(), it->accum_md.end());
                it->accum.swap(keep); it->accum_cd.swap(keep_cd); it->accum_done.swap(keep_done); it->accum_md.swap(keep_md); it->accum_bytes += bytes;
            } else { free_reads(it, it->batch, it->batch_cd); it->batch_done.clear(); it->batch_md.clear(); }
            break;
        }
        if (it->col >= it->slab_end) { if (load_slab(it) != 0) { it->error = true; *_n = -1; return nullptr; } }
        while (it->col < it->slab_end) {
            const uint32_t n = it->col_n[(size_t)(it->col - it->slab_beg)];
            const int64_t c = it->col++;
            if (!n) continue;
            if (it->plp.size() < n) it->plp.resize(n);
            for (uint32_t k = 0; k < n; ++k) {
                const b200_pileup1_t &e = it->ents[it->ent_pos + k];
                bam_pileup1_t &p = it->plp[k];
                memset(&p, 0, sizeof p);
                p.b = it->batch[(size_t)e.read]; p.cd = it->batch_cd[(size_t)e.read]; p.qpos = e.qpos; p.indel = e.indel; p.cigar_ind = e.cigar_ind;
                p.is_del = e.is_del; p.is_head = e.is_head; p.is_tail = e.is_tail; p.is_refskip = e.is_refskip;
            }
            it->ent_pos += n;
            *_tid = it->tid; *_pos = it->win_base + c; *_n = (int)n;
            return it->plp.data();
        }
    }
    return nullptr;
}

// the collected contig becomes the served one
static int start_serving(b200_plp *it)
{
    it->batch.swap(it->accum); it->batch_cd.swap(it->accum_cd); it->batch_done.swap(it->accum_done); it->batch_md.swap(it->accum_md);
    it->accum.clear(); it->accum_cd.clear(); it->accum_done.clear(); it->accum_md.clear(); it->accum_bytes = 0;
    if (it->batch.empty()) return 0;
    it->tid = it->batch[0]->core.tid;
    // the previous window of this reference sequence ended at next_beg; this one ends at the start of the read that cut it
    it->serve_beg = it->next_beg;
    it->serve_end = it->cut ? it->pending->core.pos : kPosMax;
    it->next_beg = it->cut ? it->serve_end : -1;
    if (stage_batch(it) != 0) { it->error = true; return -1; }
    it->serving = true;
    return 0;
}

extern "C" {

bam_plp_t bam_plp_init(bam_plp_auto_f func, void *data)
{
    b200_plp *it = new b200_plp();
    it->func = func; it->data = data;
    int dev = 0;
    if (const char *s = getenv("B200_DEVICE")) dev = atoi(s);
    if (b200_engine_create(dev, &it->eng) != 0) { delete it; return nullptr; }
    it->tmp = bam_init1();
    if (const char *s = getenv("B200_PLP_WINDOW_BYTES")) { const long long v = atoll(s); if (v > 0) it->budget = (size_t)v; }
    return it;
}

void bam_plp_destroy(bam_plp_t it)
{
    if (!it) return;
    free_reads(it, it->accum, it->accum_cd); free_reads(it, it->batch, it->batch_cd);
    free_pending(it); bam_destroy1(it->tmp);
    b200_engine_destroy(it->eng);
    delete it;
}

void bam_plp_reset(bam_plp_t it)
{
    free_reads(it, it->accum, it->accum_cd); free_reads(it, it->batch, it->batch_cd);
    free_pending(it);
    it->serving = false; it->eof = false; it->error = false; it->last_tid = -1; it->last_pos = -1;
    it->cut = false; it->serve_beg = -1; it->serve_end = kPosMax; it->next_beg = -1; it->accum_bytes = 0;
    it->accum_done.clear(); it->batch_done.clear(); it->accum_md.clear(); it->batch_md.clear();
}

void bam_plp_set_maxcnt(bam_plp_t it, int maxcnt) { it->maxcnt = maxcnt; }
void bam_plp_constructor(bam_plp_t it, bam_plp_cd_f func) { it->construct = func; }
void bam_plp_destructor(bam_plp_t it, bam_plp_cd_f func) { it->destruct = func; }

int bam_plp_push(bam_plp_t it, const bam1_t *b)
{
    if (it->error) return -1;
    if (!b) { it->eof = true; return 0; }
    if (b->core.tid < 0 || (b->core.flag & 4)) return 0;   // unmapped reads are ignored
    if (b->core.tid < it->last_tid || (b->core.tid == it->last_tid && b->core.pos < it->last_pos)) {
        fprintf(stderr, "[b200 bam_plp] The input is not sorted\n");
        it->error = true;
        return -1;
    }
    it->last_tid = b->core.tid; it->last_pos = b->core.pos;
    bam1_t *c = bam_init1();
    if (!c || !bam_copy1(c, b)) { it->error = true; return -1; }
    bam_pileup_cd cd; cd.i = 0;
    const bool new_tid = !it->accum.empty() && it->accum[0]->core.tid != c->core.tid;
    // a window is cut at this read when the budget is spent and the read opens a new position (all reads starting before it
    // are in hand) beyond the start of the window under collection
    const bool over = !new_tid && !it->accum.empty() && it->accum_bytes >= it->budget && c->core.pos > it->accum.back()->core.pos &&
                      c->core.pos > (it->next_beg >= 0 ? it->next_beg : it->accum[0]->core.pos);
    if (new_tid || over) {
        // it waits until the window under collection has been handed out
        if (it->pending) { it->error = true; bam_destroy1(c); return -1; }
        if (it->construct) it->construct(it->data, c, &cd);
        it->pending = c; it->pending_cd = cd; it->cut = over;
    } else {
        if (it->construct) it->construct(it->data, c, &cd);
        it->accum.push_back(c); it->accum_cd.push_back(cd); it->accum_done.push_back(0); it->accum_md.push_back(0); it->accum_bytes += (size_t)c->core.l_qseq;
    }
    return 0;
}

const bam_pileup1_t *bam_plp64_next(bam_plp_t it, int *_tid, hts_pos_t *_pos, int *_n)
{
    if (it->error) { *_n = -1; return nullptr; }
    *_n = 0;
    for (;;) {
        if (const bam_pileup1_t *p = serve(it, _tid, _pos, _n)) return p;
        if (it->error) { *_n = -1; return nullptr; }
        // a contig is complete when a read of another contig has arrived, or at end of input
        if (it->pending || (it->eof && !it->accum.empty())) {
            if (start_serving(it) != 0) { *_n = -1; return nullptr; }
            if (it->pending) {
                it->accum.push_back(it->pending); it->accum_cd.push_back(it->pending_cd); it->accum_done.push_back(0); it->accum_md.push_back(0);
                it->accum_bytes += (size_t)it->pending->core.l_qseq; it->pending = nullptr; it->cut = false;
            }
            continue;
        }
        return nullptr;
    }
}

const bam_pileup1_t *bam_plp64_auto(bam_plp_t it, int *_tid, hts_pos_t *_pos, int *_n)
{
    if (!it->func || it->error) { *_n = -1; return nullptr; }
    for (;;) {
        if (const bam_pileup1_t *p = bam_plp64_next(it, _tid, _pos, _n)) return p;
        if (it->error) { *_n = -1; return nullptr; }
        *_n = 0;
        if (it->eof) return nullptr;
        // pull until the current contig is complete
        while (!it->pending && !it->eof) {
            int ret = it->func(it->data, it->tmp);
            if (ret >= 0) { if (bam_plp_push(it, it->tmp) < 0) { *_n = -1; return nullptr; } }
            else if (ret == -1) bam_plp_push(it, nullptr);
            else { it->error = true; *_n = -1; return nullptr; }
        }
    }
}

const bam_pileup1_t *bam_plp_next(bam_plp_t it, int *_tid, int *_pos, int *_n)
{
    hts_pos_t p = 0;
    const bam_pileup1_t *r = bam_plp64_next(it, _tid, &p, _n);
    *_pos = p < INT_MAX ? (int)p : INT_MAX;
    return r;
}

const bam_pileup1_t *bam_plp_auto(bam_plp_t it, int *_tid, int *_pos, int *_n)
{
    hts_pos_t p = 0;
    const bam_pileup1_t *r = bam_plp64_auto(it, _tid, &p, _n);
    *_pos = p < INT_MAX ? (int)p : INT_MAX;
    return r;
}

}  // extern "C"

// ---- multi-file merge (htslib bam_mplp64_auto; SURVEY.md Appendix A4)
struct b200_mplp {
    int n = 0;
    std::vector<b200_plp *> it;
    std::vector<uint32_t> tid; std::vector<uint64_t> pos; std::vector<int> n_plp; std::vector<const bam_pileup1_t *> plp;
    uint32_t min_tid = (uint32_t)-1; uint64_t min_pos = (uint64_t)-1;
};

extern "C" {

bam_mplp_t bam_mplp_init(int n, bam_plp_auto_f func, void **data)
{
    b200_mplp *m = new b200_mplp();
    m->n = n;
    for (int i = 0; i < n; ++i) {
        b200_plp *p = bam_plp_init(func, data[i]);
        if (!p) { for (b200_plp *q : m->it) bam_plp_destroy(q); delete m; return nullptr; }
        m->it.push_back(p);
    }
    m->tid.assign((size_t)n, (uint32_t)-1); m->pos.assign((size_t)n, (uint64_t)-1); m->n_plp.assign((size_t)n, 0); m->plp.assign((size_t)n, nullptr);
    return m;
}
int bam_mplp_init_overlaps(bam_mplp_t m) { for (b200_plp *p : m->it) p->overlaps = true; return 0; }
void bam_mplp_set_maxcnt(bam_mplp_t m, int maxcnt) { for (b200_plp *p : m->it) p->maxcnt = maxcnt; }
void bam_mplp_destroy(bam_mplp_t m) { if (!m) return; for (b200_plp *p : m->it) bam_plp_destroy(p); delete m; }
void bam_mplp_constructor(bam_mplp_t m, bam_plp_cd_f func) { for (b200_plp *p : m->it) p->construct = func; }
void bam_mplp_destructor(bam_mplp_t m, bam_plp_cd_f func) { for (b200_plp *p : m->it) p->destruct = func; }
void bam_mplp_reset(bam_mplp_t m)
{
    for (b200_plp *p : m->it) bam_plp_reset(p);
    std::fill(m->tid.begin(), m->tid.end(), (uint32_t)-1); std::fill(m->pos.begin(), m->pos.end(), (uint64_t)-1);
    std::fill(m->n_plp.begin(), m->n_plp.end(), 0); std::fill(m->plp.begin(), m->plp.end(), nullptr);
    m->min_tid = (uint32_t)-1; m->min_pos = (uint64_t)-1;
}

int bam_mplp64_auto(bam_mplp_t m, int *_tid, hts_pos_t *_pos, int *n_plp, const bam_pileup1_t **plp)
{
    uint64_t new_pos = (uint64_t)-1; uint32_t new_tid = (uint32_t)-1;
    for (int i = 0; i < m->n; ++i) {
        if (m->pos[(size_t)i] == m->min_pos && m->tid[(size_t)i] == m->min_tid) {
            int tid; hts_pos_t pos;
            m->plp[(size_t)i] = bam_plp64_auto(m->it[(size_t)i], &tid, &pos, &m->n_plp[(size_t)i]);
            if (m->it[(size_t)i]->error) return -1;
            if (m->plp[(size_t)i]) { m->tid[(size_t)i] = (uint32_t)tid; m->pos[(size_t)i] = (uint64_t)pos; }
            else { m->tid[(size_t)i] = 0; m->pos[(size_t)i] = 0; }
        }
        if (m->plp[(size_t)i]) {
            if (m->tid[(size_t)i] < new_tid) { new_tid = m->tid[(size_t)i]; new_pos = m->pos[(size_t)i]; }
            else if (m->tid[(size_t)i] == new_tid && m->pos[(size_t)i] < new_pos) new_pos = m->pos[(size_t)i];
        }
    }
    m->min_pos = new_pos; m->min_tid = new_tid;
    if (new_pos == (uint64_t)-1) return 0;
    *_tid = (int)new_tid; *_pos = (hts_pos_t)new_pos;
    int ret = 0;
    for (int i = 0; i < m->n; ++i) {
        if (m->pos[(size_t)i] == m->min_pos && m->tid[(size_t)i] == m->min_tid) { n_plp[i] = m->n_plp[(size_t)i]; plp[i] = m->plp[(size_t)i]; ++ret; }
        else { n_plp[i] = 0; plp[i] = nullptr; }
    }
    return ret;
}

int bam_mplp_auto(bam_mplp_t m, int *_tid, int *_pos, int *n_plp, const bam_pileup1_t **plp)
{
    hts_pos_t p = 0;
    int r = bam_mplp64_auto(m, _tid, &p, n_plp, plp);
    *_pos = p < INT_MAX ? (int)p : INT_MAX;
    return r;
}

// insertion text after a column (htslib bam_plp_insertion, without base modifications; SURVEY.md A3)
int b200_plp_insertion(const bam_pileup1_t *p, char *ins, int cap, int *del_len)
{
    if (cap > 0) ins[0] = 0;
    if (p->indel <= 0) return 0;
    if (del_len) *del_len = 0;
    const bam1_t *b = p->b;
    const uint32_t *cg = bam_get_cigar(b);
    int n = 0, j = 1;
    for (int k = p->cigar_ind + 1; k < (int)b->core.n_cigar; ++k) {
        const int op = cg[k] & 0xf, l = (int)(cg[k] >> 4);
        if (op == 6) { for (int i = 0; i < l; ++i, ++n) if (n + 1 < cap) ins[n] = '*'; }
        else if (op == 1) {
            for (int i = 0; i < l; ++i, ++j, ++n) {
                const int q = p->qpos + j - (int)p->is_del;
                if (n + 1 < cap) ins[n] = q < b->core.l_qseq ? "=ACMGRSVTWYHKDBN"[bam_seqi(bam_get_seq(b), q)] : 'N';
            }
        } else { if (op == 2 && del_len) *del_len = l; break; }
    }
    if (cap > 0) ins[n < cap ? n : cap - 1] = 0;
    return n;
}

// htslib's signature: the kstring is grown as needed (bam_plp_insertion, sam.h)
int bam_plp_insertion(const bam_pileup1_t *p, kstring_t *ins, int *del_len)
{
    if (!p || !ins) return -1;
    int dl = 0;
    const int n = b200_plp_insertion(p, nullptr, 0, &dl);          // length only
    if (ins->m < (size_t)n + 1) {
        char *t = (char *)realloc(ins->s, (size_t)n + 1);
        if (!t) return -1;
        ins->s = t; ins->m = (size_t)n + 1;
    }
    b200_plp_insertion(p, ins->s, (int)ins->m, &dl);
    ins->s[n] = 0; ins->l = (size_t)n;
    if (del_len && p->indel > 0) *del_len = dl;          // htslib leaves *del_len untouched when the column has no insertion
    return n;
}

}  // extern "C"
