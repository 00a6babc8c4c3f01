// mpileup_indel.cuh -- per-column indel alleles of the mpileup column stage (b200_mpileup_indels / b200_fetch_indels) and
// their quality and read-position sums (b200_indel_qsums, b200_indel_psums).
// Included by engine.cu.
//
// The distinct "+n..." / "-n" tokens the text prints after the entries of one (column, file) that pass -Q, with strand-split
// support, as a table in HBM (plp_core.h mp_entry_indel, ins_symbols, indel_key, indel_allele_equal).  Rows are ordered by
// column, then file, then first appearance in the line (file order of the reads; a read's insertion before its deletion).
//
//   1. k_ind_walk<false>: one warp per (file, 32-column group), lane = column, walks the group's reads in file order like
//      k_mp_counts.  A simple read ([S]M[S]) has no indel and is skipped after its descriptor's first half; the other reads
//      resolve their cursor at the lane's column.  Counts the events of every (column, file).
//   2. launch_scan: event offsets, segment = column * n_files + file, so that the events land in table order.
//   3. k_ind_walk<true>: the same walk writes the events from the segment's offset on (a group without events returns at
//      once), and their symbol counts; a scan of these gives every event its symbol bytes.
//   4. k_ind_syms: thread per event, writes its symbols and key.
//   5. k_ind_insert: thread per event, open addressing in a table of 2m slots per segment of m events (so a segment never
//      fills up).  The first event to claim a slot owns it; an event that finds its allele lowers the slot's owner to the
//      first appearance (atomicMin) and counts itself on its strand.  Equality is decided on length and bytes; the key only
//      filters.  A deep column of one shared allele costs one probe per event, not a pass over the allele list.
//   6. k_ind_mark + two scans: an event that owns its slot starts an allele; allele index and symbol offset.
//   7. k_ind_emit: the table rows and their symbols.
// b200_indel_qsums and b200_indel_psums run k_ind_qsums / k_ind_psums later over the same events, which stay in HBM until
// the next stage.
// Every event kernel is launched over the stage's bound on the events (ind_bounds) and reads the real count from HBM, so
// the call synchronises with the host once, at the end.
constexpr int IND_WARPS = 4;

struct IndelEv {
    int32_t col, file, len, read, k, qpos;
    uint32_t fl;        // bit 0: reverse strand, bit 1: the entry is a deletion (ins_symbols' query offset)
    uint32_t lo, m;     // first event of the (column, file) and how many it has
};

template <bool EMIT>
__global__ void __launch_bounds__(IND_WARPS * 32) k_ind_walk(View v, int32_t min_baseQ, int32_t n_groups, uint32_t *cnt,
                                                               const uint32_t *off, IndelEv *ev, uint32_t *ev_len, uint32_t cap)
{
    const int lane = threadIdx.x & 31;
    const int64_t w = (int64_t)blockIdx.x * IND_WARPS + (threadIdx.x >> 5);
    if (w >= (int64_t)n_groups * v.n_files) return;        // whole warps
    const int f = (int)(w / n_groups), g = (int)(w % n_groups);
    const int32_t c = g * 32 + lane;
    const bool live = c < v.ncols;
    const int64_t seg = (int64_t)c * v.n_files + f;
    uint32_t o = 0, m = 0;
    if (EMIT) {
        if (live) { o = off[seg]; m = off[seg + 1] - o; }
        if (!__any_sync(0xffffffffu, m != 0)) return;
    }
    uint32_t n = 0;
    const ReadRange rr = read_range(v, f, g);
    for (int32_t t = 0; t < rr.n; ++t) {
        const int32_t i = range_at(rr, t);
        ReadDesc d = load_hot(v.desc + i);
        if (d.fl & RD_SIMPLE) continue;                      // the same descriptor on every lane: no divergence
        if (!live || (uint32_t)(c - d.rpos) >= (uint32_t)(d.rend - d.rpos)) continue;
        load_cold(d, v.desc + i);
        Ent e;
        resolve(v, d, c, e);
        if (!e.indel || ent_qual(v, d, e) < min_baseQ) continue;
        const uint32_t *cg = v.cigar + d.cig_off;
        int del_len;
        const int ins = mp_entry_indel(d, cg, e, del_len);
        for (int x = 0; x < 2; ++x) {
            const int len = x == 0 ? ins : -del_len;
            if (x == 0 ? ins < 0 : del_len == 0) continue;
            if (EMIT && o + n < cap) {
                IndelEv r;
                r.col = c; r.file = f; r.len = len; r.read = i; r.k = e.k; r.qpos = e.qpos;
                r.fl = ((d.fl & RD_REV) ? 1u : 0u) | (e.is_del ? 2u : 0u); r.lo = o; r.m = m;
                ev[o + n] = r;
                ev_len[o + n] = len > 0 ? (uint32_t)len : 0u;
            }
            ++n;
        }
    }
    if (!EMIT && live) cnt[seg] = n;
}

__device__ __forceinline__ uint32_t ind_count(const uint32_t *n_ev, uint32_t cap) { const uint32_t n = *n_ev; return n < cap ? n : cap; }

__global__ void k_ind_syms(View v, const IndelEv *ev, const uint32_t *n_ev, uint32_t cap, const uint64_t *sym_off, uint64_t sym_cap,
                           char *sym, uint64_t key_mask, uint64_t *key)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ind_count(n_ev, cap)) return;
    const IndelEv x = ev[j];
    char *p = sym + sym_off[j];
    if (sym_off[j] + (uint64_t)(x.len > 0 ? x.len : 0) > sym_cap) return;   // over the bound: the call reports it
    if (x.len > 0) {
        const ReadDesc d = load_desc(v.desc + x.read);
        Ent e; e.qpos = x.qpos; e.k = x.k; e.is_del = (uint8_t)((x.fl >> 1) & 1u);
        ins_symbols(v, d, v.cigar + d.cig_off, e, false, '*', p);
    }
    key[j] = indel_key(x.len, p, key_mask);
}

__device__ __forceinline__ uint64_t ind_mix(uint64_t k)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return k;
}

// tbl: 2 slots per event, -1 = free; tcnt: forward / reverse support per slot
__global__ void k_ind_insert(const IndelEv *ev, const uint32_t *n_ev, uint32_t cap, const uint64_t *key, const uint64_t *sym_off,
                             const char *sym, int32_t *tbl, uint32_t *tcnt, uint32_t *slot)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ind_count(n_ev, cap)) return;
    const IndelEv x = ev[j];
    if (x.lo + x.m > cap) return;                            // a segment over the bound: the call reports it
    const uint64_t kj = key[j];
    const char *sj = sym + sym_off[j];
    const uint32_t size = 2 * x.m;
    int32_t *t = tbl + 2 * (size_t)x.lo;
    uint32_t h = (uint32_t)(ind_mix(kj) % size);
    for (;;) {
        int32_t s = *(volatile int32_t *)(t + h);
        if (s < 0) { s = atomicCAS(t + h, -1, (int32_t)j); if (s < 0) break; }
        if (key[s] == kj && indel_allele_equal(x.len, sj, ev[s].len, sym + sym_off[s])) { atomicMin(t + h, (int32_t)j); break; }
        h = h + 1 == size ? 0 : h + 1;
    }
    atomicAdd(tcnt + 2 * (2 * (size_t)x.lo + h) + (x.fl & 1u), 1u);
    slot[j] = h;
}

// over all `cap` events: first[j] = 1 where event j owns its slot (the first appearance of an allele), bytes[j] its symbols
__global__ void k_ind_mark(const IndelEv *ev, const uint32_t *n_ev, uint32_t cap, const int32_t *tbl, const uint32_t *slot,
                           uint32_t *first, uint32_t *bytes)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= cap) return;
    uint32_t a = 0, b = 0;
    if (j < ind_count(n_ev, cap)) {
        const IndelEv x = ev[j];
        a = x.lo + x.m <= cap && tbl[2 * (size_t)x.lo + slot[j]] == (int32_t)j;
        b = a && x.len > 0 ? (uint32_t)x.len : 0u;
    }
    first[j] = a; bytes[j] = b;
}

__global__ void k_ind_emit(const IndelEv *ev, const uint32_t *n_ev, uint32_t cap, const uint32_t *tcnt, const uint32_t *slot,
                           const uint32_t *first, const uint32_t *a_idx, const uint64_t *a_seq, const uint64_t *sym_off,
                           const char *sym, b200_indel_t *out, char *seq)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ind_count(n_ev, cap) || !first[j]) return;
    const IndelEv x = ev[j];
    const size_t s = 2 * (2 * (size_t)x.lo + slot[j]);
    b200_indel_t r;
    r.col = x.col; r.file = x.file; r.len = x.len; r.fwd = tcnt[s]; r.rev = tcnt[s + 1]; r.pad = 0; r.seq_off = a_seq[j];
    out[a_idx[j]] = r;
    const char *src = sym + sym_off[j];
    for (int32_t i = 0; i < x.len; ++i) seq[a_seq[j] + (uint64_t)i] = src[i];
}

// b200_indel_qsums / b200_indel_psums: thread per event of the table.  The allele's row is the row of its slot's owner (the
// first appearance, k_ind_insert); add(x, d, e, row, owner) adds what the event's entry contributes: e is the cursor of the
// entry the token follows, with the query position and is_del bit the walk kept in the event.
template <class Add>
__device__ __forceinline__ void ind_event_sums(const View &v, const IndelEv *ev, uint32_t n_ev, const int32_t *tbl, const uint32_t *slot,
                                               const uint32_t *a_idx, Add add)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_ev) return;
    const IndelEv x = ev[j];
    const int32_t owner = tbl[2 * (size_t)x.lo + slot[j]];
    const uint32_t row = a_idx[owner];
    const ReadDesc d = load_desc(v.desc + x.read);
    Ent e; e.qpos = x.qpos; e.is_del = (uint8_t)((x.fl >> 1) & 1u);   // all ent_qual and qpos5_of read of the cursor
    add(x, d, e, row, owner == (int32_t)j);
}

// the event adds its entry's BQ / MQ / MQ0 (plp_core.h mp_entry_qs) on its strand.  qs: the rows, zeroed by the caller.
// deep: set where an allele has more than QS_MAX_DEPTH entries on one strand (a sum could wrap).
__global__ void k_ind_qsums(View v, const IndelEv *ev, uint32_t n_ev, const int32_t *tbl, const uint32_t *slot, const uint32_t *a_idx,
                            const b200_indel_t *tab, b200_indel_qsum_t *qs, unsigned long long *deep)
{
    ind_event_sums(v, ev, n_ev, tbl, slot, a_idx, [&](const IndelEv &x, const ReadDesc &d, const Ent &e, uint32_t row, bool owner) {
        const EntQs q = mp_entry_qs(ent_qual(v, d, e), d);
        uint32_t *o = reinterpret_cast<uint32_t *>(qs + row) + (x.fl & 1u);
        atomicAdd(o, q.bq); atomicAdd(o + 2, q.mq); atomicAdd(o + 4, q.mq0);
        if (owner && (tab[row].fwd > QS_MAX_DEPTH || tab[row].rev > QS_MAX_DEPTH)) *deep = 1ull;
    });
}

// the event adds its entry's BP-5 and its square (plp_core.h mp_entry_ps) on its strand.  ps: the rows, zeroed by the caller.
// ovf: set where a sum of squares would exceed INT64_MAX (ps_sq_over on the value the atomicAdd found).
__global__ void k_ind_psums(View v, const IndelEv *ev, uint32_t n_ev, const int32_t *tbl, const uint32_t *slot, const uint32_t *a_idx,
                            b200_indel_psum_t *ps, unsigned long long *ovf)
{
    ind_event_sums(v, ev, n_ev, tbl, slot, a_idx, [&](const IndelEv &x, const ReadDesc &d, const Ent &e, uint32_t row, bool) {
        const EntPs p = mp_entry_ps(d, e);
        unsigned long long *o = reinterpret_cast<unsigned long long *>(ps + row) + (x.fl & 1u);
        atomicAdd(o, (unsigned long long)p.bp5);              // two's complement: the signed sum
        if (ps_sq_over(atomicAdd(o + 2, (unsigned long long)p.sq), p.sq)) *ovf = 1ull;
    });
}
