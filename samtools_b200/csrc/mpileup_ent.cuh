// mpileup_ent.cuh -- default single-file mpileup text path: entry strings + gather.
//
//   k_mp_entries  READ-MAJOR, one warp per 32 consecutive reads.  First LANE = READ: each lane loads its read's
//                 descriptor (one coalesced 512-byte load per warp), clips it to the window, adds its coverage
//                 difference and counts its eight-base groups; a warp scan of the counts numbers the warp's groups.
//                 Then LANE = GROUP: the warp walks its groups 32 at a time (two steps per iteration, loads issued
//                 together), each lane finding the read that owns its group by a binary search over the scanned counts
//                 (shuffles).  A group is eight consecutive query bases of a simple read ([S]<n>M[S]) -- one aligned
//                 8-byte quality load, one aligned 4-byte base load -- turned into eight 16-bit entries (plp_core.h
//                 "entry strings": sequence character, quality character, "^"/"$" flags; 0 = fails -Q) and stored with
//                 one 16-byte store at the index of the quality bytes.  So no lane idles on a read shorter than 256
//                 bases and a 40-kb read is spread over all 32 lanes.  Other reads (~3 %) go column by column through
//                 the generic cursor into slices of a second array, the warp taking them one by one; their slices come
//                 from one cursor atomic per warp.  The same pass feeds the line-length sums of mpileup_ss.cuh (coverage
//                 difference array, failing bases and extra bytes per column): it IS the size pass.
//   k_mp_gather   COLUMN-MAJOR, one thread per reference position: derives its line's length and layout from the column's
//                 sums, walks the reads of its 32-column slice in file order and appends the non-empty entries to its line
//                 (2 bytes per entry, no decoding, no CIGAR walk); the tile leaves through TMA bulk stores at the offset
//                 k_mp_place (mpileup_ss.cuh) gave it.
// Replaces the per-(read, column) formatting loop of the round-1 write kernel (~100 instructions per pair).
#pragma once

__device__ __forceinline__ uint32_t ref_nt16_at(const View &v, const uint8_t *refc, int32_t c)
{
    if ((int64_t)c < v.ref_len_rel) { const int64_t ri = (int64_t)c - v.ref_off; if (ri >= 0 && ri < v.ref_n) return (uint32_t)refc[ri] & 0xfu; }
    return 15u;
}


// reference codes of columns c .. c+7 as eight nibbles (nibble k = column c + k), 15 beyond the staged sequence
__device__ __forceinline__ uint32_t ref_nt16_x8(const View &v, const uint8_t *refc, int32_t c)
{
    const int64_t ri = (int64_t)c - v.ref_off;
    uint32_t x, y;
    if (c >= 0 && (int64_t)c + 8 <= v.ref_len_rel && ri >= 0 && ri + 8 <= v.ref_n) {
        const unsigned long long a = (unsigned long long)(refc + ri);
        const uint2 *p = reinterpret_cast<const uint2 *>(a & ~7ull);
        const uint2 lo = __ldg(p), hi = __ldg(p + 1);
        const uint32_t sh = (uint32_t)(a & 7ull) * 8u;
        const uint64_t l = (uint64_t)lo.y << 32 | lo.x, h = (uint64_t)hi.y << 32 | hi.x;
        const uint64_t wv = sh ? (l >> sh) | (h << (64u - sh)) : l;
        x = (uint32_t)wv & 0x0f0f0f0fu; y = (uint32_t)(wv >> 32) & 0x0f0f0f0fu;
    } else {
        x = 0; y = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) { x |= ref_nt16_at(v, refc, c + k) << (8 * k); y |= ref_nt16_at(v, refc, c + 4 + k) << (8 * k); }
    }
    x = (x | x >> 4) & 0x00ff00ffu; x = (x | x >> 8) & 0xffffu;
    y = (y | y >> 4) & 0x00ff00ffu; y = (y | y >> 8) & 0xffffu;
    return x | y << 16;
}

// eight consecutive bases of a simple read that all lie inside the read and the window: no range tests, the "^" / "$"
// flags are patched in afterwards by the one lane that holds the read's first / last base
template <bool HAS_REF>
__device__ __forceinline__ uint32_t ent_group8(const View &v, const uint8_t *refc, uint2 qq, uint32_t s4, int32_t c_of_g, uint32_t rev, int minq,
                                               const uint8_t *tab, uint32_t (&ent)[8])
{
    uint32_t failmask = 0;
    const uint8_t *t = tab + rev * 16u;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t q = ((k < 4 ? qq.x : qq.y) >> (8 * (k & 3))) & 0xffu;
        uint32_t code = (s4 >> (8 * (k >> 1) + ((k & 1) ? 0 : 4))) & 0xfu;
        if (HAS_REF) { if (code == ref_nt16_at(v, refc, c_of_g + k)) code = 0; }
        uint32_t x = (uint32_t)t[code] | umin32(q + 33u, 126u) << 8;
        if ((int)q < minq) { x = 0; failmask |= 1u << k; }
        ent[k] = x;
    }
    return failmask;
}

// What a lane needs to format one eight-base group of a simple read, fetched from the lane that owns the read.  Query
// index g of the group and column c = g + cq of its first base; everything else is in columns: [a, b) the read's columns
// inside the window, fl its strand (GF_REV) and whether its first / last base lies inside the window (GF_HEAD / GF_TAIL:
// "^" / "$" go on those).
struct EntGrp { uint32_t g; int32_t c, a, b; uint32_t fl; };
enum { GF_REV = 1, GF_HEAD = 2, GF_TAIL = 4 };

// Group t of the warp's 32 reads: t counts the groups of lane 0's read first, then lane 1's, ...; incl is this lane's
// inclusive prefix sum of the group counts.  The owner is the first lane whose prefix exceeds t (a read without groups has
// the same prefix as its predecessor, so it never owns one): a five-step binary search over the lanes' registers.
__device__ __forceinline__ EntGrp ent_grp_at(uint32_t t, uint32_t incl, uint32_t gb, uint32_t cq, int32_t a, int32_t b, uint32_t fl)
{
    int j = 0;
#pragma unroll
    for (int s = 16; s; s >>= 1) { const uint32_t e = __shfl_sync(0xffffffffu, incl, j + s - 1); if (e <= t) j += s; }
    EntGrp r;
    r.g = __shfl_sync(0xffffffffu, gb, j) + 8u * t;      // gb = first group's query index - 8 x (groups before the read)
    r.c = (int32_t)(r.g + __shfl_sync(0xffffffffu, cq, j));
    r.a = __shfl_sync(0xffffffffu, a, j); r.b = __shfl_sync(0xffffffffu, b, j);
    r.fl = __shfl_sync(0xffffffffu, fl, j);
    return r;
}

// One group: all eight bases are formatted (bytes beyond the read's ends belong to its neighbours in the arrays and are
// harmless to read); the ones inside [a, b) are kept.  A group at a read's end shares its aligned 16-byte segment of E with
// the neighbouring read's group (possibly in another lane): both write only their own entries, with 2-byte stores.
template <bool HAS_REF>
__device__ __forceinline__ void ent_grp_emit(const View &v, const uint8_t *refc, const EntGrp &q, uint2 qq, uint32_t s4, bool swar, bool ends,
                                             int minq, uint32_t minq4, const uint8_t *s_tab, uint32_t *fail, uint32_t *extra, uint16_t *E)
{
    const uint32_t rev = q.fl & GF_REV;
    uint32_t w[4], failmask;
    if (swar) {
        uint32_t r8 = 0;
        if (HAS_REF) r8 = ref_nt16_x8(v, refc, q.c);
        failmask = ent_group8_swar(qq.x, qq.y, s4, HAS_REF, r8, ent_tab(rev), minq4, w);
    } else {
        uint32_t ent[8];
        failmask = ent_group8<HAS_REF>(v, refc, qq, s4, q.c, rev, minq, s_tab, ent);
#pragma unroll
        for (int k = 0; k < 4; ++k) w[k] = ent[2 * k] | ent[2 * k + 1] << 16;
    }
    const uint32_t kb = q.a > q.c ? (uint32_t)(q.a - q.c) : 0u, ke = (uint32_t)(q.b - q.c) < 8u ? (uint32_t)(q.b - q.c) : 8u;
    const uint32_t vmask = ((1u << ke) - 1u) & ~((1u << kb) - 1u);
    failmask &= vmask;
    if (ends) {   // "^"+mapq at the read's first base, "$" at its last: at most one group each
        const uint32_t kh = (q.fl & GF_HEAD) ? (uint32_t)(q.a - q.c) : 8u, kt = (q.fl & GF_TAIL) ? (uint32_t)(q.b - 1 - q.c) : 8u;
        const uint32_t okm = vmask & ~failmask;
        // flag f of entry k: word k >> 1, half k & 1 -- selected with compares so that w[] stays in registers
        if (kh < 8u && ((okm >> kh) & 1u)) {
            const uint32_t f = 0x80u << (16u * (kh & 1u)), j = kh >> 1;
            w[0] |= j == 0u ? f : 0u; w[1] |= j == 1u ? f : 0u; w[2] |= j == 2u ? f : 0u; w[3] |= j == 3u ? f : 0u;
            atomicAdd(&extra[q.c + (int32_t)kh], 2u);
        }
        if (kt < 8u && ((okm >> kt) & 1u)) {
            const uint32_t f = 0x8000u << (16u * (kt & 1u)), j = kt >> 1;
            w[0] |= j == 0u ? f : 0u; w[1] |= j == 1u ? f : 0u; w[2] |= j == 2u ? f : 0u; w[3] |= j == 3u ? f : 0u;
            atomicAdd(&extra[q.c + (int32_t)kt], 1u);
        }
    }
    while (failmask) { const int k = __ffs(failmask) - 1; failmask &= failmask - 1u; atomicAdd(&fail[q.c + k], 1u); }
    if (vmask == 0xffu) {
        *reinterpret_cast<uint4 *>(E + q.g) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) if ((vmask >> k) & 1u) E[q.g + (uint32_t)k] = (uint16_t)(w[k >> 1] >> (16 * (k & 1)));
    }
}

// steps of 32 groups whose loads k_mp_entries issues together: 2 fits 48 / 58 registers (no spills); 1 measured 1 % slower
constexpr int ENT_STEPS = 2;

template <bool HAS_REF>
__global__ void __launch_bounds__(256) k_mp_entries(View v, MpConf cf, int64_t n_reads, const uint8_t *refc /* per staged reference byte: nt16 code | 0..4 code << 4 */,
                                                    int32_t *diff, uint32_t *fail, uint32_t *extra, uint16_t *E, uint16_t *E2,
                                                    unsigned long long *e2_cursor, ReadDesc *desc_rw)
{
    __shared__ uint8_t s_tab[32];
    if (threadIdx.x < 32) s_tab[threadIdx.x] = (uint8_t)".ACMGRSVTWYHKDBN,acmgrsvtwyhkdbn"[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const bool ends = !cf.no_ends;
    const int minq = cf.min_baseQ;
    const bool swar = minq <= 127;                              // the SIMD-in-word formatter takes 0 <= -Q <= 127 (anything else: scalar route)
    const uint32_t minq4 = (uint32_t)(minq > 0 ? minq : 0) * 0x01010101u;
    for (int64_t i0 = warp * 32; i0 < n_reads; i0 += n_warps * 32) {
        // ---- lane = read: descriptor (one coalesced 512-byte load per warp), window clip, coverage difference
        const int64_t i = i0 + lane;
        ReadDesc d;
        if (i < n_reads) d = load_hot(v.desc + i);
        else { d.rpos = 0; d.rend = 0; }
        const int32_t a = d.rpos > 0 ? d.rpos : 0, b = d.rend < v.ncols ? d.rend : v.ncols;   // columns inside the window
        const bool live = d.rend > d.rpos && a < b;             // not filtered, overlaps the window
        if (live) { atomicAdd(&diff[a], 1); atomicAdd(&diff[b], -1); }
        const bool simple = live && (d.fl & RD_SIMPLE);
        // simple read: its eight-base groups [lo & ~7, hi) in query indices, lo / hi = query index of column a / b
        uint32_t n_g = 0, gb = 0, cq = 0, fl = 0;
        if (simple) {
            const uint32_t q0 = d.qoff + (uint32_t)d.qstart;                 // query index of column rpos
            const uint32_t lo = q0 + (uint32_t)(a - d.rpos), hi = q0 + (uint32_t)(b - d.rpos);
            n_g = (hi - (lo & ~7u) + 7u) >> 3;
            gb = lo & ~7u;
            cq = (uint32_t)d.rpos - q0;                                       // column = query index + cq (mod 2^32)
            fl = ((d.fl & RD_REV) ? (uint32_t)GF_REV : 0u) | (d.rpos == a ? (uint32_t)GF_HEAD : 0u) | (d.rend == b ? (uint32_t)GF_TAIL : 0u);
        }
        // ---- warp scan of the group counts.  The total fits 32 bits: every group holds at least one staged quality
        // byte of its own, and the staged qualities are limited to 4 GiB.
        uint32_t incl = n_g;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, incl, s); if (lane >= s) incl += y; }
        const uint32_t T = __shfl_sync(0xffffffffu, incl, 31);
        gb -= 8u * (incl - n_g);
        // ---- lane = group: ENT_STEPS steps of 32 groups per iteration, their loads issued together
        for (uint32_t t0 = 0; t0 < T; t0 += 32u * ENT_STEPS) {
            EntGrp q[ENT_STEPS]; uint2 qq[ENT_STEPS]; uint32_t s4[ENT_STEPS];
#pragma unroll
            for (int u = 0; u < ENT_STEPS; ++u) {
                const uint32_t t = t0 + 32u * u + (uint32_t)lane;
                if (u == 0 || t0 + 32u * u < T) q[u] = ent_grp_at(t, incl, gb, cq, a, b, fl);   // warp-uniform test
                if (t < T) { qq[u] = __ldg(reinterpret_cast<const uint2 *>(v.qual + q[u].g)); s4[u] = __ldg(reinterpret_cast<const uint32_t *>(v.seq4 + (q[u].g >> 1))); }
            }
#pragma unroll
            for (int u = 0; u < ENT_STEPS; ++u)
                if (t0 + 32u * u + (uint32_t)lane < T) ent_grp_emit<HAS_REF>(v, refc, q[u], qq[u], s4[u], swar, ends, minq, minq4, s_tab, fail, extra, E);
        }
        // ---- other reads (indels, pads, skips): the warp walks them one by one, lanes along the columns.  Their slices of
        // E2 come from one cursor atomic per warp; the gather finds a read's slice through its descriptor's pad_.
        const bool gen = live && !simple;
        uint32_t gm = __ballot_sync(0xffffffffu, gen);
        if (gm) {
            unsigned long long span = gen ? (unsigned long long)(uint32_t)(d.rend - d.rpos) : 0ull, ex = span;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, ex, s); if (lane >= s) ex += y; }
            unsigned long long base = 0;
            if (lane == 31) base = atomicAdd(e2_cursor, ex);
            base = __shfl_sync(0xffffffffu, base, 31);
            while (gm) {
                const int r = __ffs(gm) - 1; gm &= gm - 1u;
                const int64_t ir = i0 + r;
                ReadDesc dr = load_hot(v.desc + ir);
                load_cold(dr, v.desc + ir);
                const unsigned long long eo = __shfl_sync(0xffffffffu, base + ex - span, r);
                const int32_t ar = __shfl_sync(0xffffffffu, a, r), br = __shfl_sync(0xffffffffu, b, r);
                for (int32_t c = ar + lane; c < br; c += 32) {
                    const uint32_t rb = HAS_REF ? ref_nt16_at(v, refc, c) : 0x10u;
                    uint32_t xb;
                    const uint32_t x = ent_generic(v, cf, dr, c, rb, s_tab, xb);
                    E2[eo + (uint32_t)(c - dr.rpos)] = (uint16_t)x;
                    if (!x) atomicAdd(&fail[c], 1u);
                    else if (xb) atomicAdd(&extra[c], xb);
                }
            }
            if (gen) desc_rw[i].pad_ = (uint32_t)(base + ex - span);
        }
    }
}

struct MpEntFmt {
    View v; MpConf cf; const uint16_t *E, *E2;
    typedef MpFileSz State;
    __device__ __forceinline__ void write(int32_t c, const State &s, char *p) const { mp_line_write_ent(v, cf, c, s, p, E, E2); }
};

// Both entry arrays carry ENT_PAD entries in front of index 0: the gather addresses "the entry of the first column of a
// 32-column group" of every read over the group, which lies up to 31 entries before the read's first entry.
constexpr int ENT_PAD = 64;

// ---- the gather: one warp per 32-column group ------------------------------------------------------------------------
// The kernel issues every tile-level load (the column's n_plp / fail / extra sums, the tile's output offset, the warp's read
// range) at entry, before the block scan, so that they cost one round trip together.  Then two phases per round of 32 slice positions
// of the group's read range, with shared memory as the transpose buffer:
//   fetch   LANES ALONG THE READS: each lane loads its read's whole 32-byte descriptor (one sector: the second-array offset
//           of a read with indels does not wait on its flags).  Reads that reach the group get a row (ballot compaction, file
//           order kept); the 32 entries of a read over the group -- 64 contiguous bytes of its entry string -- go straight
//           from global memory into its row with five aligned 16-byte cp.async copies, not through registers.  A row header
//           carries where column c0's entry sits in the row, which columns the read covers, and its mapq / flags word.  So a
//           round waits on two round trips (descriptors, entries), three for a group with far-reaching reads (their index list).
//   append  LANES ALONG THE COLUMNS: the warp walks the rows in file order; lane c picks its entry out of the row with a
//           2-byte shared-memory load (one row = 16 consecutive banks: conflict free) and appends the sequence / quality
//           characters to its own line through cursors it keeps in registers.  No global-memory latency inside this loop,
//           so it needs no software pipelining: ~15 instructions per row.
// Entries that carry indel text (ENT_SPECIAL) go through ONE out-of-line copy of the generic formatter.
// Same bytes as mp_line_write_ent (plp_core.h), which stays the reference implementation (emulation harness, deep tiles).

// cold paths read the View / configuration from a copy in global memory: taking the address of the kernel parameter for an
// out-of-line call would make every thread copy the whole parameter block to local memory
// Length and quality come back as separate fields: the text of a deletion entry includes the deleted reference bases, so a
// long deletion's entry is longer than 16 bits.
struct SpecialEnt { uint32_t n; int q; };
__device__ __noinline__ SpecialEnt ent_special_g(const MpEntFmt *g, int32_t i, int32_t c, char *ps)
{
    SpecialEnt r;
    r.n = (uint32_t)ent_special(g->v, g->cf, i, c, ps, r.q);
    return r;
}

// Row buffer of a warp: one row of GROW bytes per slice position of a round.  GROW is a multiple of 16 (cp.async needs
// 16-byte aligned destinations); with 80 = 5 x 16 the eight 16-byte copies of a quarter warp land in distinct bank groups.
// 4 warps x 32 rows x (80 + 16 header) bytes = 12 KB per CTA; with the ~16 KB text budget at 30x / 150 bp, 7 CTAs per SM.
constexpr int GROW = 80, GROWS = 32;
struct GHdr { uint32_t off, vm, pk; int32_t i; };   // byte offset of column c0's entry in the warp's row buffer, columns covered, qstart|mapq|flags, read index

__device__ __forceinline__ void sts8(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(saddr), "r"(v) : "memory"); }

// one slice position of a round: the aligned start of the read's 80 bytes of entry string around column c0 + the row
// header fields; vm == 0: the read does not reach the group (or t is past the range)
struct GRead { const uint4 *q; uint32_t vm, pk, o; int32_t i; };

__device__ __forceinline__ GRead gather_read(const MpEntFmt &fmt, const ReadRange &rr, int32_t c0, int32_t t)
{
    const uint32_t kSimple = (uint32_t)RD_SIMPLE << 24;
    GRead f;
    f.q = nullptr; f.vm = 0; f.pk = 0; f.o = 0; f.i = 0;
    if (t < rr.n) {
        f.i = range_at(rr, t);
        const uint4 *dp = reinterpret_cast<const uint4 *>(fmt.v.desc + f.i);
        const uint4 d = __ldg(dp), d2 = __ldg(dp + 1);       // hot and cold half of the descriptor: one 32-byte sector
        const int32_t rpos = (int32_t)d.x, rend = (int32_t)d.y;
        f.pk = d.w;
        const int32_t lo_c = rpos > c0 ? rpos - c0 : 0, hi_c = rend - c0 < 32 ? rend - c0 : 32;
        if (hi_c > lo_c) {
            f.vm = (hi_c >= 32 ? 0xffffffffu : (1u << hi_c) - 1u) & ~((1u << lo_c) - 1u);
            const uint16_t *src = (f.pk & kSimple) ? fmt.E + (d.z + (f.pk & 0xffffu)) : fmt.E2 + d2.w;   // d2.w: pad_
            src += c0 - rpos;                                  // entry of column c0 (before the read's first entry when the read starts inside the group)
            const unsigned long long a = (unsigned long long)src;
            f.q = reinterpret_cast<const uint4 *>(a & ~15ull);
            f.o = (uint32_t)(a & 15ull);                       // bytes between the aligned address and column c0's entry
        }
    }
    return f;
}

// row `row` of the warp's buffer: the read's 80 bytes through cp.async (in flight until the caller's wait), then its header
__device__ __forceinline__ void gather_row(uint32_t rows_s, GHdr *hdr, uint32_t row, const GRead &f)
{
    const uint32_t s = rows_s + row * GROW;
#pragma unroll
    for (int k = 0; k < GROW / 16; ++k) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s + 16u * k), "l"(f.q + k) : "memory");
    GHdr h; h.off = row * GROW + f.o; h.vm = f.vm; h.pk = f.pk; h.i = f.i;
    *reinterpret_cast<uint4 *>(hdr + row) = *reinterpret_cast<const uint4 *>(&h);
}

template <bool OUT_MAPQ>
__device__ __forceinline__ void gather_group(const MpEntFmt &fmt, const MpEntFmt *gfmt, const ReadRange &rr, int32_t c0, bool on,
                                             uint32_t so, uint32_t qo, uint32_t mo, char *sb, unsigned char *rows, GHdr *hdr)
{
    const uint32_t sb_s = (uint32_t)__cvta_generic_to_shared(sb);
    so += sb_s; qo += sb_s; mo += sb_s;
    const int lane = threadIdx.x & 31;
    const uint32_t lt = (1u << lane) - 1u;
    const int32_t c = c0 + lane;
    const uint32_t rows_base = (uint32_t)__cvta_generic_to_shared(rows);
    for (int32_t t0 = 0; t0 < rr.n; t0 += GROWS) {
        const GRead f = gather_read(fmt, rr, c0, t0 + lane);
        // ---- rows of this round: lane = read
        const uint32_t live = __ballot_sync(0xffffffffu, f.vm != 0u);
        if (!live) continue;
        __syncwarp();                                              // the previous round's rows have been consumed
        if (f.vm) gather_row(rows_base, hdr, (uint32_t)__popc(live & lt), f);
        asm volatile("cp.async.wait_all;" ::: "memory");           // this lane's copies have landed ...
        __syncwarp();                                              // ... and every lane's: the rows are complete
        // ---- append: lane = column (cursors are 32-bit shared-memory addresses: plain st.shared, no generic-address arithmetic)
        const int nrows = __popc(live);
        if (on) {
            const uint32_t rows_s = rows_base + 2u * (uint32_t)lane;
            for (int r = 0; r < nrows; ++r) {
                const uint4 hw = *reinterpret_cast<const uint4 *>(hdr + r);          // broadcast
                uint32_t e;
                asm volatile("ld.shared.u16 %0, [%1];" : "=r"(e) : "r"(rows_s + hw.x));
                const bool has = ((hw.y >> lane) & 1u) && e != 0u;
                if (has) {
                    const uint32_t mapq = (hw.z >> 16) & 0xffu;
                    if (e & 0x8080u) {                                   // "^" / "$" decorations or indel text: rare
                        if (e == ENT_SPECIAL) {
                            const SpecialEnt se = ent_special_g(gfmt, (int32_t)hw.w, c, sb + (so - sb_s));
                            so += se.n;
                            const int q = se.q;
                            sts8(qo++, (uint32_t)(q + 33 < 126 ? q + 33 : 126));
                        } else {
                            if (e & 0x80u) { sts8(so++, (uint32_t)'^'); sts8(so++, umin32(mapq + 33u, 126u)); }
                            sts8(so++, e & 0x7fu);
                            if (e & 0x8000u) sts8(so++, (uint32_t)'$');
                            sts8(qo++, (e >> 8) & 0x7fu);
                        }
                    } else {
                        sts8(so++, e); sts8(qo++, e >> 8);
                    }
                    if (OUT_MAPQ) sts8(mo++, umin32(mapq + 33u, 126u));
                }
            }
        }
    }
}

template <int MIN_CTAS, bool OUT_MAPQ>
__global__ void __launch_bounds__(TILE, MIN_CTAS) k_mp_gather(MpEntFmt fmt, const MpEntFmt *gfmt, const int32_t *nplp, const uint32_t *fail, const uint32_t *extra,
                                                              const uint64_t *tile_base, char *out, uint32_t smem_cap)
{
    extern __shared__ __align__(16) char s_text[];
    __shared__ uint32_t s_ws[TILE / 32];
    __shared__ __align__(16) unsigned char s_rows[TILE / 32][GROWS * GROW];
    __shared__ __align__(16) GHdr s_hdr[TILE / 32][GROWS];
    const int32_t ncols = fmt.v.ncols;
    const int32_t c = (int32_t)blockIdx.x * TILE + (int32_t)threadIdx.x;
    const int32_t c0 = (int32_t)(blockIdx.x * TILE + (threadIdx.x & ~31u));
    // Every tile-level load goes out here, before the block scan, so that they share one round trip: the column's sums
    // (k_mp_place, k_mp_entries), the tile's output offset, and the warp's read range (a warp past the window reads the
    // last group's).  The line's length and state follow from the sums as in k_mp_place.
    int32_t np = 0; uint32_t nf = 0, nx = 0;
    if (c < ncols) { np = nplp[c]; nf = fail[c]; nx = extra[c]; }
    const uint64_t base = tile_base[blockIdx.x];
    const ReadRange rr = read_range(fmt.v, 0, min(c0 >> 5, fmt.v.n_tiles - 1));   // the same for the 32 lanes
    MpFileSz stt;
    const uint32_t len = c < ncols ? mp_sums_line_size(fmt.v, fmt.cf, c, np, nf, nx, &stt) : 0u;
    uint32_t total;
    const uint32_t off = block_excl_scan<TILE, ScanSum>(len, s_ws, total);
    if (total == 0) return;
    const uint32_t phase = (uint32_t)(base & 15);
    if (total + phase <= smem_cap) {
        char *sb = s_text + phase;
        // every line's fixed parts (header, count, separators, place holders, newline) by the column's own thread ...
        const int wi = threadIdx.x >> 5;
        uint32_t so = 0, qo = 0, mo = 0;
        bool on = false;
        if (len) {
            const EntCur k = ent_layout(fmt.v, fmt.cf, c, stt, sb + off);
            if (k.ps) { on = true; so = (uint32_t)(k.ps - sb); qo = (uint32_t)(k.pq - sb); mo = OUT_MAPQ ? (uint32_t)(k.pm - sb) : 0u; }
        }
        // ... then the entries of the warp's 32 columns
        if (__any_sync(0xffffffffu, on)) gather_group<OUT_MAPQ>(fmt, gfmt, rr, c0, on, so, qo, mo, sb, s_rows[wi], s_hdr[wi]);
        // Each warp stores its own 32 lines (contiguous in the tile) as soon as it has them: no block-wide barrier at the end,
        // so a warp with a deep column does not hold the other three.
        const uint32_t wbeg = __shfl_sync(0xffffffffu, off, 0);
        const uint32_t wend = __shfl_sync(0xffffffffu, off + len, 31);
        store_staged<32>(out + base, sb, wbeg, wend - wbeg, phase);
    } else if (len) {
        mp_line_write_ent(gfmt->v, gfmt->cf, c, stt, out + base + off, gfmt->E, gfmt->E2);   // very deep tile: format straight into HBM
    }
}
