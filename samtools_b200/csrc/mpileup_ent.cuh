// mpileup_ent.cuh -- default single-file mpileup text path: entry strings + gather.
//
//   k_mp_entries  READ-MAJOR, one warp per read, lanes along the read.  Simple reads ([S]<n>M[S]): each lane takes
//                 eight consecutive query bases -- one aligned 8-byte quality load, one aligned 4-byte base load --
//                 turns them into eight 16-bit entries (plp_core.h "entry strings": sequence character, quality
//                 character, "^"/"$" flags; 0 = fails -Q) and stores them with one 16-byte store at the index of the
//                 quality bytes.  Other reads go column by column through the generic cursor into a slice of a second
//                 array.  The same pass feeds the line-length sums of mpileup_ss.cuh (coverage difference array,
//                 failing bases and extra bytes per column): it IS the size pass.
//   k_mp_gather   COLUMN-MAJOR, one thread per reference position: walks the reads of its 32-column slice in file
//                 order and appends the non-empty entries to its line (2 bytes per entry, no decoding, no CIGAR walk);
//                 the tile leaves through the TMA bulk store of text_write_tile.
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
    for (int64_t i = warp; i < n_reads; i += n_warps) {
        ReadDesc d = load_hot(v.desc + i);
        if (d.rend <= d.rpos) continue;                         // filtered read
        const int32_t a = d.rpos > 0 ? d.rpos : 0, b = d.rend < v.ncols ? d.rend : v.ncols;   // columns inside the window
        if (a >= b) continue;
        if (lane == 0) { atomicAdd(&diff[a], 1); atomicAdd(&diff[b], -1); }
        const uint32_t rev = (d.fl & RD_REV) ? 1u : 0u;
        if (d.fl & RD_SIMPLE) {
            const uint32_t q0 = d.qoff + (uint32_t)d.qstart;                 // query index of column rpos
            const uint32_t lo = q0 + (uint32_t)(a - d.rpos), hi = q0 + (uint32_t)(b - d.rpos);
            const uint32_t qtail = q0 + (uint32_t)(d.rend - d.rpos) - 1u;
            const EntTab tab = ent_tab(rev);
            for (uint32_t g = (lo & ~7u) + 8u * (uint32_t)lane; g < hi; g += 256u) {
                const uint2 qq = __ldg(reinterpret_cast<const uint2 *>(v.qual + g));
                const uint32_t s4 = __ldg(reinterpret_cast<const uint32_t *>(v.seq4 + (g >> 1)));
                const int32_t c_of_g = d.rpos + (int32_t)(g - q0);          // column of query index g
                // all eight bases of the group are formatted (bytes beyond the read's ends belong to its neighbours in the
                // arrays and are harmless to read); the ones inside [lo,hi) are kept
                uint32_t w[4], failmask;
                if (swar) {
                    uint32_t r8 = 0;
                    if (HAS_REF) r8 = ref_nt16_x8(v, refc, c_of_g);
                    failmask = ent_group8_swar(qq.x, qq.y, s4, HAS_REF, r8, tab, minq4, w);
                } else {
                    uint32_t ent[8];
                    failmask = ent_group8<HAS_REF>(v, refc, qq, s4, c_of_g, rev, minq, s_tab, ent);
#pragma unroll
                    for (int k = 0; k < 4; ++k) w[k] = ent[2 * k] | ent[2 * k + 1] << 16;
                }
                const uint32_t kb = lo > g ? lo - g : 0u, ke = hi - g < 8u ? hi - g : 8u;
                const uint32_t vmask = ((1u << ke) - 1u) & ~((1u << kb) - 1u);
                failmask &= vmask;
                if (ends) {   // "^"+mapq at the read's first base, "$" at its last: at most one lane each
                    const uint32_t kh = q0 - g, kt = qtail - g;
                    const uint32_t okm = vmask & ~failmask;
                    // flag f of entry k: word k >> 1, half k & 1 -- selected with compares so that w[] stays in registers
                    if (kh < 8u && ((okm >> kh) & 1u)) {
                        const uint32_t f = 0x80u << (16u * (kh & 1u)), j = kh >> 1;
                        w[0] |= j == 0u ? f : 0u; w[1] |= j == 1u ? f : 0u; w[2] |= j == 2u ? f : 0u; w[3] |= j == 3u ? f : 0u;
                        atomicAdd(&extra[c_of_g + (int32_t)kh], 2u);
                    }
                    if (kt < 8u && ((okm >> kt) & 1u)) {
                        const uint32_t f = 0x8000u << (16u * (kt & 1u)), j = kt >> 1;
                        w[0] |= j == 0u ? f : 0u; w[1] |= j == 1u ? f : 0u; w[2] |= j == 2u ? f : 0u; w[3] |= j == 3u ? f : 0u;
                        atomicAdd(&extra[c_of_g + (int32_t)kt], 1u);
                    }
                }
                while (failmask) { const int k = __ffs(failmask) - 1; failmask &= failmask - 1u; atomicAdd(&fail[c_of_g + k], 1u); }
                if (vmask == 0xffu) {
                    *reinterpret_cast<uint4 *>(E + g) = make_uint4(w[0], w[1], w[2], w[3]);
                } else {
#pragma unroll
                    for (int k = 0; k < 8; ++k) if ((vmask >> k) & 1u) E[g + (uint32_t)k] = (uint16_t)(w[k >> 1] >> (16 * (k & 1)));
                }
            }
        } else {
            load_cold(d, v.desc + i);
            unsigned long long eo = 0;
            if (lane == 0) { eo = atomicAdd(e2_cursor, (unsigned long long)(uint32_t)(d.rend - d.rpos)); desc_rw[i].pad_ = (uint32_t)eo; }
            eo = __shfl_sync(0xffffffffu, eo, 0);
            for (int32_t c = a + lane; c < b; c += 32) {
                const uint32_t rb = HAS_REF ? ref_nt16_at(v, refc, c) : 0x10u;
                uint32_t xb;
                const uint32_t x = ent_generic(v, cf, d, c, rb, s_tab, xb);
                E2[eo + (uint32_t)(c - d.rpos)] = (uint16_t)x;
                if (!x) atomicAdd(&fail[c], 1u);
                else if (xb) atomicAdd(&extra[c], xb);
            }
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
// Two phases per chunk of 32 reads of the group's slice, with shared memory as the transpose buffer:
//   fetch   LANES ALONG THE READS: each lane brings in the 32 entries of its read that lie over the group -- 64 contiguous
//           bytes of the read's entry string -- with five aligned 16-byte loads (all in flight at once, no dependent chain) and
//           parks them in its row of the warp's buffer; reads that do not reach the group get no row (ballot compaction,
//           file order kept).  A row header carries where column c0's entry sits in the row, which columns the read covers,
//           and its mapq / flags word.
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

constexpr int GROW = 88;                       // bytes per row: 80 fetched + 8 so that 8-byte stores of consecutive lanes hit distinct banks
struct GHdr { uint32_t off, vm, pk; int32_t i; };   // byte offset of column c0's entry in the warp's row buffer, columns covered, qstart|mapq|flags, read index

__device__ __forceinline__ void sts8(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(saddr), "r"(v) : "memory"); }

// what one lane brings in for its read of a chunk: 80 bytes of the read's entry string around column c0 + the row header fields
struct GFetch { uint4 A0, A1, A2, A3, A4; uint32_t vm, pk, o; int32_t i; };

__device__ __forceinline__ GFetch gather_fetch(const MpEntFmt &fmt, const ReadRange &rr, int32_t c0, int32_t t0)
{
    const int lane = threadIdx.x & 31;
    const View &v = fmt.v;
    const uint32_t kSimple = (uint32_t)RD_SIMPLE << 24;
    GFetch f;
    f.A0 = f.A1 = f.A2 = f.A3 = f.A4 = make_uint4(0u, 0u, 0u, 0u);
    f.vm = 0; f.pk = 0; f.o = 0; f.i = 0;
    const int32_t t = t0 + lane;
    if (t < rr.n) {
        f.i = range_at(rr, t);
        const uint4 d = __ldg(reinterpret_cast<const uint4 *>(v.desc + f.i));
        const int32_t rpos = (int32_t)d.x, rend = (int32_t)d.y;
        f.pk = d.w;
        const int32_t lo_c = rpos > c0 ? rpos - c0 : 0, hi_c = rend - c0 < 32 ? rend - c0 : 32;
        if (hi_c > lo_c) {
            f.vm = (hi_c >= 32 ? 0xffffffffu : (1u << hi_c) - 1u) & ~((1u << lo_c) - 1u);
            const uint16_t *src = (f.pk & kSimple) ? fmt.E + (d.z + (f.pk & 0xffffu)) : fmt.E2 + __ldg(&v.desc[f.i].pad_);
            src += c0 - rpos;                                  // entry of column c0 (before the read's first entry when the read starts inside the group)
            const unsigned long long a = (unsigned long long)src;
            const uint4 *q = reinterpret_cast<const uint4 *>(a & ~15ull);
            f.o = (uint32_t)(a & 15ull);                       // bytes between the aligned address and column c0's entry
            f.A0 = __ldg(q); f.A1 = __ldg(q + 1); f.A2 = __ldg(q + 2); f.A3 = __ldg(q + 3); f.A4 = __ldg(q + 4);
        }
    }
    return f;
}

template <bool OUT_MAPQ>
__device__ __forceinline__ void gather_group(const MpEntFmt &fmt, const MpEntFmt *gfmt, int32_t c0, bool on,
                                             uint32_t so, uint32_t qo, uint32_t mo, char *sb, unsigned char *rows, GHdr *hdr)
{
    const uint32_t sb_s = (uint32_t)__cvta_generic_to_shared(sb);
    so += sb_s; qo += sb_s; mo += sb_s;
    const int lane = threadIdx.x & 31;
    const uint32_t lt = (1u << lane) - 1u;
    const int32_t c = c0 + lane;
    const ReadRange rr = read_range(fmt.v, 0, c0 >> 5);            // the same for the 32 lanes
    for (int32_t t0 = 0; t0 < rr.n; t0 += 32) {
        const GFetch f = gather_fetch(fmt, rr, c0, t0);
        // ---- rows of this chunk: lane = read
        const uint32_t live = __ballot_sync(0xffffffffu, f.vm != 0u);
        if (!live) continue;
        __syncwarp();                                              // the previous chunk's rows have been consumed
        if (f.vm) {
            const uint32_t row = (uint32_t)__popc(live & lt);
            uint2 *w = reinterpret_cast<uint2 *>(rows + row * GROW);
            w[0] = make_uint2(f.A0.x, f.A0.y); w[1] = make_uint2(f.A0.z, f.A0.w); w[2] = make_uint2(f.A1.x, f.A1.y); w[3] = make_uint2(f.A1.z, f.A1.w);
            w[4] = make_uint2(f.A2.x, f.A2.y); w[5] = make_uint2(f.A2.z, f.A2.w); w[6] = make_uint2(f.A3.x, f.A3.y); w[7] = make_uint2(f.A3.z, f.A3.w);
            w[8] = make_uint2(f.A4.x, f.A4.y); w[9] = make_uint2(f.A4.z, f.A4.w);
            GHdr h; h.off = row * GROW + f.o; h.vm = f.vm; h.pk = f.pk; h.i = f.i;
            *reinterpret_cast<uint4 *>(hdr + row) = *reinterpret_cast<const uint4 *>(&h);
        }
        __syncwarp();
        // ---- append: lane = column (cursors are 32-bit shared-memory addresses: plain st.shared, no generic-address arithmetic)
        const int nrows = __popc(live);
        if (on) {
            const uint32_t rows_s = (uint32_t)__cvta_generic_to_shared(rows) + 2u * (uint32_t)lane;
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
__global__ void __launch_bounds__(TILE, MIN_CTAS) k_mp_gather(MpEntFmt fmt, const MpEntFmt *gfmt, const uint32_t *len_in, const MpFileSz *st_in, const uint64_t *tile_base,
                                                              char *out, uint32_t smem_cap, int use_tma)
{
    extern __shared__ __align__(16) char s_text[];
    __shared__ uint32_t s_ws[TILE / 32];
    __shared__ __align__(16) unsigned char s_rows[TILE / 32][32 * GROW];
    __shared__ __align__(16) GHdr s_hdr[TILE / 32][32];
    const int32_t ncols = fmt.v.ncols;
    const int32_t c = (int32_t)blockIdx.x * TILE + (int32_t)threadIdx.x;
    MpFileSz stt;
    uint32_t len = 0;
    if (c < ncols) { len = len_in[c]; if (len) stt = st_in[c]; }
    uint32_t total;
    const uint32_t off = block_excl_scan<TILE>(len, s_ws, total);
    if (total == 0) return;
    const uint64_t base = tile_base[blockIdx.x];
    const uint32_t phase = (uint32_t)(base & 15);
    if (total + phase <= smem_cap) {
        char *sb = s_text + phase;
        // every line's fixed parts (header, count, separators, place holders, newline) by the column's own thread ...
        const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const int32_t c0 = (int32_t)(blockIdx.x * TILE + (threadIdx.x & ~31u));
        uint32_t so = 0, qo = 0, mo = 0;
        bool on = false;
        if (len) {
            const EntCur k = ent_layout(fmt.v, fmt.cf, c, stt, sb + off);
            if (k.ps) { on = true; so = (uint32_t)(k.ps - sb); qo = (uint32_t)(k.pq - sb); mo = OUT_MAPQ ? (uint32_t)(k.pm - sb) : 0u; }
        }
        // ... then the entries of the warp's 32 columns
        if (__any_sync(0xffffffffu, on)) gather_group<OUT_MAPQ>(fmt, gfmt, c0, on, so, qo, mo, sb, s_rows[wi], s_hdr[wi]);
        // Each warp stores its own 32 lines (contiguous in the tile) as soon as it has them: no block-wide barrier at the end,
        // so a warp with a deep column does not hold the other three.  Ragged head (to the next 16 B boundary of the
        // destination) and tail by the lanes, the aligned body through one TMA bulk store (shared memory is laid out with the
        // destination's 16-byte phase).
        const uint32_t wbeg = __shfl_sync(0xffffffffu, off, 0);
        const uint32_t wend = __shfl_sync(0xffffffffu, off + len, 31);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // this lane's text bytes -> visible to the bulk-copy engine
        __syncwarp();
        if (wend > wbeg) {
            char *g = out + base;
            const uint32_t wlen = wend - wbeg;
            const uint32_t head = min(wlen, (16u - ((phase + wbeg) & 15u)) & 15u);
            const uint32_t body = (wlen - head) & ~15u;
            const uint32_t tail = wlen - head - body;
            if ((uint32_t)lane < head) g[wbeg + lane] = sb[wbeg + lane];
            if ((uint32_t)lane < tail) g[wbeg + head + body + lane] = sb[wbeg + head + body + lane];
            if (body) {
                if (use_tma) {
                    if (lane == 0) bulk_store_s2g(g + wbeg + head, sb + wbeg + head, body);
                } else {
                    const uint4 *src = reinterpret_cast<const uint4 *>(sb + wbeg + head);
                    uint4 *dst = reinterpret_cast<uint4 *>(g + wbeg + head);
                    for (uint32_t i = lane; i < body / 16; i += 32) dst[i] = src[i];
                }
            }
        }
    } else if (len) {
        mp_line_write_ent(gfmt->v, gfmt->cf, c, stt, out + base + off, gfmt->E, gfmt->E2);   // very deep tile: format straight into HBM
    }
}
