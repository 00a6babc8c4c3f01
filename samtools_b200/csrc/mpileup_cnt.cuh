// mpileup_cnt.cuh -- per-column base and indel counts of the mpileup column stage (b200_mpileup_counts).
// Included by engine.cu.
//
// What a parser of the "--reverse-del" text would count, kept as numbers in HBM: per file CNT_PLANES planes of uint32
// (plp_core.h mp_entry_channel), out[f][plane][c] over the columns [0, ncols) of the window.
//
// One warp per (file, 32-column group), lane = column: the warp walks the group's reads (read_range, far-reaching reads
// included) and every lane loads the same descriptor (a broadcast).  A simple read resolves by arithmetic, so the lanes'
// quality and base loads are consecutive bytes / nibbles of one read; other reads go through the CIGAR cursor.  The
// counters live in shared memory, [plane][lane] per warp: each lane owns one column of every plane (no atomics, no bank
// conflicts), and a plane index never selects a register (local memory, DESIGN section 7).  The planes leave as coalesced
// 128-byte rows.
constexpr int CNT_WARPS = 4;

__global__ void __launch_bounds__(CNT_WARPS * 32) k_mp_counts(View v, int32_t min_baseQ, int32_t n_groups, uint32_t *out)
{
    __shared__ uint32_t s_cnt[CNT_WARPS][CNT_PLANES][32];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int64_t w = (int64_t)blockIdx.x * CNT_WARPS + wl;
    if (w >= (int64_t)n_groups * v.n_files) return;        // whole warps: nothing below synchronises across warps
    const int f = (int)(w / n_groups), g = (int)(w % n_groups);
    uint32_t (*s)[32] = s_cnt[wl];
    for (int k = 0; k < CNT_PLANES; ++k) s[k][lane] = 0;
    const int32_t c = g * 32 + lane;
    const ReadRange rr = read_range(v, f, g);
    uint32_t nplp = 0;
    for (int32_t t = 0; t < rr.n; ++t) {
        const int32_t i = range_at(rr, t);
        const ReadDesc d = load_desc(v.desc + i);
        if ((uint32_t)(c - d.rpos) >= (uint32_t)(d.rend - d.rpos)) continue;
        ++nplp;
        Ent e;
        resolve(v, d, c, e);
        if (ent_qual(v, d, e) < min_baseQ) continue;
        const int x = mp_entry_channel(v, d, v.cigar + d.cig_off, e, c);
        const int o = (d.fl & RD_REV) ? CNT_REV : 0;
        ++s[o + (x & 15)][lane];
        if (x & CNT_BIT_INS) ++s[o + CNT_INS_NEXT][lane];
        if (x & CNT_BIT_DEL) ++s[o + CNT_DEL_NEXT][lane];
    }
    s[CNT_NPLP][lane] = nplp;
    if (c >= v.ncols) return;
    uint32_t *p = out + (int64_t)f * CNT_PLANES * v.ncols + c;
#pragma unroll
    for (int k = 0; k < CNT_PLANES; ++k) p[(int64_t)k * v.ncols] = s[k][lane];
}
