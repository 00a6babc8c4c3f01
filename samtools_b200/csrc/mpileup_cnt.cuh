// mpileup_cnt.cuh -- per-column planes of the mpileup column stage: base and indel counts (b200_mpileup_counts), quality
// sums (b200_mpileup_qsums) and read-position sums (b200_mpileup_psums).  Included by engine.cu.
//
// What a parser of the "--reverse-del" text would count, or add up from its "-s" or "--output-BP-5" text, kept as numbers
// in HBM: per file CNT_PLANES (plp_core.h mp_entry_channel) or QS_PLANES (mp_entry_qs) planes of uint32, or PS_PLANES
// (mp_entry_ps) planes of int64, out[f][plane][c] over the columns [0, ncols) of the window.
//
// One warp per (file, 32-column group), lane = column: the warp walks the group's reads (read_range, far-reaching reads
// included) and every lane loads the same descriptor (a broadcast).  A simple read resolves by arithmetic, so the lanes'
// quality and base loads are consecutive bytes / nibbles of one read; other reads go through the CIGAR cursor.  The
// counters live in shared memory, [plane][lane] per warp: each lane owns one column of every plane (no atomics, no bank
// conflicts), and a plane index never selects a register (local memory, DESIGN section 7).  The planes leave as coalesced
// 128-byte rows (256-byte rows of int64).  The kernels run the one walk mp_col_planes; they differ in what an entry that passes -Q adds (`add`)
// and in what the lane does at the end of its column c with the column's n_plp (`fin`).
constexpr int CNT_WARPS = 4;

template <class T, int P, class Add, class Fin>
__device__ __forceinline__ void mp_col_planes(const View &v, int32_t min_baseQ, int32_t n_groups, T *out, T (*s_all)[P][32],
                                              Add add, Fin fin)
{
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int64_t w = (int64_t)blockIdx.x * CNT_WARPS + wl;
    if (w >= (int64_t)n_groups * v.n_files) return;        // whole warps: nothing below synchronises across warps
    const int f = (int)(w / n_groups), g = (int)(w % n_groups);
    T (*s)[32] = s_all[wl];
    for (int k = 0; k < P; ++k) s[k][lane] = 0;
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
        const int q = ent_qual(v, d, e);
        if (q < min_baseQ) continue;
        add(s, lane, d, e, c, q);
    }
    fin(s, lane, c, nplp);
    if (c >= v.ncols) return;
    T *p = out + (int64_t)f * P * v.ncols + c;
#pragma unroll
    for (int k = 0; k < P; ++k) p[(int64_t)k * v.ncols] = s[k][lane];
}

__global__ void __launch_bounds__(CNT_WARPS * 32) k_mp_counts(View v, int32_t min_baseQ, int32_t n_groups, uint32_t *out)
{
    __shared__ uint32_t s_cnt[CNT_WARPS][CNT_PLANES][32];
    mp_col_planes<uint32_t, CNT_PLANES>(v, min_baseQ, n_groups, out, s_cnt,
        [&](uint32_t (*s)[32], int lane, const ReadDesc &d, const Ent &e, int32_t c, int) {
            const int x = mp_entry_channel(v, d, v.cigar + d.cig_off, e, c);
            const int o = (d.fl & RD_REV) ? CNT_REV : 0;
            ++s[o + (x & 15)][lane];
            if (x & CNT_BIT_INS) ++s[o + CNT_INS_NEXT][lane];
            if (x & CNT_BIT_DEL) ++s[o + CNT_DEL_NEXT][lane];
        },
        [&](uint32_t (*s)[32], int lane, int32_t, uint32_t nplp) { s[CNT_NPLP][lane] = nplp; });
}

// deep: set where a column has more than QS_MAX_DEPTH reads (a sum could wrap); the call then fails
__global__ void __launch_bounds__(CNT_WARPS * 32) k_mp_qsums(View v, int32_t min_baseQ, int32_t n_groups, uint32_t *out,
                                                             unsigned long long *deep)
{
    __shared__ uint32_t s_qs[CNT_WARPS][QS_PLANES][32];
    mp_col_planes<uint32_t, QS_PLANES>(v, min_baseQ, n_groups, out, s_qs,
        [&](uint32_t (*s)[32], int lane, const ReadDesc &d, const Ent &e, int32_t c, int q) {
            const EntQs x = mp_entry_qs(q, d);
            const int k = ((d.fl & RD_REV) ? QS_REV : 0) + (mp_entry_channel(v, d, v.cigar + d.cig_off, e, c) & 15);
            s[k][lane] += x.bq;
            s[QS_MQ + k][lane] += x.mq;
            s[QS_MQ0 + k][lane] += x.mq0;
        },
        [&](uint32_t (*)[32], int, int32_t, uint32_t nplp) { if (nplp > QS_MAX_DEPTH) *deep = 1ull; });
}

// ovf: set where a sum of squares of a column of the window would exceed INT64_MAX (plp_core.h ps_sq_over; a lane past the
// window's last column walks reads too, but its cells are not stored); the call then fails.  The int64 cells make 28 KB of
// shared memory per block.
__global__ void __launch_bounds__(CNT_WARPS * 32) k_mp_psums(View v, int32_t min_baseQ, int32_t n_groups, int64_t *out,
                                                             unsigned long long *ovf)
{
    __shared__ int64_t s_ps[CNT_WARPS][PS_PLANES][32];
    bool over = false;
    mp_col_planes<int64_t, PS_PLANES>(v, min_baseQ, n_groups, out, s_ps,
        [&](int64_t (*s)[32], int lane, const ReadDesc &d, const Ent &e, int32_t c, int) {
            const EntPs x = mp_entry_ps(d, e);
            const int k = ((d.fl & RD_REV) ? PS_REV : 0) + (mp_entry_channel(v, d, v.cigar + d.cig_off, e, c) & 15);
            s[k][lane] += x.bp5;
            const uint64_t old = (uint64_t)s[PS_SQ + k][lane];
            over |= ps_sq_over(old, x.sq);
            s[PS_SQ + k][lane] = (int64_t)(old + x.sq);
        },
        [&](int64_t (*)[32], int, int32_t c, uint32_t) { if (over && c < v.ncols) *ovf = 1ull; });
}
