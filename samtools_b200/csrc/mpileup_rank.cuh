// mpileup_rank.cuh -- per-column rank sums of the mpileup column stage (b200_mpileup_ranksums).  Included by engine.cu.
//
// The Mann-Whitney U of BQ, MQ and the BP-5 (capped at RS_POS_CAP), ref-class entries against alt-class ones, and its tie
// term, per column and file (plp_core.h mp_entry_rank, rank_from_hist): RS_PLANES int64 planes out[f][plane][c].  Every
// size -- shared memory, buffers, grids -- is known on the host before the first launch, whatever the depth of a column or
// the length of its reads, and the call synchronises with the host once, at the end.
//   1. k_rank_counts: the walk of k_mp_counts (mp_col_planes, a fourth instance) counts each column's class entries into
//      planes 0-1 and stores planes 2-7 as zeros, so no memset precedes it.  A (file, column) whose two classes both have
//      entries is active (act[f * ncols + c] = 1); a column of the window with more class entries than rank_depth_over
//      allows raises `deep`.  launch_scan and k_rank_list compact the active pairs into a list; its length stays in HBM.
//   2. k_rank_hist: a fixed grid of warps loops over the list.  Each warp owns a ref and an alt histogram of RS_BINS uint32
//      in shared memory (9.5 KB).  Its lanes walk the group's reads (lanes along the reads), skip those that do not cover
//      the column, resolve it, apply -Q and add the class entry's three bins with shared-memory atomics.  Then, per value, a
//      warp prefix of the ref counts over runs of bins lets every lane run rank_from_hist on its run; lane 0 stores the
//      warp's sums of U2 and T into planes 2-7.
constexpr int RS_WARPS = 4;
constexpr int RS_BLOCKS_PER_SM = 5;   // 5 x 38.8 KB of histograms per SM

__global__ void __launch_bounds__(CNT_WARPS * 32) k_rank_counts(View v, int32_t min_baseQ, int32_t n_groups, int64_t *out,
                                                                uint32_t *act, unsigned long long *deep)
{
    __shared__ int64_t s_rc[CNT_WARPS][RS_PLANES][32];
    mp_col_planes<int64_t, RS_PLANES>(v, min_baseQ, n_groups, out, s_rc,
        [&](int64_t (*s)[32], int lane, const ReadDesc &d, const Ent &e, int32_t c, int q) {
            const int cls = mp_entry_rank(v, d, e, c, q).cls;
            if (cls != RS_NONE) ++s[RS_NREF + cls - RS_REF][lane];
        },
        [&](int64_t (*s)[32], int lane, int32_t c, uint32_t) {
            if (c >= v.ncols) return;
            const int f = (int)(((int64_t)blockIdx.x * CNT_WARPS + (threadIdx.x >> 5)) / n_groups);
            const int64_t nr = s[RS_NREF][lane], na = s[RS_NALT][lane];
            act[(int64_t)f * v.ncols + c] = (nr > 0 && na > 0) ? 1u : 0u;
            if (rank_depth_over((uint64_t)(nr + na))) *deep = 1ull;
        });
}

// list[off[i]] = i for every active pair i (off: the exclusive scan of act)
__global__ void k_rank_list(const uint32_t *act, const uint32_t *off, int64_t n, int32_t *list)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && act[i]) list[off[i]] = (int32_t)i;
}

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t x)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// list[0, *n_list): active pairs f * ncols + c; out: the planes, 0-1 written by k_rank_counts
__global__ void __launch_bounds__(RS_WARPS * 32) k_rank_hist(View v, int32_t min_baseQ, const int32_t *list, const uint32_t *n_list,
                                                             int64_t *out)
{
    __shared__ uint32_t s_h[RS_WARPS][2][RS_BINS];
    const int lane = threadIdx.x & 31;
    uint32_t (*h)[RS_BINS] = s_h[threadIdx.x >> 5];          // h[0]: ref, h[1]: alt
    const int64_t n = *n_list, stride = (int64_t)gridDim.x * RS_WARPS;
    for (int64_t j = (int64_t)blockIdx.x * RS_WARPS + (threadIdx.x >> 5); j < n; j += stride) {
        const int32_t p = list[j];
        const int f = p / v.ncols;
        const int32_t c = p - f * v.ncols;
        for (int b = lane; b < RS_BINS; b += 32) { h[0][b] = 0; h[1][b] = 0; }
        __syncwarp();
        const ReadRange rr = read_range(v, f, c >> 5);
        for (int32_t t = lane; t < rr.n; t += 32) {
            const ReadDesc d = load_desc(v.desc + range_at(rr, t));
            if ((uint32_t)(c - d.rpos) >= (uint32_t)(d.rend - d.rpos)) continue;
            Ent e;
            resolve(v, d, c, e);
            const int q = ent_qual(v, d, e);
            if (q < min_baseQ) continue;
            const EntRank r = mp_entry_rank(v, d, e, c, q);
            if (r.cls == RS_NONE) continue;
            uint32_t *hc = h[r.cls - RS_REF];
            atomicAdd(&hc[r.bin[0]], 1u); atomicAdd(&hc[r.bin[1]], 1u); atomicAdd(&hc[r.bin[2]], 1u);
        }
        __syncwarp();
        int64_t *o = out + ((int64_t)f * RS_PLANES + RS_U2) * v.ncols + c;
#pragma unroll
        for (int var = 0; var < 3; ++var) {
            const int nb = rs_nbins(var), per = (nb + 31) / 32;
            const int lo = min(nb, lane * per), hi = min(nb, lo + per);
            const uint32_t *ref = h[0] + var * RS_QBINS, *alt = h[1] + var * RS_QBINS;
            uint32_t r = 0;
            for (int b = lo; b < hi; ++b) r += ref[b];
            uint32_t x = r;                                   // inclusive warp prefix of the runs' ref counts
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, s); if (lane >= s) x += y; }
            uint64_t u2 = 0, tt = 0;
            rank_from_hist(ref + lo, alt + lo, hi - lo, u2, tt, x - r);
            u2 = warp_sum_u64(u2); tt = warp_sum_u64(tt);
            if (lane == 0) { o[(int64_t)(2 * var) * v.ncols] = (int64_t)u2; o[(int64_t)(2 * var + 1) * v.ncols] = (int64_t)tt; }
        }
        __syncwarp();                                         // the next pair zeroes the histograms
    }
}
