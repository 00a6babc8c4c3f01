// mpileup_ss.cuh -- order-free line sizing for the standard single-file mpileup line.
//
// The byte length of a pileup line does not depend on the order of the reads in the column,
// only on sums: n_plp (reads over the column), cnt (entries with base quality >= -Q) and the
// extra bytes of special entries ("^"+mapq at a read's first column, "$" at its last, indel
// text).  So the size pass can be read-major with no ordering constraint at all:
//   k_mp_entries (mpileup_ent.cuh) one warp per 32 reads, lanes over their bases: a coverage difference array gets
//                +1/-1 per read, only FAILING bases and special entries touch per-column counters (sparse atomics)
//   k_mp_place   one pass over the sums: prefix sum of the difference array -> n_plp per column, the line length of every
//                column (plp_core.h mp_sums_line_size), and the byte offset of every 128-column tile of the gather; both
//                prefixes cross blocks through the look-back of scan.cuh
// The gather re-derives each column's length and state from the same three sums, so no per-column line state is stored.
// Equivalent to mp_line_size (the general path); `test_c2_size_properties` checks that both paths agree.
#pragma once

// Sizes and places the gather's tiles.  A block owns PLACE_COLS consecutive columns (PLACE_COLS / TILE tiles).  It is bound by
// the latency of its round trips (ticket, loads, two look-backs), not by bandwidth, so what sets its speed is how many
// columns an SM holds in flight: the block's diff / fail / extra go into shared memory with cp.async (24 KB per block, not
// 24 registers per thread), eight blocks of 2048 columns per SM.  Then PLACE_ROUNDS rounds of 256 consecutive columns, one
// column per thread (conflict-free 4-byte shared-memory loads); the block's warp segments of 32 columns are in column order
// at index round * 8 + warp, so one warp scans them for the block.  Blocks are ticketed: the predecessors a look-back waits
// on have started.  Two look-backs: the coverage difference total (st_cov; mod-2^32 as ScanSum in scan.cuh, since partial
// sums of the difference array can be negative) gives n_plp, the byte total (st_len) the tile offsets.  Outputs: nplp[c] for
// c < ncols, col_off[t] for every tile t < nt, and col_off[nt], the text length, from the block that owns the last tile.
// The three input arrays must be readable up to column ncols + 2 (they are: the entry pass writes diff[ncols]).
constexpr int PLACE_ROUNDS = 8, PLACE_COLS = 256 * PLACE_ROUNDS;
__global__ void __launch_bounds__(256) k_mp_place(View v, MpConf cf, const int32_t *diff, const uint32_t *fail, const uint32_t *extra,
                                                  int32_t *nplp, uint64_t *col_off, int32_t nt, uint64_t *st_cov, uint64_t *st_len, uint32_t *ticket)
{
    constexpr int R = PLACE_ROUNDS, NSEG = R * 8, NTILE = PLACE_COLS / TILE, SEG_PER_TILE = TILE / 32;
    static_assert(NSEG == 64 && NTILE <= 32, "warp 0 takes two segments per lane and at most one tile per lane");
    __shared__ __align__(16) uint32_t s_in[3][PLACE_COLS];     // diff, fail, extra of the block's columns
    __shared__ uint32_t s_cov[NSEG];                            // per warp segment: coverage sum, then its exclusive prefix
    __shared__ uint32_t s_len[NSEG];                            // per warp segment: text bytes
    __shared__ int s_blk;
    if (threadIdx.x == 0) s_blk = (int)atomicAdd(ticket, 1u);
    __syncthreads();
    const int t = s_blk;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int32_t ncols = v.ncols;
    const int32_t cblk = t * PLACE_COLS;
    // ---- stage the inputs: 16-byte copies, zero-filled from the first one that starts at or past ncols
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const uint32_t *src = a == 0 ? reinterpret_cast<const uint32_t *>(diff) : a == 1 ? fail : extra;
#pragma unroll
        for (int j = 0; j < PLACE_COLS / 4 / 256; ++j) {
            const int q = 4 * ((int)threadIdx.x + 256 * j);
            const bool live = cblk + q < ncols;
            const uint32_t sa = (uint32_t)__cvta_generic_to_shared(&s_in[a][q]);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(sa), "l"(live ? src + cblk + q : src), "r"(live ? 16u : 0u) : "memory");
        }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    // ---- coverage: inclusive scan within each warp segment, then the segments (warp 0) and the look-back
    uint32_t x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int k = 256 * r + (int)threadIdx.x;
        x[r] = cblk + k < ncols ? s_in[0][k] : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x[r], o); if (lane >= o) x[r] += y; }
        if (lane == 31) s_cov[r * 8 + w] = x[r];
    }
    __syncthreads();
    if (w == 0) {                                               // lane l: segments 2l, 2l + 1
        const uint32_t a = s_cov[2 * lane], b = s_cov[2 * lane + 1], pair = a + b;
        uint32_t s = pair;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
        const uint32_t base = (uint32_t)lookback<ScanSum>(st_cov, t, (uint64_t)__shfl_sync(0xffffffffu, s, 31));
        const uint32_t e = base + s - pair;
        s_cov[2 * lane] = e; s_cov[2 * lane + 1] = e + a;
    }
    __syncthreads();
    // ---- line lengths (0 beyond ncols), summed per warp segment
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int k = 256 * r + (int)threadIdx.x;
        const int32_t c = cblk + k;
        uint32_t len = 0;
        if (c < ncols) {
            const int32_t np = (int32_t)(s_cov[r * 8 + w] + x[r]);
            MpFileSz s;
            len = mp_sums_line_size(v, cf, c, np, s_in[1][k], s_in[2][k], &s);
            nplp[c] = np;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) len += __shfl_xor_sync(0xffffffffu, len, o);
        if (lane == 0) s_len[r * 8 + w] = len;
    }
    __syncthreads();
    // ---- bytes: lane l < NTILE sums tile l of the block (segments 4l .. 4l+3); 64-bit prefix over the tiles, then the look-back
    if (w == 0) {
        uint64_t tl = 0;
        if (lane < NTILE) {
#pragma unroll
            for (int k = 0; k < SEG_PER_TILE; ++k) tl += s_len[SEG_PER_TILE * lane + k];
        }
        uint64_t s = tl;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
        const uint64_t total = __shfl_sync(0xffffffffu, s, 31);
        const uint64_t base = lookback<ScanSum>(st_len, t, total);
        const int32_t tile0 = t * NTILE, tile = tile0 + lane;
        if (lane < NTILE && tile < nt) col_off[tile] = base + s - tl;
        if (lane == 0 && tile0 <= nt - 1 && nt - 1 < tile0 + NTILE) col_off[nt] = base + total;
    }
}
