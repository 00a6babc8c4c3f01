// mpileup_ss.cuh -- order-free line sizing for the standard single-file mpileup line.
//
// The byte length of a pileup line does not depend on the order of the reads in the column,
// only on sums: n_plp (reads over the column), cnt (entries with base quality >= -Q) and the
// extra bytes of special entries ("^"+mapq at a read's first column, "$" at its last, indel
// text).  So the size pass can be read-major with no ordering constraint at all:
//   k_mp_entries (mpileup_ent.cuh) one warp per 32 reads, lanes over their bases: a coverage difference array gets
//                +1/-1 per read, only FAILING bases and special entries touch per-column counters (sparse atomics)
//   k_ss_scan    prefix sum of the difference array -> n_plp per column
//   k_ss_cols    per column: MpFileSz and line length from the sums (plp_core.h mp_sums_line_size),
//                128-column tile totals (what the write kernel and the offset scan consume)
// Equivalent to mp_line_size (the general path); `test_c2_size_properties` checks that both paths agree.
#pragma once

// inclusive prefix sum of int32 (coverage), single pass with decoupled look-back
__global__ void k_ss_scan(const int32_t *in, int32_t *out, int32_t n, uint64_t *st, uint32_t *ticket)
{
    constexpr int T = 256, IPT = 4;
    __shared__ uint32_t s_ws[T / 32];
    __shared__ int s_tile; __shared__ uint64_t s_base;
    if (threadIdx.x == 0) s_tile = (int)atomicAdd(ticket, 1u);
    __syncthreads();
    const int t = s_tile;
    const int32_t i0 = (t * T + (int32_t)threadIdx.x) * IPT;
    int32_t x[IPT]; uint32_t sum = 0;
#pragma unroll
    for (int j = 0; j < IPT; ++j) { x[j] = i0 + j < n ? in[i0 + j] : 0; sum += (uint32_t)x[j]; x[j] = (int32_t)sum; }   // mod-2^32 arithmetic: partial sums may be negative
    uint32_t total;
    const uint32_t off = block_excl_scan<T>(sum, s_ws, total);
    if (threadIdx.x < 32) { const uint64_t b = lookback_sum(st, t, (uint64_t)total); if (threadIdx.x == 0) s_base = b; }
    __syncthreads();
    const uint32_t base = (uint32_t)s_base + off;
#pragma unroll
    for (int j = 0; j < IPT; ++j) if (i0 + j < n) out[i0 + j] = (int32_t)(base + (uint32_t)x[j]);
}

__global__ void __launch_bounds__(TILE) k_ss_cols(View v, MpConf cf, const int32_t *nplp, const uint32_t *fail, const uint32_t *extra,
                                                  uint32_t *len_out, MpFileSz *fsz, uint32_t *tile_total)
{
    __shared__ uint32_t s_ws[TILE / 32];
    const int32_t c = (int32_t)blockIdx.x * TILE + (int32_t)threadIdx.x;
    uint32_t len = 0;
    if (c < v.ncols) {
        len = mp_sums_line_size(v, cf, c, nplp[c], fail[c], extra[c], fsz + c);
        len_out[c] = len;
    }
    uint32_t x = len;
#pragma unroll
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) s_ws[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t t = 0; for (int k = 0; k < TILE / 32; ++k) t += s_ws[k]; tile_total[blockIdx.x] = t; }
}
