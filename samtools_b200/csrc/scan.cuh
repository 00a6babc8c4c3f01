// scan.cuh -- single-pass prefix scans with decoupled look-back: the status words, the warp look-back, the block scan and
// the one scan kernel every stage launches.
//
// A block publishes one 64-bit status word: flag (bits 62-63: 0 nothing yet, 1 the block's aggregate, 2 its inclusive
// prefix) and a 62-bit value.  Blocks take their index from a ticket, so the predecessors a look-back waits on have started.
#pragma once

// status words are self-contained (flag + value in one 64-bit word), so polling
// needs no acquire: relaxed gpu-scope accesses go to L2 and, unlike ld.acquire,
// do not invalidate the SM's L1 (CCTL.IVALL) under the feet of the other warps.
__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t *p)
{
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(uint64_t *p, uint64_t v)
{
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
#define ST_FLAG(w) ((w) >> 62)
#define ST_VAL(w) ((w) & 0x3fffffffffffffffULL)

// The combine ops.  Each has the identity 0 in the look-back's 62-bit value field and gives the scan kernel:
//   V, id   the type of the values a block scans and its identity;
//   excl    a lane's exclusive prefix in the block from its warp's prefix `base`, its inclusive prefix x in the warp and its
//           value v (a sum takes v back off, with no shuffle: that keeps k_mp_gather at its registers and spills; a max
//           takes the left lane's x);
//   agg     a block aggregate as a look-back value;
//   out     a block's exclusive prefix P from the look-back combined with a value inside the block.
//   ScanSum  sums of u32 values, mod 2^32 inside a block; the block totals are carried in 64 bits across blocks.
//            Exclusive scans need each block's sum below 2^32 (their totals may pass it); an int32 output of an inclusive
//            scan takes the sum mod 2^32, so partial sums of a +1 / -1 difference array may be negative.
//   ScanMax  max over int32 with INT32_MIN as the empty value; the look-back holds the values biased by -INT32_MIN.
struct ScanSum {
    typedef uint32_t V;
    static constexpr V id = 0;
    template <class X> __device__ __forceinline__ static X op(X a, X b) { return a + b; }
    __device__ __forceinline__ static V excl(V base, V x, V v, int lane) { return base + x - v; }
    __device__ __forceinline__ static uint64_t agg(V v) { return v; }
    __device__ __forceinline__ static uint64_t out(uint64_t p, V v) { return p + v; }
};
struct ScanMax {
    typedef int32_t V;
    static constexpr V id = INT32_MIN;
    template <class X> __device__ __forceinline__ static X op(X a, X b) { return a > b ? a : b; }
    __device__ __forceinline__ static V excl(V base, V x, V v, int lane) { const V l = __shfl_up_sync(0xffffffffu, x, 1); return lane ? op(base, l) : base; }
    __device__ __forceinline__ static uint64_t agg(V v) { return (uint64_t)((int64_t)v - INT32_MIN); }
    __device__ __forceinline__ static int64_t out(uint64_t p, V v) { return max((int64_t)p + INT32_MIN, (int64_t)v); }
};

// decoupled look-back, executed by ONE FULL WARP: 32 predecessors are inspected
// per round.  Publishes block t's aggregate `agg`, then its inclusive prefix;
// returns the exclusive prefix of block t (all lanes; 0 for block 0).
template <class Op>
__device__ uint64_t lookback(uint64_t *st, int t, uint64_t agg)
{
    const int lane = threadIdx.x & 31;
    if (t == 0) { if (lane == 0) st_relaxed_u64(&st[0], (2ULL << 62) | agg); return 0; }
    if (lane == 0) st_relaxed_u64(&st[t], (1ULL << 62) | agg);
    uint64_t excl = 0;
    for (int base = t - 1;; base -= 32) {
        const int j = base - lane;
        uint64_t w;
        unsigned m2, need;
        for (;;) {
            w = j >= 0 ? ld_relaxed_u64(&st[j]) : (2ULL << 62);      // before block 0: inclusive prefix 0
            m2 = __ballot_sync(0xffffffffu, ST_FLAG(w) == 2);
            need = m2 ? ((2u << (__ffs(m2) - 1)) - 1u) : 0xffffffffu;  // lanes up to the nearest inclusive prefix
            if ((__ballot_sync(0xffffffffu, ST_FLAG(w) == 0) & need) == 0) break;
            __nanosleep(40);
        }
        uint64_t x = ((need >> lane) & 1u) ? ST_VAL(w) : 0;
#pragma unroll
        for (int o = 16; o; o >>= 1) x = Op::op(x, __shfl_xor_sync(0xffffffffu, x, o));
        excl = Op::op(excl, x);
        if (m2) break;
    }
    if (lane == 0) st_relaxed_u64(&st[t], (2ULL << 62) | Op::op(excl, agg));
    return excl;
}

// exclusive scan of one value per thread over a block of T threads (Op::id for thread 0); `total` gets the block's
// aggregate.  Must be called by every thread of the block.
template <int T, class Op>
__device__ __forceinline__ typename Op::V block_excl_scan(typename Op::V v, typename Op::V *warp_sums, typename Op::V &total)
{
    typedef typename Op::V V;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    V x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const V y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x = Op::op(x, y); }
    if (lane == 31) warp_sums[w] = x;
    __syncthreads();
    if (w == 0) {
        V s = lane < T / 32 ? warp_sums[lane] : Op::id;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const V y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s = Op::op(s, y); }
        if (lane < T / 32) warp_sums[lane] = s;
    }
    __syncthreads();
    total = warp_sums[T / 32 - 1];
    const V base = w ? warp_sums[w - 1] : Op::id;
    return Op::excl(base, x, v, lane);
}

// Single-pass scan of in[0, n) into out[]: each of SCAN_T threads takes IPT consecutive items, blocks are ticketed.
// INCL: out[i] = in[0] op ... op in[i].  Otherwise exclusive (out[0] = the identity) with the total in out[n].
// `st` (one status word per block) and `*ticket` must be zero at launch; n + SCAN_T * IPT must fit an int32.
constexpr int SCAN_T = 256;
template <class Op, int IPT, bool INCL, class In, class Out>
__global__ void __launch_bounds__(SCAN_T) k_scan(const In *in, Out *out, int32_t n, uint64_t *st, uint32_t *ticket)
{
    typedef typename Op::V V;
    __shared__ V s_ws[SCAN_T / 32];
    __shared__ int s_blk; __shared__ uint64_t s_base;
    if (threadIdx.x == 0) s_blk = (int)atomicAdd(ticket, 1u);
    __syncthreads();
    const int t = s_blk;
    const int32_t i0 = (t * SCAN_T + (int32_t)threadIdx.x) * IPT;
    V x[IPT], acc = Op::id;                                 // x[j]: inclusive prefix of the thread's items 0..j
#pragma unroll
    for (int j = 0; j < IPT; ++j) { acc = Op::op(acc, i0 + j < n ? (V)in[i0 + j] : Op::id); x[j] = acc; }
    V total;
    const V off = block_excl_scan<SCAN_T, Op>(acc, s_ws, total);
    if (threadIdx.x < 32) { const uint64_t b = lookback<Op>(st, t, Op::agg(total)); if (threadIdx.x == 0) s_base = b; }
    __syncthreads();
    const uint64_t p = s_base;
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
        if (i0 + j >= n) break;
        const V prev = INCL ? x[j] : j ? x[j - 1] : Op::id;
        out[i0 + j] = (Out)Op::out(p, Op::op(off, prev));
        if (!INCL && i0 + j == n - 1) out[n] = (Out)Op::out(p, Op::op(off, x[j]));
    }
}
