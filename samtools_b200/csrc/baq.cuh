// baq.cuh -- per-base alignment quality on the device.
//
// Replaces htslib sam_prob_realn (realn.c) + probaln_glocal (probaln.c) as
// called at bam_plcmd.c:451 with flag 3 (APPLY|EXTEND) or 7 (-E, recompute).
// Semantics: SURVEY.md section 8a rows a2/a3, Appendix A6.
//
// Bit-exactness rules this kernel obeys:
//   * IEEE double, every product/sum in the association order of the C source;
//     this translation unit is compiled with -fmad=false (no FMA contraction,
//     the reference is a plain x86-64 -O2 build, Makefile:29);
//   * the within-row D-state recurrence and every row sum are evaluated
//     sequentially in k, exactly like the scalar loop;
//   * pow(10,-q/10) comes from a host table (libm), rounded to float per base
//     like the reference's `float qual[]`;
//   * (int)(-4.343*log(1-max)+.499) is not evaluated with a device log: the
//     host pre-computes, with its own libm, the 101 break points of that
//     monotone step function and the device counts how many it passes.
//
// Mapping: one warp per read.  Lanes own the cells of the band (2*bw+1 = 15 by
// default) for the parallel M/I terms; the sequential D chain and the ordered
// row sums run as a lane-uniform loop over a per-warp shared-memory copy of the row.  The forward matrix
// lives in an HBM slab per resident warp (L2-resident); backward keeps two rows.
#pragma once
#include "baq_reg.h"

struct BaqPlan { int64_t xb; int32_t l_ref, bw; };

#define BAQ_EI .25
#define BAQ_EM .33333333333

__device__ __forceinline__ int ref_code(const RawSoA &r, int64_t p)
{
    const int64_t i = p - r.ref_beg;
    const char ch = (i >= 0 && i < r.ref_n) ? r.ref[i] : 'N';
    return nt16_int_of(nt16_of((unsigned char)ch));
}

// which reads need the HMM, their reference window and band (sam_prob_realn prologue)
constexpr int BAQR_MAX_LQ = 512;     // longest read the register-band kernel takes (its slab grows with the longest read)

__global__ void k_baq_plan(RawSoA r, b200_stage_conf_t cf, const uint8_t *state, BaqPlan *plan, int32_t *idx, int32_t *idx2, int use_reg,
                           unsigned long long *counters /* [0]=count, [1]=max slab doubles, [2]=max lq, [3]=count2, [4]=max lq of list 2 */)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    if (state[i] != ST_ALIVE) return;
    if (r.rbits && (r.rbits[i] & B200_RB_BAQ_DONE)) return;
    const int lq = r.l_qseq[i];
    const uint8_t *qual = r.qual + r.qual_off[i];
    if ((r.flag[i] & 4) || lq == 0 || qual[0] == 0xff) return;
    const uint32_t *cg = r.cigar + r.cigar_off[i];
    int64_t x = r.pos[i], xb = -1, xe = -1;
    int y = 0, yb = -1, ye = -1;
    for (int k = 0; k < (int)r.n_cigar[i]; ++k) {
        const int op = cg[k] & 0xf, l = (int)(cg[k] >> 4);
        if (is_mop(op)) { if (yb < 0) yb = y; if (xb < 0) xb = x; ye = y + l; xe = x + l; x += l; y += l; }
        else if (op == OP_S || op == OP_I) y += l;
        else if (op == OP_D) x += l;
        else if (op == OP_N) return;
    }
    if (xb == -1) return;
    int bw = 7;
    int64_t dd = (xe - xb) - (ye - yb); if (dd < 0) dd = -dd;
    if (dd > bw) bw = (int)dd + 3;
    const int cbw = bw;
    xb -= yb + bw / 2; if (xb < 0) xb = 0;
    xe += lq - ye + bw / 2;
    if (xe - xb - lq > bw) { xb += (xe - xb - lq - bw) / 2; xe -= (xe - xb - lq - bw) / 2; }
    if (xe > r.ref_len) xe = r.ref_len;   // "i >= ref_len" truncation of the translated reference
    const int64_t l_ref = xe - xb;
    if (l_ref <= 0) return;               // probaln_glocal returns before touching anything
    // probaln_glocal band
    int b2 = (int)(l_ref > lq ? l_ref : lq);
    if (b2 > cbw) b2 = cbw;
    int64_t d2 = l_ref - lq; if (d2 < 0) d2 = -d2;
    if (b2 < d2) b2 = (int)d2;
    BaqPlan p; p.xb = xb; p.l_ref = (int32_t)l_ref; p.bw = b2;
    plan[i] = p;
    if (use_reg && b2 == baqr::BW && lq <= BAQR_MAX_LQ) {     // band 7 (every read whose aligned spans differ by <= 7): one thread per read, k_baq_reg
        const unsigned long long slot2 = atomicAdd(&counters[3], 1ULL);
        idx2[slot2] = (int32_t)i;
        atomicMax(&counters[4], (unsigned long long)lq);
        return;
    }
    const unsigned long long slot = atomicAdd(&counters[0], 1ULL);
    idx[slot] = (int32_t)i;
    const unsigned long long stride = (unsigned long long)(2 * b2 + 1) * 3 + 6;
    const unsigned long long slab = (unsigned long long)(lq + 1) * stride + 2 * stride + (unsigned long long)lq + 2 + (unsigned long long)lq + 8;
    atomicMax(&counters[1], slab);
    atomicMax(&counters[2], (unsigned long long)lq);
}

__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

__device__ __forceinline__ double emis(int rc, int qc, double ql)
{
    return (rc > 3 || qc > 3) ? 1. : (rc == qc ? 1. - ql : ql * BAQ_EM);
}

__global__ void __launch_bounds__(128) k_baq(RawSoA r, const BaqPlan *plan, const int32_t *idx, int64_t n_idx, double *slabs,
                                             unsigned long long slab_doubles, const double *q2p, const double *qthr,
                                             unsigned long long *work, int extend)
{
    // per-warp exchange rows: the ordered (sequential-in-k) parts read the band cells of the row from
    // shared memory (broadcast loads that pipeline) instead of one shuffle round trip per cell
    __shared__ double s_x[4][2][32];
    double (*sx)[32] = s_x[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    double *slab = slabs + (size_t)gw * slab_doubles;
    for (;;) {
        unsigned long long wi = 0;
        if (lane == 0) wi = atomicAdd(work, 1ULL);
        wi = __shfl_sync(0xffffffffu, wi, 0);
        if ((int64_t)wi >= n_idx) return;
        const int64_t ri = idx[wi];
        const BaqPlan pl = plan[ri];
        const int lq = r.l_qseq[ri], l_ref = pl.l_ref, bw = pl.bw, bw2 = bw * 2 + 1;
        const int stride = bw2 * 3 + 6;
        uint8_t *qual = r.qual + r.qual_off[ri];
        const uint64_t qoff = r.qual_off[ri];
        double *F = slab;                                   // (lq+1) rows
        double *Bb = F + (size_t)(lq + 1) * stride;         // 2 rows
        double *S = Bb + 2 * (size_t)stride;                // lq+2
        int32_t *stv = (int32_t *)(S + lq + 2);             // lq ints  (fits: lq+8 doubles reserved)
        // transitions
        const double cd = 0.001, ce = 0.1;
        const double sM = 1. / (2 * lq + 2), sI = sM;
        double m[9];
        m[0] = (1 - cd - cd) * (1 - sM); m[1] = m[2] = cd * (1 - sM);
        m[3] = (1 - ce) * (1 - sI); m[4] = ce * (1 - sI); m[5] = 0.;
        m[6] = 1 - ce; m[7] = 0.; m[8] = ce;
        const double bM = (1 - cd) / l_ref, bI = cd / l_ref;
        const double EIm1 = BAQ_EI * m[1], EIm4 = BAQ_EI * m[4];
        if (lane == 0) S[0] = 1.;
        // ---------------- forward, row 1
        {
            double *fi = F + stride;
            const int beg = 1, end = l_ref < bw + 1 ? l_ref : bw + 1;
            const int qc = nt16_int_of(base4(r.seq4, qoff, 0));
            const double ql = (double)(float)q2p[qual[0]];
            double sum = 0.;
            for (int kb = beg; kb <= end; kb += 32) {
                const int k = kb + lane; const bool act = k <= end;
                double M = 0., I = 0.;
                if (act) { M = emis(ref_code(r, pl.xb + k - 1), qc, ql) * bM; I = BAQ_EI * bI; }
                const int cnt = min(32, end - kb + 1);
                sx[0][lane] = M; sx[1][lane] = I; __syncwarp();
                for (int j = 0; j < cnt; ++j) sum += sx[0][j] + sx[1][j];
                __syncwarp();
                if (act) { const int u = (k + 1) * 3; fi[u] = M; fi[u + 1] = I; fi[u + 2] = 0.; }
            }
            __syncwarp();
            if (lane == 0) S[1] = sum;
            for (int kb = beg; kb <= end; kb += 32) {
                const int k = kb + lane;
                if (k <= end) { const int u = (k + 1) * 3; fi[u] /= sum; fi[u + 1] /= sum; fi[u + 2] /= sum; }
            }
            __syncwarp();
        }
        // ---------------- forward, rows 2..lq
        for (int i = 2; i <= lq; ++i) {
            double *fi = F + (size_t)i * stride; const double *f1 = F + (size_t)(i - 1) * stride;
            const int x = i - bw > 0 ? i - bw : 0, x1 = i - 1 - bw > 0 ? i - 1 - bw : 0;
            const int beg = i - bw > 1 ? i - bw : 1, end = i + bw < l_ref ? i + bw : l_ref;
            const int beg1 = i - 1 - bw > 1 ? i - 1 - bw : 1, end1 = (i - 1 + bw < l_ref ? i - 1 + bw : l_ref);
            const int end1r = (i - 1 == 1) ? (l_ref < bw + 1 ? l_ref : bw + 1) : end1;   // row 1 has its own band end
            const int qc = nt16_int_of(base4(r.seq4, qoff, i - 1));
            const double ql = (double)(float)q2p[qual[i - 1]];
            double sum = 0., Dc = 0., tc = m[2] * 0.;
            for (int kb = beg; kb <= end; kb += 32) {
                const int k = kb + lane; const bool act = k <= end;
                double M = 0., I = 0.;
                if (act) {
                    double a0 = 0., a1 = 0., a2 = 0., c0 = 0., c1 = 0.;
                    if (k - 1 >= beg1 && k - 1 <= end1r) { const int v = (k - 1 - x1 + 1) * 3; a0 = f1[v]; a1 = f1[v + 1]; a2 = f1[v + 2]; }
                    if (k >= beg1 && k <= end1r) { const int v = (k - x1 + 1) * 3; c0 = f1[v]; c1 = f1[v + 1]; }
                    const double e = emis(ref_code(r, pl.xb + k - 1), qc, ql);
                    M = e * (m[0] * a0 + m[3] * a1 + m[6] * a2);
                    I = BAQ_EI * (m[1] * c0 + m[4] * c1);
                }
                const int cnt = min(32, end - kb + 1);
                double myD = 0.;
                sx[0][lane] = M; sx[1][lane] = I; __syncwarp();
                for (int j = 0; j < cnt; ++j) {
                    const double Mj = sx[0][j], Ij = sx[1][j];
                    const double Dj = tc + m[8] * Dc;
                    sum += Mj + Ij + Dj;
                    if (lane == j) myD = Dj;
                    tc = m[2] * Mj; Dc = Dj;
                }
                __syncwarp();
                if (act) { const int u = (k - x + 1) * 3; fi[u] = M; fi[u + 1] = I; fi[u + 2] = myD; }
            }
            __syncwarp();
            if (lane == 0) S[i] = sum;
            const double inv = 1. / sum;
            for (int kb = beg; kb <= end; kb += 32) {
                const int k = kb + lane;
                if (k <= end) { const int u = (k - x + 1) * 3; fi[u] *= inv; fi[u + 1] *= inv; fi[u + 2] *= inv; }
            }
            __syncwarp();
        }
        // band of row lq (row 1 is special)
        const int xl = lq - bw > 0 ? lq - bw : 0;
        const int begl = lq - bw > 1 ? lq - bw : 1;
        const int endl = (lq == 1) ? (l_ref < bw + 1 ? l_ref : bw + 1) : (lq + bw < l_ref ? lq + bw : l_ref);
        // ---------------- termination
        double s_last;
        {
            const double *fl = F + (size_t)lq * stride;
            double sum = 0.;
            for (int kb = begl; kb <= endl; kb += 32) {
                const int k = kb + lane;
                double t = 0.;
                if (k <= endl) { const int u = (k - xl + 1) * 3; t = fl[u] * sM + fl[u + 1] * sI; }
                const int cnt = min(32, endl - kb + 1);
                sx[0][lane] = t; __syncwarp();
                for (int j = 0; j < cnt; ++j) sum += sx[0][j];
                __syncwarp();
            }
            s_last = sum;
            if (lane == 0) S[lq + 1] = sum;
        }
        __syncwarp();
        // ---------------- backward + MAP, row lq first
        double *bcur = Bb, *bnext = Bb + stride;
        {
            const double s_lq = S[lq];
            for (int kb = begl; kb <= endl; kb += 32) {
                const int k = kb + lane;
                if (k <= endl) { const int u = (k - xl + 1) * 3; bcur[u] = sM / s_lq / s_last; bcur[u + 1] = sI / s_lq / s_last; bcur[u + 2] = 0.; }
            }
        }
        __syncwarp();
        for (int i = lq; i >= 1; --i) {
            const int x = i - bw > 0 ? i - bw : 0;
            const int beg = i - bw > 1 ? i - bw : 1;
            const int end = (i == 1) ? (l_ref < bw + 1 ? l_ref : bw + 1) : (i + bw < l_ref ? i + bw : l_ref);
            if (i < lq) {
                // bnext holds row i+1 (scaled); compute row i into bcur
                const int x1 = i + 1 - bw > 0 ? i + 1 - bw : 0;
                const int beg1 = i + 1 - bw > 1 ? i + 1 - bw : 1, end1 = i + 1 + bw < l_ref ? i + 1 + bw : l_ref;
                // rows 2..lq-1 use the general band; row 1 computed here uses the GENERAL band too in the reference
                const int bbeg = i - bw > 1 ? i - bw : 1, bend = i + bw < l_ref ? i + bw : l_ref;
                const double y = (i > 1) ? 1. : 0.;
                const int qc = nt16_int_of(base4(r.seq4, qoff, i));
                const double ql = (double)(float)q2p[qual[i]];
                double Dn = 0.;   // bi[(i,k+1)+2]; zero beyond the band end
                // descending k, chunks of 32 from the top
                for (int kt = bend; kt >= bbeg; kt -= 32) {
                    const int k = kt - lane; const bool act = k >= bbeg;
                    double e = 0., p0 = 0., p1 = 0.;
                    if (act) {
                        double b11 = 0., b10 = 0.;
                        if (k + 1 >= beg1 && k + 1 <= end1) b11 = bnext[(k + 1 - x1 + 1) * 3];
                        if (k >= beg1 && k <= end1) b10 = bnext[(k - x1 + 1) * 3 + 1];
                        e = (k >= l_ref ? 0. : emis(ref_code(r, pl.xb + k), qc, ql)) * b11;
                        p0 = e * m[0] + EIm1 * b10;
                        p1 = e * m[3] + EIm4 * b10;
                    }
                    const int cnt = min(32, kt - bbeg + 1);
                    double myD = 0., myDn = 0.;
                    sx[0][lane] = e; __syncwarp();
                    for (int j = 0; j < cnt; ++j) {
                        const double ej = sx[0][j];
                        const double Dj = (ej * m[6] + m[8] * Dn) * y;
                        if (lane == j) { myD = Dj; myDn = Dn; }
                        Dn = Dj;
                    }
                    __syncwarp();
                    if (act) { const int u = (k - x + 1) * 3; bcur[u] = p0 + m[2] * myDn; bcur[u + 1] = p1; bcur[u + 2] = myD; }
                }
                __syncwarp();
                const double inv = 1. / S[i];
                for (int kb = bbeg; kb <= bend; kb += 32) {
                    const int k = kb + lane;
                    if (k <= bend) { const int u = (k - x + 1) * 3; bcur[u] *= inv; bcur[u + 1] *= inv; bcur[u + 2] *= inv; }
                }
                __syncwarp();
            }
            // MAP for row i over the general band (probaln.c MAP loop)
            {
                const int mbeg = i - bw > 1 ? i - bw : 1, mend = i + bw < l_ref ? i + bw : l_ref;
                const double *fi = F + (size_t)i * stride;
                double sum = 0., mx = 0.; int max_k = -1;
                for (int kb = mbeg; kb <= mend; kb += 32) {
                    const int k = kb + lane;
                    double z0 = 0., z1 = 0.;
                    if (k <= mend) {
                        const int u = (k - x + 1) * 3;
                        // cells outside the band actually written for this row read as zero
                        const bool inF = k >= beg && k <= end;
                        const bool inB = (i == lq) ? (k >= begl && k <= endl) : true;
                        const double f0 = inF ? fi[u] : 0., f1v = inF ? fi[u + 1] : 0.;
                        const double b0 = inB ? bcur[u] : 0., b1 = inB ? bcur[u + 1] : 0.;
                        z0 = f0 * b0; z1 = f1v * b1;
                    }
                    const int cnt = min(32, mend - kb + 1);
                    sx[0][lane] = z0; sx[1][lane] = z1; __syncwarp();
                    for (int j = 0; j < cnt; ++j) {
                        const double a = sx[0][j], b = sx[1][j];
                        if (a > mx) { mx = a; max_k = (kb + j - 1) << 2 | 0; }
                        sum += a;
                        if (b > mx) { mx = b; max_k = (kb + j - 1) << 2 | 1; }
                        sum += b;
                    }
                    __syncwarp();
                }
                if (lane == 0) {
                    mx /= sum;
                    stv[i - 1] = max_k;
                    const double xx = 1. - mx;
                    int kq;
                    if (!(xx > 0.)) kq = 0;            // log(0) / NaN: x86 cvttsd2si gives INT_MIN, stored as uint8 0
                    else {
                        int lo_ = 0, hi_ = 101;        // count thresholds T[1..101] with xx <= T[j]
                        while (lo_ < hi_) { const int mid = (lo_ + hi_ + 1) >> 1; if (xx <= qthr[mid]) lo_ = mid; else hi_ = mid - 1; }
                        kq = lo_ > 100 ? 99 : lo_;
                    }
                    ((uint8_t *)(stv + lq))[i - 1] = (uint8_t)kq;
                }
            }
            __syncwarp();
            double *t = bcur; bcur = bnext; bnext = t;   // row i becomes "next"
        }
        __syncwarp();
        // ---------------- BAQ from the MAP path (sam_prob_realn epilogue, EXTEND+APPLY)
        if (lane == 0) {
            const uint8_t *qv = (const uint8_t *)(stv + lq);
            uint8_t *bq = (uint8_t *)(stv + lq) + lq;       // lq bytes
            uint8_t *left = bq + lq, *rght = left + lq;      // 2*lq bytes (slab reserves them)
            for (int j = 0; j < lq; ++j) bq[j] = qual[j];
            const uint32_t *cg = r.cigar + r.cigar_off[ri];
            int64_t x = r.pos[ri]; int y = 0;
            for (int k = 0; k < (int)r.n_cigar[ri]; ++k) {
                const int op = cg[k] & 0xf; int l = (int)(cg[k] >> 4);
                if (is_mop(op)) {
                    if (l > lq - y) l = lq - y;
                    if (l > 0) {
                        for (int j = y; j < y + l; ++j)
                            bq[j] = ((stv[j] & 3) != 0 || (int64_t)(stv[j] >> 2) != x - pl.xb + (j - y)) ? 0 : qv[j];
                        if (extend) {
                            left[y] = bq[y];
                            for (int j = y + 1; j < y + l; ++j) left[j] = bq[j] > left[j - 1] ? bq[j] : left[j - 1];
                            rght[y + l - 1] = bq[y + l - 1];
                            for (int j = y + l - 2; j >= y; --j) rght[j] = bq[j] > rght[j + 1] ? bq[j] : rght[j + 1];
                            for (int j = y; j < y + l; ++j) bq[j] = left[j] < rght[j] ? left[j] : rght[j];
                        }
                    }
                    x += l; y += l;
                } else if (op == OP_S || op == OP_I) { if (l > lq - y) l = lq - y; y += l; }
                else if (op == OP_D) x += l;
            }
            for (int j = 0; j < lq; ++j) {
                const int adj = qual[j] <= bq[j] ? 0 : qual[j] - bq[j];   // bq' = 64 + adj ; qual -= bq' - 64
                qual[j] = (uint8_t)(qual[j] - adj);
            }
        }
        __syncwarp();
    }
}


// ---------------------------------------------------------------------------------------------
// Register-band BAQ (baq_reg.h): one thread per read of band 7, the band row in registers.  Per row a thread
// writes the scaled forward M/I states (15 x 16 B) and the row's 1/s (8 B) into its lane's column of the warp's
// slab -- slot s of row i of lane l lives at ((i-1)*16 + s)*32 + l (16-byte units), so a warp store is one
// contiguous 512-byte request -- and reads them back once, in reverse, through cp.async into a double-buffered
// per-thread shared-memory stage one row ahead of the MAP step that consumes them.
struct BaqDevMem {
    double2 *rows;             // this lane's slot 0 of row 1
    int32_t *words;            // this lane's per-base scratch word 0
    double2 *stage;            // this thread's slot 0 of stage buffer 0 (shared memory)
    const uint8_t *refc; int64_t ref_lo, ref_n;
    __device__ __forceinline__ int ref_code(int p) const { const int64_t a = ref_lo + p; return (a >= 0 && a < ref_n) ? (int)(refc[a] >> 4) : 4; }
    // codes of window positions p..p+7, one per byte (the high nibble of the staged code bytes); 4 outside the staged sequence
    __device__ __forceinline__ uint64_t ref8(int p) const
    {
        const int64_t a = ref_lo + p;
        if (a >= 0 && a + 8 <= ref_n) return (baqr::ld8(refc + a) >> 4) & 0x0f0f0f0f0f0f0f0full;
        uint64_t w = 0;
        for (int k = 0; k < 8; ++k) w |= (uint64_t)((a + k >= 0 && a + k < ref_n) ? (refc[a + k] >> 4) : 4) << (8 * k);
        return w;
    }
    __device__ __forceinline__ size_t row_of(int i) const { return (size_t)(i - 1) * (16 * 32); }
    __device__ __forceinline__ void put_row(int i, const double (&M)[baqr::NB], const double (&I)[baqr::NB], double inv)
    {
        double2 *r = rows + row_of(i);
#pragma unroll
        for (int j = 0; j < baqr::NB; ++j) r[j * 32] = make_double2(M[j], I[j]);
        reinterpret_cast<double *>(r + 15 * 32)[0] = inv;
    }
    __device__ __forceinline__ void fence() { __threadfence_block(); }
    __device__ __forceinline__ void fetch(int i)
    {
        const double2 *r = rows + row_of(i);
        const uint32_t s = (uint32_t)__cvta_generic_to_shared(stage + (i & 1) * (16 * 128));
#pragma unroll
        for (int k = 0; k < 16; ++k)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s + k * (128 * 16)), "l"(r + k * 32) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    __device__ __forceinline__ void wait(int pending)
    {
        if (pending) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __device__ __forceinline__ void get(int i, int j, double &a, double &b) const { const double2 v = stage[((i & 1) * 16 + j) * 128]; a = v.x; b = v.y; }
    __device__ __forceinline__ double inv(int i) const { return stage[((i & 1) * 16 + 15) * 128].x; }
    __device__ __forceinline__ void put_word(int j, int32_t w) { words[(size_t)j * 32] = w; }
    __device__ __forceinline__ int32_t get_word(int j) const { return words[(size_t)j * 32]; }
};

// reference bases -> codes, once per staged reference: low nibble = 4-bit IUPAC code (what pileup_seq compares a
// read base with), high nibble = 0..3 / 4 (ambiguous) (what the BAQ HMM compares)
__global__ void k_ref_codes(const char *ref, int64_t n, uint8_t *codes)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const int c16 = nt16_of((unsigned char)ref[i]); codes[i] = (uint8_t)(c16 | nt16_int_of(c16) << 4); }
}

constexpr int BAQR_THREADS = 128;
constexpr int BAQR_STAGE_BYTES = 2 * 16 * BAQR_THREADS * 16;

__global__ void __launch_bounds__(BAQR_THREADS, 3) k_baq_reg(RawSoA r, const BaqPlan *plan, const int32_t *idx, int64_t n_idx, double2 *slabs,
                                                             unsigned long long slab_units, int lqmax, const uint8_t *refc,
                                                             const double *q2p, const double *qthr, int extend)
{
    extern __shared__ __align__(16) unsigned char s_dyn[];
    __shared__ double s_q2pf[256];
    __shared__ double s_qthr[102];
    for (int t = threadIdx.x; t < 256; t += BAQR_THREADS) s_q2pf[t] = (double)(float)q2p[t];
    for (int t = threadIdx.x; t < 102; t += BAQR_THREADS) s_qthr[t] = qthr[t];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_thr = (int64_t)gridDim.x * blockDim.x;
    BaqDevMem mem;
    mem.rows = slabs + (size_t)gw * slab_units + lane;
    mem.words = reinterpret_cast<int32_t *>(slabs + (size_t)gw * slab_units + (size_t)lqmax * (16 * 32)) + lane;
    mem.stage = reinterpret_cast<double2 *>(s_dyn) + threadIdx.x;
    mem.refc = refc; mem.ref_n = r.ref_n;
    for (int64_t wi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; wi < n_idx; wi += n_thr) {
        const int64_t ri = idx[wi];
        const BaqPlan pl = plan[ri];
        mem.ref_lo = pl.xb - r.ref_beg;
        baqr::baq_read(mem, r.qual + r.qual_off[ri], r.seq4, (uint32_t)r.qual_off[ri], r.l_qseq[ri], pl.l_ref, r.pos[ri], pl.xb,
                       r.cigar + r.cigar_off[ri], (int)r.n_cigar[ri], s_q2pf, s_qthr, extend != 0);
    }
}

// host: tables with the box's own libm (what the reference binary would use here)
static void baq_host_tables(double *q2p, double *qthr) { baqr::host_tables(q2p, qthr); }

int launch_baq(b200_engine *e, const RawSoA &r, const b200_stage_conf_t &cf)
{
    const int64_t n = r.n;
    if (!e->d_q2p) {
        double q2p[256], qthr[102];
        baq_host_tables(q2p, qthr);
        CK(cudaMalloc((void **)&e->d_q2p, sizeof q2p)); CK(cudaMalloc((void **)&e->d_qthr, sizeof qthr));
        CK(cudaMemcpyAsync(e->d_q2p, q2p, sizeof q2p, cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->d_qthr, qthr, sizeof qthr, cudaMemcpyHostToDevice, e->stream));
        CK(cudaStreamSynchronize(e->stream));
    }
    // plan array + two index lists share one buffer
    size_t plan_bytes = (size_t)(n + 1) * sizeof(BaqPlan);
    const int64_t nr = (n + 1 + 3) & ~3LL;
    if (ensure(e, e->baq_idx, e->cap_baq_idx, (size_t)(2 * nr) + plan_bytes / 4 + 4)) return -1;
    int32_t *idx = e->baq_idx, *idx2 = e->baq_idx + nr;
    BaqPlan *plan = (BaqPlan *)(e->baq_idx + 2 * nr);
    // band-7 reads run on the register kernel (k_baq_reg), everything else (wide bands, very long reads) on the warp kernel;
    // B200_BAQ_REG=0 (read per handle when it is created) sends every read to the warp kernel (cross-check)
    CK(cudaMemsetAsync(e->d_misc + MISC_BAQ, 0, 16 * 8, e->stream));
    k_baq_plan<<<nblk(n, 256), 256, 0, e->stream>>>(r, cf, e->state, plan, idx, idx2, e->baq_reg, e->d_misc + MISC_BAQ); e->launches++;
    unsigned long long h[5];
    CK(cudaMemcpyAsync(h, e->d_misc + MISC_BAQ, sizeof h, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaGetLastError());
    const int64_t n_idx = (int64_t)h[0], n_idx2 = (int64_t)h[3];
    if (n_idx2 > 0) {   // band 7: one thread per read, band row in registers
        const int lqmax = (int)h[4];
        // per warp: lqmax rows of 16 slots x 32 lanes x 16 B, then one scratch word per base and lane
        const unsigned long long slab_units = (unsigned long long)lqmax * (16 * 32) + ((unsigned long long)lqmax * 32 * 4 + 15) / 16 + 32;
        int64_t warps = (int64_t)e->n_sm * 3 * (BAQR_THREADS / 32);
        const int64_t cap = (int64_t)((24ULL << 30) / (slab_units * 16));
        if (warps > cap) warps = cap;
        if (warps > (n_idx2 + 31) / 32) warps = (n_idx2 + 31) / 32;
        if (warps < 1) warps = 1;
        const int blocks = (int)((warps + BAQR_THREADS / 32 - 1) / (BAQR_THREADS / 32));
        warps = (int64_t)blocks * (BAQR_THREADS / 32);
        if (ensure(e, e->baq_f, e->cap_baq_f, (size_t)warps * slab_units * 2)) return -1;
        // per device (function attributes are), so once per engine handle -- not once per process: a second GPU's handle needs it too
        if (!e->baq_attr_set) { CK(cudaFuncSetAttribute(k_baq_reg, cudaFuncAttributeMaxDynamicSharedMemorySize, BAQR_STAGE_BYTES)); e->baq_attr_set = true; }
        k_baq_reg<<<blocks, BAQR_THREADS, BAQR_STAGE_BYTES, e->stream>>>(r, plan, idx2, n_idx2, (double2 *)e->baq_f, slab_units, lqmax, e->ref_codes, e->d_q2p, e->d_qthr, cf.baq != 3); e->launches++;
        CK(cudaGetLastError());
    }
    if (n_idx > 0) {    // wide bands / long reads: one warp per read
        const unsigned long long slab = h[1] + 2 * h[2] / 8 + 8;   // + left/right byte rows
        int64_t warps = (int64_t)e->n_sm * 12 * 4;
        const int64_t cap = (int64_t)((6ULL << 30) / (slab * 8));
        if (warps > cap) warps = cap;
        if (warps > n_idx) warps = n_idx;
        if (warps < 1) warps = 1;
        const int blocks = (int)((warps + 3) / 4);
        warps = (int64_t)blocks * 4;
        if (n_idx2 > 0) CK(cudaStreamSynchronize(e->stream));   // the slab buffer is shared by the two kernels
        if (ensure(e, e->baq_f, e->cap_baq_f, (size_t)warps * slab)) return -1;
        k_baq<<<blocks, 128, 0, e->stream>>>(r, plan, idx, n_idx, e->baq_f, slab, e->d_q2p, e->d_qthr, e->d_misc + MISC_BAQ + 11, cf.baq != 3); e->launches++;
    }
    CK(cudaGetLastError());
    return 0;
}
