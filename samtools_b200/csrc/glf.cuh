// glf.cuh -- genotype likelihoods per column on the device.
//
// Replaces bcf_call_glfgen (bam2bcf.c:65-123: per-read filter, quality caps,
// packing q<<5|strand<<4|base, qsum) and htslib errmod_cal / errmod_init
// (errmod.c; tables fk, beta, lhet; ks_shuffle over hts_drand48 when a column
// holds more than 255 usable bases; ascending sort consumed from the top).
// Semantics: SURVEY.md section 8a rows a16/a17.  One warp per (column, file).
// No reference test pins these numbers ("parity unpinned"); parity is against
// the CPU oracle's restatement.
#pragma once
#include <math.h>

#define GL_CAP 4096   // usable bases per (column,file) kept in shared memory

__device__ __forceinline__ uint64_t lcg_jump(uint64_t s, uint64_t k)
{
    // s_{n+1} = A*s_n + C (mod 2^48); advance k steps by repeated squaring
    uint64_t A = 0x5DEECE66DULL, C = 0xBULL, accA = 1, accC = 0;
    const uint64_t M = 0xffffffffffffULL;
    while (k) {
        if (k & 1) { accC = (accC * A + C) & M; accA = (accA * A) & M; }
        C = ((A + 1) * C) & M; A = (A * A) & M;
        k >>= 1;
    }
    return (accA * s + accC) & M;
}

// pass 1: usable bases per (column,file) -> random draws ks_shuffle will consume
// one read of a column -> packed code q<<5 | strand<<4 | base (bam2bcf.c:88-112): q = base quality (0 past the read's
// end), b4 = 4-bit base or -1 past the end, capQ = bca->capQ (60)
__device__ __forceinline__ bool gl_pack(int q, int mapq, int b4, int rev, int rb4, int min_baseQ, int capQ, uint16_t &code, int &qv, int &bv)
{
    if (q < min_baseQ) return false;
    int mapQ = mapq < 255 ? mapq : 20;
    if (q > 99) q = 99;
    if (mapQ > capQ) mapQ = capQ;
    if (q > mapQ) q = mapQ;
    if (q > 63) q = 63;
    if (q < 4) q = 4;
    const int b = b4 >= 0 ? nt16_int_of(b4 ? b4 : rb4) : 4;
    code = (uint16_t)(q << 5 | (rev ? 1 : 0) << 4 | b);
    qv = q; bv = b;
    return true;
}
__device__ __forceinline__ bool gl_code(const View &v, const ReadDesc &d, int32_t c, int min_baseQ, int rb4, uint16_t &code, int &qv, int &bv)
{
    Ent e; resolve(v, d, c, e);
    if (e.is_del || e.is_refskip) return false;
    const bool in = e.qpos < d.l_qseq;
    const int q = in ? (int)v.qual[d.qoff + (uint64_t)e.qpos] : 0;
    return gl_pack(q, d.mapq, in ? base4(v.seq4, d.qoff, e.qpos) : -1, (d.fl & RD_REV) != 0, rb4, min_baseQ, 60, code, qv, bv);
}

// errmod_cal (htslib errmod.c) by ONE WARP on n packed codes in shared memory bs[] (room for max(n, 256) entries):
// n > 255 -> ks_shuffle with the drand48 state `rng` (advanced by n-1 draws) and keep 255; ascending sort; accumulate
// from the top; q[m*m] written by lane 0.  m <= 16 alleles (samtools uses 5, phase / targetcut 4).
__device__ void errmod_cal_warp(uint16_t *bs, int n, int m, uint64_t *rng, const double *fk, const double *beta, const double *lhet, float *q)
{
    const int lane = threadIdx.x & 31;
    if (n == 0) {                                   // errmod_cal: "if (n == 0) return 0" with q cleared
        for (int i = lane; i < m * m; i += 32) q[i] = 0.f;
        __syncwarp();
        return;
    }
    if (n > 255) {
        if (lane == 0) {
            uint64_t s = *rng;
            for (int i = n; i > 1; --i) {
                s = (s * 0x5DEECE66DULL + 0xBULL) & 0xffffffffffffULL;
                const int j = (int)(((double)s / 281474976710656.0) * i);
                const uint16_t t = bs[j]; bs[j] = bs[i - 1]; bs[i - 1] = t;
            }
            *rng = s;
        }
        n = 255;
        __syncwarp();
    }
    // ascending sort of n <= 255 codes: pad to 256 and bitonic-sort in shared memory
    for (int i = n + lane; i < 256; i += 32) bs[i] = 0xffff;
    __syncwarp();
    for (int k = 2; k <= 256; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = lane; t < 256; t += 32) {
                const int p = t ^ j;
                if (p > t) {
                    const uint16_t a = bs[t], b = bs[p];
                    const bool up = (t & k) == 0;
                    if ((a > b) == up) { bs[t] = b; bs[p] = a; }
                }
            }
            __syncwarp();
        }
    if (lane == 0) {
        double fsum[16], bsum[16];
        int cc[16], w[32];
        for (int i = 0; i < 16; ++i) { fsum[i] = 0.; bsum[i] = 0.; cc[i] = 0; }
        for (int i = 0; i < 32; ++i) w[i] = 0;
        for (int j = n - 1; j >= 0; --j) {
            const uint16_t b = bs[j];
            int qual = (b >> 5) < 4 ? 4 : (b >> 5);
            if (qual > 63) qual = 63;
            const int basestrand = b & 0x1f, base = b & 0xf;
            const double fkw = fk[w[basestrand]];
            fsum[base] += fkw;
            bsum[base] += fkw * beta[qual << 16 | n << 8 | cc[base]];
            ++cc[base]; ++w[basestrand];
        }
        for (int i = 0; i < m * m; ++i) q[i] = 0.f;
        for (int j = 0; j < m; ++j) {
            float tmp1 = 0.f; int tmp2 = 0;
            for (int k = 0; k < m; ++k) { if (k == j) continue; tmp1 = (float)((double)tmp1 + bsum[k]); tmp2 += cc[k]; }
            if (tmp2) q[j * m + j] = tmp1;
            for (int k = j + 1; k < m; ++k) {
                const int cjk = cc[j] + cc[k];
                tmp1 = 0.f; tmp2 = 0;
                for (int i = 0; i < m; ++i) { if (i == j || i == k) continue; tmp1 = (float)((double)tmp1 + bsum[i]); tmp2 += cc[i]; }
                const float val = tmp2 ? (float)(-4.343 * lhet[cjk << 8 | cc[k]] + (double)tmp1) : (float)(-4.343 * lhet[cjk << 8 | cc[k]]);
                q[j * m + k] = q[k * m + j] = val;
            }
            for (int k = 0; k < m; ++k) if (q[j * m + k] < 0.0f) q[j * m + k] = 0.0f;
        }
    }
    __syncwarp();
}

__global__ void k_gl_count(View v, int min_baseQ, uint32_t *draws, int32_t *nplp_any)
{
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)v.ncols * v.n_files) return;
    const int32_t c = (int32_t)(idx / v.n_files); const int f = (int)(idx % v.n_files);
    const int g = c >> 5;
    const ReadRange rr = read_range(v, f, g);
    int rb4 = 15;
    { const char rc = ref_char(v, c); rb4 = (v.ref && (int64_t)c < v.ref_len_rel) ? nt16_of((unsigned char)rc) : 15; }
    uint32_t n = 0, np = 0;
    for (int32_t t_ = 0; t_ < rr.n; ++t_) {
        const ReadDesc d = v.desc[range_at(rr, t_)];
        if (c < d.rpos || c >= d.rend) continue;
        ++np;
        uint16_t code; int q, b;
        if (gl_code(v, d, c, min_baseQ, rb4, code, q, b)) ++n;
    }
    draws[idx] = n > 255 ? n - 1 : 0;
    if (np) atomicOr(&nplp_any[c], 1);
}

__global__ void __launch_bounds__(128) k_gl(View v, int min_baseQ, const uint64_t *draw_off, uint64_t rng_base_draws,
                                             const double *fk, const double *beta, const double *lhet,
                                             int32_t *out_n, float *out_qp /* 29 floats */, uint32_t *overflow)
{
    __shared__ uint16_t s_b[4][GL_CAP];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int64_t idx = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (idx >= (int64_t)v.ncols * v.n_files) return;
    const int32_t c = (int32_t)(idx / v.n_files); const int f = (int)(idx % v.n_files);
    const int g = c >> 5;
    const ReadRange rr = read_range(v, f, g);
    uint16_t *bs = s_b[wl];
    int rb4;
    { const char rc = ref_char(v, c); rb4 = (v.ref && (int64_t)c < v.ref_len_rel) ? nt16_of((unsigned char)rc) : 15; }
    int n = 0, nplp = 0;
    float qsum[4] = {0, 0, 0, 0};   // exact small integers, order-independent below 2^24
    for (int32_t base = 0; base < rr.n; base += 32) {
        const int32_t t_ = base + lane;
        bool ok = false, cov = false; uint16_t code = 0; int q = 0, b = 4;
        if (t_ < rr.n) {
            const ReadDesc d = v.desc[range_at(rr, t_)];
            if (c >= d.rpos && c < d.rend) { cov = true; ok = gl_code(v, d, c, min_baseQ, rb4, code, q, b); }
        }
        const unsigned mk = __ballot_sync(0xffffffffu, ok);
        nplp += __popc(__ballot_sync(0xffffffffu, cov));
        if (ok) { const int slot = n + __popc(mk & ((1u << lane) - 1)); if (slot < GL_CAP) bs[slot] = code; }
        n += __popc(mk);
#pragma unroll
        for (int bb = 0; bb < 4; ++bb) {
            float x = (ok && b == bb) ? (float)q : 0.f;
            for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            qsum[bb] += x;
        }
    }
    __syncwarp();
    float *o = out_qp + idx * 29;
    if (nplp == 0) { if (lane == 0) out_n[idx] = -1; if (lane < 29) o[lane] = 0.f; return; }
    if (n > GL_CAP) { if (lane == 0) atomicOr(overflow, 1u); n = GL_CAP; }
    const int n_used = n;
    uint64_t rng = 0;
    if (n > 255 && lane == 0) rng = lcg_jump(0x330EULL, rng_base_draws + draw_off[idx]);   // the process-wide drand48 stream at this column
    __shared__ float s_q[4][25];
    errmod_cal_warp(bs, n, 5, &rng, fk, beta, lhet, s_q[wl]);
    if (lane == 0) {
        out_n[idx] = n_used;
        for (int i = 0; i < 4; ++i) o[i] = qsum[i];
        for (int i = 0; i < 25; ++i) o[4 + i] = s_q[wl][i];
    }
}

// errmod_init(depcorr = 1 - 0.83) tables, built once with the host libm (long double exp/log as upstream)
static void errmod_host_tables(std::vector<double> &fk, std::vector<double> &beta, std::vector<double> &lhet)
{
    const double depcorr = 1. - 0.83, eta = 0.03;
    fk.assign(256, 0.); beta.assign((size_t)256 * 256 * 64, 0.); lhet.assign(256 * 256, 0.);
    fk[0] = 1.0;
    for (int n = 1; n < 256; ++n) fk[n] = pow(1. - depcorr, n) * (1.0 - eta) + eta;
    std::vector<double> lC(256 * 256, 0.);
    for (int n = 1; n != 256; ++n) {
        const double lgn = lgamma(n + 1);
        for (int k = 1; k <= n; ++k) lC[n << 8 | k] = lgn - lgamma(k + 1) - lgamma(n - k + 1);
    }
    for (int q = 1; q != 64; ++q) {
        const double e = pow(10.0, -q / 10.0), le = log(e), le1 = log(1.0 - e);
        for (int n = 1; n <= 255; ++n) {
            // binomial tail ratio in LOG space with long double accumulators (htslib errmod.c cal_coef); in plain space the
            // running sums underflow to 0/0 for the deep k of a high-quality column (n = 167, q = 40, k >= 100)
            double *b = beta.data() + (q << 16 | n << 8);
            long double sum, sum1;
            sum1 = lC[n << 8 | n] + n * le;
            b[n] = HUGE_VAL;
            for (int k = n - 1; k >= 0; --k, sum1 = sum) {
                sum = sum1 + log1pl(expl(lC[n << 8 | k] + k * le + (n - k) * le1 - sum1));
                b[k] = -10. / M_LN10 * (double)(sum1 - sum);
            }
        }
    }
    for (int n = 0; n < 256; ++n)
        for (int k = 0; k < 256; ++k) lhet[n << 8 | k] = lC[n << 8 | k] - M_LN2 * n;
}

static int errmod_tables(b200_engine *e, double depcorr);

extern "C" int b200_glf(b200_engine_t *e, int32_t min_baseQ, int64_t *n_cols, int64_t *col_pos, int32_t *n_bases,
                        float *qsum, float *p25, size_t cap_cols)
{
    if (!e || !e->staged) { if (e) snprintf(e->err, sizeof e->err, "no staged batch"); return -1; }
    CK(cudaSetDevice(e->device));
    if (errmod_tables(e, 1. - 0.83)) return -1;
    View v; fill_view(e, v, nullptr, nullptr, 0, 0, 0);
    *n_cols = 0;
    const int64_t tot = (int64_t)v.ncols * v.n_files;
    if (tot == 0) return 0;
    ENSURE(col_n, (size_t)tot + 1); ENSURE(col_off, (size_t)tot + 2); ENSURE(gl_n, (size_t)tot + 1);
    ENSURE(gl_out, (size_t)tot * 29 + 1); ENSURE(gl_flag, (size_t)v.ncols + 2);
    CK(cudaMemsetAsync(e->gl_flag, 0, ((size_t)v.ncols + 2) * 4, e->stream));
    CK(cudaEventRecord(e->ev0, e->stream));
    k_gl_count<<<nblk(tot, 256), 256, 0, e->stream>>>(v, min_baseQ, e->col_n, (int32_t *)e->gl_flag); e->launches++;
    if (launch_scan<ScanSum, 1, false>(e, e->col_n, e->col_off, tot)) return -1;
    uint32_t *ovf = (uint32_t *)(e->gl_flag + v.ncols);
    k_gl<<<nblk(tot * 32, 128), 128, 0, e->stream>>>(v, min_baseQ, e->col_off, e->gl_rng_draws, e->d_fk, e->d_beta, e->d_lhet,
                                                    e->gl_n, e->gl_out, ovf); e->launches++;
    CK(cudaEventRecord(e->ev1, e->stream));
    uint64_t total_draws = 0;
    CK(cudaMemcpyAsync(&total_draws, e->col_off + tot, 8, cudaMemcpyDeviceToHost, e->stream));
    if (!col_pos) {   // device-only: the likelihoods stay in HBM
        uint32_t h_ovf = 0;
        CK(cudaMemcpyAsync(&h_ovf, ovf, 4, cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaGetLastError());
        float ms0 = 0; cudaEventElapsedTime(&ms0, e->ev0, e->ev1); e->last_kernel_ms = ms0;
        e->gl_rng_draws += total_draws;
        if (h_ovf) { snprintf(e->err, sizeof e->err, "GL: a column holds more than %d usable bases", GL_CAP); return -1; }
        *n_cols = v.ncols;
        return 0;
    }
    std::vector<uint32_t> flag((size_t)v.ncols + 1);
    std::vector<int32_t> hn((size_t)tot);
    std::vector<float> ho((size_t)tot * 29);
    CK(cudaMemcpyAsync(flag.data(), e->gl_flag, ((size_t)v.ncols + 1) * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hn.data(), e->gl_n, (size_t)tot * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(ho.data(), e->gl_out, (size_t)tot * 29 * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaGetLastError());
    float ms = 0; cudaEventElapsedTime(&ms, e->ev0, e->ev1); e->last_kernel_ms = ms;
    e->gl_rng_draws += total_draws;
    if (flag[(size_t)v.ncols]) { snprintf(e->err, sizeof e->err, "GL: a column holds more than %d usable bases", GL_CAP); return -1; }
    int64_t k = 0;
    for (int32_t c = 0; c < v.ncols; ++c) {
        if (!flag[(size_t)c]) continue;
        if ((size_t)k >= cap_cols) { snprintf(e->err, sizeof e->err, "GL output capacity too small"); return -2; }
        col_pos[k] = e->win_base + c;
        for (int f = 0; f < v.n_files; ++f) {
            const size_t s = (size_t)c * v.n_files + f, d = (size_t)k * v.n_files + f;
            n_bases[d] = hn[s];
            memcpy(qsum + d * 4, ho.data() + s * 29, 16);
            memcpy(p25 + d * 25, ho.data() + s * 29 + 4, 100);
        }
        ++k;
    }
    *n_cols = k;
    return 0;
}

// ---- the htslib / bam2bcf per-column entry points (tier T1: errmod_cal, bcf_call_glfgen) --------------------------
// One column per call: a correctness surface for callers that own their pileup loop (bam_tview.c:197, phase.c:754,
// cut_target.c:84), not a fast path -- the batch path is b200_glf().
__global__ void __launch_bounds__(32) k_errmod_one(uint16_t *bases, int n, int m, uint64_t rng_draws, const double *fk, const double *beta,
                                                   const double *lhet, float *q)
{
    extern __shared__ uint16_t s_bs[];
    const int lane = threadIdx.x;
    for (int i = lane; i < n; i += 32) s_bs[i] = bases[i];
    __syncwarp();
    uint64_t rng = 0;
    if (n > 255 && lane == 0) rng = lcg_jump(0x330EULL, rng_draws);
    __shared__ float s_q[256];
    errmod_cal_warp(s_bs, n, m, &rng, fk, beta, lhet, s_q);
    for (int i = lane; i < m * m; i += 32) q[i] = s_q[i];
    const int ns = n > 255 ? 255 : n;                  // errmod_cal leaves the (first 255, shuffled) codes sorted in place
    for (int i = lane; i < ns; i += 32) bases[i] = s_bs[i];
}

// bcf_call_glfgen for one column: per read q (base quality at qpos, 0 past the end), mapq, b4 (4-bit base, 0xff past the end),
// fl bit 0 = skip (is_del | is_refskip | unmapped), bit 1 = reverse strand
__global__ void __launch_bounds__(32) k_glfgen_one(const uint8_t *rq, const uint8_t *rmapq, const uint8_t *rb4, const uint8_t *rfl, int n_in,
                                                   int ref_base, int min_baseQ, int capQ, uint64_t rng_draws, const double *fk, const double *beta,
                                                   const double *lhet, int32_t *n_out, float *qsum_out, float *p_out, int cap)
{
    extern __shared__ uint16_t s_bs[];
    const int lane = threadIdx.x;
    int n = 0;
    float qsum[4] = {0, 0, 0, 0};
    for (int base = 0; base < n_in; base += 32) {
        const int t = base + lane;
        bool ok = false; uint16_t code = 0; int q = 0, b = 4;
        if (t < n_in && !(rfl[t] & 1)) ok = gl_pack((int)rq[t], (int)rmapq[t], rb4[t] == 0xff ? -1 : (int)rb4[t], (rfl[t] & 2) != 0, ref_base, min_baseQ, capQ, code, q, b);
        const unsigned mk = __ballot_sync(0xffffffffu, ok);
        if (ok) { const int slot = n + __popc(mk & ((1u << lane) - 1)); if (slot < cap) s_bs[slot] = code; }
        n += __popc(mk);
#pragma unroll
        for (int bb = 0; bb < 4; ++bb) {
            float x = (ok && b == bb) ? (float)q : 0.f;
            for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            qsum[bb] += x;
        }
    }
    __syncwarp();
    if (lane == 0) { *n_out = n; for (int i = 0; i < 4; ++i) qsum_out[i] = qsum[i]; }
    if (n > cap) n = cap;
    uint64_t rng = 0;
    if (n > 255 && lane == 0) rng = lcg_jump(0x330EULL, rng_draws);
    __shared__ float s_q[32];
    errmod_cal_warp(s_bs, n, 5, &rng, fk, beta, lhet, s_q);
    if (lane < 25) p_out[lane] = s_q[lane];
}

static int errmod_tables(b200_engine *e, double depcorr)
{
    if (!e->d_beta) {
        std::vector<double> fk, beta, lhet;
        errmod_host_tables(fk, beta, lhet);
        CK(cudaMalloc((void **)&e->d_fk, fk.size() * 8)); CK(cudaMalloc((void **)&e->d_beta, beta.size() * 8)); CK(cudaMalloc((void **)&e->d_lhet, lhet.size() * 8));
        CK(cudaMemcpy(e->d_fk, fk.data(), fk.size() * 8, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(e->d_beta, beta.data(), beta.size() * 8, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(e->d_lhet, lhet.data(), lhet.size() * 8, cudaMemcpyHostToDevice));
        e->fk_depcorr = 1. - 0.83;
    }
    if (depcorr != e->fk_depcorr) {   // only fk depends on the dependency coefficient (errmod_init)
        double fk[256]; fk[0] = 1.0;
        for (int n = 1; n < 256; ++n) fk[n] = pow(1. - depcorr, n) * (1.0 - 0.03) + 0.03;
        CK(cudaMemcpy(e->d_fk, fk, sizeof fk, cudaMemcpyHostToDevice));
        e->fk_depcorr = depcorr;
    }
    return 0;
}

extern "C" int b200_errmod_cal(b200_engine_t *e, double depcorr, int32_t n, int32_t m, uint16_t *bases, float *q)
{
    if (!e || n < 0 || m < 1 || m > 16) { if (e) snprintf(e->err, sizeof e->err, "errmod_cal: bad arguments"); return -1; }
    CK(cudaSetDevice(e->device));
    for (int i = 0; i < m * m; ++i) q[i] = 0.f;
    if (n == 0) return 0;
    if (errmod_tables(e, depcorr)) return -1;
    const size_t nb = (size_t)std::max(n, 256);
    ENSURE(col_n, nb / 2 + 64 + 256);              // bases (u16) followed by the m*m floats
    uint16_t *d_b = (uint16_t *)e->col_n; float *d_q = (float *)(e->col_n + nb / 2 + 32);
    CK(cudaMemcpyAsync(d_b, bases, (size_t)n * 2, cudaMemcpyHostToDevice, e->stream));
    if (nb * 2 > 48 * 1024) CK(cudaFuncSetAttribute(k_errmod_one, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(nb * 2)));
    if (nb * 2 > 200 * 1024) { snprintf(e->err, sizeof e->err, "errmod_cal: %d bases exceed the per-column capacity", n); return -1; }
    k_errmod_one<<<1, 32, nb * 2, e->stream>>>(d_b, n, m, e->gl_rng_draws, e->d_fk, e->d_beta, e->d_lhet, d_q); e->launches++;
    CK(cudaMemcpyAsync(q, d_q, (size_t)m * m * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(bases, d_b, (size_t)std::min(n, 255) * 2, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaGetLastError());
    if (n > 255) e->gl_rng_draws += (uint64_t)(n - 1);
    return 0;
}

extern "C" int b200_glfgen(b200_engine_t *e, double depcorr, int32_t n, const uint8_t *q, const uint8_t *mapq, const uint8_t *base4, const uint8_t *fl,
                           int32_t ref_base, int32_t min_baseQ, int32_t capQ, float *qsum, float *p25)
{
    if (!e || n < 0) return -1;
    CK(cudaSetDevice(e->device));
    for (int i = 0; i < 4; ++i) qsum[i] = 0.f;
    for (int i = 0; i < 25; ++i) p25[i] = 0.f;
    if (n == 0) return -1;                                   // bcf_call_glfgen: "_n <= 0 -> -1"
    if (errmod_tables(e, depcorr)) return -1;
    const size_t nb = (size_t)std::max(n, 256);
    if (nb * 2 > 200 * 1024) { snprintf(e->err, sizeof e->err, "glfgen: %d reads exceed the per-column capacity", n); return -1; }
    ENSURE(col_n, (size_t)n + 256);
    uint8_t *d = (uint8_t *)e->col_n;                        // q | mapq | base4 | fl, then n_out + qsum + p
    float *d_out = (float *)(e->col_n + (size_t)n + 64);
    CK(cudaMemcpyAsync(d, q, (size_t)n, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(d + n, mapq, (size_t)n, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(d + 2 * (size_t)n, base4, (size_t)n, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(d + 3 * (size_t)n, fl, (size_t)n, cudaMemcpyHostToDevice, e->stream));
    if (nb * 2 > 48 * 1024) CK(cudaFuncSetAttribute(k_glfgen_one, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(nb * 2)));
    k_glfgen_one<<<1, 32, nb * 2, e->stream>>>(d, d + n, d + 2 * (size_t)n, d + 3 * (size_t)n, n, ref_base, min_baseQ, capQ, e->gl_rng_draws,
                                               e->d_fk, e->d_beta, e->d_lhet, (int32_t *)d_out, d_out + 1, d_out + 5, (int)nb); e->launches++;
    float h[30];
    CK(cudaMemcpyAsync(h, d_out, sizeof h, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaGetLastError());
    int32_t n_used; memcpy(&n_used, h, 4);
    memcpy(qsum, h + 1, 16); memcpy(p25, h + 5, 100);
    if (n_used > 255) e->gl_rng_draws += (uint64_t)(n_used - 1);
    return n_used;
}

// sam_cap_mapq of every read of the staged batch (stage it with capq_thres = 0 so that nothing was applied yet)
__global__ void k_cap_mapq(RawSoA r, int thres, int32_t *out)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < r.n) out[i] = cap_mapq(r, i, thres);
}
extern "C" int b200_cap_mapq(b200_engine_t *e, int32_t thres, int32_t *out, size_t n)
{
    if (!e || !e->staged) { if (e) snprintf(e->err, sizeof e->err, "no staged batch"); return -1; }
    CK(cudaSetDevice(e->device));
    if (!e->has_ref) { snprintf(e->err, sizeof e->err, "sam_cap_mapq needs the reference"); return -1; }
    n = std::min(n, (size_t)e->n);
    if (n == 0) return 0;
    ENSURE(col_n, n + 1);
    RawSoA r;
    r.pos = e->pos; r.flag = e->flag; r.mapq = e->mapq; r.l_qseq = e->l_qseq; r.n_cigar = e->n_cigar;
    r.cigar_off = e->cigar_off; r.qual_off = e->qual_off; r.mtid = e->mtid; r.mpos = e->mpos; r.isize = e->isize;
    r.prev = nullptr; r.rbits = nullptr; r.cigar = e->cigar; r.seq4 = e->seq4; r.qual = e->qual;
    r.ref = e->ref; r.ref_beg = e->ref_beg; r.ref_n = e->ref_n; r.ref_len = e->ref_len; r.n = e->n; r.tid = e->tid;
    k_cap_mapq<<<nblk(e->n, 128), 128, 0, e->stream>>>(r, thres, (int32_t *)e->col_n); e->launches++;
    CK(cudaMemcpyAsync(out, e->col_n, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaGetLastError());
    return 0;
}
