// overlap.cuh -- read-pair overlap handling on the device.
//
// mpileup (htslib sam.c overlap_push / tweak_overlap_quality / overlap_remove,
// enabled at bam_plcmd.c:586; rule text doc/samtools-mpileup.1:353-365):
// the reference keeps a qname -> buffered-read hash while it streams reads.
// Here the host supplies, for every record, the index of the previous record
// with the same name (prev_same_name); the device turns that into forward
// chains and one thread replays the hash's state machine along each chain
// (chains are independent; typical length 2).  The quality rewrite itself walks
// both CIGARs in lock-step over the shared reference span.
//
// depth -s (bam2depth.c:598-623): same chains, but the state is just the first
// mate's end position, which becomes the second mate's clip coordinate.
#pragma once

__global__ void k_link_next(const int64_t *prev, int64_t *next, int64_t n)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t p = prev[i];
    if (p >= 0 && p < n) next[p] = i;
}

__global__ void k_overlap(RawSoA r, const int64_t *next, const uint8_t *state, const int32_t *rlen,
                          const int64_t *file_start, int n_files, int32_t *pairs, unsigned int *n_pairs)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < r.n) overlap_chain(r, i, next, state, rlen, file_start, n_files, pairs, n_pairs);
}
// the quality tweak of every collected pair (the count stays on the device: no host round trip).  One WARP per pair: two
// mates of the simple shape share a span in which every position is independent (plp_stage.h overlap_span_simple), so the
// lanes take every 32nd position; any other pair is walked in lock-step by lane 0 (tweak_overlap).
__global__ void __launch_bounds__(128) k_overlap_tweak(RawSoA r, const ReadDesc *desc, const int32_t *rlen, const int32_t *pairs, const unsigned int *n_pairs)
{
    const unsigned int n = *n_pairs;
    const int lane = threadIdx.x & 31;
    const unsigned int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    for (unsigned int k = warp; k < n; k += n_warps) {
        const int64_t ia = pairs[2 * (size_t)k], ib = pairs[2 * (size_t)k + 1];
        const ReadDesc da = load_hot(desc + ia), db = load_hot(desc + ib);
        if ((da.fl & RD_SIMPLE) && (db.fl & RD_SIMPLE)) {
            const OvSpan sp = overlap_span_simple(r, da, db, rlen, ia, ib);
            uint8_t *aq = r.qual + r.qual_off[ia], *bq = r.qual + r.qual_off[ib];
            const uint64_t aoff = r.qual_off[ia], boff = r.qual_off[ib];
            const int amul = (r.rbits && (r.rbits[ia] & B200_RB_NAME_ODD)) ? 1 : 0;
            for (int32_t j = lane; j < sp.n; j += 32) tweak_pos(r.seq4, aq, bq, aoff, boff, sp.a0 + j, sp.b0 + j, amul);
        } else if (lane == 0) tweak_overlap(r, ia, ib);
    }
}
__global__ void k_depth_clip(RawSoA r, const int64_t *next, const uint8_t *state, const int32_t *rlen, int32_t *clip, int64_t win_base)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < r.n) depth_clip_chain(r, i, next, state, rlen, clip, win_base);
}

__global__ void k_fill_i64(int64_t *p, int64_t v, int64_t n) { int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = v; }
__global__ void k_fill_i32(int32_t *p, int32_t v, int64_t n) { int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = v; }

static int link_chains(b200_engine *e, const RawSoA &r)
{
    const int64_t n = r.n;
    if (ensure(e, e->next, e->cap_next, (size_t)n + 1)) return -1;
    k_fill_i64<<<nblk(n, 256), 256, 0, e->stream>>>(e->next, -1, n); e->launches++;
    k_link_next<<<nblk(n, 256), 256, 0, e->stream>>>(r.prev, e->next, n); e->launches++;
    return 0;
}

int launch_overlap(b200_engine *e, const RawSoA &r)
{
    if (link_chains(e, r)) return -1;
    if (ensure(e, e->ov_pairs, e->cap_ov_pairs, (size_t)r.n + 2)) return -1;      // at most n/2 pairs of two indices
    CK(cudaMemsetAsync(e->d_misc + MISC_OVERLAP, 0, 8, e->stream));
    k_overlap<<<nblk(r.n, 128), 128, 0, e->stream>>>(r, e->next, e->state, e->rlen, e->file_start, e->n_files, e->ov_pairs, (unsigned int *)(e->d_misc + MISC_OVERLAP)); e->launches++;
    const int gt = (int)std::min<int64_t>(nblk((r.n / 2 + 1) * 32, 128), (int64_t)e->n_sm * 16);
    k_overlap_tweak<<<gt, 128, 0, e->stream>>>(r, e->desc, e->rlen, e->ov_pairs, (const unsigned int *)(e->d_misc + MISC_OVERLAP)); e->launches++;
    CK(cudaGetLastError());
    return 0;
}

int launch_depth_clip(b200_engine *e, const RawSoA &r)
{
    if (link_chains(e, r)) return -1;
    if (ensure(e, e->clip, e->cap_clip, (size_t)r.n + 1)) return -1;
    k_fill_i32<<<nblk(r.n, 256), 256, 0, e->stream>>>(e->clip, INT32_MIN, r.n); e->launches++;
    k_depth_clip<<<nblk(r.n, 128), 128, 0, e->stream>>>(r, e->next, e->state, e->rlen, e->clip, e->win_base); e->launches++;
    CK(cudaGetLastError());
    e->has_clip = true;
    return 0;
}
