"""Seeded synthetic workloads of SURVEY.md section 8(d), as SoA batches (and SAM text).

One contig of `length` bp at `depth`x with `read_len` bp paired reads:
  reference  uniform ACGT, 0.1 % of positions inside short N runs
  pairs      insert size ~ N(400, 50), proper-pair flags 99/147 (and 83/163),
             so ~15 % of pairs overlap; both mates on this contig
  mapq       60 for 90 % of reads, uniform 0..59 otherwise
  qualities  Illumina-like: Q37 plateau decaying towards Q20 at the 3' end, +-3 noise, floor 2
  bases      reference with substitutions at the per-base error rate (+0.1 % SNPs)
  CIGAR      97 % <L>M, 1.5 % one insertion (<=10), 1.5 % one deletion (<=10),
             2 % soft-clipped end, 0.1 % ref-skip (N)  (fractions configurable)
  flags      0.5 % get DUP / SECONDARY / QCFAIL to exercise the filters
Everything derives from numpy Generator(seed); the same seed gives the same
batch on every machine.  `write_sam()` writes the identical records as SAM text
so the CPU oracle (or a real samtools) reads the same data.
"""
import numpy as np

NT16 = {'A': 1, 'C': 2, 'G': 4, 'T': 8, 'N': 15}
_CODE2CH = np.frombuffer(b'=ACMGRSVTWYHKDBN', dtype=np.uint8)


def make_reference(length, seed=1, n_frac=0.001):
    rng = np.random.default_rng(seed)
    ref = np.frombuffer(b'ACGT', dtype=np.uint8)[rng.integers(0, 4, size=length)]
    n_runs = max(1, int(length * n_frac / 20)) if n_frac > 0 else 0
    for s in rng.integers(0, max(1, length - 20), size=n_runs):
        ref[s:s + int(rng.integers(5, 35))] = ord('N')
    return ref


def _name_odd(pair_id, width=9):
    """__ac_Wang_hash(__ac_X31_hash_string("p%0*d")) & 1, vectorised (uint32 wraparound)."""
    h = np.full(pair_id.shape, ord('p'), dtype=np.uint32)
    div = 10 ** (width - 1)
    with np.errstate(over='ignore'):
        for _ in range(width):
            d = ((pair_id // div) % 10).astype(np.uint32) + np.uint32(ord('0'))
            h = h * np.uint32(31) + d
            div //= 10
        h = h + ~(h << np.uint32(15)); h ^= (h >> np.uint32(10)); h = h + (h << np.uint32(3)); h ^= (h >> np.uint32(6))
        h = h + ~(h << np.uint32(11)); h ^= (h >> np.uint32(16))
    return (h & 1).astype(np.uint8)


def make_batch(length=1_000_000, depth=30, read_len=150, seed=2, ref=None, ref_seed=1, with_ref=True, tid=0,
               tid_name='chr1', frac_ins=0.015, frac_del=0.015, frac_clip=0.02, frac_skip=0.001, frac_flag=0.005,
               paired=True, n_pairs=None, start_lo=0, start_span=None):
    """Returns a dict with the b200_batch_t arrays (+ 'pair_id', 'ref' ...).
    n_pairs / start_lo / start_span override the uniform whole-contig placement (used by make_panel: the
    leftmost mates start inside [start_lo, start_lo + start_span))."""
    rng = np.random.default_rng(seed)
    L = read_len
    if ref is None:
        ref = make_reference(length, ref_seed)
    if n_pairs is None:
        n_pairs = int(round(depth * length / (2.0 * L)))
    isize = np.clip(rng.normal(400, 50, n_pairs).round().astype(np.int64), L, 1000)
    if start_span is None:
        start_span = max(1, length - 3200 - start_lo)                               # reads (even with a 2 kb N skip) stay inside the contig
    start = (start_lo + rng.integers(0, max(1, start_span), size=n_pairs)).astype(np.int64)
    # which mate is first / forward
    fwd_first = rng.random(n_pairs) < 0.5
    n = 2 * n_pairs
    pair_id = np.repeat(np.arange(n_pairs, dtype=np.int64), 2)
    is_second = np.tile(np.array([0, 1], dtype=np.int8), n_pairs)          # 0: leftmost mate, 1: rightmost
    pos = np.where(is_second == 0, np.repeat(start, 2), np.repeat(start + isize - L, 2))
    rev = is_second.astype(bool)                                           # rightmost mate is the reverse one
    read1 = np.where(np.repeat(fwd_first, 2), is_second == 0, is_second == 1)
    flag = np.full(n, 1 | 2, dtype=np.uint16)
    flag |= np.where(rev, 16, 32).astype(np.uint16)
    flag |= np.where(read1, 64, 128).astype(np.uint16)
    if not paired:
        flag = np.where(rev, 16, 0).astype(np.uint16)
    # CIGAR class: 0 M, 1 ins, 2 del, 3 clip-left, 4 clip-right, 5 ref-skip
    u = rng.random(n)
    cls = np.zeros(n, dtype=np.int8)
    edges = np.cumsum([frac_ins, frac_del, frac_clip / 2, frac_clip / 2, frac_skip])
    cls[u < edges[4]] = 5; cls[u < edges[3]] = 4; cls[u < edges[2]] = 3; cls[u < edges[1]] = 2; cls[u < edges[0]] = 1
    k = np.minimum(rng.geometric(0.4, n), 10).astype(np.int64)              # indel / clip length
    k = np.where(cls == 5, rng.integers(200, 2000, n), k)
    k = np.where((cls == 3) | (cls == 4), rng.integers(1, 30, n), k)
    a = rng.integers(10, L - 20, n).astype(np.int64)                       # bases before the event
    # query index -> reference index (or -1 = random base); only the ~6 % non-<L>M reads need fixing up
    j = np.arange(L, dtype=np.int32)[None, :]
    refidx = pos.astype(np.int32)[:, None] + j
    sp = np.nonzero(cls != 0)[0]
    if len(sp):
        A, K, P, CL = a[sp, None].astype(np.int32), k[sp, None].astype(np.int32), pos[sp, None].astype(np.int32), cls[sp, None]
        r = P + j
        r = np.where((CL == 1) & (j >= A) & (j < A + K), -1, r)
        r = np.where((CL == 1) & (j >= A + K), P + j - K, r)
        r = np.where(((CL == 2) | (CL == 5)) & (j >= A), P + j + K, r)
        r = np.where((CL == 3) & (j < K), -1, r)
        r = np.where((CL == 3) & (j >= K), P + j - K, r)
        r = np.where((CL == 4) & (j >= L - K), -1, r)
        refidx[sp] = r
    # qualities
    prof = np.where(np.arange(L) < L * 0.6, 37.0, 37.0 - 17.0 * (np.arange(L) - L * 0.6) / (L * 0.4)).astype(np.float32)
    q = np.clip(np.rint(prof[None, :] + 3.0 * rng.standard_normal((n, L), dtype=np.float32)), 2, 41).astype(np.uint8)
    q[rev] = q[rev, ::-1]                                                  # 3' end is the left end of a reverse read
    # bases
    base = ref[np.clip(refidx, 0, length - 1)]
    perr = (10.0 ** (-np.arange(64, dtype=np.float32) / 10.0) + 0.001).astype(np.float32)[q]
    mut = rng.random((n, L), dtype=np.float32) < perr
    mut |= (refidx < 0) | (refidx >= length)
    nm = int(mut.sum())
    base[mut] = np.frombuffer(b'ACGT', dtype=np.uint8)[rng.integers(0, 4, size=nm, dtype=np.uint8)]
    lut = np.full(256, 15, dtype=np.uint8)
    for ch, v in NT16.items():
        lut[ord(ch)] = v
    code = lut[base]
    # mapq + flags
    mapq = np.where(rng.random(n) < 0.9, 60, rng.integers(0, 60, n)).astype(np.uint8)
    ff = rng.random(n)
    flag = flag | np.where(ff < frac_flag / 3, 1024, 0).astype(np.uint16)
    flag = flag | np.where((ff >= frac_flag / 3) & (ff < 2 * frac_flag / 3), 256, 0).astype(np.uint16)
    flag = flag | np.where((ff >= 2 * frac_flag / 3) & (ff < frac_flag), 512, 0).astype(np.uint16)
    # sort by position (stable: keeps pair order for ties)
    order = np.argsort(pos, kind='stable')
    pos, flag, mapq, cls, k, a, pair_id, code, q = pos[order], flag[order], mapq[order], cls[order], k[order], a[order], pair_id[order], code[order], q[order]
    # CIGAR ops
    n_cigar = np.where(cls == 0, 1, np.where((cls == 3) | (cls == 4), 2, 3)).astype(np.uint32)
    cigar_off = np.concatenate([[0], np.cumsum(n_cigar)[:-1]]).astype(np.uint64)
    cigar = np.zeros(int(n_cigar.sum()), dtype=np.uint32)
    M, I, D, N_, S = 0, 1, 2, 3, 4
    o = cigar_off.astype(np.int64)
    m0 = cls == 0; cigar[o[m0]] = (L << 4) | M
    for c_, op in ((1, I), (2, D), (5, N_)):
        m = cls == c_
        cigar[o[m]] = (a[m].astype(np.uint32) << 4) | M
        cigar[o[m] + 1] = (k[m].astype(np.uint32) << 4) | op
        rest = (L - a[m] - (k[m] if c_ == 1 else 0)).astype(np.uint32)
        cigar[o[m] + 2] = (rest << 4) | M
    m = cls == 3; cigar[o[m]] = (k[m].astype(np.uint32) << 4) | S; cigar[o[m] + 1] = ((L - k[m]).astype(np.uint32) << 4) | M
    m = cls == 4; cigar[o[m]] = ((L - k[m]).astype(np.uint32) << 4) | M; cigar[o[m] + 1] = (k[m].astype(np.uint32) << 4) | S
    rlen = np.where(cls == 1, L - k, np.where((cls == 2) | (cls == 5), L + k, np.where((cls == 3) | (cls == 4), L - k, L))).astype(np.int64)
    # mates
    by_pair = np.argsort(pair_id, kind='stable')
    first, second = by_pair[0::2], by_pair[1::2]
    prev = np.full(n, -1, dtype=np.int64)
    prev[second] = first
    mpos = np.zeros(n, dtype=np.int64); mpos[first] = pos[second]; mpos[second] = pos[first]
    tl = np.zeros(n, dtype=np.int64)
    span = np.maximum(pos[second] + rlen[second], pos[first] + rlen[first]) - pos[first]
    tl[first] = span; tl[second] = -span
    if not paired:
        prev[:] = -1; mpos[:] = -1; tl[:] = 0
    # pack
    lq = L + (L & 1)
    qual = np.zeros((n, lq), dtype=np.uint8); qual[:, :L] = q
    cpad = np.zeros((n, lq), dtype=np.uint8); cpad[:, :L] = code
    seq4 = ((cpad[:, 0::2] << 4) | cpad[:, 1::2]).reshape(-1)
    qual_off = (np.arange(n, dtype=np.uint64) * np.uint64(lq))
    rbits = (_name_odd(pair_id) * 2).astype(np.uint8)
    return dict(file_start=np.array([0, n], dtype=np.int64), pos=pos.astype(np.int64), flag=flag, mapq=mapq,
                l_qseq=np.full(n, L, dtype=np.int32), n_cigar=n_cigar, cigar_off=cigar_off, qual_off=qual_off,
                mtid=np.full(n, tid if paired else -1, dtype=np.int32), mpos=mpos, isize=tl, prev_same_name=prev, rbits=rbits,
                cigar=cigar, seq4=np.ascontiguousarray(seq4), qual=np.ascontiguousarray(qual.reshape(-1)),
                tid=tid, tid_len=length, tid_name=tid_name, ref=ref if with_ref else None, ref_beg=0, ref_len=length,
                pair_id=pair_id, read_len=L, ref_full=ref)


def make_region(length, depth=30, read_len=150, seed=2, chunk=1_000_000, with_ref=False, tid_name='chr1', **kw):
    """A `length`-bp window built from independent `chunk`-sized pieces (bounded generator memory).
    Reads never cross a chunk edge, so the concatenation stays coordinate sorted."""
    parts, off = [], 0
    i = 0
    while off < length:
        ln = min(chunk, length - off)
        parts.append((off, make_batch(length=ln, depth=depth, read_len=read_len, seed=seed * 1000 + i, ref_seed=seed * 1000 + i + 500,
                                      with_ref=True, tid_name=tid_name, **kw)))
        off += ln; i += 1
    out = {}
    nread = np.cumsum([0] + [len(p['pos']) for _, p in parts])
    ncig = np.cumsum([0] + [len(p['cigar']) for _, p in parts])
    nq = np.cumsum([0] + [len(p['qual']) for _, p in parts])
    npair = np.cumsum([0] + [int(p['pair_id'].max()) + 1 if len(p['pair_id']) else 0 for _, p in parts])
    cat = lambda key, add=None: np.concatenate([(p[key] + (add[i] if add is not None else 0)).astype(p[key].dtype) for i, (_, p) in enumerate(parts)])
    offs = [o for o, _ in parts]
    out['pos'] = cat('pos', offs); out['mpos'] = cat('mpos', offs)
    for k_ in ('flag', 'mapq', 'l_qseq', 'n_cigar', 'mtid', 'isize', 'cigar', 'seq4', 'qual'):
        out[k_] = cat(k_)
    out['cigar_off'] = cat('cigar_off', [np.uint64(x) for x in ncig[:-1]]); out['qual_off'] = cat('qual_off', [np.uint64(x) for x in nq[:-1]])
    out['prev_same_name'] = np.concatenate([np.where(p['prev_same_name'] >= 0, p['prev_same_name'] + nread[i], -1) for i, (_, p) in enumerate(parts)])
    out['pair_id'] = cat('pair_id', list(npair[:-1]))
    out['rbits'] = (_name_odd(out['pair_id']) * 2).astype(np.uint8)
    out['file_start'] = np.array([0, nread[-1]], dtype=np.int64)
    ref = np.concatenate([p['ref_full'] for _, p in parts])
    out.update(tid=0, tid_len=length, tid_name=tid_name, ref=ref if with_ref else None, ref_beg=0, ref_len=length, read_len=read_len, ref_full=ref)
    return out


def algorithmic_bytes_in(soa, overlap=True):
    """SURVEY 8(d): sum over reads of ceil(l/2) + l + 4*n_cigar + 24 (+24 mate fields) (+ ref bytes touched)."""
    l = soa['l_qseq'].astype(np.int64)
    b = int(((l + 1) // 2 + l + 4 * soa['n_cigar'].astype(np.int64) + 24 + (24 if overlap else 0)).sum())
    return b


def write_fasta(path, name, ref, width=60):
    with open(path, 'w') as f:
        f.write(f'>{name}\n')
        s = ref.tobytes().decode()
        for i in range(0, len(s), width):
            f.write(s[i:i + width] + '\n')


def write_sam(path, soa, max_reads=None):
    """The same records as SAM text (names p%09d, so the name-hash bit matches rbits).
    A list of batches (one per contig, as make_long_set returns) or a batch of variable-length reads goes through
    _write_sam_var."""
    if isinstance(soa, (list, tuple)) or soa.get('read_len') is None:
        return _write_sam_var(path, soa if isinstance(soa, (list, tuple)) else [soa])
    name = soa['tid_name']; L = soa['read_len']
    lq = L + (L & 1)
    n = len(soa['pos']) if max_reads is None else min(max_reads, len(soa['pos']))
    seq4 = soa['seq4'].reshape(-1, lq // 2); qual = soa['qual'].reshape(-1, lq)
    ops = 'MIDNSHP=XB'
    with open(path, 'w') as f:
        f.write(f'@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:{name}\tLN:{soa["tid_len"]}\n')
        for i in range(n):
            co = int(soa['cigar_off'][i]); nc = int(soa['n_cigar'][i])
            cg = ''.join(f'{int(c) >> 4}{ops[int(c) & 15]}' for c in soa['cigar'][co:co + nc])
            nib = np.empty(lq, dtype=np.uint8); nib[0::2] = seq4[i] >> 4; nib[1::2] = seq4[i] & 15
            seq = _CODE2CH[nib[:L]].tobytes().decode()
            ql = (qual[i, :L] + 33).tobytes().decode()
            paired = bool(soa['flag'][i] & 1)
            f.write(f'p{int(soa["pair_id"][i]):09d}\t{int(soa["flag"][i])}\t{name}\t{int(soa["pos"][i]) + 1}\t{int(soa["mapq"][i])}\t{cg}\t'
                    f'{"=" if paired else "*"}\t{int(soa["mpos"][i]) + 1}\t{int(soa["isize"][i])}\t{seq}\t{ql}\n')


def ref_span(soa):
    """bam_cigar2rlen per read (reference bases consumed: M, D, N, =, X)."""
    cg = soa['cigar']
    op = cg & 0xf
    ln = np.where((op == 0) | (op == 2) | (op == 3) | (op == 7) | (op == 8), cg >> 4, 0).astype(np.int64)
    cs = np.concatenate([[0], np.cumsum(ln)])
    o = soa['cigar_off'].astype(np.int64)
    return cs[o + soa['n_cigar'].astype(np.int64)] - cs[o]


def _gather_ranges(off, cnt):
    """indices off[i] .. off[i]+cnt[i]-1 for every i, concatenated."""
    cnt = cnt.astype(np.int64)
    tot = int(cnt.sum())
    if tot == 0:
        return np.zeros(0, dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    return np.repeat(off.astype(np.int64) - starts, cnt) + np.arange(tot, dtype=np.int64)


def take_reads(soa, idx):
    """Sub-batch holding reads `idx` (ascending batch indices, or a permutation), payload re-packed; name links that
    leave the selection become -1.  All reads must have the same l_qseq (true of this generator)."""
    idx = np.asarray(idx, dtype=np.int64)
    n0 = len(soa['pos'])
    if soa.get('read_len') is None:
        return _take_reads_var(soa, idx)
    L = soa['read_len']; lq = L + (L & 1)
    out = dict(soa)
    for k in ('pos', 'flag', 'mapq', 'l_qseq', 'n_cigar', 'mtid', 'mpos', 'isize', 'rbits', 'pair_id'):
        out[k] = np.ascontiguousarray(soa[k][idx])
    inv = np.full(n0 + 1, -1, dtype=np.int64)
    inv[idx] = np.arange(len(idx), dtype=np.int64)
    prev = soa['prev_same_name'][idx]
    out['prev_same_name'] = np.where(prev >= 0, inv[np.where(prev >= 0, prev, n0)], -1).astype(np.int64)
    rows = (soa['qual_off'][idx] // np.uint64(lq)).astype(np.int64)
    out['qual'] = np.ascontiguousarray(soa['qual'].reshape(-1, lq)[rows].reshape(-1))
    out['seq4'] = np.ascontiguousarray(soa['seq4'].reshape(-1, lq // 2)[rows].reshape(-1))
    out['qual_off'] = np.arange(len(idx), dtype=np.uint64) * np.uint64(lq)
    out['cigar'] = np.ascontiguousarray(soa['cigar'][_gather_ranges(soa['cigar_off'][idx], out['n_cigar'])])
    out['cigar_off'] = np.concatenate([[0], np.cumsum(out['n_cigar'].astype(np.int64))[:-1]]).astype(np.uint64)
    out['file_start'] = np.array([0, len(idx)], dtype=np.int64)
    return out


def make_panel(n_targets=500, target_len=2000, depth=200, n_hot=20, hot_depth=2000, hot_span=100, spacing=10_000,
               read_len=150, seed=4, with_ref=True, tid_name='chr1', **kw):
    """BASELINE config 4 shape (SURVEY.md 8d): `n_targets` targets of `target_len` bp at `depth`x mean, `n_hot` of them
    carrying a hotspot where another `hot_depth`x of pairs start inside `hot_span` bp (columns with thousands of reads,
    i.e. errmod_cal's n > 255 shuffle path).  One contig, targets `spacing` bp apart; coordinate sorted."""
    L = read_len
    length = n_targets * spacing
    rng = np.random.default_rng(seed)
    hot = set(rng.choice(n_targets, size=min(n_hot, n_targets), replace=False).tolist()) if n_hot else set()
    ref = make_reference(length, seed * 1000 + 1)
    parts = []
    npair = 0
    for t in range(n_targets):
        off = t * spacing
        sub = ref[off:off + spacing]
        pieces = [dict(n_pairs=int(round(depth * target_len / (2.0 * L))), start_lo=200, start_span=target_len, seed=seed * 100003 + 2 * t)]
        if t in hot:
            pieces.append(dict(n_pairs=int(round(hot_depth * (hot_span + L) / (2.0 * L))), start_lo=200 + target_len // 2, start_span=hot_span,
                               seed=seed * 100003 + 2 * t + 1))
        for pc in pieces:
            b = make_batch(length=spacing, read_len=L, ref=sub, with_ref=True, tid_name=tid_name, **pc, **kw)
            parts.append((off, b, npair))
            npair += int(b['pair_id'].max()) + 1 if len(b['pair_id']) else 0
    nread = np.cumsum([0] + [len(p['pos']) for _, p, _ in parts])
    ncig = np.cumsum([0] + [len(p['cigar']) for _, p, _ in parts])
    nq = np.cumsum([0] + [len(p['qual']) for _, p, _ in parts])
    out = {}
    out['pos'] = np.concatenate([p['pos'] + o for o, p, _ in parts]); out['mpos'] = np.concatenate([p['mpos'] + o for o, p, _ in parts])
    for k_ in ('flag', 'mapq', 'l_qseq', 'n_cigar', 'mtid', 'isize', 'cigar', 'seq4', 'qual'):
        out[k_] = np.concatenate([p[k_] for _, p, _ in parts])
    out['cigar_off'] = np.concatenate([p['cigar_off'] + np.uint64(ncig[i]) for i, (_, p, _) in enumerate(parts)])
    out['qual_off'] = np.concatenate([p['qual_off'] + np.uint64(nq[i]) for i, (_, p, _) in enumerate(parts)])
    out['prev_same_name'] = np.concatenate([np.where(p['prev_same_name'] >= 0, p['prev_same_name'] + nread[i], -1) for i, (_, p, _) in enumerate(parts)])
    out['pair_id'] = np.concatenate([p['pair_id'] + base for _, p, base in parts])
    out['rbits'] = (_name_odd(out['pair_id']) * 2).astype(np.uint8)
    out['file_start'] = np.array([0, nread[-1]], dtype=np.int64)
    out.update(tid=0, tid_len=length, tid_name=tid_name, ref=ref if with_ref else None, ref_beg=0, ref_len=length, read_len=L, ref_full=ref)
    order = np.argsort(out['pos'], kind='stable')              # hotspot pieces interleave with their target's reads
    res = take_reads(out, order)
    res['hot_targets'] = sorted(hot)
    return res


def _reg2bin(beg, end):
    """SAMv1 5.3 reg2bin, vectorised (end exclusive)."""
    end = end - 1
    b = np.zeros(len(beg), dtype=np.int64)
    done = np.zeros(len(beg), dtype=bool)
    for shift, base in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        m = ~done & ((beg >> shift) == (end >> shift))
        b[m] = base + (beg[m] >> shift)
        done |= m
    return b.astype(np.uint16)


def write_bam(path, soa, level=1, block=0xff00):
    """The same records as a coordinate-sorted BAM (BGZF, SAMv1 4.2): what `samtools mpileup` really reads.
    Names are p%09d like write_sam().  No index is written (the readers here scan).
    A list of batches or a batch of variable-length reads goes through _write_bam_var."""
    if isinstance(soa, (list, tuple)) or soa.get('read_len') is None:
        return _write_bam_var(path, soa if isinstance(soa, (list, tuple)) else [soa], level, block)
    import struct
    import zlib
    name = soa['tid_name'].encode(); L = soa['read_len']; lq = L + (L & 1)
    n = len(soa['pos'])
    text = f'@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:{soa["tid_name"]}\tLN:{soa["tid_len"]}\n'.encode()
    hdr = b'BAM\1' + struct.pack('<i', len(text)) + text + struct.pack('<i', 1) + struct.pack('<i', len(name) + 1) + name + b'\0' + \
        struct.pack('<i', int(soa['tid_len']))
    ncg = soa['n_cigar'].astype(np.int64)
    fixed = 32 + 11 + (L + 1) // 2 + L
    size = fixed + 4 * ncg                                   # block_size field excluded
    off = np.concatenate([[0], np.cumsum(size + 4)])
    buf = np.zeros(int(off[-1]), dtype=np.uint8)
    rl = ref_span(soa)
    pos = soa['pos'].astype(np.int64)
    core = np.zeros(n, dtype=np.dtype([('bs', '<i4'), ('tid', '<i4'), ('pos', '<i4'), ('lname', 'u1'), ('mapq', 'u1'), ('bin', '<u2'), ('ncig', '<u2'),
                                        ('flag', '<u2'), ('lseq', '<i4'), ('mtid', '<i4'), ('mpos', '<i4'), ('tlen', '<i4')]))
    core['bs'] = size; core['tid'] = soa.get('tid', 0); core['pos'] = pos; core['lname'] = 11; core['mapq'] = soa['mapq']
    core['bin'] = _reg2bin(pos, pos + np.maximum(rl, 1)); core['ncig'] = ncg; core['flag'] = soa['flag']; core['lseq'] = L
    core['mtid'] = soa['mtid']; core['mpos'] = soa['mpos']; core['tlen'] = soa['isize']
    cb = core.view(np.uint8).reshape(n, 36)
    digits = np.zeros((n, 11), dtype=np.uint8); digits[:, 0] = ord('p')
    pid = soa['pair_id'].astype(np.int64)
    for k in range(9):
        digits[:, 9 - k] = ord('0') + (pid // 10 ** k) % 10
    rows = (soa['qual_off'] // np.uint64(lq)).astype(np.int64)
    seq = soa['seq4'].reshape(-1, lq // 2)[rows][:, :(L + 1) // 2].copy()
    if L & 1:
        seq[:, -1] &= 0xf0
    qual = soa['qual'].reshape(-1, lq)[rows][:, :L]
    o = off[:-1]
    for cols, at in ((cb, 0), (digits, 36)):
        buf[(o[:, None] + at + np.arange(cols.shape[1])[None, :]).reshape(-1)] = cols.reshape(-1)
    cig_bytes = soa['cigar'].astype('<u4').view(np.uint8)
    dst = np.repeat(o + 47, 4 * ncg) + (np.arange(int(4 * ncg.sum())) - np.repeat(np.concatenate([[0], np.cumsum(4 * ncg)[:-1]]), 4 * ncg))
    src = _gather_ranges(4 * soa['cigar_off'].astype(np.int64), 4 * ncg)
    buf[dst] = cig_bytes[src]
    so = o + 47 + 4 * ncg
    buf[(so[:, None] + np.arange(seq.shape[1])[None, :]).reshape(-1)] = seq.reshape(-1)
    qo = so + seq.shape[1]
    buf[(qo[:, None] + np.arange(L)[None, :]).reshape(-1)] = qual.reshape(-1)
    _write_bgzf(path, hdr + buf.tobytes(), level, block)


def _write_bgzf(path, data, level, block):
    import struct
    import zlib
    with open(path, 'wb') as f:
        for i in range(0, len(data), block):
            chunk = data[i:i + block]
            c = zlib.compressobj(level, zlib.DEFLATED, -15)
            comp = c.compress(chunk) + c.flush()
            f.write(b'\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0' + struct.pack('<H', len(comp) + 25) + comp +
                    struct.pack('<II', zlib.crc32(chunk) & 0xffffffff, len(chunk)))
        f.write(bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000'))


# ---------------------------------------------------------------------------------------------------------- long reads
# Variable-length batches: 'read_len' is None, every read has its own l_qseq; qualities start on even offsets (qual_off) and
# the bases are the nibbles qual_off.. of seq4, as b200_batch_t requires.
_OPS = 'MIDNSHP=XB'
_QCONS = np.array([1, 1, 0, 0, 1, 0, 0, 1, 1, 0], dtype=bool)      # M I D N S H P = X B: consumes query
_RCONS = np.array([1, 0, 1, 1, 0, 0, 0, 1, 1, 0], dtype=bool)      # consumes reference


def parse_cigar(s):
    """'300M2I10D' -> (lengths, op codes) as int64 arrays"""
    import re
    t = re.findall(r'(\d+)([MIDNSHP=XB])', s)
    return np.array([int(l) for l, _ in t], dtype=np.int64), np.array([_OPS.index(o) for _, o in t], dtype=np.int64)


def baq_band(pos, lens, ops, lq, ref_len):
    """Band probaln_glocal runs with for one read under sam_prob_realn's window rule (None: the read gets no HMM -- an N
    skip, or no M op).  Restated here for the generator's self-checks: it classifies inputs, it does not compute answers."""
    x = int(pos); xb = xe = -1; y = 0; yb = ye = -1
    for l, op in zip(lens.tolist(), ops.tolist()):
        if op in (0, 7, 8):
            if yb < 0: yb = y
            if xb < 0: xb = x
            ye = y + l; xe = x + l; x += l; y += l
        elif op in (1, 4): y += l
        elif op == 2: x += l
        elif op == 3: return None
    if xb == -1:
        return None
    bw = 7
    dd = abs((xe - xb) - (ye - yb))
    if dd > bw: bw = dd + 3
    xb = max(xb - (yb + bw // 2), 0)
    xe += lq - ye + bw // 2
    if xe - xb - lq > bw:
        xb += (xe - xb - lq - bw) // 2
        xe -= (xe - xb - lq - bw) // 2
    xe = min(xe, ref_len)
    l_ref = xe - xb
    if l_ref <= 0:
        return None
    return max(min(max(l_ref, lq), bw), abs(l_ref - lq))


def _realise(rng, ref, pos, lens, ops, sub_rate=0.03, n_rate=0.002):
    """query bases of a read with this CIGAR at `pos`: the reference under aligned ops (plus substitutions), random bases in
    insertions / soft clips / past the contig end, some N"""
    ql = np.where(_QCONS[ops], lens, 0); rl = np.where(_RCONS[ops], lens, 0)
    rstart = pos + np.concatenate([[0], np.cumsum(rl)[:-1]])
    qstart = np.concatenate([[0], np.cumsum(ql)[:-1]])
    n = int(ql.sum())
    ridx = np.repeat(rstart - qstart, ql) + np.arange(n)
    ok = np.repeat(np.isin(ops, (0, 7, 8)), ql) & (ridx >= 0) & (ridx < len(ref))
    acgt = np.frombuffer(b'ACGT', dtype=np.uint8)
    base = acgt[rng.integers(0, 4, n)]
    base[ok] = ref[ridx[ok]]
    sub = ok & (rng.random(n) < sub_rate)
    base[sub] = acgt[rng.integers(0, 4, int(sub.sum()))]
    base[rng.random(n) < n_rate] = ord('N')
    return base


def _long_quals(rng, n, mode='ont'):
    if mode == 'star':
        return np.full(n, 0xff, dtype=np.uint8)
    if mode == 'wide':
        return (np.arange(n) % 94).astype(np.uint8)
    q = np.clip(np.rint(rng.normal(18.0, 8.0, n)), 0, 93).astype(np.uint8)
    u = rng.random(n)
    q[u < 0.02] = 93; q[u > 0.99] = 0
    return q


def _ont_cigar(rng, span, indel_rate=0.03, del_bias=0.0, max_run=6):
    """M runs separated by single I / D events (geometric lengths <= max_run) covering ~span reference bases.
    del_bias in (-1, 1) tilts the events towards deletions (> 0) or insertions (< 0): the net indel difference, and with it
    the BAQ band, grows with |del_bias|."""
    n_ev = int(span * indel_rate * 1.5) + 8
    m = rng.geometric(indel_rate, n_ev).astype(np.int64)
    is_del = rng.random(n_ev) < 0.5 * (1.0 + del_bias)
    il = np.minimum(rng.geometric(0.55, n_ev), max_run).astype(np.int64)
    k = min(int(np.searchsorted(np.cumsum(m + np.where(is_del, il, 0)), span)) + 1, n_ev)
    lens = np.empty(2 * k - 1, dtype=np.int64); ops = np.zeros(2 * k - 1, dtype=np.int64)
    lens[0::2] = m[:k]
    lens[1::2] = il[:k - 1]; ops[1::2] = np.where(is_del[:k - 1], 2, 1)
    return lens, ops


def _rec(rng, ref, pos, lens, ops, flag=0, name=None, qmode='ont', mapq=60, **kw):
    seq = _realise(rng, ref, pos, lens, ops, **kw)
    return dict(pos=int(pos), lens=lens, ops=ops, flag=int(flag), name=name, mapq=int(mapq), seq=seq, qual=_long_quals(rng, len(seq), qmode))


def _pack(recs, ref, length, tid, tid_name, name_base=0):
    """records -> variable-length SoA (coordinate sorted, stable); names p%09d of name_base + record['name'] (reads without a
    name get a fresh one); mates are the records sharing a name (their mate fields point at the next one, cyclically)"""
    nxt = max([r['name'] for r in recs if r['name'] is not None] + [-1]) + 1
    for r in recs:
        if r['name'] is None:
            r['name'] = nxt; nxt += 1
    recs = sorted(recs, key=lambda r: r['pos'])
    n = len(recs)
    pos = np.array([r['pos'] for r in recs], dtype=np.int64)
    lq = np.array([len(r['seq']) for r in recs], dtype=np.int32)
    ncig = np.array([len(r['lens']) for r in recs], dtype=np.uint32)
    cigar = np.concatenate([(r['lens'] << 4) | r['ops'] for r in recs]).astype(np.uint32)
    cigar_off = np.concatenate([[0], np.cumsum(ncig.astype(np.int64))[:-1]]).astype(np.uint64)
    padded = lq.astype(np.int64) + (lq & 1)
    qo = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
    tot = int(padded.sum())
    qual = np.zeros(tot + 2, dtype=np.uint8); nib = np.zeros(tot + 2, dtype=np.uint8)
    lut = np.full(256, 15, dtype=np.uint8)
    for ch, v in NT16.items():
        lut[ord(ch)] = v
    for i, r in enumerate(recs):
        qual[qo[i]:qo[i] + lq[i]] = r['qual']; nib[qo[i]:qo[i] + lq[i]] = lut[r['seq']]
    seq4 = (nib[0::2] << 4) | nib[1::2]
    pair_id = np.array([name_base + r['name'] for r in recs], dtype=np.int64)
    flag = np.array([r['flag'] for r in recs], dtype=np.uint16)
    rlen = np.array([int(r['lens'][_RCONS[r['ops']]].sum()) for r in recs], dtype=np.int64)
    prev = np.full(n, -1, dtype=np.int64); mtid = np.full(n, -1, dtype=np.int32)
    mpos = np.full(n, -1, dtype=np.int64); isize = np.zeros(n, dtype=np.int64)
    groups = {}
    for i in range(n):
        g = groups.setdefault(int(pair_id[i]), [])
        if g:
            prev[i] = g[-1]
        g.append(i)
    for g in groups.values():
        if len(g) < 2:
            continue
        lo = min(pos[g]); hi = max(pos[g] + rlen[g])
        for k, i in enumerate(g):
            if flag[i] & 1:
                j = g[(k + 1) % len(g)]
                mtid[i] = tid; mpos[i] = pos[j]
                isize[i] = (hi - lo) if pos[i] == lo and k == 0 else -(hi - lo)
    return dict(file_start=np.array([0, n], dtype=np.int64), pos=pos, flag=flag, mapq=np.array([r['mapq'] for r in recs], dtype=np.uint8),
                l_qseq=lq, n_cigar=ncig, cigar_off=cigar_off, qual_off=qo.astype(np.uint64), mtid=mtid, mpos=mpos, isize=isize,
                prev_same_name=prev, rbits=(_name_odd(pair_id) * 2).astype(np.uint8), cigar=cigar, seq4=np.ascontiguousarray(seq4),
                qual=qual, tid=tid, tid_len=length, tid_name=tid_name, ref=ref, ref_beg=0, ref_len=length, pair_id=pair_id,
                read_len=None, ref_full=ref)


def _band_cigar(pos, ref_len, target):
    """300M<k>D300M or 300M<k>I300M whose BAQ band is exactly `target`"""
    for k in range(1, 1000):
        for op in 'DI':
            s = f'300M{k}{op}300M'
            lens, ops = parse_cigar(s)
            if baq_band(pos, lens, ops, 600 + (k if op == 'I' else 0), ref_len) == target:
                return s
    raise ValueError(target)


def _name_with_parity(start, parity):
    i = start
    while int(_name_odd(np.array([i]))[0]) != parity:
        i += 1
    return i


def _planted(rng, ref, length):
    """the long-read edge cases (positions inside a contig of >= 160 kb)"""
    P = []
    add = lambda pos, cig, **kw: P.append(_rec(rng, ref, pos, *parse_cigar(cig), **kw))
    # l_qseq 1 / 8 / 9 / 511 / 512 / 513 (band 7: 512 on the register kernel, 513 on the warp kernel)
    for k, l in enumerate((1, 8, 9, 511, 512, 513)):
        add(5000 + 700 * k, f'{l}M')
    # n_cigar 8 and 9 (hard + soft clips)
    add(10_000, '10S100M2I100M3D100M1I90M', flag=16)
    add(10_050, '5H10S100M2I100M3D100M1I90M')
    # reference spans 511 / 512 / 513 / 544, simple and with an insertion / a deletion
    for k, s in enumerate((511, 512, 513, 544)):
        add(11_000 + 97 * k, f'{s}M')
        add(11_010 + 97 * k, f'200M3I{s - 200}M', flag=16)
        add(11_020 + 97 * k, f'200M4D{s - 204}M')
    # BAQ bands of 15 / 16 / 31 / 32 / 100 (2*bw+1 = 31 / 33 / 63 / 65 / 201 cells: both sides of the 32- and 64-cell edges)
    for k, b in enumerate((15, 16, 31, 32, 100)):
        add(13_000 + 1500 * k, _band_cigar(13_000 + 1500 * k, length, b))
    # leading soft clips of 65535 / 65536 on <n>M reads (the clip decides the simple-read qstart)
    add(100_000, '65535S400M')
    add(100_500, '65536S400M', flag=16)
    # hard clips
    add(21_000, '30H500M'); add(21_100, '500M40H', flag=16); add(21_200, '10H20S400M15S10H')
    # deletions of >= 512 bases (the 1000-base one covers whole 32-column groups as '*' only)
    add(22_000, '300M1000D300M'); add(22_100, '200M600D200M', flag=16)
    # N skips of several kb (no BAQ)
    add(24_000, '500M3000N500M'); add(24_200, '400M5000N300M', flag=16)
    # an insertion of 2 kb
    add(30_500, '300M2100I300M')
    # qualities 0..93, '*' qualities, N bases
    add(31_000, '700M', qmode='wide'); add(31_100, '800M', qmode='star'); add(31_200, '600M', n_rate=0.1)
    # position 0, and a read running past the contig end
    add(0, '300M'); add(0, '20S300M', flag=16); add(length - 150, '400M')
    # overlapping long mates: both simple, one with indels, both with indels; both name-hash parities; one name triplet
    nm = 900_000
    for k, (a, b, par) in enumerate((('3000M', '3000M', 0), ('3000M', '3000M', 1), ('1000M5D1000M3I997M', '2500M', 0),
                                     ('2500M', '1200M8I1300M', 1), (None, None, 0), (None, None, 1))):
        nm = _name_with_parity(nm + 1, par)
        p0 = 40_000 + 8000 * k
        la, oa = parse_cigar(a) if a else _ont_cigar(rng, 4000)
        lb, ob = parse_cigar(b) if b else _ont_cigar(rng, 4000)
        f0, f1 = (99, 147) if k % 2 == 0 else (163, 83)
        P.append(_rec(rng, ref, p0, la, oa, flag=f0, name=nm))
        P.append(_rec(rng, ref, p0 + 1500, lb, ob, flag=f1, name=nm))
    nm = _name_with_parity(nm + 1, 0)
    for k, (cig, f) in enumerate((('2000M', 99), ('1500M10D500M', 147), ('2000M', 2048 | 97))):
        add(90_000 + 600 * k, cig, flag=f, name=nm)
    return P


def make_long_reads(length=200_000, depth=12, seed=31, ref=None, ref_seed=None, tid=0, tid_name='chr1', del_bias=0.0,
                    indel_rate=0.03, sub_rate=0.03, median_len=2500, sigma=0.8, max_len=40_000, frac_pair=0.12,
                    plant=True, name_base=0):
    """ONT/PacBio-like reads on one contig, as a variable-length SoA (read_len None; see make_batch for the fields).
      lengths    log-normal around median_len, clipped to 513 .. max_len
      errors     substitutions (sub_rate) and single I / D runs of <= 6 bases (indel_rate per base, del_bias tilts them)
      clips      20 % soft clip on each side (10..500 bases), 5 % hard clips
      qualities  ~N(18, 8) clipped to 0..93 with spikes at 0 and 93; 2 % of reads '*'; 0.2 % N bases
      mates      frac_pair of the reads get an overlapping long mate (99/147 or 163/83)
      plant      adds every edge case of _planted (needs length >= 160 kb)
    Seeded: the same arguments give the same batch."""
    rng = np.random.default_rng(seed)
    if ref is None:
        ref = make_reference(length, seed * 7 + 3 if ref_seed is None else ref_seed)
    recs = _planted(rng, ref, length) if plant else []
    n_reads = int(round(depth * length / float(median_len) / np.exp(sigma * sigma / 2)))
    for _ in range(n_reads):
        span = int(np.clip(rng.lognormal(np.log(median_len), sigma), 513, max_len))
        span = min(span, length - 10)
        pos = int(rng.integers(0, max(1, length - span)))
        lens, ops = _ont_cigar(rng, span, indel_rate, del_bias)
        if rng.random() < 0.2: lens, ops = np.concatenate([[rng.integers(10, 500)], lens]), np.concatenate([[4], ops])
        if rng.random() < 0.2: lens, ops = np.concatenate([lens, [rng.integers(10, 500)]]), np.concatenate([ops, [4]])
        if rng.random() < 0.05: lens, ops = np.concatenate([[rng.integers(1, 2000)], lens]), np.concatenate([[5], ops])
        u = rng.random()
        flag = 1024 if u < 0.005 else 256 if u < 0.01 else 0
        qmode = 'star' if rng.random() < 0.02 else 'ont'
        mapq = 60 if rng.random() < 0.9 else int(rng.integers(0, 60))
        if rng.random() < frac_pair:
            nm = len(recs) + 1_000_000
            mp = pos + int(span * rng.uniform(0.1, 0.9))
            mspan = min(int(np.clip(rng.lognormal(np.log(median_len), sigma), 513, max_len)), length - 10 - mp)
            f0, f1 = (99, 147) if rng.random() < 0.5 else (163, 83)
            recs.append(_rec(rng, ref, pos, lens, ops, flag=f0, name=nm, qmode=qmode, mapq=mapq, sub_rate=sub_rate))
            if mspan > 50:
                ml, mo = _ont_cigar(rng, mspan, indel_rate, del_bias)
                recs.append(_rec(rng, ref, mp, ml, mo, flag=f1, name=nm, mapq=mapq, sub_rate=sub_rate))
            continue
        recs.append(_rec(rng, ref, pos, lens, ops, flag=flag | (16 if rng.random() < 0.5 else 0), qmode=qmode, mapq=mapq, sub_rate=sub_rate))
    return _pack(recs, ref, length, tid, tid_name, name_base)


def make_long_set(seed=31, lengths=(200_000, 120_000), **kw):
    """two contigs of long reads (chr1 carries the planted edge cases); write_sam / write_bam take the list"""
    out = []
    plant = kw.pop('plant', True)
    for t, L in enumerate(lengths):
        out.append(make_long_reads(length=L, seed=seed + 1000 * t, tid=t, tid_name=f'chr{t + 1}', plant=plant and t == 0,
                                   name_base=10_000_000 * t, **kw))
    return out


def make_long_deletion(seed=41, length=100_000, del_len=70_000):
    """a small input whose one read carries a `del_len`-base deletion (its mpileup entry is longer than 64 KiB), at low depth
    around it.  Only for -B: with BAQ on, that read's band would need gigabytes."""
    rng = np.random.default_rng(seed)
    ref = make_reference(length, seed * 7 + 3)
    recs = [_rec(rng, ref, 10_000, *parse_cigar(f'300M{del_len}D300M'))]
    recs[0]['qual'][:] = 30                   # its entry before the deletion passes the default -Q 13
    for k in range(40):
        p = int(rng.integers(0, length - 700))
        recs.append(_rec(rng, ref, p, *parse_cigar('600M'), flag=16 if k & 1 else 0))
    return _pack(recs, ref, length, 0, 'chr1')


def make_long_cigar(seed=43, length=120_000, n_rep=16_500):
    """a small input with one read of 4 * n_rep > 65535 CIGAR ops (write_bam stores it as CG:B,I behind the
    <l_qseq>S<rlen>N placeholder), plus a few long reads around it"""
    rng = np.random.default_rng(seed)
    ref = make_reference(length, seed * 7 + 3)
    lens = np.tile(np.array([2, 1, 2, 1], dtype=np.int64), n_rep); ops = np.tile(np.array([0, 1, 0, 2], dtype=np.int64), n_rep)
    recs = [_rec(rng, ref, 1000, lens, ops)]
    for k in range(30):
        span = int(rng.integers(600, 6000))
        l, o = _ont_cigar(rng, span)
        recs.append(_rec(rng, ref, int(rng.integers(0, length - span)), l, o, flag=16 if k & 1 else 0))
    return _pack(recs, ref, length, 0, 'chr1')


def _nibbles(soa):
    s = soa['seq4']
    nib = np.empty(2 * len(s), dtype=np.uint8); nib[0::2] = s >> 4; nib[1::2] = s & 15
    return nib


def _write_sam_var(path, soas):
    with open(path, 'w') as f:
        f.write('@HD\tVN:1.6\tSO:coordinate\n' + ''.join(f'@SQ\tSN:{s["tid_name"]}\tLN:{s["tid_len"]}\n' for s in soas))
        for soa in soas:
            name = soa['tid_name']; nib = _nibbles(soa)
            for i in range(len(soa['pos'])):
                co = int(soa['cigar_off'][i]); nc = int(soa['n_cigar'][i])
                c = soa['cigar'][co:co + nc]
                cg = ''.join(f'{l}{_OPS[o]}' for l, o in zip((c >> 4).tolist(), (c & 15).tolist()))
                qo = int(soa['qual_off'][i]); l = int(soa['l_qseq'][i])
                seq = _CODE2CH[nib[qo:qo + l]].tobytes().decode() if l else '*'
                q = soa['qual'][qo:qo + l]
                ql = '*' if l == 0 or q[0] == 0xff else (q + 33).tobytes().decode()
                mt = int(soa['mtid'][i])
                f.write(f'p{int(soa["pair_id"][i]):09d}\t{int(soa["flag"][i])}\t{name}\t{int(soa["pos"][i]) + 1}\t{int(soa["mapq"][i])}\t{cg}\t'
                        f'{"*" if mt < 0 else "="}\t{int(soa["mpos"][i]) + 1}\t{int(soa["isize"][i])}\t{seq}\t{ql}\n')


def _write_bam_var(path, soas, level, block):
    """write_bam for variable-length reads; a CIGAR of more than 65535 ops goes into CG:B,I behind <l_qseq>S<rlen>N (SAMv1 4.2.2)"""
    import struct
    text = ('@HD\tVN:1.6\tSO:coordinate\n' + ''.join(f'@SQ\tSN:{s["tid_name"]}\tLN:{s["tid_len"]}\n' for s in soas)).encode()
    out = [b'BAM\1' + struct.pack('<i', len(text)) + text + struct.pack('<i', len(soas))]
    for s in soas:
        nm = s['tid_name'].encode()
        out.append(struct.pack('<i', len(nm) + 1) + nm + b'\0' + struct.pack('<i', int(s['tid_len'])))
    for s in soas:
        nib = _nibbles(s); rl = ref_span(s)
        for i in range(len(s['pos'])):
            co = int(s['cigar_off'][i]); nc = int(s['n_cigar'][i]); l = int(s['l_qseq'][i]); qo = int(s['qual_off'][i])
            cig = s['cigar'][co:co + nc].astype('<u4')
            aux = b''
            if nc > 65535:
                aux = b'CGBI' + struct.pack('<I', nc) + cig.tobytes()
                cig = np.array([(l << 4) | 4, (int(rl[i]) << 4) | 3], dtype='<u4')
            nb = nib[qo:qo + l].copy()
            if l & 1:
                nb = np.append(nb, 0)
            seq = ((nb[0::2] << 4) | nb[1::2]).astype(np.uint8).tobytes()
            p = int(s['pos'][i])
            name = f'p{int(s["pair_id"][i]):09d}'.encode() + b'\0'
            body = struct.pack('<iiBBHHHiiii', int(s['tid']), p, len(name), int(s['mapq'][i]),
                               int(_reg2bin(np.array([p]), np.array([p + max(int(rl[i]), 1)]))[0]), len(cig), int(s['flag'][i]), l,
                               int(s['mtid'][i]), int(s['mpos'][i]), int(s['isize'][i]))
            body += name + cig.tobytes() + seq + s['qual'][qo:qo + l].tobytes() + aux
            out.append(struct.pack('<i', len(body)) + body)
    _write_bgzf(path, b''.join(out), level, block)


def _take_reads_var(soa, idx):
    """take_reads for variable-length batches (qualities / bases re-packed read by read)"""
    n0 = len(soa['pos'])
    out = dict(soa)
    for k in ('pos', 'flag', 'mapq', 'l_qseq', 'n_cigar', 'mtid', 'mpos', 'isize', 'rbits', 'pair_id'):
        out[k] = np.ascontiguousarray(soa[k][idx])
    inv = np.full(n0 + 1, -1, dtype=np.int64)
    inv[idx] = np.arange(len(idx), dtype=np.int64)
    prev = soa['prev_same_name'][idx]
    out['prev_same_name'] = np.where(prev >= 0, inv[np.where(prev >= 0, prev, n0)], -1).astype(np.int64)
    lq = out['l_qseq'].astype(np.int64); padded = lq + (lq & 1)
    qo = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
    src = _gather_ranges(soa['qual_off'][idx], lq); dst = _gather_ranges(qo, lq)
    qual = np.zeros(int(padded.sum()) + 2, dtype=np.uint8); qual[dst] = soa['qual'][src]
    nib = np.zeros(len(qual), dtype=np.uint8); nib[dst] = _nibbles(soa)[src]
    out['qual'] = qual; out['seq4'] = np.ascontiguousarray((nib[0::2] << 4) | nib[1::2])
    out['qual_off'] = qo.astype(np.uint64)
    out['cigar'] = np.ascontiguousarray(soa['cigar'][_gather_ranges(soa['cigar_off'][idx], out['n_cigar'])])
    out['cigar_off'] = np.concatenate([[0], np.cumsum(out['n_cigar'].astype(np.int64))[:-1]]).astype(np.uint64)
    out['file_start'] = np.array([0, len(idx)], dtype=np.int64)
    return out
