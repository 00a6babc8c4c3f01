"""Warp-boundary composition of the mpileup entry pass (k_mp_entries), byte for byte against the oracle.

The entry pass hands each warp 32 consecutive reads, one per lane, then spreads the warp's eight-base groups over the lanes:
one group can belong to a read held by another lane, one aligned 16-byte segment of the entry array can hold the tail of
one read and the head of the next, and the other reads (indels, skips, clips) take the warp's one cursor atomic for their
slices.  Which reads share a warp is set by their index, so every set below is staged again with k = 0 .. 31 unmapped reads
(flag 4, filtered) in front of the first read: every read moves through every lane and warp position.  Sets:
  mixed   make_batch with indels, soft clips and N skips, plus reads clipped on both ends
  long    the same with every 32nd read a long read of make_long_reads (as generated, or as one [S]<n>M[S] run)
  short   the same with a third of the reads cut to l_qseq 1 .. 9 (groups straddling two reads, odd lengths)
compared as `mpileup -a` without a FASTA and with one (-B -f), at -Q 0, 13 and 200 (above 127: the scalar formatter), and
in three column windows whose edges cut reads."""
import subprocess
import numpy as np
import pytest
from test_gpu_parity import _same

pytestmark = pytest.mark.gpu

LENGTH = 30_000
WINDOWS = [(0, 9001), (9001, 21013), (21013, LENGTH)]


def _records(soa):
    """the reads of a batch as synth._pack records (bases as text, names kept: mates stay mates)"""
    from samtools_b200 import synth
    nib = synth._nibbles(soa)
    out = []
    for i in range(len(soa['pos'])):
        co, nc = int(soa['cigar_off'][i]), int(soa['n_cigar'][i])
        c = soa['cigar'][co:co + nc].astype(np.int64)
        qo, l = int(soa['qual_off'][i]), int(soa['l_qseq'][i])
        out.append(dict(pos=int(soa['pos'][i]), lens=c >> 4, ops=c & 15, flag=int(soa['flag'][i]), name=int(soa['pair_id'][i]),
                        mapq=int(soa['mapq'][i]), seq=synth._CODE2CH[nib[qo:qo + l]].copy(), qual=soa['qual'][qo:qo + l].copy()))
    return out


def _base_records(rng):
    from samtools_b200 import synth
    soa = synth.make_batch(length=LENGTH, depth=30, seed=7, frac_ins=0.05, frac_del=0.05, frac_clip=0.08, frac_skip=0.01)
    recs = _records(soa)
    for r in recs[5::23]:                                # soft clips on both ends: still a simple read
        if len(r['lens']) == 1:
            a, b = int(rng.integers(1, 12)), int(rng.integers(1, 12))
            r['lens'] = np.array([a, 150 - a - b, b]); r['ops'] = np.array([4, 0, 4])
    return soa['ref_full'], recs


def _with_long(rng, ref, recs):
    """every 32nd read gets a long read of make_long_reads placed just before it (same position); every other one of
    those is turned into a single aligned run with soft clips (a long simple read: all 32 lanes format its groups)"""
    from samtools_b200 import synth
    pool = [r for r in _records(synth.make_long_reads(length=LENGTH, depth=3, seed=5, ref=ref, plant=False))]
    out, k = [], 0
    for j, r in enumerate(recs):
        if j % 32 == 31:
            lr = dict(pool[k % len(pool)]); k += 1
            lr['pos'] = r['pos']; lr['name'] = None; lr['flag'] = int(lr['flag']) & 16
            n = len(lr['seq'])
            if k & 1:
                s = int(rng.integers(0, 40))
                m = min(n - s, LENGTH - r['pos'] - 1)
                if m > 0:
                    lr['lens'] = np.array([s, m, n - s - m]) if s else np.array([m, n - m]); lr['ops'] = np.array([4, 0, 4]) if s else np.array([0, 4])
                    lr['lens'], lr['ops'] = lr['lens'][lr['lens'] > 0], lr['ops'][lr['lens'] > 0]
            rspan = int(lr['lens'][np.isin(lr['ops'], (0, 2, 3, 7, 8))].sum())
            if r['pos'] + rspan <= LENGTH:
                out.append(lr)
        out.append(r)
    return out


def _with_short(rng, recs):
    """a third of the reads cut to 1 .. 9 bases: M, S+M, M+S or S+M+S"""
    out = []
    for j, r in enumerate(recs):
        if j % 3 == 1:
            l = 1 + (j // 3) % 9
            r = dict(r, seq=r['seq'][:l].copy(), qual=r['qual'][:l].copy(), name=None, flag=int(r['flag']) & 16)
            shape = j % 4 if l >= 3 else 0
            a = 1 if shape in (1, 3) else 0
            b = 1 if shape in (2, 3) else 0
            lens = [x for x in (a, l - a - b, b) if x]; ops = [o for x, o in zip((a, l - a - b, b), (4, 0, 4)) if x]
            r['lens'], r['ops'] = np.array(lens), np.array(ops)
        out.append(r)
    return out


def _pack(ref, recs, k):
    """the records behind k unmapped reads at the first read's position (stable sort: they come first)"""
    from samtools_b200 import synth
    p0 = min(r['pos'] for r in recs)
    unm = [dict(pos=p0, lens=np.array([20]), ops=np.array([0]), flag=4, name=None, mapq=0,
                seq=np.frombuffer(b'ACGTACGTACGTACGTACGT', np.uint8).copy(), qual=np.full(20, 30, np.uint8)) for _ in range(k)]
    return synth._pack([dict(r) for r in unm + recs], ref, LENGTH, 0, 'chr1')


@pytest.fixture(scope='module', params=['mixed', 'long', 'short'])
def entry_set(request, tmp_path_factory):
    from samtools_b200 import synth
    rng = np.random.default_rng(17)
    ref, recs = _base_records(rng)
    if request.param == 'long':
        recs = _with_long(rng, ref, recs)
    elif request.param == 'short':
        recs = _with_short(rng, recs)
    d = tmp_path_factory.mktemp('entry_' + request.param)
    soas = [_pack(ref, recs, k) for k in range(32)]
    for k in (0, 31):                                    # the unmapped reads change nothing the oracle prints
        synth.write_sam(str(d / f'k{k}.sam'), soas[k])
    synth.write_fasta(str(d / 'ref.fa'), 'chr1', ref)
    return request.param, d, soas


def _oracle(oracle_bin, d, *args):
    return subprocess.run([oracle_bin, *args], cwd=d, capture_output=True, check=True).stdout


CASES = [(ref, q) for ref in (False, True) for q in (0, 13, 200)]


def test_entry_pass_warp_composition(entry_set, oracle_bin):
    from samtools_b200 import engine
    name, d, soas = entry_set
    e = engine.Engine(0)
    for with_ref, q in CASES:
        args = ['mpileup', '-a', '-Q', str(q)] + (['-B', '-f', 'ref.fa'] if with_ref else [])
        want = _oracle(oracle_bin, d, *args, 'k0.sam')
        assert len(want) > 100_000
        assert _oracle(oracle_bin, d, *args, 'k31.sam') == want
        sconf = engine.default_stage_conf(engine.MODE_MPILEUP, **({'baq': 0} if with_ref else {}))
        for k, soa in enumerate(soas):
            s = dict(soa)
            if not with_ref:
                s['ref'] = None
            e.stage(s, sconf)
            _same(e.mpileup_text(all=1, min_baseQ=q), want, f'{name}, k={k}, ' + ' '.join(args))
    e.close()


def test_entry_pass_windows(entry_set, oracle_bin):
    """three column windows whose edges cut reads: reads starting before the window or ending after it"""
    from samtools_b200 import engine, shard
    name, d, soas = entry_set
    want = _oracle(oracle_bin, d, 'mpileup', '-a', 'k0.sam')
    e = engine.Engine(0)
    for k in (0, 7, 19, 31):
        s = dict(soas[k]); s['ref'] = None
        got = []
        for beg, end in WINDOWS:
            e.stage(shard.select_window(s, beg, end), engine.default_stage_conf(engine.MODE_MPILEUP, beg=beg, end=end))
            got.append(e.mpileup_text(all=1))
        _same(b''.join(got), want, f'{name}, k={k}, windows {WINDOWS}')
    e.close()
