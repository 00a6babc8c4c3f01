"""Slice rounds of the mpileup gather (k_mp_gather), byte for byte against the oracle.

The gather takes a 32-column group's read slice 32 positions per round: lane l holds position t0 + l, a ballot gives the
rows of the reads that reach the group, their entries arrive in the rows through cp.async, and a longer slice loops.
Each case below is its own small contig, so that its text fits the shared-memory budget that the engine sizes from the
average tile:
  stack<N>  N reads starting at the first column of the contig's second group (the first is empty), N in
            {1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 2000}: the slice holds exactly N reads.  Lengths 1 .. 32 (8 .. 32
            for 2000), so "^" sits on the group's first column and "$" on every column up to its last; both strands;
            reads with an insertion or a deletion (second entry array) at slice positions 0, 31, 32, 63, 64 and 65.
  pmax      a long read raises the running maximum end, so the slice starts with it and also holds reads that end before
            the group: they get no row.  Such reads sit on both sides of the round edges at positions 32, 64 and 128.
  reach     deletions and N skips longer than 512 bases over a stacked group: far-reaching reads (listed ahead of the
            slice proper), plus one that starts inside the reach window.
Compared as `mpileup -a` at -Q 0 and -Q 13, with -s, and with a FASTA (-B -f), with the engine created under the
default environment, with the direct-to-HBM path for every tile (B200_PLP_SMEM_TEXT=1024) and with a budget large enough
for the 2000-read stack (B200_PLP_SMEM_TEXT=196608)."""
import subprocess
import numpy as np
import pytest
from test_gpu_parity import _same

pytestmark = pytest.mark.gpu

M, I, D, N, S = 0, 1, 2, 3, 4
STACKS = [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 2000]
E2_AT = (0, 31, 32, 63, 64, 65)
ENVS = {'default': {}, 'direct': {'B200_PLP_SMEM_TEXT': '1024'},
        'wide': {'B200_PLP_SMEM_TEXT': '196608'}}
CONFS = [(['-Q', '0'], {'min_baseQ': 0}, False), (['-Q', '13'], {'min_baseQ': 13}, False),
         (['-s'], {'out_mapq': 1}, False), (['-B', '-f', 'ref.fa'], {}, True)]


def _read(rng, pos, cig, rev=None):
    lens = np.array([n for n, _ in cig], np.int64); ops = np.array([o for _, o in cig], np.int64)
    lq = int(lens[np.isin(ops, (M, I, S))].sum())
    seq = np.frombuffer(b'ACGTN', np.uint8)[rng.choice(5, size=lq, p=[0.24, 0.24, 0.24, 0.24, 0.04])].copy()
    rev = bool(rng.integers(0, 2)) if rev is None else rev
    return dict(pos=int(pos), lens=lens, ops=ops, flag=16 if rev else 0, name=None, mapq=int(rng.integers(0, 61)),
                seq=seq, qual=rng.integers(0, 41, size=lq).astype(np.uint8))


def _indel_cigar(rng, span, k):
    """a cigar over `span` reference columns with one insertion (k even) or deletion (k odd) inside"""
    span = max(span, 4)
    a = int(rng.integers(1, span - 2))
    return [(a, M), (int(rng.integers(1, 4)), I), (span - a, M)] if k % 2 == 0 else [(a, M), (2, D), (span - a - 2, M)]


def _stack(rng, n, g):
    lo, hi = (8, 32) if n > 1000 else (1, 32)
    recs = []
    for t in range(n):
        span = lo + (t * 7) % (hi - lo + 1)
        cig = _indel_cigar(rng, span, t) if t in E2_AT else [(span, M)]
        if t % 5 == 3 and t not in E2_AT:          # soft clips keep a read simple
            cig = [(2, S)] + cig + [(1, S)]
        recs.append(_read(rng, g, cig))
    return recs


def _pmax(rng, g):
    recs = [_read(rng, g - 400, [(450, M)])]        # slice position 0: raises the running maximum end past g
    dead = {30, 31, 32, 33, 34, 62, 63, 64, 65, 66, 96, 97, 126, 127, 128, 129}
    for j in range(140):
        t = 1 + j
        p = g - 100 + (j * 100) // 140
        if t in dead:
            cig = [(g - p - int(rng.integers(0, g - p)), M)]                 # ends at or before g: no row
        elif t % 9 == 4:
            cig = _indel_cigar(rng, g - p + int(rng.integers(1, 40)), t)
        else:
            cig = [(g - p + int(rng.integers(1, 40)), M)]
        recs.append(_read(rng, p, cig))
    return recs + _stack(rng, 10, g)


def _reach(rng, g):
    recs = [_read(rng, 0, [(20, M), (1100, N), (20, M)]), _read(rng, 100, [(30, M), (950, D), (30, M)]),
            _read(rng, 300, [(10, M), (700, N), (40, M)]), _read(rng, g - 544, [(20, M), (600, D), (10, M)]),
            _read(rng, g - 400, [(20, M), (500, N), (20, M)])]   # the last starts within reach: in the slice proper
    return recs + _stack(rng, 70, g)


def _cases():
    rng = np.random.default_rng(23)
    out = [(f'stack{n}', 128, _stack(rng, n, 32)) for n in STACKS]
    out.append(('pmax', 640, _pmax(rng, 512)))
    out.append(('reach', 1280, _reach(rng, 1024)))
    return out


@pytest.fixture(scope='module')
def gather_cases(tmp_path_factory):
    from samtools_b200 import synth
    out = []
    for name, length, recs in _cases():
        ref = synth.make_reference(length, seed=len(recs))
        soa = synth._pack(recs, ref, length, 0, 'chr1')
        d = tmp_path_factory.mktemp('gather_' + name)
        synth.write_sam(str(d / 'g.sam'), soa)
        synth.write_fasta(str(d / 'ref.fa'), 'chr1', ref)
        out.append((name, d, soa))
    return out


def _oracle(oracle_bin, d, *args):
    return subprocess.run([oracle_bin, *args], cwd=d, capture_output=True, check=True).stdout


@pytest.mark.parametrize('env', list(ENVS))
def test_gather_slice_rounds(gather_cases, oracle_bin, env, monkeypatch):
    from samtools_b200 import engine
    for k, v in ENVS[env].items():
        monkeypatch.setenv(k, v)
    e = engine.Engine(0)                                # the variables are read here
    try:
        for name, d, soa in gather_cases:
            for args, kw, with_ref in CONFS:
                want = _oracle(oracle_bin, d, 'mpileup', '-a', *args, 'g.sam')
                s = dict(soa)
                if not with_ref:
                    s['ref'] = None
                e.stage(s, engine.default_stage_conf(engine.MODE_MPILEUP, **({'baq': 0} if with_ref else {})))
                _same(e.mpileup_text(all=1, **kw), want, f'{name}, {env}, mpileup -a ' + ' '.join(args))
    finally:
        e.close()
