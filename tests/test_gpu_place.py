"""Line sizing and tile placement of the default mpileup path (k_mp_place), byte for byte against the general path and the oracle.

k_mp_place stages 2048 columns per block in shared memory and takes them in eight rounds of 256; it scans the coverage
difference array into n_plp with one decoupled look-back and the line lengths into the 128-column tile offsets with a second
one; the block that owns the last tile writes the text length.  The cases aim at its edges:
  widths   windows of 1, 127, 128, 129, 1023 .. 1025, 2047 .. 2049 and 32 * 1024 + 1 columns, at the contig start and inside it
  digits   windows with beg > 0 in which the position goes from 9999 to 10000 and from 99999 to 100000 mid-block
  deep     stacks of reads that start just before a block edge and end just after it (or one block further): n_plp in the
           thousands carried from block to block, and blocks whose coverage-difference total is negative
  gaps     runs of empty blocks between two covered stretches and after them, and a window without any read
  big      one window of several thousand blocks
  bed      a BED region whose intervals cross block and tile edges, single positions included
Every case runs as `mpileup -a`, `mpileup -a -s` and `mpileup` (no -a), on the default path, on the default path with
every tile formatted straight into HBM (B200_PLP_SMEM_TEXT=1024) and on the general path (B200_PLP_GENERAL=1).  Each text
must equal the oracle's, its returned length the text length, and stay within b200_mpileup_text_bound."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from test_gpu_parity import _same
from test_gpu_gather import _read, M

pytestmark = pytest.mark.gpu

ENVS = {'default': {}, 'direct': {'B200_PLP_SMEM_TEXT': '1024'}, 'general': {'B200_PLP_GENERAL': '1'}}
CONFS = [(['-a'], {'all': 1}), (['-a', '-s'], {'all': 1, 'out_mapq': 1}), ([], {})]
WIDTHS = [1, 127, 128, 129, 1023, 1024, 1025, 2047, 2048, 2049, 32 * 1024 + 1]
BLOCK = 2048


def _deep(rng):
    """about 2500 reads over each block edge: starts 1 .. 6 columns before it, ends 1 .. 60 columns after it or one block on"""
    length = 8 * BLOCK + 300
    recs = []
    for k in range(1, 8):
        edge = k * BLOCK
        for j in range(2500):
            p = edge - 1 - j % 6
            end = edge + 1 + (j * 7) % 60 + (BLOCK if j % 11 == 0 else 0)
            recs.append(_read(rng, p, [(min(end, length) - p, M)]))
    return length, recs


def _gaps(rng):
    """reads only in [0, 3000) and [20000, 23000) of a 40 kb contig"""
    length = 40_000
    recs = []
    for lo in (0, 20_000):
        for j in range(600):
            p = lo + int(rng.integers(0, 3000 - 150))
            cig = [(150, M)] if j % 13 else [(60, M), (2, 2), (88, M)]
            recs.append(_read(rng, p, cig))
    return length, recs


@pytest.fixture(scope='module')
def place_cases(tmp_path_factory, oracle_bin):
    """name -> (directory, soa, {oracle args: text}); the oracle runs once per contig and configuration"""
    from samtools_b200 import synth
    rng = np.random.default_rng(41)
    contigs = {'base': synth.make_batch(length=140_000, depth=12, seed=31),
               'big': synth.make_batch(length=6_200_000, depth=2, seed=37)}
    for name, (length, recs) in (('deep', _deep(rng)), ('gaps', _gaps(rng))):
        ref = synth.make_reference(length, seed=len(recs))
        contigs[name] = synth._pack(recs, ref, length, 0, 'chr1')
    out = {}
    for name, soa in contigs.items():
        d = tmp_path_factory.mktemp('place_' + name)
        synth.write_sam(str(d / 'p.sam'), soa)
        s = dict(soa); s['ref'] = None
        want = {}
        for args, _ in CONFS:
            want[tuple(args)] = subprocess.run([oracle_bin, 'mpileup', *args, 'p.sam'], cwd=d, capture_output=True, check=True).stdout
        out[name] = (d, s, want)
    return out


class _Engines:
    """one engine per entry of ENVS (each reads its environment when it is created)"""
    def __enter__(self):
        from samtools_b200 import engine
        self.e = {}
        for name, env in ENVS.items():
            old = {k: os.environ.get(k) for k in env}
            os.environ.update(env)
            try:
                self.e[name] = engine.Engine(0)
            finally:
                for k, v in old.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
        return self.e

    def __exit__(self, *exc):
        for e in self.e.values():
            e.close()


def _check(engines, soa, sconf, kw, want, what, bed=None):
    """stage on every engine and compare; bed: (beg, end) int64 arrays of disjoint sorted 0-based intervals"""
    from samtools_b200 import engine
    for env, e in engines.items():
        e.stage(soa, sconf)
        conf = engine.mpileup_conf(**kw)
        if bed is not None:
            conf.bed_beg, conf.bed_end = bed[0].ctypes.data, bed[1].ctypes.data
            conf.n_bed, conf.bed_active = len(bed[0]), 1
        got = e.mpileup_text(conf)
        _same(got, want, f'{what}, {env}')
        n = e.mpileup_text(conf, fetch=False)
        e.lib.b200_mpileup_text_bound.restype = C.c_uint64
        bound = e.lib.b200_mpileup_text_bound(e.h, C.byref(conf))
        assert n == len(got) <= bound, f'{what}, {env}: length {n}, text {len(got)}, bound {bound}'


def _index(text):
    """1-based position and starting byte offset of every line"""
    lines = text.split(b'\n')[:-1]
    pos = np.array([int(l.split(b'\t', 2)[1]) for l in lines], np.int64)
    off = np.concatenate([[0], np.cumsum([len(l) + 1 for l in lines], dtype=np.int64)])
    return pos, off


def _slice(text, index, beg, end):
    """the lines of the 0-based columns [beg, end)"""
    pos, off = index
    a, b = np.searchsorted(pos, beg + 1), np.searchsorted(pos, end + 1)
    return text[off[a]:off[b]]


def _windows(place_cases, name, wins):
    from samtools_b200 import engine, shard
    d, soa, want = place_cases[name]
    idx = {k: _index(t) for k, t in want.items()}
    with _Engines() as engines:
        for beg, end in wins:
            s = shard.select_window(soa, beg, end)
            sconf = engine.default_stage_conf(engine.MODE_MPILEUP, beg=beg, end=end)
            for args, kw in CONFS:
                w = _slice(want[tuple(args)], idx[tuple(args)], beg, end)
                _check(engines, s, sconf, kw, w, f'{name} [{beg}, {end}) mpileup ' + ' '.join(args))


def _whole(place_cases, name):
    from samtools_b200 import engine
    d, soa, want = place_cases[name]
    with _Engines() as engines:
        for args, kw in CONFS:
            _check(engines, soa, engine.default_stage_conf(engine.MODE_MPILEUP), kw, want[tuple(args)], f'{name} mpileup ' + ' '.join(args))


def test_place_window_widths(place_cases):
    _windows(place_cases, 'base', [(b, b + w) for b in (0, 70_001) for w in WIDTHS])


def test_place_digit_changes(place_cases):
    _windows(place_cases, 'base', [(9_500, 11_500), (99_300, 100_800)])


def test_place_deep_block_edges(place_cases):
    _whole(place_cases, 'deep')
    _windows(place_cases, 'deep', [(BLOCK - 3, 3 * BLOCK + 5), (2 * BLOCK + 1, 5 * BLOCK)])


def test_place_empty_blocks(place_cases):
    _whole(place_cases, 'gaps')
    _windows(place_cases, 'gaps', [(5_000, 5_000 + 2 * BLOCK + 1), (2_000, 21_000)])


def test_place_several_thousand_blocks(place_cases):
    _whole(place_cases, 'big')


def test_place_bed_region(place_cases, oracle_bin):
    from samtools_b200 import engine
    d, soa, _ = place_cases['base']
    iv = [(0, 1), (1_000, 1_030), (2_040, 4_100), (10_200, 10_201), (50_000, 83_000), (139_000, 140_000)]
    (d / 'r.bed').write_text(''.join(f'chr1\t{a}\t{b}\n' for a, b in iv))
    bed = (np.array([a for a, _ in iv], np.int64), np.array([b for _, b in iv], np.int64))
    with _Engines() as engines:
        for args, kw in CONFS:
            want = subprocess.run([oracle_bin, 'mpileup', *args, '-l', 'r.bed', 'p.sam'], cwd=d, capture_output=True, check=True).stdout
            _check(engines, soa, engine.default_stage_conf(engine.MODE_MPILEUP), kw, want, 'base, BED, mpileup ' + ' '.join(args), bed)
