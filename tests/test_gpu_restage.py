"""b200_restage repeats the read stage on the device-resident batch.  Before it does, it undoes what the previous stage
edited in the qualities: everything after BAQ, -6 or a new upload (a full copy from the pristine image), only the mates of
the overlapping pairs after the overlap tweak, nothing when no stage wrote to them.  Every restage must give what a fresh
b200_stage of the same batch gives: text, qualities, mapq and per-read verdicts, counts, depth and coverage."""
import ctypes as C
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

REPEATS = 5


def _region(seed, paired=True, seq_star=0):
    """300 kb at 30x of 175 bp pairs: with inserts of 400 +- 50 about 16 % of the pairs overlap; 4 % of the reads have
    an insertion and 4 % a deletion, so both the per-position and the lock-step tweak run.  seq_star: that many second
    mates of overlapping pairs lose their sequence (l_qseq 0, SEQ '*'), whose CIGAR walk the tweak still follows."""
    from samtools_b200 import synth
    soa = synth.make_region(300_000, read_len=175, seed=seed, chunk=100_000, with_ref=True, paired=paired,
                            frac_ins=0.04, frac_del=0.04)
    if seq_star:
        pick = np.random.default_rng(seed).choice(_overlapping_second_mates(soa)[0], seq_star, replace=False)
        soa['l_qseq'] = soa['l_qseq'].copy(); soa['l_qseq'][pick] = 0
    return soa


def _overlapping_second_mates(soa):
    """(second mates that start before their first mate ends, number of pairs)"""
    from samtools_b200 import synth
    second = np.nonzero(soa['prev_same_name'] >= 0)[0]
    end = soa['pos'] + synth.ref_span(soa)
    return second[soa['pos'][second] < end[soa['prev_same_name'][second]]], len(second)


def _overlap_fraction(soa):
    over, pairs = _overlapping_second_mates(soa)
    return len(over) / pairs if pairs else 0.0


def _conf(mode=None, **kw):
    from samtools_b200 import engine
    kw.setdefault('baq', 0)
    return engine.default_stage_conf(engine.MODE_MPILEUP if mode is None else mode, **kw)


def _stats(st):
    return tuple(getattr(st, k) for k, _ in st._fields_)


def _outputs(e, soa):
    """everything a caller can read back of the read stage and the mpileup column stage"""
    n = len(soa['pos'])
    mapq, keep = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    assert e.lib.b200_fetch_mapq_keep(e.h, mapq.ctypes.data_as(C.c_void_p), keep.ctypes.data_as(C.c_void_p), n) == 0
    return {'text': e.mpileup_text(all=1), 'qual': e.fetch_qual(len(soa['qual'])), 'mapq': mapq, 'keep': keep,
            'counts': e.mpileup_counts(min_baseQ=13)}


def _fresh(soa, conf, out=_outputs):
    from samtools_b200 import engine
    e = engine.Engine(0)
    st = e.stage(soa, conf)
    got = out(e, soa)
    e.close()
    return _stats(st), got


def _same(got, want, what):
    assert got.keys() == want.keys()
    for k in want:
        if isinstance(want[k], np.ndarray):
            assert np.array_equal(got[k], want[k]), f'{what}: {k} differs'
        else:
            assert got[k] == want[k], f'{what}: {k} differs'


@pytest.fixture(scope='module')
def region():
    soa = _region(7, seq_star=40)
    assert 0.10 < _overlap_fraction(soa) < 0.25
    return soa


@pytest.mark.parametrize('kw', [{}, {'baq': 1}, {'illumina13': 1}, {'capq_thres': 50}, {'overlaps': 0}],
                         ids=['overlap_tweak', 'baq', 'illumina13', 'capq50', 'no_overlap'])
def test_restage_matches_fresh_stage(region, kw):
    """five restages in a row, each equal to a fresh stage: the first restage after the upload takes the full copy, the
    next ones whatever the previous restage left (pairs to restore, nothing, or the full copy again)"""
    from samtools_b200 import engine
    conf = _conf(**kw)
    st_want, want = _fresh(region, conf)
    e = engine.Engine(0); e.set_keep_raw(True)
    assert _stats(e.stage(region, conf)) == st_want
    _same(_outputs(e, region), want, 'stage')
    for k in range(REPEATS):
        assert _stats(e.restage()) == st_want
        _same(_outputs(e, region), want, f'restage {k}')
    e.close()


@pytest.mark.parametrize('first,then', [({}, {'baq': 1}), ({'baq': 1}, {}), ({}, {'capq_thres': 50})],
                         ids=['tweak_then_baq', 'baq_then_tweak', 'tweak_then_capq'])
def test_restage_after_new_stage(region, first, then):
    """a b200_stage with another conf (same batch) uploads the qualities again: the restages after it start over from the
    pristine image, not from the pairs the earlier conf's tweak listed"""
    from samtools_b200 import engine
    e = engine.Engine(0); e.set_keep_raw(True)
    e.stage(region, _conf(**first)); e.restage(); e.restage()
    st_want, want = _fresh(region, _conf(**then))
    assert _stats(e.stage(region, _conf(**then))) == st_want
    for k in range(3):
        assert _stats(e.restage()) == st_want
        _same(_outputs(e, region), want, f'restage {k}')
    e.close()


def test_restage_after_new_batch(region):
    """a new batch replaces the pairs list of the old one: its restages must not restore by the old list"""
    from samtools_b200 import engine
    other = _region(8)
    conf = _conf()
    e = engine.Engine(0); e.set_keep_raw(True)
    e.stage(region, conf); e.restage()
    st_want, want = _fresh(other, conf)
    assert _stats(e.stage(other, conf)) == st_want
    for k in range(3):
        assert _stats(e.restage()) == st_want
        _same(_outputs(e, other), want, f'restage {k}')
    e.close()


def test_restage_without_overlapping_pairs():
    """unpaired reads: the tweak runs and lists no pair, so the restore has a count of 0"""
    from samtools_b200 import engine
    soa = _region(9, paired=False)
    assert _overlap_fraction(soa) == 0.0
    conf = _conf()
    st_want, want = _fresh(soa, conf)
    e = engine.Engine(0); e.set_keep_raw(True)
    e.stage(soa, conf)
    for k in range(REPEATS):
        assert _stats(e.restage()) == st_want
        _same(_outputs(e, soa), want, f'restage {k}')
    e.close()


def _depth_out(e, soa):
    return {'text': e.depth_text(all=1)}


def _cov_out(e, soa):
    return {'sums': e.coverage(min_baseQ=0, min_depth=1)}


@pytest.mark.parametrize('mode,kw,out', [('depth', {}, _depth_out), ('depth', {'d_remove_overlaps': 1}, _depth_out),
                                         ('coverage', {}, _cov_out)], ids=['depth', 'depth_s', 'coverage'])
def test_restage_other_modes(region, mode, kw, out):
    from samtools_b200 import engine
    m = {'depth': engine.MODE_DEPTH, 'coverage': engine.MODE_COVERAGE}[mode]
    conf = engine.default_stage_conf(m, **kw)
    st_want, want = _fresh(region, conf, out)
    e = engine.Engine(0); e.set_keep_raw(True)
    e.stage(region, conf)
    for k in range(3):
        assert _stats(e.restage()) == st_want
        _same(out(e, region), want, f'{mode} restage {k}')
    e.close()
