"""Long reads through the CUDA path (the inputs of tests/test_longread.py), byte for byte against the oracle: the C ABI per
contig (BAQ on multi-chunk bands and 40-kb reads, long mate overlaps, far-reaching read lists, GL at every column), the
BAQ warp kernel against the register kernel, the CLI on SAM and BAM (CG:B,I), a deletion whose mpileup entry is longer
than 64 KiB through the shared-memory gather, and the iterator tier with windows cutting long reads."""
import os, subprocess
import numpy as np
import pytest
from conftest import ROOT
from test_longread import write_long_inputs, run_cases, LONG_CASES
from test_fuzz_emul import run_all

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')


@pytest.fixture(scope='module')
def long_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp('glong')
    return d, write_long_inputs(d)


def _oracle(oracle_bin, d, *args):
    return subprocess.run([oracle_bin, *args], cwd=d, capture_output=True, check=True).stdout


def _engine_text(soas, conf_kw, text_kw, what='mpileup', env=None):
    """one engine handle (created under `env`), every contig staged in turn, texts concatenated"""
    from samtools_b200 import engine
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        e = engine.Engine(0)
    finally:
        for k, v in old.items():
            if v is None: os.environ.pop(k)
            else: os.environ[k] = v
    out = []
    mode = engine.MODE_MPILEUP if what == 'mpileup' else engine.MODE_DEPTH
    for s in soas:
        e.stage(s, engine.default_stage_conf(mode, **conf_kw))
        out.append(e.mpileup_text(**text_kw) if what == 'mpileup' else e.depth_text(**text_kw))
    e.close()
    return b''.join(out)


def _same(got, want, what):
    from test_gpu_parity import _same as same
    assert len(want) > 1000, what
    same(got, want, what)


@pytest.mark.parametrize('conf,text,args', [
    ({}, {}, ['mpileup', '-f', 'long.fa', 'long.sam']),
    ({'baq': 2}, {}, ['mpileup', '-E', '-f', 'long.fa', 'long.sam']),
    ({}, {'all': 1, 'out_mapq': 1}, ['mpileup', '-a', '-s', '-f', 'long.fa', 'long.sam']),
    ({'baq': 0}, {'all': 1, 'min_baseQ': 0}, ['mpileup', '-B', '-a', '-Q', '0', '-f', 'long.fa', 'long.sam']),
], ids=['f', 'E', 'a_s', 'B_a_Q0'])
def test_cabi_mpileup_long(conf, text, args, long_dir, oracle_bin):
    d, soas = long_dir
    _same(_engine_text(soas, conf, text), _oracle(oracle_bin, d, *args), ' '.join(args))


def test_baq_warp_kernel_matches_register_kernel(long_dir, oracle_bin, tmp_path):
    """B200_BAQ_REG=0 sends every read to k_baq: same text as the default split and as the oracle, on the long set and on
    BASELINE C2 (200 000 band-7 150-bp reads through k_baq)"""
    from samtools_b200 import synth
    d, soas = long_dir
    want = _oracle(oracle_bin, d, 'mpileup', '-f', 'long.fa', 'long.sam')
    a = _engine_text(soas, {}, {})
    b = _engine_text(soas, {}, {}, env={'B200_BAQ_REG': '0'})
    _same(a, want, 'long, default'); _same(b, want, 'long, B200_BAQ_REG=0')
    c2 = synth.make_batch(length=1_000_000, depth=30, seed=2)
    sam, fa = str(tmp_path / 'c2.sam'), str(tmp_path / 'c2.fa')
    synth.write_sam(sam, c2); synth.write_fasta(fa, c2['tid_name'], c2['ref_full'])
    want = _oracle(oracle_bin, tmp_path, 'mpileup', '-f', fa, sam)
    a = _engine_text([c2], {}, {})
    b = _engine_text([c2], {}, {}, env={'B200_BAQ_REG': '0'})
    _same(a, want, 'C2, default'); _same(b, want, 'C2, B200_BAQ_REG=0')


def test_cabi_depth_coverage_gl_long(long_dir, oracle_bin):
    from samtools_b200 import engine
    d, soas = long_dir
    _same(_engine_text(soas, {}, {'all': 1}, 'depth'), _oracle(oracle_bin, d, 'depth', '-a', 'long.sam'), 'depth -a')
    _same(_engine_text(soas, {'d_remove_overlaps': 1}, {}, 'depth'), _oracle(oracle_bin, d, 'depth', '-s', 'long.sam'), 'depth -s')
    rows = _oracle(oracle_bin, d, 'coverage', 'long.sam').split(b'\n')[1:-1]
    gl = _oracle(oracle_bin, d, 'gl', '-B', '-f', 'long.fa', 'long.sam').decode().split('\n')[:-1]
    e = engine.Engine(0)
    k = 0
    for s, row in zip(soas, rows):
        row = row.split(b'\t')
        st = e.stage(s, engine.default_stage_conf(engine.MODE_COVERAGE, rflag_filter=4 | 256 | 512 | 1024, end=s['tid_len']))
        cv = e.coverage(min_baseQ=0, min_depth=1)
        L = float(s['tid_len'])
        assert int(row[3]) == st.n_selected_reads and int(row[4]) == cv['n_covered_bases']
        assert row[5] == (b'%g' % (100.0 * cv['n_covered_bases'] / L)) and row[6] == (b'%g' % (cv['summed_coverage'] / L))
        st = e.stage(s, engine.default_stage_conf(engine.MODE_MPILEUP, baq=0))
        pos, n, qs, p25 = e.glf(13, int(st.n_cols) + 16)
        mine = [l for l in gl if l.split('\t', 1)[0] == s['tid_name']]
        assert len(mine) == len(pos) > 1000
        want = np.array([[np.float32(x) for x in l.split('\t')[3:33]] for l in mine], dtype=np.float32)
        assert (np.array([int(l.split('\t')[1]) for l in mine]) == pos + 1).all()
        assert (np.maximum(n[:, 0], 0) == want[:, 0].astype(np.int64)).all()
        assert (qs[:, 0, :] == want[:, 1:5]).all() and (p25[:, 0, :] == want[:, 5:30]).all()
        k += 1
    e.close()
    assert k == 2


def test_read_ops_long(long_dir):
    """sam_prob_realn (flags 3, 1, 0, 2) on every long read through the per-read launch path"""
    d, _ = long_dir
    exe = os.path.join(ROOT, 'tests', 'compat', '_build', 'read_ops_check')
    r = subprocess.run([exe, str(d / 'long.sam'), str(d / 'long.fa'), '100000'], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


CLI_CASES = [('mpileup', '-f long.fa long.sam'), ('mpileup', '-f long.fa long.bam'), ('mpileup', '-f cg.fa cg.bam'),
             ('depth', '-a long.sam'), ('depth', '-a long.bam'), ('depth', '-a cg.bam'), ('coverage', 'long.sam'), ('coverage', 'cg.bam')]


@pytest.mark.parametrize('env', [{}, {'B200_WINDOW_COLS': '4099'}, {'B200_DEVICES': '0,0'}], ids=['default', 'win4099', 'devices00'])
def test_cli_long(env, long_dir, oracle_bin):
    d, _ = long_dir
    bad = run_cases(CLI, oracle_bin, d, CLI_CASES, env)
    assert not bad, bad[:3]


def test_cli_long_noBAQ_options(long_dir, oracle_bin):
    d, _ = long_dir
    bad = run_cases(CLI, oracle_bin, d, LONG_CASES)
    assert not bad, bad[:3]


@pytest.mark.parametrize('env', [{}, {'B200_PLP_SMEM_TEXT': '204000'}, {'B200_PLP_SMEM_TEXT': '204000', 'B200_PLP_GENERAL': '1'}],
                         ids=['default', 'smem204000', 'general'])
def test_entry_longer_than_64k(env, long_dir, oracle_bin):
    """a 70 000-base deletion: its mpileup entry carries 70 000 deleted reference bases.  The tile's shared-memory text budget
    is 9/8 of the average tile's bound, at most B200_PLP_SMEM_TEXT: with a region of a few dozen columns around the deletion
    the average tile is that one tile, so with the raised budget it goes through the shared-memory gather, whose cursor must
    not wrap at 16 bits (the whole-contig runs format it straight into HBM)"""
    d, _ = long_dir
    for args in ('-B -f del.fa del.sam', '-B -Q 0 del.sam', '-B -a -s -f del.fa del.sam', '-B -r chr1:10280-10330 -f del.fa del.sam',
                 '-B -Q 0 -r chr1:10295-10305 del.sam', '-B -s -r chr1:10290-10310 -f del.fa del.sam'):
        bad = run_cases(CLI, oracle_bin, d, [('mpileup', args)], env)
        assert not bad, bad
    want = _oracle(oracle_bin, d, 'mpileup', '-B', '-f', 'del.fa', 'del.sam')
    assert max(len(l) for l in want.split(b'\n')) > 70_000


def test_iterator_tier_long_windows(long_dir, oracle_bin, monkeypatch):
    d, _ = long_dir
    monkeypatch.setenv('B200_PLP_WINDOW_BYTES', '262144')
    exe = os.path.join(ROOT, 'tests', 'compat', '_build', 'plp_dump')
    for files in (['long.sam'], ['long.sam', 'long2.sam'], ['cg.bam']):
        paths = [str(d / f) for f in files]
        got = subprocess.run([exe, *paths], capture_output=True)
        want = subprocess.run([oracle_bin, 'pileup-dump', *paths], capture_output=True)
        assert got.returncode == 0, got.stderr[-300:]
        assert got.stdout == want.stdout and len(want.stdout) > 1000, files
