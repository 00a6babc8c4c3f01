"""GPU parity tests: the CUDA path, through the C ABI / the CLI, against
(1) every golden vector of the reference's test-suite, (2) the CPU oracle on
seeded synthetic batches, (3) size-independent properties at BASELINE C2 size."""
import hashlib, os, subprocess
import numpy as np
import pytest
import golden_cases
from conftest import ROOT

pytestmark = pytest.mark.gpu
CASES = golden_cases.all_cases()
CLI = os.environ.get('B200_TEST_CLI') or os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')


@pytest.fixture(scope='module')
def cli():
    assert os.path.exists(CLI), 'samtools_b200/bin/b200samtools missing: run python samtools_b200/build.py'
    return CLI


@pytest.fixture(scope='module')
def golden_results(cli, oracle_bin, corpus):
    """All golden command lines, run once up front with a few processes in flight (each CLI process pays ~1 s of CUDA
    context creation; serially the 160+ cases take four minutes).  Lines that write a scratch file into the corpus
    directory (`sed ... > sample1.sam; ...`) run one at a time afterwards.  Results are checked per case below."""
    from concurrent.futures import ThreadPoolExecutor

    def run(c):
        try:
            return golden_cases.run_case(c, cli, oracle_bin, corpus)
        except Exception as e:          # timeout etc.: reported by the case's own test
            return e
    todo = [c for c in CASES if not c['skip']]
    par = [c for c in todo if '>' not in c['cmd']]
    ser = [c for c in todo if '>' in c['cmd']]
    res = {}
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        for c, r in zip(par, ex.map(run, par)):
            res[c['id']] = r
    for c in ser:
        res[c['id']] = run(c)
    return res


@pytest.mark.parametrize('case', CASES, ids=[c['id'] for c in CASES])
def test_reference_golden_on_gpu(case, golden_results):
    if case['skip']:
        pytest.skip(case['skip'])
    r = golden_results[case['id']]
    if isinstance(r, Exception):
        raise r
    ok, out, err = r
    if not ok and b'not available on the device path' in err:
        pytest.skip('--output-extra/QNAME/mods: host-string columns not on the device path yet')
    assert ok, f"{case['cmd']}\nstderr: {err[-400:]!r}\nstdout head: {out[:300]!r}"


def test_column_windows_on_gpu(cli, oracle_bin, corpus, monkeypatch):
    """the drivers' column windows (halo reads staged again, tests/test_emul_golden.py::test_column_windows_with_halo) through
    the CUDA engine: every golden case with 97-column windows, BAQ included"""
    from concurrent.futures import ThreadPoolExecutor
    monkeypatch.setenv('B200_WINDOW_COLS', '97')
    todo = [c for c in CASES if not c['skip'] and '>' not in c['cmd']]

    def run(c):
        ok, out, err = golden_cases.run_case(c, cli, oracle_bin, corpus)
        if not ok and b'not available on the device path' in err:
            return None
        return None if ok else (c['id'], c['cmd'], err[-200:])
    with ThreadPoolExecutor(max_workers=6) as ex:
        bad = [r for r in ex.map(run, todo) if r]
    assert not bad, bad[:3]


# ---------------------------------------------------------------- synthetic, C ABI vs oracle
@pytest.fixture(scope='module')
def synth_set(tmp_path_factory, oracle_bin):
    from samtools_b200 import synth
    td = tmp_path_factory.mktemp('synth')
    soa = synth.make_batch(length=60_000, depth=30, seed=7)
    sam, fa = str(td / 's.sam'), str(td / 's.fa')
    synth.write_sam(sam, soa); synth.write_fasta(fa, soa['tid_name'], soa['ref_full'])
    return dict(soa=soa, sam=sam, fa=fa, oracle=oracle_bin)


@pytest.fixture(scope='module')
def eng():
    from samtools_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()


def oracle_out(s, *args):
    return subprocess.run([s['oracle'], *args], capture_output=True, check=True).stdout


def noref(soa):
    d = dict(soa); d['ref'] = None
    return d


def test_mpileup_a_noref(synth_set, eng):
    from samtools_b200 import engine
    eng.stage(noref(synth_set['soa']), engine.default_stage_conf(engine.MODE_MPILEUP))
    assert eng.mpileup_text(all=1) == oracle_out(synth_set, 'mpileup', '-a', synth_set['sam'])


def test_mpileup_noBAQ_ref_options(synth_set, eng):
    from samtools_b200 import engine
    eng.stage(synth_set['soa'], engine.default_stage_conf(engine.MODE_MPILEUP, baq=0, overlaps=0, min_mq=20))
    got = eng.mpileup_text(min_baseQ=20, out_mapq=1, out_qpos=1, out_qpos5=1, rev_del=1)
    want = oracle_out(synth_set, 'mpileup', '-B', '-x', '-q', '20', '-Q', '20', '-s', '-O', '--output-BP-5', '--reverse-del',
                      '-f', synth_set['fa'], synth_set['sam'])
    assert got == want


def test_mpileup_BAQ_overlap(synth_set, eng):
    from samtools_b200 import engine
    eng.stage(synth_set['soa'], engine.default_stage_conf(engine.MODE_MPILEUP))
    assert eng.mpileup_text() == oracle_out(synth_set, 'mpileup', '-f', synth_set['fa'], synth_set['sam'])


def test_mpileup_capq(synth_set, eng):
    from samtools_b200 import engine
    eng.stage(synth_set['soa'], engine.default_stage_conf(engine.MODE_MPILEUP, baq=0, capq_thres=50))
    assert eng.mpileup_text() == oracle_out(synth_set, 'mpileup', '-B', '-C', '50', '-f', synth_set['fa'], synth_set['sam'])


def test_depth_variants(synth_set, eng):
    from samtools_b200 import engine
    eng.stage(synth_set['soa'], engine.default_stage_conf(engine.MODE_DEPTH))
    assert eng.depth_text(all=1) == oracle_out(synth_set, 'depth', '-a', synth_set['sam'])
    assert eng.depth_text(min_qual=30, count_del=1) == oracle_out(synth_set, 'depth', '-q', '30', '-J', synth_set['sam'])
    eng.stage(synth_set['soa'], engine.default_stage_conf(engine.MODE_DEPTH, d_remove_overlaps=1, d_min_mapq=10))
    assert eng.depth_text() == oracle_out(synth_set, 'depth', '-s', '-Q', '10', synth_set['sam'])


def test_coverage_sums(synth_set, eng):
    from samtools_b200 import engine
    soa = synth_set['soa']
    st = eng.stage(soa, engine.default_stage_conf(engine.MODE_COVERAGE, min_mq=5, end=soa['tid_len']))
    s = eng.coverage(min_baseQ=10, min_depth=2)
    row = oracle_out(synth_set, 'coverage', '-q', '5', '-Q', '10', '--min-depth', '2', synth_set['sam']).split(b'\n')[1].split(b'\t')
    L = float(soa['tid_len'])
    fmt = lambda x, f: (f % x).encode()
    assert int(row[3]) == st.n_selected_reads and int(row[4]) == s['n_covered_bases']
    assert row[5] == fmt(100.0 * s['n_covered_bases'] / L, '%g') and row[6] == fmt(s['summed_coverage'] / L, '%g')
    assert row[7] == fmt(s['summed_baseQ'] / s['quality_bases'], '%.3g') and row[8] == fmt(st.summed_mapq / st.n_selected_reads, '%.3g')


def test_glf_matches_oracle(synth_set, eng):
    from samtools_b200 import engine
    soa = synth_set['soa']
    st = eng.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, baq=0))
    pos, n, qs, p25 = eng.glf(13, int(st.n_cols) + 16)
    lines = oracle_out(synth_set, 'gl', '-B', '-f', synth_set['fa'], synth_set['sam']).decode().split('\n')[:-1]
    assert len(lines) == len(pos)
    for k in range(0, len(lines), max(1, len(lines) // 4000)):
        f = lines[k].split('\t')
        assert int(f[1]) == pos[k] + 1 and int(f[3]) == max(int(n[k, 0]), 0)
        assert [np.float32(x) for x in f[4:8]] == list(qs[k, 0]), (k, f[4:8], qs[k, 0])
        assert [np.float32(x) for x in f[8:33]] == list(p25[k, 0]), (k, f[8:33], p25[k, 0])


def test_pileup_entries_tier(synth_set, eng):
    """bam_pileup1_t fields per column == what the text is built from (depth via entries == depth -a -J style count)."""
    from samtools_b200 import engine
    soa = synth_set['soa']
    eng.stage(noref(soa), engine.default_stage_conf(engine.MODE_MPILEUP, baq=0, overlaps=0))
    col_n, ents = eng.pileup_entries(0, 1000, 3000, 200000)
    assert col_n.sum() == len(ents)
    txt = eng.mpileup_text(min_baseQ=0).split(b'\n')
    depth = {int(l.split(b'\t')[1]): int(l.split(b'\t')[3]) for l in txt if l}
    for i, c in enumerate(range(1000, 3000)):
        assert depth.get(c + 1, 0) == col_n[i]
    assert (ents['qpos'] >= 0).all() and (ents['read'] < len(soa['pos'])).all()


def test_restage_repeats_read_stage(synth_set):
    """b200_restage (device-resident repeat of the read stage, used by bench.py) gives the same bytes as a fresh b200_stage,
    also when the stage edits qualities in place (BAQ, overlap tweak, -C)."""
    from samtools_b200 import engine
    soa = synth_set['soa']
    conf = engine.default_stage_conf(engine.MODE_MPILEUP, capq_thres=50)
    e1 = engine.Engine(0); e1.stage(soa, conf); want = e1.mpileup_text(all=1); e1.close()
    e2 = engine.Engine(0); e2.set_keep_raw(True); e2.stage(soa, conf)
    got0 = e2.mpileup_text(all=1)
    e2.restage(); got1 = e2.mpileup_text(all=1)
    e2.restage(); got2 = e2.mpileup_text(all=1)
    e2.close()
    assert got0 == want and got1 == want and got2 == want


# ---------------------------------------------------------------- full-size properties (BASELINE C2)
def test_c2_size_properties():
    from samtools_b200 import engine, synth
    soa = noref(synth.make_batch(length=1_000_000, depth=30, seed=2))
    digests = {}
    for tag, env in (('default', {}), ('direct', {'B200_PLP_SMEM_TEXT': '1024'}),
                     ('general', {'B200_PLP_GENERAL': '1'}), ('general_direct', {'B200_PLP_GENERAL': '1', 'B200_PLP_SMEM_TEXT': '1024'})):
        os.environ.update(env)
        e = engine.Engine(0)
        e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
        t1 = e.mpileup_text(all=1); t2 = e.mpileup_text(all=1)
        e.close()
        for k in env:
            os.environ.pop(k)
        assert t1 == t2, 'not idempotent'
        digests[tag] = hashlib.sha256(t1).hexdigest()
        if tag == 'default':
            lines = t1.split(b'\n')
            assert len(lines) - 1 == 1_000_000                      # -a: one row per reference position
            assert lines[0].startswith(b'chr1\t1\tN\t') and lines[999_999].startswith(b'chr1\t1000000\tN\t')
            # depth column sums to the number of kept (read, column) pairs that pass -Q13; positions ascend
            pos = np.array([int(l.split(b'\t', 2)[1]) for l in lines[:-1:997]])
            assert (np.diff(pos) > 0).all()
    assert len(set(digests.values())) == 1, digests   # entry-string path / general path, TMA / direct-to-HBM stores all agree


# ---------------------------------------------------------------- BASELINE C2 size, CUDA bytes vs the oracle's bytes
@pytest.fixture(scope='module')
def c2_set(tmp_path_factory, oracle_bin):
    """BASELINE config 2: 1 Mb, 30x, 150 bp (200 000 reads).  The oracle needs ~1 s (-a), ~8 s (-f, BAQ) for it."""
    from samtools_b200 import synth
    td = tmp_path_factory.mktemp('c2')
    soa = synth.make_batch(length=1_000_000, depth=30, seed=2)
    sam, fa = str(td / 'c2.sam'), str(td / 'c2.fa')
    synth.write_sam(sam, soa); synth.write_fasta(fa, soa['tid_name'], soa['ref_full'])
    return dict(soa=soa, sam=sam, fa=fa, oracle=oracle_bin)


def _same(got, want, what):
    if got != want:
        n = min(len(got), len(want))
        a = np.frombuffer(got[:n], np.uint8); b = np.frombuffer(want[:n], np.uint8)
        d = int(np.argmax(a != b)) if (a != b).any() else n
        lo = max(0, d - 120)
        raise AssertionError(f'{what}: first difference at byte {d} of {len(want)} (got {len(got)})\n got: {got[lo:d + 80]!r}\nwant: {want[lo:d + 80]!r}')


def test_c2_mpileup_a_vs_oracle(c2_set, eng):
    from samtools_b200 import engine
    eng.stage(noref(c2_set['soa']), engine.default_stage_conf(engine.MODE_MPILEUP))
    _same(eng.mpileup_text(all=1), oracle_out(c2_set, 'mpileup', '-a', c2_set['sam']), 'mpileup -a (C2, no FASTA)')


def test_c2_mpileup_f_baq_vs_oracle(c2_set, eng):
    """the default mode of `mpileup -f`: BAQ (sam_prob_realn on every read) + mate-overlap tweak, 200 000 reads"""
    from samtools_b200 import engine
    eng.stage(c2_set['soa'], engine.default_stage_conf(engine.MODE_MPILEUP))
    _same(eng.mpileup_text(), oracle_out(c2_set, 'mpileup', '-f', c2_set['fa'], c2_set['sam']), 'mpileup -f (C2, BAQ + overlap)')
    _same(eng.mpileup_text(all=1, out_mapq=1), oracle_out(c2_set, 'mpileup', '-a', '-s', '-f', c2_set['fa'], c2_set['sam']), 'mpileup -a -s -f (C2)')


def test_c2_depth_coverage_vs_oracle(c2_set, eng):
    from samtools_b200 import engine
    soa = c2_set['soa']
    eng.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    _same(eng.depth_text(all=1), oracle_out(c2_set, 'depth', '-a', c2_set['sam']), 'depth -a (C2)')
    st = eng.stage(soa, engine.default_stage_conf(engine.MODE_COVERAGE, rflag_filter=4 | 256 | 512 | 1024, end=soa['tid_len']))
    s = eng.coverage(min_baseQ=0, min_depth=1)
    row = oracle_out(c2_set, 'coverage', c2_set['sam']).split(b'\n')[1].split(b'\t')
    L = float(soa['tid_len'])
    fmt = lambda x, f: (f % x).encode()
    assert int(row[3]) == st.n_selected_reads and int(row[4]) == s['n_covered_bases']
    assert row[5] == fmt(100.0 * s['n_covered_bases'] / L, '%g') and row[6] == fmt(s['summed_coverage'] / L, '%g')
    assert row[7] == fmt(s['summed_baseQ'] / s['quality_bases'], '%.3g') and row[8] == fmt(st.summed_mapq / st.n_selected_reads, '%.3g')


# ---------------------------------------------------------------- BASELINE C4 shape: deep columns -> GL (errmod_cal n > 255)
def test_c4_panel_gl_every_column(tmp_path, oracle_bin, eng):
    """200x targets with 2000x hotspots: every column's n, qsum[4] and p[25] against the oracle, including the columns with
    more than 255 usable bases (ks_shuffle over the hts_drand48 stream, LCG jump-ahead on the device) and the number of
    random draws consumed (the stream position a following call would continue from)."""
    from samtools_b200 import engine, synth
    soa = synth.make_panel(n_targets=12, n_hot=3, seed=4)
    sam, fa = str(tmp_path / 'c4.sam'), str(tmp_path / 'c4.fa')
    synth.write_sam(sam, soa); synth.write_fasta(fa, soa['tid_name'], soa['ref_full'])
    st = eng.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, baq=0))
    d0 = eng.gl_rng_draws
    pos, n, qs, p25 = eng.glf(13, int(st.n_cols) + 16)
    lines = subprocess.run([oracle_bin, 'gl', '-B', '-f', fa, sam], capture_output=True, check=True).stdout.decode().split('\n')[:-1]
    assert len(lines) == len(pos)
    want = np.array([[np.float32(x) for x in l.split('\t')[3:33]] for l in lines], dtype=np.float32)
    wpos = np.array([int(l.split('\t', 2)[1]) for l in lines])
    assert (wpos == pos + 1).all()
    wn = want[:, 0].astype(np.int64)
    assert (wn > 255).sum() > 500 and wn.max() > 1500, 'the panel must exercise the shuffle path'
    assert (np.maximum(n[:, 0], 0) == wn).all()
    assert (qs[:, 0, :] == want[:, 1:5]).all()
    bad = np.nonzero((p25[:, 0, :] != want[:, 5:30]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), int(wpos[bad[0]]), int(wn[bad[0]]), p25[bad[0], 0], want[bad[0], 5:30])
    assert eng.gl_rng_draws - d0 == int((wn[wn > 255] - 1).sum())
    # the text path on the same deep columns (thousands of entries per line)
    _same(eng.mpileup_text(), subprocess.run([oracle_bin, 'mpileup', '-B', '-f', fa, sam], capture_output=True, check=True).stdout, 'mpileup -B -f (C4 panel)')


# ---------------------------------------------------------------- region shards with halo == unsharded (SURVEY 8e)
def _shard_outputs(soa, L, n_shards, devices):
    """stage the `-r` window of every shard (reads overlapping it: the halo) and run the three column stages on it"""
    from samtools_b200 import engine, shard
    mp, dp, cv, nsel = [], [], None, 0
    for k, (beg, end) in enumerate(shard.plan_shards(L, n_shards)):
        e = engine.Engine(devices[k % len(devices)])
        w = shard.select_window(soa, beg, end)
        e.stage(w, engine.default_stage_conf(engine.MODE_MPILEUP, beg=beg, end=end))
        mp.append(e.mpileup_text(all=1))
        e.stage(w, engine.default_stage_conf(engine.MODE_DEPTH, beg=beg, end=end))
        dp.append(e.depth_text(all=1))
        e.stage(w, engine.default_stage_conf(engine.MODE_COVERAGE, rflag_filter=4 | 256 | 512 | 1024, beg=beg, end=end))
        s = e.coverage(min_baseQ=0, min_depth=1)
        cv = s if cv is None else {k_: cv[k_] + s[k_] for k_ in s}
        e.close()
    return b''.join(mp), b''.join(dp), cv


@pytest.mark.parametrize('n_shards', [2, 5])
def test_region_shards_concatenate_to_unsharded(n_shards, tmp_path, oracle_bin):
    """N shards of ONE contig, each staged with the reads that overlap it (bam_plcmd.c:550-554) and clipped to its columns
    (:609): the concatenation is byte-identical to the unsharded run (mpileup -a -f with BAQ and the overlap tweak,
    depth -a) and the coverage sums add up.  Runs sequentially on one GPU and, when the box has several, one shard per device."""
    import torch
    from samtools_b200 import engine, synth
    L = 300_000
    soa = synth.make_batch(length=L, depth=30, seed=5)
    sam, fa = str(tmp_path / 's.sam'), str(tmp_path / 's.fa')
    synth.write_sam(sam, soa); synth.write_fasta(fa, soa['tid_name'], soa['ref_full'])
    want_mp = subprocess.run([oracle_bin, 'mpileup', '-a', '-f', fa, sam], capture_output=True, check=True).stdout
    want_dp = subprocess.run([oracle_bin, 'depth', '-a', sam], capture_output=True, check=True).stdout
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_COVERAGE, rflag_filter=4 | 256 | 512 | 1024, end=L))
    want_cv = e.coverage(min_baseQ=0, min_depth=1)
    e.close()
    dev_sets = [[0]]
    if torch.cuda.device_count() > 1:
        dev_sets.append(list(range(min(torch.cuda.device_count(), n_shards))))
    for devs in dev_sets:
        mp, dp, cv = _shard_outputs(soa, L, n_shards, devs)
        _same(mp, want_mp, f'mpileup -a -f, {n_shards} shards on devices {devs}')
        _same(dp, want_dp, f'depth -a, {n_shards} shards on devices {devs}')
        assert cv == want_cv


# ---------------------------------------------------------------- htslib's per-read / per-column entry points (T1)
def test_htslib_read_ops_vs_oracle(tmp_path, synth_set, corpus):
    """sam_prob_realn (flags 3, 1, 0, 2), sam_cap_mapq, errmod_cal (n up to 3000: the ks_shuffle path), bcf_call_glfgen and
    bam_plp_insertion_mod as exported by libb200pileup.so with htslib's signatures, compared call by call with the oracle
    (tests/compat/read_ops_check.cpp links both)."""
    exe = os.path.join(ROOT, 'tests', 'compat', '_build', 'read_ops_check')
    assert os.path.exists(exe), 'tests/compat/_build/read_ops_check missing: run python samtools_b200/build.py'
    r = subprocess.run([exe, synth_set['sam'], synth_set['fa'], '240'], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    # reads with stored BQ:Z tags (the integer path) and odd CIGARs from the reference's own test data
    mp = os.path.join(corpus, 'test', 'mpileup')
    r = subprocess.run([exe, os.path.join(mp, 'mpileup.1.bam'), os.path.join(mp, 'mpileup.ref.fa'), '120'], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr


# ---------------------------------------------------------------- htslib-compatible iterator tier (T1)
COMPAT = os.path.join(ROOT, 'tests', 'compat', '_build', 'plp_dump')


@pytest.mark.parametrize('args,files', golden_cases.COMPAT_CASES, ids=golden_cases.COMPAT_IDS)
def test_htslib_compat_iterator(args, files, oracle_bin, corpus):
    """bam_mplp64_auto() through the GPU engine == the oracle's restatement of htslib's iterator,
    field by field (qpos, indel, is_del/head/tail/refskip, cigar_ind, quality seen through p->b, insertion text)."""
    assert os.path.exists(COMPAT), 'tests/compat/_build/plp_dump missing: run python samtools_b200/build.py'
    paths = [os.path.join(corpus, f) for f in files]
    got = subprocess.run([COMPAT, *args, *paths], capture_output=True)
    want = subprocess.run([oracle_bin, 'pileup-dump', *args, *paths], capture_output=True)
    assert got.returncode == 0, got.stderr[-300:]
    assert got.stdout == want.stdout
    assert len(got.stdout) > 100


def test_htslib_compat_hooks(oracle_bin, corpus):
    """constructor/destructor hooks + kstring bam_plp_insertion through the CUDA engine (host logic also in tests/test_emul_compat.py)"""
    paths = [os.path.join(corpus, 'test/mpileup/mp_DI.sam')]
    got = subprocess.run([COMPAT, '-c', *paths], capture_output=True)
    want = subprocess.run([oracle_bin, 'pileup-dump', *paths], capture_output=True)
    assert got.returncode == 0, got.stderr[-300:]
    assert got.stdout == want.stdout and b'bad=0' in got.stderr


# ---------------------------------------------------------------- BASELINE config 1 (examples/ex1): engine vs oracle
@pytest.mark.parametrize('cmd', golden_cases.EX1_CMDS)
def test_c1_ex1_engine_vs_oracle(cmd, cli, oracle_bin, corpus):
    """No expected output exists in-tree for examples/ex1 (SURVEY 8c): parity is oracle vs engine."""
    cwd = os.path.join(corpus, 'examples')
    want = subprocess.run(f'{oracle_bin} {cmd}', shell=True, cwd=cwd, capture_output=True)
    got = subprocess.run(f'{cli} {cmd}', shell=True, cwd=cwd, capture_output=True)
    assert got.returncode == 0 and len(want.stdout) > 1000
    assert got.stdout == want.stdout


# ---------------------------------------------------------------- coverage histogram views (coverage.c:223-304, 609-660)
def test_coverage_histogram_views_on_gpu(cli, oracle_bin, corpus, tmp_path):
    """per-bin breadth / depth counters on the device (k_coverage_hist), print_hist on the host; oracle-compared (unpinned)"""
    import hist_cases
    from samtools_b200 import synth
    soa = synth.make_batch(length=30_000, depth=12, seed=21)
    sam = str(tmp_path / 'h.sam')
    synth.write_sam(sam, soa)
    assert not hist_cases.run_all(cli, oracle_bin, corpus, tmp_path, sam)
    assert not hist_cases.run_all(cli, oracle_bin, corpus, tmp_path, sam, {'B200_WINDOW_COLS': '997'})


# ---------------------------------------------------------------- several engine handles behind one driver (B200_DEVICES / B200_HANDLES)
def test_window_workers_on_gpu(cli, oracle_bin, corpus, monkeypatch):
    """the drivers hand column windows round-robin to several handles (threads; one per listed device -- here the same device
    three times, plus a second device when the box has one) and write the text in window order: mpileup (BAQ, overlaps) and depth goldens"""
    import torch
    from concurrent.futures import ThreadPoolExecutor
    devs = ['0', '0', '0'] + (['1'] if torch.cuda.device_count() > 1 else [])      # a second device when the box has one
    monkeypatch.setenv('B200_WINDOW_COLS', '97')
    monkeypatch.setenv('B200_DEVICES', ','.join(devs))
    todo = [c for c in CASES if not c['skip'] and '>' not in c['cmd'] and ('mpileup' in c['cmd'] or 'depth' in c['cmd'])][::3]

    def run(c):
        ok, out, err = golden_cases.run_case(c, cli, oracle_bin, corpus)
        if not ok and b'not available on the device path' in err:
            return None
        return None if ok else (c['id'], c['cmd'], err[-200:])
    with ThreadPoolExecutor(max_workers=4) as ex:
        bad = [r for r in ex.map(run, todo) if r]
    assert len(todo) > 30 and not bad, bad[:3]
