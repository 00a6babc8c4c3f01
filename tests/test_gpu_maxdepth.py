"""The -d max-depth rule at real depth, through the CUDA path, against the oracle: amplicon stacks of 2x150 overlapping
pairs far over the default -d 8000, and RNA-seq-like spliced reads whose N skips of 300-20 000 bases keep thousands of them
buffered into a downstream exon stack (far-reaching read lists of thousands of reads per group).  C ABI (mpileup_text,
coverage, pileup_entries; general path, two files), the CLI with column windows cutting the stacks, the iterator tier, the
device gate next to its exact bound, and the structured window-edge inputs of tests/test_maxdepth.py through the CUDA CLI."""
import os, subprocess
import numpy as np
import pytest
from conftest import ROOT
from test_maxdepth import write_structured, structured_cases, check_cases, W, DEPTH

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')
PLP_DUMP = os.path.join(ROOT, 'tests', 'compat', '_build', 'plp_dump')

AMP_LEN = 260
K_REACH = 512        # plp_core.h kReach: a read is served through the far-reaching lists for groups from rpos + kReach on


def make_amplicons(seed=3, pairs=(9500, 11500, 3000, 12000, 2500), spacing=1000, read_len=150, length=None, ref_seed=None):
    """2x150 pairs on 260-base amplicons (the mates overlap by ~40 bases); each amplicon's pairs start at three forward and
    two reverse primer positions.  Amplicons with fewer than 8000 pairs are the controls."""
    from samtools_b200 import synth
    rng = np.random.default_rng(seed)
    length = length or 300 + spacing * len(pairs)
    ref = synth.make_reference(length, seed=ref_seed or seed)
    recs, name = [], 0
    lens, ops = np.array([read_len], dtype=np.int64), np.array([0], dtype=np.int64)
    for k, n in enumerate(pairs):
        a = 200 + k * spacing
        fwd = a + rng.choice([0, 2, 5], n)
        rev = a + AMP_LEN - read_len - rng.choice([0, 3], n)
        for i in range(n):
            recs.append(synth._rec(rng, ref, int(fwd[i]), lens, ops, flag=99, name=name))
            recs.append(synth._rec(rng, ref, int(rev[i]), lens, ops, flag=147, name=name))
            name += 1
    return synth._pack(recs, ref, length, 0, 'amp')


def make_rnaseq(seed=7, introns=(300, 2500, 20000), n_spliced=4500, n_down=5000, a=50, b=100, read_len=150, gap=1500):
    """Genes of two exons.  n_spliced reads start at three positions of exon 1 and skip the intron (N) into exon 2; n_down
    unspliced reads start at exon 2's first two bases.  The spliced reads are still buffered there, so the downstream stack
    goes over -d 8000.  Returns the batch and the first base of each exon 2."""
    from samtools_b200 import synth
    rng = np.random.default_rng(seed)
    starts, s = [], gap
    for n in introns:
        starts.append((s, s + a + n)); s += a + n + read_len + gap
    length = s + gap
    ref = synth.make_reference(length, seed=seed)
    recs = []
    for s, q in starts:
        for st in s + rng.choice([0, 2, 5], n_spliced):
            st = int(st)
            recs.append(synth._rec(rng, ref, st, np.array([a, q - st - a, b], np.int64), np.array([0, 3, 0], np.int64)))
        for st in q + rng.choice([0, 1], n_down):
            recs.append(synth._rec(rng, ref, int(st), np.array([read_len], np.int64), np.array([0], np.int64)))
    return synth._pack(recs, ref, length, 0, 'rna'), [q for _, q in starts]


def merge_files(a, b):
    """two single-file batches of the same contig as one two-file batch"""
    out = {}
    na, nqa = len(a['pos']), len(a['qual'])
    for k in ('pos', 'flag', 'mapq', 'l_qseq', 'n_cigar', 'mtid', 'mpos', 'isize', 'rbits', 'cigar', 'seq4', 'qual', 'pair_id'):
        out[k] = np.concatenate([a[k], b[k]])
    out['cigar_off'] = np.concatenate([a['cigar_off'], b['cigar_off'] + np.uint64(len(a['cigar']))])
    out['qual_off'] = np.concatenate([a['qual_off'], b['qual_off'] + np.uint64(nqa)])
    assert nqa % 2 == 0 and len(a['seq4']) * 2 == nqa
    out['prev_same_name'] = np.concatenate([a['prev_same_name'], np.where(b['prev_same_name'] >= 0, b['prev_same_name'] + na, -1)])
    out['file_start'] = np.array([0, na, na + len(b['pos'])], dtype=np.int64)
    for k in ('tid', 'tid_len', 'tid_name', 'ref', 'ref_beg', 'ref_len', 'ref_full'):
        out[k] = a[k]
    return out


def max_stack(soa):
    """largest number of reads whose closed intervals [pos, pos + rlen] share a position (numpy difference array)"""
    from samtools_b200 import synth
    pos = soa['pos'].astype(np.int64); end = pos + synth.ref_span(soa)
    diff = np.zeros(int(end.max()) + 3, np.int64)
    np.add.at(diff, pos, 1); np.add.at(diff, end + 1, -1)
    return int(np.cumsum(diff).max())


def longest_far_list(soa, win_base, ncols):
    """the longest per-group far-reaching list a stage at win_base builds (the k_ovf_count rule): a read longer than kReach
    is listed for every 32-column group from rpos + kReach to its end"""
    from samtools_b200 import synth
    rpos = soa['pos'].astype(np.int64) - win_base; rend = rpos + synth.ref_span(soa)
    far = rend - rpos > K_REACH
    a = rpos[far] + K_REACH
    g0 = np.where(a <= 0, 0, (a + 31) >> 5); g1 = np.minimum(np.where(rend[far] > 0, (rend[far] - 1) >> 5, -1), (ncols + 31) // 32)
    ok = g1 >= g0
    diff = np.zeros((ncols + 31) // 32 + 3, np.int64)
    np.add.at(diff, g0[ok], 1); np.add.at(diff, g1[ok] + 1, -1)
    return int(np.cumsum(diff).max())


@pytest.fixture(scope='module')
def amp_dir(tmp_path_factory):
    from samtools_b200 import synth
    d = tmp_path_factory.mktemp('amp')
    soa = make_amplicons()
    synth.write_sam(str(d / 'amp.sam'), soa); synth.write_fasta(str(d / 'amp.fa'), 'amp', soa['ref_full'])
    low = make_amplicons(seed=6, ref_seed=3, pairs=(1500,) * 5)      # a second file that never reaches -d
    synth.write_sam(str(d / 'ampb.sam'), low)
    one = make_amplicons(seed=4, pairs=(10000,), length=800)
    synth.write_sam(str(d / 'amp1.sam'), one)
    return d, soa, low, one


@pytest.fixture(scope='module')
def rna_dir(tmp_path_factory):
    from samtools_b200 import synth
    d = tmp_path_factory.mktemp('rna')
    soa, exon2 = make_rnaseq()
    synth.write_sam(str(d / 'rna.sam'), soa); synth.write_fasta(str(d / 'rna.fa'), 'rna', soa['ref_full'])
    small, small_exon2 = make_rnaseq(seed=8, introns=(2500,), n_spliced=400, n_down=450)
    synth.write_sam(str(d / 'rnas.sam'), small)
    return d, soa, exon2, small, small_exon2[0]


def _oracle(oracle_bin, d, *args):
    return subprocess.run([oracle_bin, *args], cwd=d, capture_output=True, check=True).stdout


def _engine(env=None):
    from samtools_b200 import engine
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        return engine.Engine(0)
    finally:
        for k, v in old.items():
            if v is None: os.environ.pop(k)
            else: os.environ[k] = v


def _text(soa, conf_kw, text_kw, env=None):
    from samtools_b200 import engine
    e = _engine(env)
    try:
        e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, **conf_kw))
        return e.mpileup_text(**text_kw), e.launches
    finally:
        e.close()


def _d0(args):
    """the same options with the rule off"""
    return (args[:args.index('-d')] + ['-d', '0'] + args[args.index('-d') + 2:]) if '-d' in args else args + ['-d', '0']


def test_inputs_are_deep(amp_dir, rna_dir):
    _, soa, low, _ = amp_dir
    assert max_stack(soa) > 2 * 8000 and max_stack(low) < 8000
    _, rna, exon2, _, _ = rna_dir
    assert max_stack(rna) > 9000
    assert longest_far_list(rna, 0, int(rna['tid_len'])) >= 4000     # thousands of reads in one group's far-reaching list


@pytest.mark.parametrize('conf,text,args,env', [
    ({}, {}, ['-f', 'amp.fa'], None),
    ({'overlaps': 0}, {}, ['-x', '-f', 'amp.fa'], None),
    ({'baq': 0}, {'all': 1, 'out_mapq': 1}, ['-B', '-a', '-s', '-f', 'amp.fa'], None),
    ({'baq': 0, 'max_depth': 2500}, {'min_baseQ': 0}, ['-B', '-d', '2500', '-Q', '0', '-f', 'amp.fa'], None),
    ({}, {}, ['-f', 'amp.fa'], {'B200_PLP_GENERAL': '1'}),
    ({'baq': 0}, {'all': 1, 'out_qpos': 1}, ['-B', '-a', '-O', '-f', 'amp.fa'], None),
], ids=['baq', 'x', 'B_a_s', 'B_d2500', 'general', 'B_a_O'])
def test_cabi_mpileup_amplicons(conf, text, args, env, amp_dir, oracle_bin):
    from test_gpu_parity import _same
    d, soa, _, _ = amp_dir
    want = _oracle(oracle_bin, d, 'mpileup', *args, 'amp.sam')
    assert _oracle(oracle_bin, d, 'mpileup', *_d0(args), 'amp.sam') != want      # the rule fires
    got, _ = _text(soa, conf, text, env)
    _same(got, want, ' '.join(args))


@pytest.mark.parametrize('env', [None, {'B200_PLP_GENERAL': '1'}], ids=['default', 'general'])
def test_cabi_two_files_one_over_the_cap(env, amp_dir, oracle_bin):
    """a deep file and one that never reaches -d, in one batch: the rule is per file"""
    from test_gpu_parity import _same
    d, soa, low, _ = amp_dir
    args = ['-B', '-f', 'amp.fa']
    want = _oracle(oracle_bin, d, 'mpileup', *args, 'amp.sam', 'ampb.sam')
    assert _oracle(oracle_bin, d, 'mpileup', *_d0(args), 'amp.sam', 'ampb.sam') != want
    got, _ = _text(merge_files(soa, low), {'baq': 0}, {}, env)
    _same(got, want, 'two files')


def test_gate_next_to_the_bound(amp_dir, oracle_bin):
    """M = the largest number of kept reads whose closed intervals share a position.  At -d M-1 the rule fires: the device
    gate must let the host sweep run, which drops reads (two more launches: the drop and the rebuilt read slices).  At -d M
    and M+1 nothing is dropped (the oracle's output equals its -d 0 output); the test sees only that the output stays right
    and that no drop was applied, not whether the gate stopped the sweep."""
    from test_gpu_parity import _same
    d, soa, _, _ = amp_dir
    M = max_stack(soa)
    off = _oracle(oracle_bin, d, 'mpileup', '-B', '-x', '-d', '0', '-f', 'amp.fa', 'amp.sam')
    got = {}
    for dd in (M - 1, M, M + 1):
        want = _oracle(oracle_bin, d, 'mpileup', '-B', '-x', '-d', str(dd), '-f', 'amp.fa', 'amp.sam')
        assert (want != off) == (dd == M - 1), dd
        got[dd] = _text(soa, {'baq': 0, 'overlaps': 0, 'max_depth': dd}, {})
        _same(got[dd][0], want, f'-d {dd}')
    assert got[M - 1][1] > got[M][1] == got[M + 1][1]


def _coverage_row(e, soa, dd):
    """the whole `coverage` row (coverage.c print_tabular_line) of one contig from the engine's sums"""
    from samtools_b200 import engine
    st = e.stage(soa, engine.default_stage_conf(engine.MODE_COVERAGE, rflag_filter=4 | 256 | 512 | 1024, max_depth=dd, end=soa['tid_len']))
    cv = e.coverage(min_baseQ=0, min_depth=1)
    L = int(soa['tid_len'])
    n_sel = st.n_selected_reads
    return ('%s\t1\t%d\t%d\t%d\t%g\t%g\t%.3g\t%.3g' % (
        soa['tid_name'], L, n_sel, cv['n_covered_bases'], 100.0 * cv['n_covered_bases'] / L, cv['summed_coverage'] / L,
        cv['summed_baseQ'] / cv['quality_bases'] if cv['quality_bases'] > 0 else 0,
        st.summed_mapq / n_sel if n_sel > 0 else 0)).encode()


@pytest.mark.parametrize('which', ['amp', 'rna'])
def test_cabi_coverage(which, amp_dir, rna_dir, oracle_bin):
    d, soa = (amp_dir[0], amp_dir[1]) if which == 'amp' else (rna_dir[0], rna_dir[1])
    e = _engine()
    try:
        for dd in (8000, 3000):
            row = _oracle(oracle_bin, d, 'coverage', '-d', str(dd), f'{which}.sam').split(b'\n')[1]
            assert row != _oracle(oracle_bin, d, 'coverage', '-d', '0', f'{which}.sam').split(b'\n')[1], dd
            assert _coverage_row(e, soa, dd) == row, dd
    finally:
        e.close()


@pytest.mark.parametrize('baq', [0, 1], ids=['B', 'baq'])
def test_cabi_mpileup_rnaseq(baq, rna_dir, oracle_bin):
    """each gene's exon-2 stack as a region: the spliced reads reach it from thousands of columns before (far-reaching
    lists of thousands of reads per group) and push it over -d 8000"""
    from test_gpu_parity import _same
    from samtools_b200 import engine
    d, soa, exon2, _, _ = rna_dir
    e = _engine()
    try:
        for q in exon2:
            beg, end = q - 40, q + 170
            args = (['-B'] if not baq else []) + ['-r', f'rna:{beg + 1}-{end}', '-f', 'rna.fa']
            want = _oracle(oracle_bin, d, 'mpileup', *args, 'rna.sam')
            assert _oracle(oracle_bin, d, 'mpileup', *_d0(args), 'rna.sam') != want, q
            e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, baq=baq, beg=beg, end=end))
            _same(e.mpileup_text(), want, f'exon 2 at {q}')
        assert longest_far_list(soa, exon2[-1] - 40, 210) >= 4000
    finally:
        e.close()


def _dump_columns(text, beg, end):
    """pileup-dump lines of columns [beg, end): {pos: [name/qpos/indel/flags/cigar_ind/qual, ...]}"""
    out = {}
    for line in text.split(b'\n'):
        if not line:
            continue
        tid, pos, rest = line.split(b'\t', 2)
        pos = int(pos)
        if beg <= pos < end:
            out[pos] = [b'/'.join(x.split(b'/')[:6]) for x in rest.split(b' ')[1:]]
    return out


def _entries_columns(soa, e, beg, end, cap):
    col_n, ents = e.pileup_entries(0, beg, end, cap)
    out, k = {}, 0
    for c in range(end - beg):
        n = int(col_n[c])
        if n:
            rows = []
            for x in ents[k:k + n]:
                i = int(x['read']); qp = int(x['qpos']); bits = int(x['bits'])
                q = int(soa['qual'][int(soa['qual_off'][i]) + qp]) if qp < int(soa['l_qseq'][i]) else -1
                rows.append(b'p%09d/%d/%d/%d%d%d%d/%d/%d' % (int(soa['pair_id'][i]), qp, int(x['indel']), bits & 1, (bits >> 1) & 1,
                                                             (bits >> 2) & 1, (bits >> 3) & 1, int(x['cigar_ind']), q))
            out[beg + c] = rows
        k += n
    return out


@pytest.mark.parametrize('which', ['amp1', 'rnas'])
def test_cabi_pileup_entries(which, amp_dir, rna_dir, oracle_bin):
    """b200_pileup_entries (every bam_pileup1_t field but the read's text) over the stacked columns vs the oracle's
    iterator: the deep amplicon at -d 8000, the small spliced set (intron columns of reference skips) at -d 600"""
    from samtools_b200 import engine
    if which == 'amp1':
        d, soa, dd = amp_dir[0], amp_dir[3], 8000
        beg, end = 200 + AMP_LEN - 150 - 20, 200 + AMP_LEN - 150 + 40
    else:
        d, soa, q, dd = rna_dir[0], rna_dir[3], rna_dir[4], 600
        beg, end = q - 40, q + 20
    want = _oracle(oracle_bin, d, 'pileup-dump', '-d', str(dd), f'{which}.sam')
    assert want != _oracle(oracle_bin, d, 'pileup-dump', '-d', '0', f'{which}.sam')
    want = _dump_columns(want, beg, end)
    e = _engine()
    try:
        e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, baq=0, overlaps=0, max_depth=dd, rflag_filter=0, no_orphan=0))
        got = _entries_columns(soa, e, beg, end, 2_000_000)
    finally:
        e.close()
    assert sorted(got) == sorted(want) and len(want) == end - beg
    for c in want:
        assert got[c] == want[c], c


@pytest.mark.parametrize('env', [{'B200_WINDOW_COLS': '97'}, {'B200_WINDOW_COLS': '97', 'B200_DEVICES': '0,0'}, {}],
                         ids=['win97', 'win97_devices00', 'default'])
def test_cli_amplicons_windows(env, amp_dir, oracle_bin):
    """97-column windows cut every amplicon's stacks: halo reads carry their verdicts, reads ending at a window start count"""
    d = amp_dir[0]
    cases = [('mpileup -B -f amp.fa amp.sam', True), ('mpileup -B -x -d 5000 amp.sam', True), ('coverage -d 6000 amp.sam', True),
             ('mpileup -B amp.sam ampb.sam', True)]
    bad = check_cases(CLI, oracle_bin, d, cases, env)
    assert not bad, bad[:3]


def test_cli_rnaseq_windows(rna_dir, oracle_bin):
    """97-column windows over each exon-2 region (the spliced reads are halo reads of every window) and 4099-column windows
    over the whole contig (the spliced reads are staged again by every window their intron crosses)"""
    d = rna_dir[0]
    cases = [(f'mpileup -B -r rna:{q - 39}-{q + 170} rna.sam', True) for q in rna_dir[2]]
    bad = check_cases(CLI, oracle_bin, d, cases, {'B200_WINDOW_COLS': '97'})        # edges at q+57 and q+154 of each region
    bad += check_cases(CLI, oracle_bin, d, [('coverage -d 8000 rna.sam', True)], {'B200_WINDOW_COLS': '4099'})
    assert not bad, bad[:3]


@pytest.mark.parametrize('budget', ['1000000', '100000'])
def test_iterator_tier_amplicon(budget, amp_dir, oracle_bin):
    """plp_dump -d 8000 -o on one deep amplicon, windows cut inside its stacks"""
    d = amp_dir[0]
    p = str(d / 'amp1.sam')
    want = subprocess.run([oracle_bin, 'pileup-dump', '-o', '-d', '8000', p], capture_output=True)
    off = subprocess.run([oracle_bin, 'pileup-dump', '-o', '-d', '0', p], capture_output=True)
    assert want.returncode == 0 and want.stdout != off.stdout
    del off
    got = subprocess.run([PLP_DUMP, '-o', '-d', '8000', p], capture_output=True, env=dict(os.environ, B200_PLP_WINDOW_BYTES=budget))
    assert got.returncode == 0, got.stderr[-300:]
    assert got.stdout == want.stdout


@pytest.fixture(scope='module')
def sdir(tmp_path_factory):
    d = tmp_path_factory.mktemp('gmaxdepth')
    write_structured(d)
    return d


@pytest.mark.parametrize('env', [{'B200_WINDOW_COLS': str(W)}, {'B200_WINDOW_COLS': str(W), 'B200_DEVICES': '0,0'},
                                 {'B200_WINDOW_COLS': str(W), 'B200_PLP_GENERAL': '1'}], ids=['win97', 'win97_devices00', 'win97_general'])
def test_cli_structured_windows(env, sdir, oracle_bin):
    cases = [(c, True) for c in structured_cases()] + [(f'mpileup -d {DEPTH} -f x.fa st.sam', True)]
    bad = check_cases(CLI, oracle_bin, sdir, cases, env)
    assert not bad, f'{len(bad)} of {len(cases)}: {bad[:3]}'
