"""Per-column rank-sum bias statistics (`b200samtools counts --ranksums`, b200_mpileup_ranksums, Engine.mpileup_ranksums,
engine.ranksum_z) against the Mann-Whitney U that scipy computes from the oracle's `mpileup --reverse-del -s --output-BP-5`
text of the same options: entry i of a file's sequence column pairs with character i of its quality and mapq columns and
number i of its BP-5 column; '.' / ',' entries are the ref class, A C G T letters the alt class.  CPU through the emulation
harness (plain and under the address and undefined-behaviour sanitizers), and the CUDA path (BAQ included) under -m gpu."""
import os, re, subprocess
import numpy as np
import pytest
from scipy import stats
from conftest import ROOT
import test_counts
import test_qsums
import test_psums
from test_counts import GOLDEN, fuzz_jobs
from test_qsums import golden_jobs, build_emul

CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')
PLANES = 8
CNT = test_counts.PLANES
QS = test_qsums.PLANES
PS = test_psums.PLANES
POS_CAP = 1024
MAX_DEPTH = (1 << 21) - 1


# ---------------------------------------------------------------- the text -> rank sums parser
def files_of(line):
    """chr, pos, ref and per file (cnt, seq, qual, mapq, bp5) of one `-s --output-BP-5` line"""
    f = line.split('\t')
    return f[:3], [f[3 + 5 * k: 8 + 5 * k] for k in range((len(f) - 3) // 5)]


def class_entries(seq, qual, mq, bp, ref):
    """[(cls, BQ, MQ, BP-5 capped at 1024)] of one file's columns, cls 'r' for '.' / ',' on an A C G T reference and 'a' for
    an A C G T letter; every other entry (deletions, skips, N and IUPAC bases) is left out"""
    out = []
    pos = [int(x) for x in bp.split(',')]
    ref_acgt = ref.upper() in 'ACGT'
    i, n = 0, -1
    while i < len(seq):
        ch = seq[i]
        if ch == '^':                 # "^" + a mapq character, which may itself be '$', '+', '-', '.' or ','
            i += 2
        elif ch == '$':
            i += 1
        elif ch in '+-':
            m = re.match(r'\d+', seq[i + 1:])
            i += 1 + len(m.group(0)) + int(m.group(0))
        else:
            n += 1
            cls = ('r' if ref_acgt else None) if ch in '.,' else 'a' if ch.upper() in 'ACGT' else None
            if cls:
                out.append((cls, ord(qual[n]) - 33, ord(mq[n]) - 33, min(pos[n], POS_CAP)))
            i += 1
    assert n + 1 == len(qual) == len(mq) == len(pos), (seq, qual, mq, bp)
    return out


def rank_planes(entries, fast=False):
    """the 8 planes of one (column, file): n_ref, n_alt, then U2 (scipy's U of the alt sample, times 2) and T (numpy.unique
    counts) of BQ, MQ and BP-5.  fast: U2 by counting, per alt value, the ref values below and equal (numpy.searchsorted)"""
    ref = np.array([e[1:] for e in entries if e[0] == 'r'], np.int64).reshape(-1, 3)
    alt = np.array([e[1:] for e in entries if e[0] == 'a'], np.int64).reshape(-1, 3)
    p = [len(ref), len(alt)] + [0] * 6
    if len(ref) and len(alt):
        for v in range(3):
            if fast:
                r = np.sort(ref[:, v])
                u = int((np.searchsorted(r, alt[:, v], 'left') + np.searchsorted(r, alt[:, v], 'right')).sum())
            else:
                u = stats.mannwhitneyu(alt[:, v], ref[:, v]).statistic * 2
                assert u == round(u)
            t = np.unique(np.concatenate([ref[:, v], alt[:, v]]), return_counts=True)[1].astype(np.int64)
            p[2 + 2 * v], p[3 + 2 * v] = int(round(u)), int((t ** 3 - t).sum())
    return p


def count_rows(text_rs, base, per_file, seen=None, fast=False):
    """the `counts --ranksums` rows: each row of `base` (chr, pos, ref, then per_file values per file) with the 8 rank
    planes after each file's values.  seen: a dict that collects what the columns exercise; fast: see rank_planes"""
    brow = base.decode().split('\n')[:-1]
    rrow = text_rs.decode().split('\n')[:-1]
    assert len(brow) == len(rrow)
    out = []
    for lb, lr in zip(brow, rrow):
        head, files = files_of(lr)
        b = lb.split('\t')
        assert b[:3] == head
        vals = []
        for k, (cnt, seq, qual, mq, bp) in enumerate(files):
            ent = class_entries(seq, qual, mq, bp, head[2]) if int(cnt) else []
            rp = rank_planes(ent, fast)
            if seen is not None and ent:
                both = rp[0] and rp[1]
                seen['both'] = seen.get('both', 0) + bool(both)
                seen['one_empty'] = seen.get('one_empty', 0) + (not both)
                r = {e[1:] for e in ent if e[0] == 'r'}
                seen['tie_across'] = seen.get('tie_across', 0) + any(e[1 + v] in {x[v] for x in r} for e in ent if e[0] == 'a' for v in range(3))
                seen['pos_capped'] = seen.get('pos_capped', 0) + any(e[3] == POS_CAP for e in ent)
            vals += b[3 + per_file * k: 3 + per_file * (k + 1)] + [str(x) for x in rp]
        out.append('\t'.join(head + vals) + '\n')
    return ''.join(out).encode()


def test_parser_on_hand_made_column():
    # '.' / ',' refs, letters of both cases, N, '*', a deletion token, '^' with the meta-characters '.' and ',' as mapq,
    # BP-5 above 1024 (capped) and at 1024
    seq, qual, mq, bp = '^.,A$^,.c*N-1a,', 'I5+!?I#', '<<!~<<A', '3,1500,1,1024,7,2,1025'
    ent = class_entries(seq, qual, mq, bp, 'G')
    assert ent == [('r', 40, 27, 3), ('a', 20, 27, 1024), ('r', 10, 0, 1), ('a', 0, 93, 1024), ('r', 2, 32, 1024)]
    #   BQ: alt {20, 0} vs ref {40, 10, 2}: 20 beats two -> U2 4, no ties; MQ: alt {27, 93} vs {27, 0, 32}: 27 beats one and
    #   ties one, 93 beats three -> U2 9, 27 twice -> T 6; BP-5: alt {1024, 1024} vs {3, 1, 1024}: 2 * (2 + 2 + 1) -> 10, T 24
    assert rank_planes(ent) == [3, 2, 4, 0, 9, 6, 10, 24]
    assert rank_planes(ent, fast=True) == [3, 2, 4, 0, 9, 6, 10, 24]
    rng = np.random.default_rng(7)                 # the counting U2 is scipy's on random samples with many ties
    for _ in range(200):
        ent = [('ra'[int(rng.integers(2))], *(int(x) for x in rng.integers(0, 6, 3))) for _ in range(int(rng.integers(2, 40)))]
        assert rank_planes(ent, fast=True) == rank_planes(ent)
    # on an N reference '.' is not a class entry, and an N base never is
    assert class_entries('.,N', '!!!', '!!!', '1,1,1', 'N') == []
    line = 'c\t5\tA\t2\t.C\tI5\t<<\t1,2\t0\t*\t*\t*\t*\n'
    assert count_rows(line.encode(), b'c\t5\tA\tx\ty\n', 1) == b'c\t5\tA\tx\t1\t1\t0\t0\t1\t6\t2\t0\ty\t0\t0\t0\t0\t0\t0\t0\t0\n'


# ---------------------------------------------------------------- command lines
def run_pair(tool, oracle, cwd, args, prefix='', env=None, sums=False, seen=None, fast=False):
    """None when `tool counts --ranksums <args>` (with sums: `counts --qsums --psums --ranksums`) prints the rows parsed
    from the oracle's text, 'baq' when the emulation harness cannot stage the case, else a description of the difference"""
    pre = re.sub(r'\$samtools\s+view', oracle + ' view', prefix).replace('$samtools', oracle)
    sh = lambda line: subprocess.run(pre + line, shell=True, cwd=cwd, capture_output=True, env=env, timeout=900)
    got = sh(f'{tool} counts {"--qsums --psums " if sums else ""}--ranksums {args}')
    if got.returncode != 0 and b'BAQ kernel is not emulated' in got.stderr:
        return 'baq'
    text, text_q0 = sh(f'{oracle} mpileup --reverse-del {args}').stdout, sh(f'{oracle} mpileup --reverse-del {args} -Q 0').stdout
    base, per_file = test_counts.rows_from_text(text, text_q0), CNT
    if sums:
        base = test_qsums.count_rows(sh(f'{oracle} mpileup --reverse-del -s {args}').stdout, text, text_q0)
        base = test_psums.count_rows(sh(f'{oracle} mpileup --reverse-del --output-BP-5 {args}').stdout, base, CNT + QS)
        per_file = CNT + QS + PS
    exp = count_rows(sh(f'{oracle} mpileup --reverse-del -s --output-BP-5 {args}').stdout, base, per_file, seen, fast)
    if got.returncode != 0 or got.stdout != exp:
        return (args, got.returncode, got.stderr[-300:], exp[:300], got.stdout[:300])
    return None


def run_many(tool, oracle, jobs, env=None, sums=False, fast=False):
    """every job, (cwd, args) or (cwd, args, prefix): the differences, how many matched, and what the columns exercised"""
    from concurrent.futures import ThreadPoolExecutor
    seen = [dict() for _ in jobs]
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        res = list(ex.map(lambda k: run_pair(tool, oracle, jobs[k][0], jobs[k][1], jobs[k][2] if len(jobs[k]) > 2 else '', env, sums, seen[k], fast),
                          range(len(jobs))))
    total = {}
    for s in seen:
        for k, v in s.items():
            total[k] = total.get(k, 0) + v
    return [r for r in res if r not in (None, 'baq')], sum(r is None for r in res), total


def check_invariant(rows, n_files, per_file):
    """n_ref + n_alt of each file equals its A C G T count planes of both strands (rows of `counts [...] --ranksums`)"""
    for ln in rows.decode().split('\n')[:-1]:
        f = [int(x) for x in ln.split('\t')[3:]]
        for k in range(n_files):
            v = f[k * per_file: (k + 1) * per_file]
            assert v[-8] + v[-7] == sum(v[0:4]) + sum(v[9:13]), ln


def write_deep_column(d, n):
    """one column of n one-base reads on a contig 'A' of length 1: alternately 'A' (ref) and 'C' (alt), all of BQ 40, MQ 60
    and BP-5 1, so every value is one tie of all n entries"""
    with open(os.path.join(d, 'deep.fa'), 'w') as f:
        f.write('>c\nA\n')
    name = f'deep{n}.sam'
    with open(os.path.join(d, name), 'w') as f:
        f.write('@SQ\tSN:c\tLN:1\n')
        f.writelines(f'r{i}\t0\tc\t1\t60\t1M\t*\t0\t0\t{"AC"[i & 1]}\tI\n' for i in range(n))
    return name


def check_depth_boundary(tool, d):
    """2^21 - 1 class entries give exact planes (T = n^3 - n, the largest tie term); 2^21 fail with a message"""
    n = MAX_DEPTH
    r = subprocess.run(f'{tool} counts --ranksums -B -d 0 -f deep.fa {write_deep_column(d, n)}', shell=True, cwd=d, capture_output=True, timeout=1800)
    nr, na = (n + 1) // 2, n // 2
    cnt = [0] * CNT
    cnt[0], cnt[1], cnt[CNT - 1] = nr, na, n
    rk = [nr, na] + [nr * na, n ** 3 - n] * 3
    assert n ** 3 - n < 1 << 63
    want = '\t'.join(['c', '1', 'A'] + [str(x) for x in cnt + rk]) + '\n'
    assert r.returncode == 0 and r.stdout == want.encode(), (r.stderr[-300:], r.stdout[:300])
    r = subprocess.run(f'{tool} counts --ranksums -B -d 0 -f deep.fa {write_deep_column(d, n + 1)}', shell=True, cwd=d, capture_output=True, timeout=1800)
    assert r.returncode != 0 and b'more than 2097151 reference and non-reference bases' in r.stderr, (r.returncode, r.stderr[-300:])


# ---------------------------------------------------------------- emulation harness (no GPU)
@pytest.fixture(scope='module')
def emul_bin(tmp_path_factory):
    """the CLI on the emulation harness with every numeric output, rank sums included (emul_ranksums.cpp)"""
    return build_emul(tmp_path_factory, 'ranksums')


@pytest.fixture(scope='module')
def emul_psums(tmp_path_factory):
    """the CLI on the harness build with the position sums (emul_psums.cpp), which has no rank sums"""
    return build_emul(tmp_path_factory, 'psums')


@pytest.fixture(scope='module')
def emul_asan(tmp_path_factory):
    """emul_ranksums.cpp and the CLI built under -fsanitize=address,undefined -fno-sanitize-recover"""
    exe = str(tmp_path_factory.mktemp('emul_asan') / 'b200samtools_emul_asan')
    host = os.path.join(ROOT, 'samtools_b200', 'csrc', 'host')
    subprocess.run(['g++', '-std=c++17', '-O1', '-g', '-fno-omit-frame-pointer', '-fsanitize=address,undefined', '-fno-sanitize-recover',
                    '-Wall', '-Wno-unused-function', '-Wno-parentheses', '-o', exe, os.path.join(host, 'cli.cpp'), os.path.join(host, 'hts_io.cpp'),
                    os.path.join(ROOT, 'tests', 'emul', 'emul_ranksums.cpp'), '-lz'], check=True)
    return exe


def test_rank_rules_under_sanitizers(tmp_path):
    """rank_from_hist against the pairwise definition, whole and in runs, and rank_depth_over at 2^21 - 1 against 2^21"""
    exe = str(tmp_path / 'rank_check')
    subprocess.run(['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address,undefined', '-fno-sanitize-recover', '-Wall', '-Wno-parentheses',
                    '-o', exe, os.path.join(ROOT, 'tests', 'emul', 'rank_check.cpp')], check=True)
    r = subprocess.run([exe], capture_output=True)
    assert r.returncode == 0 and r.stdout == b'ok\n', (r.stdout, r.stderr[-500:])


def test_engine_without_ranksums_refuses(emul_psums, corpus):
    """an engine build without the rank sums: --ranksums stops with a message, and `counts` with its other sums still runs"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    r = subprocess.run([emul_psums, 'counts', '--ranksums', 'mpileup.1.bam'], cwd=cwd, capture_output=True)
    assert r.returncode != 0 and r.stdout == b'' and b'this engine build has no rank sums' in r.stderr, r.stderr
    r = subprocess.run([emul_psums, 'counts', '--qsums', '--psums', 'mpileup.1.bam'], cwd=cwd, capture_output=True)
    assert r.returncode == 0 and r.stdout, r.stderr


def test_ranksums_is_an_option_of_counts_only(emul_bin, corpus):
    cwd = os.path.join(corpus, 'test', 'mpileup')
    for cmd in ('mpileup', 'indels'):
        r = subprocess.run([emul_bin, cmd, '--ranksums', 'mpileup.1.bam'], cwd=cwd, capture_output=True)
        assert r.returncode != 0 and r.stdout == b'' and b'--ranksums is an option of `counts`' in r.stderr, (cmd, r.stderr)


def test_without_flag_unchanged_emul(emul_bin, emul_psums, corpus):
    """`counts` without --ranksums (with and without the other sums) prints what the harness build without rank sums prints"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    for args in (['-B', 'mpileup.1.bam', 'mpileup.2.bam'], ['-B', '-Q', '0', '-a', 'mpileup.3.bam'], ['-B', '-f', 'mpileup.ref.fa', 'mpileup.3.bam'],
                 ['--qsums', '--psums', '-B', '-f', 'mpileup.ref.fa', 'mpileup.1.bam']):
        a = subprocess.run([emul_psums, 'counts'] + args, cwd=cwd, capture_output=True)
        b = subprocess.run([emul_bin, 'counts'] + args, cwd=cwd, capture_output=True)
        assert a.returncode == 0 and a.stdout and a.stdout == b.stdout


@pytest.mark.parametrize('case', GOLDEN, ids=[c['id'] for c in GOLDEN])
def test_golden_ranksums_emul(case, emul_bin, oracle_bin, corpus):
    r = run_pair(emul_bin, oracle_bin, os.path.join(corpus, case['cwd']), case['args'], case['prefix'])
    if r == 'baq':
        pytest.skip('needs the BAQ kernel (covered by -m gpu)')
    assert r is None, r


def test_golden_ranksums_windows_emul(emul_bin, oracle_bin, corpus):
    """97-column windows: every case crosses window edges (halo reads, -a rows, BED) and must print the same rows"""
    bad, ok, seen = run_many(emul_bin, oracle_bin, golden_jobs(corpus), dict(os.environ, B200_WINDOW_COLS='97'))
    assert not bad and ok > 30, bad[:2]
    assert seen.get('both', 0) > 0, seen


def test_all_sums_together_emul(emul_bin, oracle_bin, corpus):
    """--qsums --psums --ranksums: per file the counts, the quality sums, the position sums, then the rank planes"""
    mp = os.path.join(corpus, 'test', 'mpileup')
    for args in ('-B -f mpileup.ref.fa mpileup.1.bam mpileup.2.bam mpileup.3.bam', '-Q 0 -B -f mpileup.ref.fa mpileup.1.bam', 'output-BP.sam'):
        assert run_pair(emul_bin, oracle_bin, mp, args, sums=True) is None


FUZZ_SEEDS = test_psums.FUZZ_SEEDS


def test_fuzz_ranksums_emul(emul_bin, oracle_bin, tmp_path):
    """the fuzz SAMs: columns with both classes, with one class empty, and with a value tied across the classes all occur"""
    bad, ok, seen = run_many(emul_bin, oracle_bin, fuzz_jobs(tmp_path, FUZZ_SEEDS, need_noBAQ=True))
    assert not bad and ok > 100, bad[:2]
    assert seen.get('both', 0) > 0 and seen.get('one_empty', 0) > 0 and seen.get('tie_across', 0) > 0, seen


def test_invariant_class_counts_emul(emul_bin, corpus):
    """n_ref + n_alt equals the A C G T count planes of both strands at the same -Q"""
    mp = os.path.join(corpus, 'test', 'mpileup')
    for args, nf in ((['-B', '-f', 'mpileup.ref.fa', 'mpileup.1.bam', 'mpileup.2.bam'], 2), (['-B', '-Q', '0', 'mpileup.3.bam'], 1),
                     (['-Q', '30', '-B', '-f', 'mpileup.ref.fa', 'mpileup.3.bam'], 1)):
        r = subprocess.run([emul_bin, 'counts', '--ranksums'] + args, cwd=mp, capture_output=True, check=True)
        assert r.stdout
        check_invariant(r.stdout, nf, CNT + PLANES)


def test_golden_and_fuzz_under_sanitizers(emul_asan, oracle_bin, corpus, tmp_path):
    """the golden cases and the fuzz SAMs through the harness built with the address and undefined-behaviour sanitizers"""
    env = dict(os.environ, ASAN_OPTIONS='detect_leaks=0', UBSAN_OPTIONS='print_stacktrace=1')
    jobs = golden_jobs(corpus) + fuzz_jobs(tmp_path, (1, 4, 15, 20), need_noBAQ=True)
    bad, ok, _ = run_many(emul_asan, oracle_bin, jobs, env)
    assert not bad and ok > 60, bad[:2]


def test_depth_boundary_emul(emul_bin, tmp_path):
    check_depth_boundary(emul_bin, str(tmp_path))


# ---------------------------------------------------------------- CUDA path
@pytest.fixture(scope='module')
def cli():
    assert os.path.exists(CLI), 'samtools_b200/bin/b200samtools missing: run python samtools_b200/build.py'
    return CLI


@pytest.mark.gpu
def test_golden_ranksums_gpu(cli, oracle_bin, corpus):
    """every golden mpileup case without text-only options, BAQ (21.out, 23.out), -6, -C and multi-file lists included (the
    97-column windows of these cases run on the emulation harness; the amplicon test runs windows on the device)"""
    jobs = golden_jobs(corpus)
    bad, ok, seen = run_many(cli, oracle_bin, jobs, fast=True)
    assert not bad and ok == len(jobs), bad[:2]
    assert seen.get('both', 0) > 0, seen


@pytest.mark.gpu
def test_multi_file_and_all_sums_gpu(cli, oracle_bin, corpus):
    mp = os.path.join(corpus, 'test', 'mpileup')
    jobs = [(mp, '-B -f mpileup.ref.fa mpileup.1.bam mpileup.2.bam mpileup.3.bam'), (mp, '-Q 0 -f mpileup.ref.fa mpileup.1.bam mpileup.2.bam mpileup.3.bam'),
            (os.path.join(corpus, 'test', 'dat'), '-B -b mpileup.bam.list')]
    for cwd, args in jobs:
        for sums in (False, True):
            assert run_pair(cli, oracle_bin, cwd, args, sums=sums, fast=True) is None
    r = subprocess.run([cli, 'counts', '--ranksums', '-B', '-f', 'mpileup.ref.fa', 'mpileup.1.bam', 'mpileup.2.bam', 'mpileup.3.bam'],
                       cwd=mp, capture_output=True, check=True)
    check_invariant(r.stdout, 3, CNT + PLANES)


@pytest.mark.gpu
def test_fuzz_ranksums_gpu(cli, oracle_bin, tmp_path):
    """fuzz SAMs under every option set without text-only options: BAQ, -C 50, -6, -E, -d, BED and regions"""
    bad, ok, seen = run_many(cli, oracle_bin, fuzz_jobs(tmp_path, (1, 15), need_noBAQ=False), fast=True)
    assert not bad and ok > 40, bad[:2]
    assert seen.get('both', 0) > 0 and seen.get('one_empty', 0) > 0 and seen.get('tie_across', 0) > 0, seen


@pytest.mark.gpu
def test_long_reads_ranksums_gpu(cli, oracle_bin, tmp_path):
    """reads of 513 b .. 40 kb with thousands of CIGAR ops (in 40-50 kb regions, BAQ on one of them): BP-5 above 1024 occurs
    and ranks as 1024"""
    from test_longread import write_long_inputs
    write_long_inputs(tmp_path)
    jobs = [(str(tmp_path), a) for a in ('-B -r chr1:1-50000 -f long.fa long.sam', '-r chr1:50001-90000 -f long.fa long.sam',
                                          '-B -Q 0 -r chr1:100000-140000 -f long.fa long.sam long2.sam', '-B -a -r chr1:90000-110000 -f long.fa long.bam',
                                          '-B -f cg.fa cg.sam', '-B -f del.fa del.sam')]
    bad, ok, seen = run_many(cli, oracle_bin, jobs, fast=True)
    assert not bad and ok == len(jobs), bad[:2]
    assert seen.get('pos_capped', 0) > 0 and seen.get('both', 0) > 0, seen


def write_amplicon(d, n_reads=20000, seed=5):
    """one amplicon of n_reads 100 bp reads over 1..100 of a random contig, half of them with a C>T (or other) change at
    column 50, random qualities and mapqs: a column of 20 000 reads above -d 8000, both classes deep"""
    rng = np.random.default_rng(seed)
    ref = ''.join(rng.choice(list('ACGT'), 300))
    with open(os.path.join(d, 'amp.fa'), 'w') as f:
        f.write(f'>amp\n{ref}\n')
    alt = {'A': 'G', 'C': 'T', 'G': 'A', 'T': 'C'}[ref[49]]
    with open(os.path.join(d, 'amp.sam'), 'w') as f:
        f.write('@SQ\tSN:amp\tLN:300\n')
        for i in range(n_reads):
            seq = list(ref[:100])
            if i & 1:
                seq[49] = alt
            q = ''.join(chr(33 + int(x)) for x in rng.integers(2, 42, 100))
            f.write(f'r{i}\t{16 if rng.random() < 0.5 else 0}\tamp\t1\t{int(rng.integers(0, 70))}\t100M\t*\t0\t0\t{"".join(seq)}\t{q}\n')


@pytest.mark.gpu
def test_amplicon_ranksums_gpu(cli, oracle_bin, tmp_path):
    """20 000 reads over one amplicon, a 50 % alt allele: above -d and below it, both classes with more than 1024 entries"""
    write_amplicon(str(tmp_path))
    jobs = [(str(tmp_path), a) for a in ('-B -d 0 -f amp.fa amp.sam', '-B -f amp.fa amp.sam', '-f amp.fa amp.sam', '-B -d 2500 -Q 0 -f amp.fa amp.sam')]
    bad, ok, _ = run_many(cli, oracle_bin, jobs, fast=True)
    assert not bad and ok == len(jobs), bad[:2]
    r = subprocess.run([cli, 'counts', '--ranksums', '-B', '-d', '0', '-r', 'amp:50-50', '-f', 'amp.fa', 'amp.sam'], cwd=str(tmp_path),
                       capture_output=True, check=True)
    v = [int(x) for x in r.stdout.split(b'\t')[3:]]
    assert v[CNT] > 1024 and v[CNT + 1] > 1024, v
    bad, ok, _ = run_many(cli, oracle_bin, jobs, dict(os.environ, B200_WINDOW_COLS='97'), fast=True)
    assert not bad and ok == len(jobs), bad[:2]


@pytest.mark.gpu
def test_depth_boundary_gpu(cli, tmp_path):
    check_depth_boundary(cli, str(tmp_path))


@pytest.fixture(scope='module')
def c2(tmp_path_factory):
    """the BASELINE C2 shape at 1 Mb: 30x, 150 bp pairs, with its FASTA (without one no base is of the ref class)"""
    from samtools_b200 import synth
    soa = synth.make_batch(length=1_000_000, depth=30, seed=2)
    d = tmp_path_factory.mktemp('c2')
    sam, fa = str(d / 'c2.sam'), str(d / 'c2.fa')
    synth.write_sam(sam, soa)
    synth.write_fasta(fa, soa['tid_name'], soa['ref_full'])
    return soa, sam, fa


C2_CHECK = 250_000   # the columns of the C2 batch compared with the oracle's text (-r), so that its parse stays short


def oracle_text(oracle, sam, fa, name):
    return subprocess.run([oracle, 'mpileup', '--reverse-del', '-s', '--output-BP-5', '-r', f'{name}:1-{C2_CHECK}', '-f', fa, sam],
                          capture_output=True, check=True).stdout


def oracle_planes(text):
    want = np.zeros((1, PLANES, C2_CHECK), np.int64)
    for ln in text.decode().split('\n')[:-1]:
        head, files = files_of(ln)
        if int(files[0][0]):
            want[0, :, int(head[1]) - 1] = rank_planes(class_entries(*files[0][1:], head[2]), fast=True)
    return want


@pytest.mark.gpu
def test_c2_ranksums_tensor_and_z(c2, oracle_bin):
    import torch
    from samtools_b200 import engine
    soa, sam, fa = c2
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n = int(e._n_cols)
    got = e.mpileup_ranksums(13)
    assert got.shape == (1, PLANES, n) and got.dtype == np.int64 and e.last_kernel_ms > 0
    text = oracle_text(oracle_bin, sam, fa, soa['tid_name'])
    assert np.array_equal(got[:, :, :C2_CHECK], oracle_planes(text))
    cnt = e.mpileup_counts(13)[0].astype(np.int64)
    assert np.array_equal(got[0, 0] + got[0, 1], cnt[0:4].sum(0) + cnt[9:13].sum(0))
    active = (got[0, 0] > 0) & (got[0, 1] > 0)
    assert active.sum() > 1000, active.sum()
    t = torch.full((1, PLANES, n), -1, dtype=torch.int64, device='cuda:0')
    assert e.mpileup_ranksums(13, out=t) is t
    assert np.array_equal(t.cpu().numpy(), got)
    with pytest.raises(ValueError):
        e.mpileup_ranksums(13, out=torch.zeros((1, PLANES, n), dtype=torch.int32, device='cuda:0'))
    with pytest.raises(ValueError):
        e.mpileup_ranksums(13, out=torch.zeros((1, PLANES, n + 1), dtype=torch.int64, device='cuda:0'))
    # z-scores: numpy and torch agree, NaN exactly where a class is empty or every value ties, and the two-sided p-values
    # are scipy's asymptotic ones without continuity correction
    z = engine.ranksum_z(got)
    zt = engine.ranksum_z(t)
    assert z.shape == (1, 3, n) and z.dtype == np.float64 and zt.is_cuda and zt.dtype == torch.float64
    assert np.array_equal(np.isnan(z), np.isnan(zt.cpu().numpy())) and np.allclose(z, zt.cpu().numpy(), rtol=1e-12, equal_nan=True)
    assert np.isnan(z[0][:, ~active]).all()
    checked = 0
    for ln in text.decode().split('\n')[:-1]:
        head, files = files_of(ln)
        c = int(head[1]) - 1
        if not int(files[0][0]) or not active[c]:
            continue
        ent = class_entries(*files[0][1:], head[2])
        ref = np.array([x[1:] for x in ent if x[0] == 'r']); alt = np.array([x[1:] for x in ent if x[0] == 'a'])
        for v in range(3):
            if len(np.unique(np.concatenate([ref[:, v], alt[:, v]]))) == 1:
                assert np.isnan(z[0, v, c])
                continue
            p = stats.mannwhitneyu(alt[:, v], ref[:, v], use_continuity=False, method='asymptotic').pvalue
            assert np.isclose(2 * stats.norm.sf(abs(z[0, v, c])), p, rtol=1e-9, atol=0), (c, v, z[0, v, c], p)
            checked += 1
        if checked > 3000:
            break
    assert checked > 3000
    e.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    with pytest.raises(RuntimeError, match='B200_MODE_MPILEUP'):
        e.mpileup_ranksums(13)
    e.close()


@pytest.mark.gpu
def test_c_abi_ranksums_errors(c2):
    import ctypes as C
    import torch
    from samtools_b200 import engine
    soa, _, _ = c2
    e = engine.Engine(0)
    n = C.c_int64(0)
    assert e.lib.b200_mpileup_ranksums(e.h, 13, None, 0, C.byref(n)) == -1                # nothing staged
    assert b'no staged batch' in e.lib.b200_last_error(e.h)
    e.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    assert e.lib.b200_mpileup_ranksums(e.h, 13, None, 0, C.byref(n)) == -1                # another mode
    assert b'B200_MODE_MPILEUP' in e.lib.b200_last_error(e.h)
    st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    assert e.lib.b200_mpileup_ranksums(e.h, 13, None, 0, C.byref(n)) == 0 and n.value == st.n_cols   # compute only
    small = np.zeros(PLANES * 16, np.int64)
    assert e.lib.b200_mpileup_ranksums(e.h, 13, small.ctypes.data_as(C.c_void_p), 16, C.byref(n)) == -2
    assert b'rank sum buffer too small' in e.lib.b200_last_error(e.h)
    if torch.cuda.device_count() > 1:
        t = torch.empty((1, PLANES, int(st.n_cols)), dtype=torch.int64, device='cuda:1')
        assert e.lib.b200_mpileup_ranksums(e.h, 13, C.c_void_p(t.data_ptr()), st.n_cols, C.byref(n)) == -1
        assert b'is on device 1' in e.lib.b200_last_error(e.h)
        with pytest.raises(ValueError):
            e.mpileup_ranksums(13, out=t)
    e.close()


@pytest.mark.gpu
def test_shard_ranksums_concatenate(c2):
    """plan_shards windows of one contig: their planes, side by side, are the planes of the whole contig"""
    from samtools_b200 import engine, shard
    soa, _, _ = c2
    L = int(soa['tid_len'])
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    whole = e.mpileup_ranksums(13)
    parts = []
    for beg, end in shard.plan_shards(L, 3):
        st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, beg=beg, end=end))
        assert st.n_cols == end - beg
        parts.append(e.mpileup_ranksums(13))
    e.close()
    assert np.array_equal(np.concatenate(parts, axis=2), whole[:, :, :L])
    assert ((whole[0, 0] > 0) & (whole[0, 1] > 0)).sum() > 1000
