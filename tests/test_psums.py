"""Per-column read-position sums (`b200samtools counts --psums` / `indels --psums`, b200_mpileup_psums / b200_indel_psums,
Engine.mpileup_psums / Engine.indel_psums) against the sums a parser takes from the oracle's
`mpileup --reverse-del --output-BP-5` text of the same options: entry i of a file's sequence column pairs with number i of
its BP-5 column, and an indel token takes the BP-5 of the entry it follows.  CPU through the emulation harness, and the
CUDA path (BAQ included) under -m gpu."""
import os, re, subprocess
import numpy as np
import pytest
from conftest import ROOT
import test_counts
import test_indels
import test_qsums
from test_counts import GOLDEN, fuzz_jobs
from test_qsums import entry_kind, files_of, golden_jobs, build_emul

CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')
PLANES = 28
CNT = test_counts.PLANES
QS = test_qsums.PLANES
L_MAX = (1 << 28) - 1          # the longest CIGAR op


# ---------------------------------------------------------------- the text -> position sums parser
def entry_psums(seq, bp, ref):
    """(28 planes, [(token, fwd, rev, bp5_fwd, bp5_rev, bp5sq_fwd, bp5sq_rev)]) of one file's sequence and BP-5 columns;
    tokens in first-appearance order, upper-cased with '#' pads as '*', on the strand of the entry they follow"""
    p = [0] * PLANES
    found = {}
    pos = [int(x) for x in bp.split(',')]
    ref_k = 'ACGT'.find(ref.upper()) if ref.upper() in 'ACGT' else 4
    i, n = 0, -1
    rev, x = False, 0
    while i < len(seq):
        ch = seq[i]
        if ch == '^':                 # "^" + a mapq character, which may itself be '$', '+', '-', '.' or ','
            i += 2
        elif ch == '$':
            i += 1
        elif ch in '+-':
            m = re.match(r'\d+', seq[i + 1:])
            j = i + 1 + len(m.group(0))
            tok = ch + m.group(0) + seq[j:j + int(m.group(0))].upper().replace('#', '*')
            a = found.setdefault(tok, [0] * 6)
            for k, y in enumerate((1, x, x * x)):
                a[2 * k + rev] += y
            i = j + int(m.group(0))
        else:
            n += 1
            rev = ch in ',#<' or ch.islower()
            x = pos[n]
            k = 7 * rev + entry_kind(ch, ref_k)
            p[k] += x; p[14 + k] += x * x
            i += 1
    assert n + 1 == len(pos), (seq, bp)
    return p, [(t, *a) for t, a in found.items()]


def bp5_values(text):
    """every BP-5 number of a `--output-BP-5` text (without -s)"""
    out = []
    for ln in text.decode().split('\n')[:-1]:
        for cnt, _, _, bp in files_of(ln)[1]:
            if int(cnt):
                out += [int(x) for x in bp.split(',')]
    return out


def count_rows(text_bp, base, per_file):
    """the `counts --psums` rows: each row of `base` (chr, pos, ref, then per_file values per file: the counts, and the
    quality sums with --qsums) with the 28 position sums after each file's values"""
    brow = base.decode().split('\n')[:-1]
    prow = text_bp.decode().split('\n')[:-1]
    assert len(brow) == len(prow)
    out = []
    for lb, lp in zip(brow, prow):
        head, files = files_of(lp)
        b = lb.split('\t')
        assert b[:3] == head
        vals = []
        for k, (cnt, seq, _, bp) in enumerate(files):
            ps = entry_psums(seq, bp, head[2])[0] if int(cnt) else [0] * PLANES
            vals += b[3 + per_file * k: 3 + per_file * (k + 1)] + [str(x) for x in ps]
        out.append('\t'.join(head + vals) + '\n')
    return ''.join(out).encode()


def allele_psums(text_bp):
    """[(chr, pos, ref, file, token, fwd, rev, bp5_fwd, bp5_rev, bp5sq_fwd, bp5sq_rev)] of the lines' indel tokens"""
    out = []
    for ln in text_bp.decode().split('\n')[:-1]:
        head, files = files_of(ln)
        for k, (cnt, seq, _, bp) in enumerate(files):
            if int(cnt):
                out += [(*head, str(k), t, *a) for t, *a in entry_psums(seq, bp, head[2])[1]]
    return out


def allele_rows(text_bp, text_s=None):
    """the `indels --psums` rows (with text_s, the `-s` text: `indels --qsums --psums`): chr, pos, ref, file, token, fwd,
    rev, [the six quality sums,] then the four position sums"""
    rows = allele_psums(text_bp)
    if text_s is None:
        return ''.join('\t'.join(str(x) for x in r) + '\n' for r in rows).encode()
    qrows = test_qsums.allele_rows(text_s).decode().split('\n')[:-1]
    assert len(qrows) == len(rows)
    out = []
    for q, r in zip(qrows, rows):
        assert q.split('\t')[:7] == [str(x) for x in r[:7]]
        out.append(q + ''.join(f'\t{x}' for x in r[7:]) + '\n')
    return ''.join(out).encode()


def test_parser_on_hand_made_columns():
    # '^' with a '+' or '$' mapq character; an insertion and a deletion after one entry; an insertion after a deletion entry
    # (whose BP-5 counts is_del); a negative and a zero BP-5 on the reverse strand
    p, a = entry_psums('^+.+1g-2tt^$,*+2AC#-1n$', '4,-2,11,0', 'c')
    want = [0] * PLANES
    for k, x in ((1, 4), (8, -2), (5, 11), (12, 0)):
        want[k] += x; want[14 + k] += x * x
    assert p == want
    assert a == [('+1G', 1, 0, 4, 0, 16, 0), ('-2TT', 1, 0, 4, 0, 16, 0), ('+2AC', 1, 0, 11, 0, 121, 0), ('-1N', 0, 1, 0, 0, 0, 0)]
    line = b'c\t5\tA\t2\t.+1g,\t5!\t3,-7\t0\t*\t*\t*\t1\t,-1c\tI\t12\n'
    assert allele_rows(line) == b'c\t5\tA\t0\t+1G\t1\t0\t3\t0\t9\t0\nc\t5\tA\t2\t-1C\t0\t1\t0\t12\t0\t144\n'
    assert bp5_values(line) == [3, -7, 12]


# ---------------------------------------------------------------- command lines
def run_pair(tool, oracle, cwd, args, prefix='', env=None, cmd='counts', qsums=False):
    """(None when `tool <cmd> --psums <args>` prints the rows parsed from the oracle's text, 'baq' when the emulation harness
    cannot stage the case, else a description of the difference; the BP-5 numbers of the text)"""
    pre = re.sub(r'\$samtools\s+view', oracle + ' view', prefix).replace('$samtools', oracle)
    sh = lambda line: subprocess.run(pre + line, shell=True, cwd=cwd, capture_output=True, env=env, timeout=900)
    text_bp = sh(f'{oracle} mpileup --reverse-del --output-BP-5 {args}').stdout
    got = sh(f'{tool} {cmd} {"--qsums " if qsums else ""}--psums {args}')
    if got.returncode != 0 and b'BAQ kernel is not emulated' in got.stderr:
        return 'baq', []
    text_s = sh(f'{oracle} mpileup --reverse-del -s {args}').stdout if qsums else None
    if cmd == 'counts':
        text, text_q0 = sh(f'{oracle} mpileup --reverse-del {args}').stdout, sh(f'{oracle} mpileup --reverse-del {args} -Q 0').stdout
        base = test_qsums.count_rows(text_s, text, text_q0) if qsums else test_counts.rows_from_text(text, text_q0)
        exp = count_rows(text_bp, base, CNT + (QS if qsums else 0))
    else:
        exp = allele_rows(text_bp, text_s)
    if got.returncode != 0 or got.stdout != exp:
        return (cmd, args, got.returncode, got.stderr[-300:], exp[:300], got.stdout[:300]), []
    return None, bp5_values(text_bp)


def run_many(tool, oracle, jobs, env=None):
    """both commands on every job, (cwd, args) or (cwd, args, prefix): the differences, how many matched, the least BP-5"""
    from concurrent.futures import ThreadPoolExecutor
    full = [(j[0], j[1], j[2] if len(j) > 2 else '', cmd) for j in jobs for cmd in ('counts', 'indels')]
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        res = list(ex.map(lambda j: run_pair(tool, oracle, *j[:3], env=env, cmd=j[3]), full))
    low = min((min(v) for _, v in res if v), default=None)
    return [r for r, _ in res if r not in (None, 'baq')], sum(r is None for r, _ in res), low


def write_long_column(d, n, ins=False):
    """n forward reads without SEQ, each one CIGAR op of the longest length L at position 1 (then 1I with ins=True), on a
    contig of length L: every entry of the last columns is an N past the read's sequence with BP-5 = its position"""
    cig = f'{L_MAX}M' + ('1I' if ins else '')
    name = f'long{n}{"i" if ins else ""}.sam'
    with open(os.path.join(d, name), 'w') as f:
        f.write(f'@SQ\tSN:c\tLN:{L_MAX}\n')
        f.writelines(f'r{i}\t0\tc\t1\t60\t{cig}\t*\t0\t0\t*\t*\n' for i in range(n))
    return name


def check_overflow_boundary(tool, d):
    """the largest read count whose sums of squares fit in int64 gives exact sums; one read more fails with a message"""
    n = ((1 << 63) - 1) // (L_MAX * L_MAX)
    assert n * L_MAX * L_MAX <= (1 << 63) - 1 < (n + 1) * L_MAX * L_MAX
    region = f'-B -Q 0 -r c:{L_MAX - 2}-{L_MAX}'
    r = subprocess.run(f'{tool} counts --psums {region} {write_long_column(d, n)}', shell=True, cwd=d, capture_output=True, timeout=600)
    want = []
    for p in range(L_MAX - 2, L_MAX + 1):
        cnt, ps = [0] * CNT, [0] * PLANES
        cnt[4] = cnt[CNT - 1] = n                     # forward N, n_plp
        ps[4], ps[14 + 4] = n * p, n * p * p
        want.append('\t'.join(['c', str(p), 'N'] + [str(x) for x in cnt + ps]) + '\n')
    assert r.returncode == 0 and r.stdout == ''.join(want).encode(), (r.stderr, r.stdout[:400])
    r = subprocess.run(f'{tool} indels --psums {region} {write_long_column(d, n, True)}', shell=True, cwd=d, capture_output=True, timeout=600)
    assert r.returncode == 0 and r.stdout == f'c\t{L_MAX}\tN\t0\t+1N\t{n}\t0\t{n * L_MAX}\t0\t{n * L_MAX * L_MAX}\t0\n'.encode(), r.stderr
    for cmd, ins in (('counts', False), ('indels', True)):
        r = subprocess.run(f'{tool} {cmd} --psums {region} {write_long_column(d, n + 1, ins)}', shell=True, cwd=d, capture_output=True, timeout=600)
        assert r.returncode != 0 and b'squared read positions would exceed 2^63 - 1' in r.stderr, (cmd, r.returncode, r.stderr)


def test_ctypes_row_matches_c(tmp_path):
    """sizeof(b200_indel_psum_t) and its field offsets from the C compiler equal the ctypes mirror"""
    import ctypes as C
    from samtools_b200 import engine
    src = tmp_path / 'sz.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200_pileup.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu\\n", sizeof(b200_indel_psum_t), offsetof(b200_indel_psum_t, bp5_fwd), '
                   'offsetof(b200_indel_psum_t, bp5_rev), offsetof(b200_indel_psum_t, bp5sq_fwd), offsetof(b200_indel_psum_t, bp5sq_rev)); return 0; }\n')
    exe = str(tmp_path / 'sz')
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', exe, str(src)], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, check=True).stdout.split()]
    assert got == [C.sizeof(engine.IndelPsum)] + [getattr(engine.IndelPsum, f).offset for f in engine.INDEL_PSUM_FIELDS]
    assert got[0] == 32 and engine.INDEL_PSUM_FIELDS == ('bp5_fwd', 'bp5_rev', 'bp5sq_fwd', 'bp5sq_rev')


# ---------------------------------------------------------------- emulation harness (no GPU)
@pytest.fixture(scope='module')
def emul_bin(tmp_path_factory):
    """the CLI on the emulation harness with the count, indel, quality-sum and position-sum outputs (emul_psums.cpp)"""
    return build_emul(tmp_path_factory, 'psums')


@pytest.fixture(scope='module')
def emul_qsums(tmp_path_factory):
    """the CLI on the harness build with the quality sums (emul_qsums.cpp), which has no position sums"""
    return build_emul(tmp_path_factory, 'qsums')


def test_engine_without_psums_refuses(emul_qsums, corpus):
    """an engine build with the quality sums but without the position sums: --psums stops with a message, and `counts`,
    `indels` and their --qsums still run"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    for cmd in ('counts', 'indels'):
        r = subprocess.run([emul_qsums, cmd, '--psums', 'mpileup.1.bam'], cwd=cwd, capture_output=True)
        assert r.returncode != 0 and r.stdout == b'' and b'this engine build has no position sums' in r.stderr, r.stderr
        for extra in ([], ['--qsums']):
            r = subprocess.run([emul_qsums, cmd] + extra + ['mpileup.1.bam'], cwd=cwd, capture_output=True)
            assert r.returncode == 0 and r.stdout, r.stderr


def test_psums_is_not_a_text_option(emul_bin, corpus):
    r = subprocess.run([emul_bin, 'mpileup', '--psums', 'mpileup.1.bam'], cwd=os.path.join(corpus, 'test', 'mpileup'), capture_output=True)
    assert r.returncode != 0 and r.stdout == b'' and b'--psums is an option of' in r.stderr


def test_without_flag_unchanged_emul(emul_bin, emul_qsums, corpus):
    """`counts` and `indels` without --psums (with and without --qsums) print what the harness build without the position
    sums prints"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    for cmd in ('counts', 'indels'):
        for args in (['-B', 'mpileup.1.bam', 'mpileup.2.bam'], ['-B', '-Q', '0', '-a', 'mpileup.3.bam'], ['--qsums', '-B', 'mpileup.1.bam']):
            a = subprocess.run([emul_qsums, cmd] + args, cwd=cwd, capture_output=True)
            b = subprocess.run([emul_bin, cmd] + args, cwd=cwd, capture_output=True)
            assert a.returncode == 0 and a.stdout and a.stdout == b.stdout


def test_oracle_bp5_is_the_golden_one(oracle_bin, corpus):
    """the oracle's --output-BP-5 column on output-BP.sam is the one of the reference's 81.out, reverse-strand deletions
    printing 11 included; the oracle's text is what the sums are taken from"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    got = subprocess.run([oracle_bin, 'mpileup', '--output-BP-5', 'output-BP.sam'], cwd=cwd, capture_output=True, check=True).stdout
    want = open(os.path.join(cwd, 'expected', '81.out'), 'rb').read()
    col = lambda t: [ln.split(b'\t')[-1] for ln in t.split(b'\n')[:-1]]
    assert col(got) == col(want) and b'11,11' in col(want)
    rd = subprocess.run([oracle_bin, 'mpileup', '--reverse-del', '--output-BP-5', 'output-BP.sam'], cwd=cwd, capture_output=True, check=True).stdout
    assert col(rd) == col(want)


def test_output_bp_psums_emul(emul_bin, oracle_bin, corpus):
    """output-BP.sam (a deletion on both strands, an insertion after it): the sums of the golden's BP-5 column"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    for args in ('output-BP.sam', '-Q 0 output-BP.sam', '-B -Q 0 -a output-BP.sam'):
        for cmd in ('counts', 'indels'):
            for qsums in (False, True):
                r, v = run_pair(emul_bin, oracle_bin, cwd, args, cmd=cmd, qsums=qsums)
                assert r is None and v, r
    rows = subprocess.run([emul_bin, 'indels', '--psums', 'output-BP.sam'], cwd=cwd, capture_output=True, check=True).stdout
    assert rows.split(b'\n')[0].split(b'\t')[4:] == [b'-3NNN', b'1', b'1', b'10', b'11', b'100', b'121']


@pytest.mark.parametrize('case', GOLDEN, ids=[c['id'] for c in GOLDEN])
def test_golden_psums_emul(case, emul_bin, oracle_bin, corpus):
    for cmd in ('counts', 'indels'):
        r, _ = run_pair(emul_bin, oracle_bin, os.path.join(corpus, case['cwd']), case['args'], case['prefix'], cmd=cmd)
        if r == 'baq':
            pytest.skip('needs the BAQ kernel (covered by -m gpu)')
        assert r is None, r


def test_golden_psums_windows_emul(emul_bin, oracle_bin, corpus):
    """97-column windows: every case crosses window edges (halo reads, -a rows, BED) and must print the same rows"""
    bad, ok, _ = run_many(emul_bin, oracle_bin, golden_jobs(corpus), dict(os.environ, B200_WINDOW_COLS='97'))
    assert not bad and ok > 60, bad[:2]


# The fuzz seeds: SEQ '*' records come with the seeds divisible by 5 (fuzz_sam.py), but those of seeds 5 and 10 are all on the
# forward strand; 15, 20 and 25 add reverse-strand ones, whose BP-5 at -Q 0 is l_qseq - qpos <= 0.
FUZZ_SEEDS = list(range(1, 13)) + [15, 20, 25]


def test_fuzz_psums_emul(emul_bin, oracle_bin, tmp_path):
    """the fuzz SAMs, SEQ '*' records at -Q 0 among them: a BP-5 <= 0 must occur, so the signed sums are exercised"""
    bad, ok, low = run_many(emul_bin, oracle_bin, fuzz_jobs(tmp_path, FUZZ_SEEDS, need_noBAQ=True))
    assert not bad and ok > 200, bad[:2]
    assert low is not None and low <= 0, low


def test_overflow_boundary_emul(emul_bin, tmp_path):
    check_overflow_boundary(emul_bin, str(tmp_path))


# ---------------------------------------------------------------- CUDA path
@pytest.fixture(scope='module')
def cli():
    assert os.path.exists(CLI), 'samtools_b200/bin/b200samtools missing: run python samtools_b200/build.py'
    return CLI


@pytest.mark.gpu
def test_golden_psums_gpu(cli, oracle_bin, corpus):
    """every golden mpileup case without text-only options, BAQ (21.out, 23.out), -6, -C and multi-file lists included, plain
    and in 97-column windows"""
    jobs = golden_jobs(corpus)
    for env in (None, dict(os.environ, B200_WINDOW_COLS='97')):
        bad, ok, _ = run_many(cli, oracle_bin, jobs, env)
        assert not bad and ok == 2 * len(jobs), bad[:2]


@pytest.mark.gpu
def test_output_bp_and_multi_file_gpu(cli, oracle_bin, corpus):
    """output-BP.sam, and multi-file lists, with --qsums beside --psums too"""
    mp = os.path.join(corpus, 'test', 'mpileup')
    jobs = [(mp, 'output-BP.sam'), (mp, '-B -Q 0 -a output-BP.sam'), (mp, '-B mpileup.1.bam mpileup.2.bam mpileup.3.bam'),
            (mp, '-Q 0 -f mpileup.ref.fa mpileup.1.bam mpileup.2.bam mpileup.3.bam'),
            (os.path.join(corpus, 'test', 'dat'), '-B -b mpileup.bam.list')]
    for cwd, args in jobs:
        for cmd in ('counts', 'indels'):
            for qsums in (False, True):
                r, v = run_pair(cli, oracle_bin, cwd, args, cmd=cmd, qsums=qsums)
                assert r is None and v, r


@pytest.mark.gpu
def test_fuzz_psums_gpu(cli, oracle_bin, tmp_path):
    """fuzz SAMs under every option set without text-only options: BAQ, -C 50, -6, -E, -d, BED and regions; seed 15 has
    reverse-strand SEQ '*' records"""
    bad, ok, low = run_many(cli, oracle_bin, fuzz_jobs(tmp_path, (1, 2, 3, 15), need_noBAQ=False))
    assert not bad and ok > 150, bad[:2]
    assert low is not None and low <= 0, low


@pytest.mark.gpu
def test_long_reads_psums_gpu(cli, oracle_bin, tmp_path):
    """reads of 513 b .. 40 kb with hundreds to thousands of CIGAR ops, one of > 65535 ops, a 70 kb deletion; sums of squares
    past 2^32"""
    from test_longread import write_long_inputs
    write_long_inputs(tmp_path)
    jobs = [(str(tmp_path), a) for a in ('-B -f long.fa long.sam', '-f long.fa long.sam', '-B -Q 0 -f long.fa long.sam long2.sam',
                                          '-B -a -r chr1:90000-110000 -f long.fa long.bam', '-B -f cg.fa cg.sam', '-B -f del.fa del.sam')]
    bad, ok, _ = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == 2 * len(jobs), bad[:2]
    text = subprocess.run(f'{oracle_bin} mpileup --reverse-del --output-BP-5 -B -f long.fa long.sam', shell=True, cwd=str(tmp_path),
                          capture_output=True, check=True).stdout
    assert max(max(entry_psums(f[1], f[3], ln.split('\t')[2])[0][14:]) for ln in text.decode().split('\n')[:-1]
               for f in files_of(ln)[1] if int(f[0])) >= 1 << 32


@pytest.mark.gpu
def test_amplicon_max_depth_psums_gpu(cli, oracle_bin, tmp_path):
    """amplicon stacks of 2500 .. 12000 pairs: -d 8000 and -d 2500 drop reads, with and without column windows"""
    from samtools_b200 import synth
    from test_gpu_maxdepth import make_amplicons
    soa = make_amplicons()
    synth.write_sam(str(tmp_path / 'amp.sam'), soa); synth.write_fasta(str(tmp_path / 'amp.fa'), 'amp', soa['ref_full'])
    jobs = [(str(tmp_path), a) for a in ('-B -f amp.fa amp.sam', '-f amp.fa amp.sam', '-B -d 2500 -Q 0 -f amp.fa amp.sam')]
    bad, ok, _ = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == 2 * len(jobs), bad[:2]
    bad, ok, _ = run_many(cli, oracle_bin, jobs, dict(os.environ, B200_WINDOW_COLS='997'))
    assert not bad and ok == 2 * len(jobs), bad[:2]


@pytest.mark.gpu
def test_overflow_boundary_gpu(cli, tmp_path):
    check_overflow_boundary(cli, str(tmp_path))


@pytest.fixture(scope='module')
def c2(tmp_path_factory):
    """the BASELINE C2 shape at 1 Mb: 30x, 150 bp pairs, no FASTA"""
    from samtools_b200 import synth
    soa = synth.make_batch(length=1_000_000, depth=30, seed=2)
    soa = dict(soa); soa['ref'] = None
    sam = str(tmp_path_factory.mktemp('c2') / 'c2.sam')
    synth.write_sam(sam, soa)
    return soa, sam


def check_cauchy_schwarz(cnt, ps, rows, ips):
    """per cell and per allele with m > 0 entries: m * sum(BP-5^2) >= sum(BP-5)^2; cnt [19, n] and ps [28, n] are one file's
    planes"""
    c = cnt.astype(np.int64)
    for r in range(2):
        for k in range(7):
            m, s, q = c[9 * r + k], ps[7 * r + k], ps[14 + 7 * r + k]
            assert ((m == 0) | (m * q >= s * s)).all() and ((m > 0) | ((s == 0) & (q == 0))).all()
    for r, f in enumerate(('fwd', 'rev')):
        m = rows[f].astype(np.int64)
        assert ((m == 0) | (m * ips[:, 2 + r] >= ips[:, r] ** 2)).all()


@pytest.mark.gpu
def test_c2_psums_and_tensor_output(c2, oracle_bin):
    import torch
    from samtools_b200 import engine
    soa, sam = c2
    e = engine.Engine(0)
    st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n = int(st.n_cols)
    got = e.mpileup_psums(13)
    assert got.shape == (1, PLANES, n) and got.dtype == np.int64 and e.last_kernel_ms > 0
    want = np.zeros((1, PLANES, n), np.int64)
    text = subprocess.run([oracle_bin, 'mpileup', '--reverse-del', '--output-BP-5', sam], capture_output=True, check=True).stdout
    for ln in text.decode().split('\n')[:-1]:
        head, files = files_of(ln)
        if int(files[0][0]):
            want[0, :, int(head[1]) - 1] = entry_psums(files[0][1], files[0][3], head[2])[0]
    assert np.array_equal(got, want)
    t = torch.full((1, PLANES, n), -1, dtype=torch.int64, device='cuda:0')
    assert e.mpileup_psums(13, out=t) is t
    assert np.array_equal(t.cpu().numpy(), got)
    with pytest.raises(ValueError):
        e.mpileup_psums(13, out=torch.zeros((1, PLANES, n), dtype=torch.int32, device='cuda:0'))
    with pytest.raises(ValueError):
        e.mpileup_psums(13, out=torch.zeros((1, PLANES, n + 1), dtype=torch.int64, device='cuda:0'))
    # the allele sums, against the parsed text and on the device
    rows, seq = e.mpileup_indels(13)
    ips = e.indel_psums()
    assert ips.shape == (len(rows), 4) and ips.dtype == np.int64 and len(rows) > 1000 and e.last_kernel_ms > 0
    from test_indels import table_rows
    lines = [a + ''.join(f'\t{x}' for x in q) + '\n' for a, q in zip(table_rows(rows, seq, soa['tid_name']).decode().split('\n')[:-1], ips)]
    assert ''.join(lines).encode() == allele_rows(text)
    tp = e.indel_psums(device=True)
    assert tp.is_cuda and tp.dtype == torch.int64 and tuple(tp.shape) == ips.shape
    assert np.array_equal(tp.cpu().numpy(), ips)
    check_cauchy_schwarz(e.mpileup_counts(13)[0], got[0], rows, ips)
    e.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    with pytest.raises(RuntimeError, match='B200_MODE_MPILEUP'):
        e.mpileup_psums(13)
    e.close()


@pytest.mark.gpu
def test_c_abi_psums_errors(c2):
    import ctypes as C
    import torch
    from samtools_b200 import engine
    soa, _ = c2
    e = engine.Engine(0)
    st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n = C.c_int64(0)
    assert e.lib.b200_mpileup_psums(e.h, 13, None, 0, C.byref(n)) == 0 and n.value == st.n_cols   # compute only
    small = np.zeros(PLANES * 16, np.int64)
    assert e.lib.b200_mpileup_psums(e.h, 13, small.ctypes.data_as(C.c_void_p), 16, C.byref(n)) == -2
    assert b'position sum buffer too small' in e.lib.b200_last_error(e.h)
    row = np.zeros((1, 4), np.int64)
    assert e.lib.b200_indel_psums(e.h, None, 0) == -1                                   # no table since the stage
    assert b'no indel table' in e.lib.b200_last_error(e.h)
    na, nb = C.c_int64(0), C.c_uint64(0)
    assert e.lib.b200_mpileup_indels(e.h, 13, C.byref(na), C.byref(nb)) == 0 and na.value > 1
    assert e.lib.b200_indel_psums(e.h, None, 0) == 0                                    # compute only
    assert e.lib.b200_indel_psums(e.h, row.ctypes.data_as(C.c_void_p), 1) == -2
    assert b'position sum buffer too small' in e.lib.b200_last_error(e.h)
    if torch.cuda.device_count() > 1:
        t = torch.empty((na.value, 4), dtype=torch.int64, device='cuda:1')
        assert e.lib.b200_indel_psums(e.h, C.c_void_p(t.data_ptr()), na.value) == -1
        assert b'is on device 1' in e.lib.b200_last_error(e.h)
        t = torch.empty((1, PLANES, int(st.n_cols)), dtype=torch.int64, device='cuda:1')
        assert e.lib.b200_mpileup_psums(e.h, 13, C.c_void_p(t.data_ptr()), st.n_cols, C.byref(n)) == -1
        assert b'is on device 1' in e.lib.b200_last_error(e.h)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    assert e.lib.b200_indel_psums(e.h, None, 0) == -1                                   # a new stage drops the table
    e.mpileup_indels(13)
    e.set_keep_raw(True)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    e.mpileup_indels(13)
    e.restage()
    with pytest.raises(RuntimeError, match='no indel table'):                            # and so does a restage
        e.indel_psums()
    e.set_keep_raw(False)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    e.mpileup_indels(13)
    e.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    with pytest.raises(RuntimeError, match='no indel table'):                            # another mode has no table
        e.indel_psums()
    e.close()


@pytest.mark.gpu
def test_shard_psums_concatenate(c2):
    """plan_shards windows of one contig: their planes, side by side, are the planes of the whole contig, and their allele
    sums follow each other as the whole contig's do"""
    from samtools_b200 import engine, shard
    soa, _ = c2
    L = int(soa['tid_len'])
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    whole = e.mpileup_psums(13)
    rows, _ = e.mpileup_indels(13)
    whole_ips = e.indel_psums()[rows['col'] < L]
    parts, iparts = [], []
    for beg, end in shard.plan_shards(L, 3):
        st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, beg=beg, end=end))
        assert st.n_cols == end - beg
        parts.append(e.mpileup_psums(13))
        e.mpileup_indels(13)
        iparts.append(e.indel_psums())
    e.close()
    assert np.array_equal(np.concatenate(parts, axis=2), whole[:, :, :L])
    assert np.array_equal(np.concatenate(iparts), whole_ips)
