"""Per-column quality sums (`b200samtools counts --qsums` / `indels --qsums`, b200_mpileup_qsums / b200_indel_qsums,
Engine.mpileup_qsums / Engine.indel_qsums) against the sums a parser takes from the oracle's `mpileup --reverse-del -s` text
of the same options: entry i of a file's sequence column pairs with character i of its quality and mapq columns.  CPU
through the emulation harness, and the CUDA path (BAQ included) under -m gpu."""
import os, re, subprocess
import numpy as np
import pytest
from conftest import ROOT
import test_counts
from test_counts import GOLDEN, fuzz_jobs

CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')
PLANES = 42
CNT = test_counts.PLANES


# ---------------------------------------------------------------- the text -> quality sums parser
def entry_kind(ch, ref_k):
    """kind 0-6 (A C G T N deletion skip) of one entry character, as test_counts.entry_counts counts it"""
    if ch in '.,':
        return ref_k
    if ch in '*#':
        return 5
    if ch in '><':
        return 6
    k = 'ACGT'.find(ch.upper())
    return 4 if k < 0 else k


def entry_qsums(seq, qual, mq, ref):
    """(42 planes, [(token, fwd, rev, bq_fwd, bq_rev, mq_fwd, mq_rev, mq0_fwd, mq0_rev)]) of one file's sequence, quality and
    -s columns; tokens in first-appearance order, upper-cased with '#' pads as '*', on the strand of the entry they follow"""
    p = [0] * PLANES
    found = {}
    ref_k = 'ACGT'.find(ref.upper()) if ref.upper() in 'ACGT' else 4
    i, n = 0, -1
    rev, bq, mqv, mq0 = False, 0, 0, 0
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
            a = found.setdefault(tok, [0] * 8)
            for k, x in enumerate((1, bq, mqv, mq0)):
                a[2 * k + rev] += x
            i = j + int(m.group(0))
        else:
            n += 1
            rev = ch in ',#<' or ch.islower()
            bq, mqv, mq0 = ord(qual[n]) - 33, ord(mq[n]) - 33, int(mq[n] == '!')
            k = 7 * rev + entry_kind(ch, ref_k)
            p[k] += bq; p[14 + k] += mqv; p[28 + k] += mq0
            i += 1
    assert n + 1 == len(qual) == len(mq), (seq, qual, mq)
    return p, [(t, *a) for t, a in found.items()]


def files_of(line):
    """chr, pos, ref and per file (cnt, seq, qual, mapq) of one `-s` line"""
    f = line.split('\t')
    return f[:3], [f[3 + 4 * k: 7 + 4 * k] for k in range((len(f) - 3) // 4)]


def count_rows(text_s, text, text_q0):
    """the `counts --qsums` rows: chr, pos, ref, then per file the 19 count planes and the 42 quality planes"""
    crow = test_counts.rows_from_text(text, text_q0).decode().split('\n')[:-1]
    srow = text_s.decode().split('\n')[:-1]
    assert len(crow) == len(srow)
    out = []
    for lc, ls in zip(crow, srow):
        head, files = files_of(ls)
        c = lc.split('\t')
        assert c[:3] == head
        vals = []
        for k, (cnt, seq, qual, mq) in enumerate(files):
            q = entry_qsums(seq, qual, mq, head[2])[0] if int(cnt) else [0] * PLANES
            vals += c[3 + CNT * k: 3 + CNT * (k + 1)] + [str(x) for x in q]
        out.append('\t'.join(head + vals) + '\n')
    return ''.join(out).encode()


def allele_rows(text_s):
    """the `indels --qsums` rows: chr, pos, ref, file, token, fwd, rev, then the six sums"""
    out = []
    for ln in text_s.decode().split('\n')[:-1]:
        head, files = files_of(ln)
        for k, (cnt, seq, qual, mq) in enumerate(files):
            if int(cnt):
                out += ['\t'.join(head + [str(k), t] + [str(x) for x in a]) + '\n' for t, *a in entry_qsums(seq, qual, mq, head[2])[1]]
    return ''.join(out).encode()


def test_parser_on_hand_made_columns():
    # '^' with a '+', ',' or '$' mapq character, an insertion and a deletion after one entry, pads, skips, N, reverse strand
    p, a = entry_qsums('^+.+2AC-1a$^,,*#><gN^$A$', '5?I~!#+0B', '~!A"#$%&(', 'c')
    want = [0] * PLANES
    for k, q, m in ((1, 20, 93), (8, 30, 0), (5, 40, 32), (12, 93, 1), (6, 0, 2), (13, 2, 3), (9, 10, 4), (4, 15, 5), (0, 33, 7)):
        want[k] += q; want[14 + k] += m; want[28 + k] += m == 0
    assert p == want
    assert a == [('+2AC', 1, 0, 20, 0, 93, 0, 0, 0), ('-1A', 1, 0, 20, 0, 93, 0, 0, 0)]
    assert allele_rows(b'c\t5\tA\t2\t.+1g,\t5!\t!~\t0\t*\t*\t*\t1\t,-1c\tI\tA\n') == \
        b'c\t5\tA\t0\t+1G\t1\t0\t20\t0\t0\t0\t1\t0\nc\t5\tA\t2\t-1C\t0\t1\t0\t40\t0\t32\t0\t0\n'


# ---------------------------------------------------------------- command lines
def run_pair(tool, oracle, cwd, args, prefix='', env=None, cmd='counts'):
    """None when `tool <cmd> --qsums <args>` prints the rows parsed from the oracle's text; 'baq' when the emulation harness
    cannot stage the case; else a description of the difference"""
    pre = re.sub(r'\$samtools\s+view', oracle + ' view', prefix).replace('$samtools', oracle)
    sh = lambda line: subprocess.run(pre + line, shell=True, cwd=cwd, capture_output=True, env=env, timeout=900)
    want_s = sh(f'{oracle} mpileup --reverse-del -s {args}')
    got = sh(f'{tool} {cmd} --qsums {args}')
    if got.returncode != 0 and b'BAQ kernel is not emulated' in got.stderr:
        return 'baq'
    if cmd == 'counts':
        exp = count_rows(want_s.stdout, sh(f'{oracle} mpileup --reverse-del {args}').stdout,
                         sh(f'{oracle} mpileup --reverse-del {args} -Q 0').stdout)
    else:
        exp = allele_rows(want_s.stdout)
    if got.returncode != 0 or got.stdout != exp:
        return (cmd, args, got.returncode, got.stderr[-300:], exp[:300], got.stdout[:300])
    return None


def run_many(tool, oracle, jobs, env=None):
    """both commands on every job, (cwd, args) or (cwd, args, prefix)"""
    from concurrent.futures import ThreadPoolExecutor
    full = [(j[0], j[1], j[2] if len(j) > 2 else '', cmd) for j in jobs for cmd in ('counts', 'indels')]
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        res = list(ex.map(lambda j: run_pair(tool, oracle, *j[:3], env=env, cmd=j[3]), full))
    return [r for r in res if r not in (None, 'baq')], sum(r is None for r in res)


def golden_jobs(corpus):
    return [(os.path.join(corpus, c['cwd']), c['args'], c['prefix']) for c in GOLDEN if '>' not in c['prefix']]


# ---------------------------------------------------------------- emulation harness (no GPU)
def build_emul(tmp_path_factory, name):
    exe = str(tmp_path_factory.mktemp(f'emul_{name}') / f'b200samtools_emul_{name}')
    host = os.path.join(ROOT, 'samtools_b200', 'csrc', 'host')
    subprocess.run(['g++', '-std=c++17', '-O1', '-g', '-ffp-contract=off', '-Wall', '-Wno-unused-function', '-Wno-parentheses', '-o', exe,
                    os.path.join(host, 'cli.cpp'), os.path.join(host, 'hts_io.cpp'), os.path.join(ROOT, 'tests', 'emul', f'emul_{name}.cpp'),
                    '-lz'], check=True)
    return exe


@pytest.fixture(scope='module')
def emul_bin(tmp_path_factory):
    """the CLI on the emulation harness with the count, indel and quality-sum outputs (tests/emul/emul_qsums.cpp)"""
    return build_emul(tmp_path_factory, 'qsums')


@pytest.fixture(scope='module')
def emul_without(tmp_path_factory):
    """the CLI on the harness builds with the count output (emul_counts.cpp) and the indel table (emul_indels.cpp), which have
    no quality sums"""
    return {name: build_emul(tmp_path_factory, name) for name in ('counts', 'indels')}


def test_engine_without_qsums_refuses(emul_without, corpus):
    """engine builds with the counts or the indel table but without the quality sums: --qsums stops with a message, and the
    commands without it still run"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    for name, exe in emul_without.items():
        r = subprocess.run([exe, name, '--qsums', 'mpileup.1.bam'], cwd=cwd, capture_output=True)
        assert r.returncode != 0 and r.stdout == b'' and b'no quality sums' in r.stderr, r.stderr
        r = subprocess.run([exe, name, 'mpileup.1.bam'], cwd=cwd, capture_output=True)
        assert r.returncode == 0 and r.stdout, r.stderr


def test_qsums_is_not_a_text_option(emul_bin, corpus):
    r = subprocess.run([emul_bin, 'mpileup', '--qsums', 'mpileup.1.bam'], cwd=os.path.join(corpus, 'test', 'mpileup'), capture_output=True)
    assert r.returncode != 0 and r.stdout == b'' and b'--qsums is an option of' in r.stderr


def test_without_flag_unchanged_emul(emul_bin, emul_without, corpus):
    """`counts` and `indels` without --qsums print what the harness builds without the quality sums print"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    for name, old in emul_without.items():
        for args in (['-B', 'mpileup.1.bam', 'mpileup.2.bam'], ['-B', '-Q', '0', '-a', 'mpileup.3.bam']):
            a = subprocess.run([old, name] + args, cwd=cwd, capture_output=True)
            b = subprocess.run([emul_bin, name] + args, cwd=cwd, capture_output=True)
            assert a.returncode == 0 and a.stdout and a.stdout == b.stdout


@pytest.mark.parametrize('case', GOLDEN, ids=[c['id'] for c in GOLDEN])
def test_golden_qsums_emul(case, emul_bin, oracle_bin, corpus):
    for cmd in ('counts', 'indels'):
        r = run_pair(emul_bin, oracle_bin, os.path.join(corpus, case['cwd']), case['args'], case['prefix'], cmd=cmd)
        if r == 'baq':
            pytest.skip('needs the BAQ kernel (covered by -m gpu)')
        assert r is None, r


def test_golden_qsums_windows_emul(emul_bin, oracle_bin, corpus):
    """97-column windows: every case crosses window edges (halo reads, -a rows, BED) and must print the same rows"""
    bad, ok = run_many(emul_bin, oracle_bin, golden_jobs(corpus), dict(os.environ, B200_WINDOW_COLS='97'))
    assert not bad and ok > 60, bad[:2]


def test_fuzz_qsums_emul(emul_bin, oracle_bin, tmp_path):
    bad, ok = run_many(emul_bin, oracle_bin, fuzz_jobs(tmp_path, range(1, 13), need_noBAQ=True))
    assert not bad and ok > 200, bad[:2]


# ---------------------------------------------------------------- CUDA path
@pytest.fixture(scope='module')
def cli():
    assert os.path.exists(CLI), 'samtools_b200/bin/b200samtools missing: run python samtools_b200/build.py'
    return CLI


@pytest.mark.gpu
def test_golden_qsums_gpu(cli, oracle_bin, corpus):
    """every golden mpileup case without text-only options, BAQ (21.out, 23.out), -6, -C and multi-file lists included, plain
    and in 97-column windows"""
    jobs = golden_jobs(corpus)
    for env in (None, dict(os.environ, B200_WINDOW_COLS='97')):
        bad, ok = run_many(cli, oracle_bin, jobs, env)
        assert not bad and ok == 2 * len(jobs), bad[:2]


@pytest.mark.gpu
def test_saturating_overlap_gpu(cli, oracle_bin, corpus):
    """the overlapping pair of dat/mpileup.out.5: its summed quality prints as '~', and BQ counts it as 93"""
    cwd = os.path.join(corpus, 'test', 'dat')
    args = '-r chr3:128814202-128814202 ../mpileup/overlap.bam'
    txt = subprocess.run(f'{oracle_bin} mpileup --reverse-del -s {args}', shell=True, cwd=cwd, capture_output=True).stdout
    assert txt.split(b'\t')[5] == b'~'
    for cmd in ('counts', 'indels'):
        assert run_pair(cli, oracle_bin, cwd, args, cmd=cmd) is None
    row = subprocess.run(f'{cli} counts --qsums {args}', shell=True, cwd=cwd, capture_output=True).stdout.split(b'\t')
    assert max(int(x) for x in row[3 + CNT: 3 + CNT + 14]) == 93


@pytest.mark.gpu
def test_fuzz_qsums_gpu(cli, oracle_bin, tmp_path):
    """fuzz SAMs under every option set without text-only options: BAQ, -C 50, -6, -E, -d, BED and regions"""
    bad, ok = run_many(cli, oracle_bin, fuzz_jobs(tmp_path, range(1, 7), need_noBAQ=False))
    assert not bad and ok > 200, bad[:2]


@pytest.mark.gpu
def test_cap_mapq_and_illumina_gpu(cli, oracle_bin, corpus):
    """-C (mapq after the cap) and -6 (qualities after the shift) on the golden BAMs"""
    cwd = os.path.join(corpus, 'test', 'mpileup')
    jobs = [(cwd, a) for a in ('-C 50 -f mpileup.ref.fa mpileup.1.bam mpileup.2.bam', '-B -C 20 -Q 0 -f mpileup.ref.fa mpileup.3.bam',
                               '-x -6 -f mpileup.ref.fa overlapIllumina.bam', '-B -6 -C 50 -Q 0 -f mpileup.ref.fa overlapIllumina.bam')]
    bad, ok = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == 2 * len(jobs), bad[:2]


@pytest.mark.gpu
def test_long_reads_qsums_gpu(cli, oracle_bin, tmp_path):
    """reads of 513 b .. 40 kb with hundreds to thousands of CIGAR ops, one of > 65535 ops, a 70 kb deletion"""
    from test_longread import write_long_inputs
    write_long_inputs(tmp_path)
    jobs = [(str(tmp_path), a) for a in ('-B -f long.fa long.sam', '-f long.fa long.sam', '-B -Q 0 -f long.fa long.sam long2.sam',
                                          '-B -a -r chr1:90000-110000 -f long.fa long.bam', '-B -f cg.fa cg.sam', '-B -f del.fa del.sam')]
    bad, ok = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == 2 * len(jobs), bad[:2]


@pytest.mark.gpu
def test_amplicon_max_depth_qsums_gpu(cli, oracle_bin, tmp_path):
    """amplicon stacks of 2500 .. 12000 pairs: -d 8000 and -d 2500 drop reads, with and without column windows"""
    from samtools_b200 import synth
    from test_gpu_maxdepth import make_amplicons
    soa = make_amplicons()
    synth.write_sam(str(tmp_path / 'amp.sam'), soa); synth.write_fasta(str(tmp_path / 'amp.fa'), 'amp', soa['ref_full'])
    jobs = [(str(tmp_path), a) for a in ('-B -f amp.fa amp.sam', '-f amp.fa amp.sam', '-B -d 2500 -Q 0 -f amp.fa amp.sam')]
    bad, ok = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == 2 * len(jobs), bad[:2]
    bad, ok = run_many(cli, oracle_bin, jobs[:1], dict(os.environ, B200_WINDOW_COLS='997'))
    assert not bad and ok == 2, bad[:2]


@pytest.fixture(scope='module')
def c2(tmp_path_factory):
    """the BASELINE C2 shape at 1 Mb: 30x, 150 bp pairs, no FASTA"""
    from samtools_b200 import synth
    soa = synth.make_batch(length=1_000_000, depth=30, seed=2)
    soa = dict(soa); soa['ref'] = None
    sam = str(tmp_path_factory.mktemp('c2') / 'c2.sam')
    synth.write_sam(sam, soa)
    return soa, sam


def check_invariants(cnt, qs, rows, iqs):
    """against the counts: an MQ0 plane <= its count plane, a BQ or MQ plane <= 93 x its count plane; per allele the MQ0
    counts <= fwd / rev and the sums <= 93 x fwd / rev; cnt [19, n] and qs [42, n] are one file's planes"""
    c = cnt.astype(np.int64)
    for r in range(2):
        for k in range(7):
            n = c[9 * r + k]
            assert (qs[28 + 7 * r + k] <= n).all() and (qs[7 * r + k] <= 93 * n).all() and (qs[14 + 7 * r + k] <= 93 * n).all()
    for r, f in enumerate(('fwd', 'rev')):
        n = rows[f].astype(np.int64)
        assert (iqs[:, 4 + r] <= n).all() and (iqs[:, r] <= 93 * n).all() and (iqs[:, 2 + r] <= 93 * n).all()


@pytest.mark.gpu
def test_c2_qsums_and_tensor_output(c2, oracle_bin):
    import torch
    from samtools_b200 import engine
    soa, sam = c2
    e = engine.Engine(0)
    st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n = int(st.n_cols)
    got = e.mpileup_qsums(13)
    assert got.shape == (1, PLANES, n) and e.last_kernel_ms > 0
    want = np.zeros((1, PLANES, n), np.uint32)
    text = subprocess.run([oracle_bin, 'mpileup', '--reverse-del', '-s', sam], capture_output=True, check=True).stdout
    for ln in text.decode().split('\n')[:-1]:
        head, files = files_of(ln)
        if int(files[0][0]):
            want[0, :, int(head[1]) - 1] = entry_qsums(*files[0][1:], head[2])[0]
    assert np.array_equal(got, want)
    t = torch.full((1, PLANES, n), -1, dtype=torch.int32, device='cuda:0')
    assert e.mpileup_qsums(13, out=t) is t
    assert np.array_equal(t.cpu().numpy().view(np.uint32), got)
    with pytest.raises(ValueError):
        e.mpileup_qsums(13, out=torch.zeros((1, PLANES, n + 1), dtype=torch.int32, device='cuda:0'))
    # the allele sums, against the parsed text and on the device
    rows, seq = e.mpileup_indels(13)
    iqs = e.indel_qsums()
    assert iqs.shape == (len(rows), 6) and iqs.dtype == np.uint32 and len(rows) > 1000 and e.last_kernel_ms > 0
    from test_indels import table_rows
    lines = [a + ''.join(f'\t{x}' for x in q) + '\n' for a, q in zip(table_rows(rows, seq, soa['tid_name']).decode().split('\n')[:-1], iqs)]
    assert ''.join(lines).encode() == allele_rows(text)
    tq = e.indel_qsums(device=True)
    assert tq.is_cuda and tq.dtype == torch.int32 and tuple(tq.shape) == iqs.shape
    assert np.array_equal(tq.cpu().numpy().view(np.uint32), iqs)
    check_invariants(e.mpileup_counts(13)[0], got[0], rows, iqs)
    e.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    with pytest.raises(RuntimeError, match='B200_MODE_MPILEUP'):
        e.mpileup_qsums(13)
    e.close()


@pytest.mark.gpu
def test_c_abi_qsums_errors(c2):
    import ctypes as C
    import torch
    from samtools_b200 import engine
    soa, _ = c2
    e = engine.Engine(0)
    st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n = C.c_int64(0)
    assert e.lib.b200_mpileup_qsums(e.h, 13, None, 0, C.byref(n)) == 0 and n.value == st.n_cols
    small = np.zeros(PLANES * 16, np.uint32)
    assert e.lib.b200_mpileup_qsums(e.h, 13, small.ctypes.data_as(C.c_void_p), 16, C.byref(n)) == -2
    assert b'quality sum buffer too small' in e.lib.b200_last_error(e.h)
    row = np.zeros((1, 6), np.uint32)
    assert e.lib.b200_indel_qsums(e.h, None, 0) == -1                                   # no table since the stage
    assert b'no indel table' in e.lib.b200_last_error(e.h)
    na, nb = C.c_int64(0), C.c_uint64(0)
    assert e.lib.b200_mpileup_indels(e.h, 13, C.byref(na), C.byref(nb)) == 0 and na.value > 1
    assert e.lib.b200_indel_qsums(e.h, None, 0) == 0                                    # compute only
    assert e.lib.b200_indel_qsums(e.h, row.ctypes.data_as(C.c_void_p), 1) == -2
    assert b'quality sum buffer too small' in e.lib.b200_last_error(e.h)
    if torch.cuda.device_count() > 1:
        t = torch.empty((na.value, 6), dtype=torch.int32, device='cuda:1')
        assert e.lib.b200_indel_qsums(e.h, C.c_void_p(t.data_ptr()), na.value) == -1
        assert b'is on device 1' in e.lib.b200_last_error(e.h)
        t = torch.empty((1, PLANES, int(st.n_cols)), dtype=torch.int32, device='cuda:1')
        assert e.lib.b200_mpileup_qsums(e.h, 13, C.c_void_p(t.data_ptr()), st.n_cols, C.byref(n)) == -1
        assert b'is on device 1' in e.lib.b200_last_error(e.h)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    assert e.lib.b200_indel_qsums(e.h, None, 0) == -1                                   # a new stage drops the table
    e.mpileup_indels(13)
    e.set_keep_raw(True)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    e.mpileup_indels(13)
    e.restage()
    with pytest.raises(RuntimeError, match='no indel table'):                            # and so does a restage
        e.indel_qsums()
    e.set_keep_raw(False)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    e.mpileup_indels(13)
    e.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    with pytest.raises(RuntimeError, match='no indel table'):                            # another mode has no table
        e.indel_qsums()
    e.close()


@pytest.mark.gpu
def test_shard_qsums_concatenate(c2):
    """plan_shards windows of one contig: their planes, side by side, are the planes of the whole contig, and their allele
    sums follow each other as the whole contig's do"""
    from samtools_b200 import engine, shard
    soa, _ = c2
    L = int(soa['tid_len'])
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    whole = e.mpileup_qsums(13)
    rows, _ = e.mpileup_indels(13)
    whole_iqs = e.indel_qsums()[rows['col'] < L]
    parts, iparts = [], []
    for beg, end in shard.plan_shards(L, 3):
        st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, beg=beg, end=end))
        assert st.n_cols == end - beg
        parts.append(e.mpileup_qsums(13))
        e.mpileup_indels(13)
        iparts.append(e.indel_qsums())
    e.close()
    assert np.array_equal(np.concatenate(parts, axis=2), whole[:, :, :L])
    assert np.array_equal(np.concatenate(iparts), whole_iqs)
