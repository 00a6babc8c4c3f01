"""Per-column indel alleles (`b200samtools indels`, b200_mpileup_indels / b200_fetch_indels, Engine.mpileup_indels) against
the alleles a parser takes from the oracle's `mpileup --reverse-del` text of the same options: CPU through the emulation
harness, and the CUDA path (BAQ included) under -m gpu."""
import os, random, re, subprocess
import numpy as np
import pytest
from conftest import ROOT
from test_counts import GOLDEN, fuzz_jobs

CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')


# ---------------------------------------------------------------- the text -> alleles parser
def entry_alleles(seq):
    """[(token, fwd, rev)] of one file's pileup sequence column, in first-appearance order: each "+n..." / "-n..." token
    upper-cased with '#' pads as '*', on the strand of the entry it follows"""
    found = {}
    i, rev = 0, False
    while i < len(seq):
        ch = seq[i]
        if ch == '^':                 # "^" + a mapq character, which may itself be '$', '+', '-', '.' or ','
            i += 2
        elif ch == '$':
            i += 1
        elif ch in '+-':
            m = re.match(r'\d+', seq[i + 1:])
            j = i + 1 + len(m.group(0))
            n = int(m.group(0))
            tok = ch + m.group(0) + seq[j:j + n].upper().replace('#', '*')
            f, r = found.get(tok, (0, 0))
            found[tok] = (f + (not rev), r + rev)
            i = j + n
        else:
            rev = ch in ',#<' or ch.islower()
            i += 1
    return [(t, f, r) for t, (f, r) in found.items()]


def rows_from_text(text):
    """the `indels` rows of mpileup's lines: chr, pos, ref, file, token, fwd, rev"""
    out = []
    for ln in text.decode().split('\n')[:-1]:
        fa = ln.split('\t')
        for f in range((len(fa) - 3) // 3):
            if int(fa[3 + 3 * f]):
                out += [f'{fa[0]}\t{fa[1]}\t{fa[2]}\t{f}\t{t}\t{a}\t{b}\n' for t, a, b in entry_alleles(fa[4 + 3 * f])]
    return ''.join(out).encode()


def test_parser_on_hand_made_columns():
    # +n then -m on one entry, pads on both strands, '^' with a '+', '-' or '$' mapq character, reverse strand, N tokens
    assert entry_alleles('.+2AC-2GT,+2ac^+.^-,+1N^$a$-2gt,+3a#c.+3A*C') == \
        [('+2AC', 1, 1), ('-2GT', 1, 1), ('+1N', 0, 1), ('+3A*C', 1, 1)]
    assert entry_alleles('*-1N#-1n<>.+3N*N') == [('-1N', 1, 1), ('+3N*N', 1, 0)]
    assert rows_from_text(b'c\t5\tA\t2\t.+1g,\t??\t0\t*\t*\t1\t,-1c\t?\n') == \
        b'c\t5\tA\t0\t+1G\t1\t0\nc\t5\tA\t2\t-1C\t0\t1\n'


# ---------------------------------------------------------------- command lines
def run_pair(tool, oracle, cwd, args, prefix='', env=None):
    """None when `tool indels <args>` prints the rows parsed from the oracle's text; 'baq' when the emulation harness
    cannot stage the case; else a description of the difference"""
    pre = re.sub(r'\$samtools\s+view', oracle + ' view', prefix).replace('$samtools', oracle)
    sh = lambda line: subprocess.run(pre + line, shell=True, cwd=cwd, capture_output=True, env=env, timeout=900)
    want = sh(f'{oracle} mpileup --reverse-del {args}')
    got = sh(f'{tool} indels {args}')
    if got.returncode != 0 and b'BAQ kernel is not emulated' in got.stderr:
        return 'baq'
    exp = rows_from_text(want.stdout)
    if got.returncode != 0 or got.stdout != exp:
        return (args, got.returncode, got.stderr[-300:], exp[:300], got.stdout[:300])
    return None


def run_many(tool, oracle, jobs, env=None):
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        res = list(ex.map(lambda j: run_pair(tool, oracle, *j, env=env), jobs))
    return [r for r in res if r not in (None, 'baq')], sum(r is None for r in res)


def write_deep(d, n_same, n_short, n_long, n_del, seed=7):
    """one column (position 160) under reads that all start at 101: n_same share the insertion +2AC, n_short carry distinct
    insertions of 1-12 symbols, n_long distinct ones of 13-40 symbols (and a tenth of them one shared 30-mer), n_del
    deletions of 1-5 bases; shuffled, a third on the reverse strand.  Writes deep.sam and deep.fa."""
    rng = random.Random(seed)
    ref = ''.join(rng.choice('ACGT') for _ in range(400))
    shared_long = ''.join(rng.choice('ACGT') for _ in range(30))
    ins, seen = [], set()
    ins += ['AC'] * n_same
    while len(seen) < n_short:
        s = ''.join(rng.choice('ACGTN') for _ in range(rng.randint(1, 12)))
        if s != 'AC' and s not in seen:
            seen.add(s); ins.append(s)
    while len(seen) < n_short + n_long:
        s = ''.join(rng.choice('ACGT') for _ in range(rng.randint(13, 40)))
        if s not in seen:
            seen.add(s); ins.append(s)
    ins += [shared_long] * (n_long // 10)
    recs = [('I', s) for s in ins] + [('D', rng.randint(1, 5)) for _ in range(n_del)]
    rng.shuffle(recs)
    lines = ['@HD\tVN:1.6\tSO:coordinate', f'@SQ\tSN:d\tLN:{len(ref)}']
    for k, (op, x) in enumerate(recs):
        if op == 'I':
            seq, cig = ref[100:160] + x + ref[160:220], f'60M{len(x)}I60M'
        else:
            seq, cig = ref[100:160] + ref[160 + x:220 + x], f'60M{x}D60M'
        lines.append(f'r{k}\t{16 if k % 3 == 0 else 0}\td\t101\t60\t{cig}\t*\t0\t0\t{seq}\t{"I" * len(seq)}')
    (d / 'deep.sam').write_text('\n'.join(lines) + '\n')
    (d / 'deep.fa').write_text('>d\n' + ref + '\n')


DEEP_ARGS = '-B -d 100000 -f deep.fa deep.sam'


# ---------------------------------------------------------------- emulation harness (no GPU)
@pytest.fixture(scope='module')
def emul_bin(tmp_path_factory):
    """the CLI on the emulation harness with the indel output (tests/emul/emul_indels.cpp), built here: pytest-xdist workers
    rebuild tests/emul/_build concurrently"""
    exe = str(tmp_path_factory.mktemp('emul_indels') / 'b200samtools_emul_indels')
    host = os.path.join(ROOT, 'samtools_b200', 'csrc', 'host')
    subprocess.run(['g++', '-std=c++17', '-O1', '-g', '-ffp-contract=off', '-Wall', '-Wno-unused-function', '-Wno-parentheses', '-o', exe,
                    os.path.join(host, 'cli.cpp'), os.path.join(host, 'hts_io.cpp'), os.path.join(ROOT, 'tests', 'emul', 'emul_indels.cpp'),
                    '-lz'], check=True)
    return exe


def test_engine_without_indel_output_refuses(corpus):
    """the harness build without b200_mpileup_indels: `indels` stops with a message instead of printing rows"""
    subprocess.run([os.path.join(ROOT, 'tests', 'emul', 'build.sh')], check=True)
    exe = os.path.join(ROOT, 'tests', 'emul', '_build', 'b200samtools_emul')
    r = subprocess.run([exe, 'indels', 'mpileup.1.bam'], cwd=os.path.join(corpus, 'test', 'mpileup'), capture_output=True)
    assert r.returncode != 0 and r.stdout == b'' and b'no indel output' in r.stderr


@pytest.mark.parametrize('case', GOLDEN, ids=[c['id'] for c in GOLDEN])
def test_golden_indels_emul(case, emul_bin, oracle_bin, corpus):
    r = run_pair(emul_bin, oracle_bin, os.path.join(corpus, case['cwd']), case['args'], case['prefix'])
    if r == 'baq':
        pytest.skip('needs the BAQ kernel (covered by -m gpu)')
    assert r is None, r


def test_golden_indels_windows_emul(emul_bin, oracle_bin, corpus):
    """97-column windows: every case crosses window edges and must print the same rows"""
    env = dict(os.environ, B200_WINDOW_COLS='97')
    jobs = [(os.path.join(corpus, c['cwd']), c['args'], c['prefix']) for c in GOLDEN if '>' not in c['prefix']]
    bad, ok = run_many(emul_bin, oracle_bin, jobs, env)
    assert not bad and ok > 30, bad[:2]


def test_fuzz_indels_emul(emul_bin, oracle_bin, tmp_path):
    bad, ok = run_many(emul_bin, oracle_bin, fuzz_jobs(tmp_path, range(1, 13), need_noBAQ=True))
    assert not bad and ok > 100, bad[:2]


def test_forced_key_collisions_emul(emul_bin, oracle_bin, corpus, tmp_path):
    """keys of 0 and 3 bits: different insertions share keys, and the rows stay the same"""
    write_deep(tmp_path, n_same=200, n_short=150, n_long=60, n_del=30)
    jobs = [(os.path.join(corpus, c['cwd']), c['args'], c['prefix']) for c in GOLDEN if '>' not in c['prefix']]
    jobs += fuzz_jobs(tmp_path, range(1, 4), need_noBAQ=True) + [(str(tmp_path), DEEP_ARGS)]
    for bits in ('0', '3'):
        bad, ok = run_many(emul_bin, oracle_bin, jobs, dict(os.environ, B200_INDEL_KEY_BITS=bits))
        assert not bad and ok > 50, (bits, bad[:2])


@pytest.mark.parametrize('opt', ['-s', '-O', '-M', '--output-QNAME', '--output-extra FLAG', '--no-output-ins', '--reverse-del',
                                 '--output-BP-5', '-aBsQ0'])
def test_indels_refuses_text_options(opt, emul_bin, corpus):
    r = subprocess.run(f'{emul_bin} indels {opt} mpileup.1.bam', shell=True, cwd=os.path.join(corpus, 'test', 'mpileup'),
                       capture_output=True)
    assert r.returncode != 0 and r.stdout == b'' and b'Usage: b200samtools indels' in r.stderr


# ---------------------------------------------------------------- CUDA path
@pytest.fixture(scope='module')
def cli():
    assert os.path.exists(CLI), 'samtools_b200/bin/b200samtools missing: run python samtools_b200/build.py'
    return CLI


@pytest.mark.gpu
def test_golden_indels_gpu(cli, oracle_bin, corpus):
    """every golden mpileup case without text-only options, BAQ and multi-file lists included, plain and in 97-column windows"""
    jobs = [(os.path.join(corpus, c['cwd']), c['args'], c['prefix']) for c in GOLDEN if '>' not in c['prefix']]
    bad, ok = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == len(jobs), bad[:2]
    bad, ok = run_many(cli, oracle_bin, jobs, dict(os.environ, B200_WINDOW_COLS='97'))
    assert not bad and ok == len(jobs), bad[:2]


@pytest.mark.gpu
def test_fuzz_indels_gpu(cli, oracle_bin, tmp_path):
    bad, ok = run_many(cli, oracle_bin, fuzz_jobs(tmp_path, range(1, 7), need_noBAQ=False))
    assert not bad and ok > 100, bad[:2]


@pytest.mark.gpu
def test_long_reads_indels_gpu(cli, oracle_bin, tmp_path):
    """reads of 513 b .. 40 kb with hundreds to thousands of CIGAR ops, a 2 kb insertion, one of > 65535 ops, a 70 kb deletion"""
    from test_longread import write_long_inputs
    write_long_inputs(tmp_path)
    jobs = [(str(tmp_path), a) for a in ('-B -f long.fa long.sam', '-f long.fa long.sam', '-B -Q 0 -f long.fa long.sam long2.sam',
                                          '-B -a -r chr1:90000-110000 -f long.fa long.bam', '-B -f cg.fa cg.sam', '-B -f del.fa del.sam',
                                          '-B del.sam')]
    bad, ok = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == len(jobs), bad[:2]


@pytest.mark.gpu
def test_amplicon_max_depth_indels_gpu(cli, oracle_bin, tmp_path):
    """amplicon stacks of 2500 .. 12000 pairs: -d 8000 and -d 2500 drop reads, with and without column windows"""
    from samtools_b200 import synth
    from test_gpu_maxdepth import make_amplicons
    soa = make_amplicons()
    synth.write_sam(str(tmp_path / 'amp.sam'), soa); synth.write_fasta(str(tmp_path / 'amp.fa'), 'amp', soa['ref_full'])
    jobs = [(str(tmp_path), a) for a in ('-B -f amp.fa amp.sam', '-f amp.fa amp.sam', '-B -d 2500 -Q 0 -f amp.fa amp.sam')]
    bad, ok = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == len(jobs), bad[:2]
    bad, ok = run_many(cli, oracle_bin, jobs[:1], dict(os.environ, B200_WINDOW_COLS='997'))
    assert not bad and ok == 1, bad[:2]


@pytest.mark.gpu
def test_deep_column_gpu(cli, oracle_bin, tmp_path):
    """one column under 9000 reads: 4000 share one insertion, 3000 distinct short and 1000 distinct long ones, 100 share a long
    one, 500 deletions; then with keys of 0 and 7 bits"""
    write_deep(tmp_path, n_same=4000, n_short=3000, n_long=1000, n_del=500)
    for env in (None, dict(os.environ, B200_INDEL_KEY_BITS='0'), dict(os.environ, B200_INDEL_KEY_BITS='7')):
        assert run_pair(cli, oracle_bin, str(tmp_path), DEEP_ARGS, env=env) is None


@pytest.fixture(scope='module')
def c2(tmp_path_factory):
    """the BASELINE C2 shape at 1 Mb: 30x, 150 bp pairs, no FASTA"""
    from samtools_b200 import synth
    soa = synth.make_batch(length=1_000_000, depth=30, seed=2)
    soa = dict(soa); soa['ref'] = None
    sam = str(tmp_path_factory.mktemp('c2') / 'c2.sam')
    synth.write_sam(sam, soa)
    return soa, sam


def table_rows(rows, seq, name, beg=0):
    """the `indels` rows of an Engine.mpileup_indels table without a FASTA"""
    out = []
    for r in rows:
        n = int(r['len'])
        tok = f'+{n}' + bytes(seq[int(r['seq_off']):int(r['seq_off']) + n]).decode() if n >= 0 else f'-{-n}' + 'N' * -n
        out.append(f"{name}\t{beg + int(r['col']) + 1}\tN\t{int(r['file'])}\t{tok}\t{int(r['fwd'])}\t{int(r['rev'])}\n")
    return ''.join(out).encode()


@pytest.mark.gpu
def test_c2_indels_counts_and_tensor_output(c2, oracle_bin):
    import torch
    from samtools_b200 import engine
    soa, sam = c2
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    rows, seq = e.mpileup_indels(13)
    assert e.last_kernel_ms > 0 and len(rows) > 1000
    want = subprocess.run([oracle_bin, 'mpileup', '--reverse-del', sam], capture_output=True, check=True).stdout
    assert table_rows(rows, seq, soa['tid_name']) == rows_from_text(want)
    # the counts invariant: per column, fwd / rev sums over insertions and deletions are planes 7, 16 and 8, 17
    cnt = e.mpileup_counts(13)
    for ins, (pf, pr) in ((True, (7, 16)), (False, (8, 17))):
        sel = rows[(rows['len'] >= 0) == ins]
        for field, plane in (('fwd', pf), ('rev', pr)):
            s = np.zeros(cnt.shape[2], np.int64)
            np.add.at(s, sel['col'], sel[field])
            assert np.array_equal(s, cnt[0, plane].astype(np.int64)), (field, plane)
    trows, tseq = e.mpileup_indels(13, device=True)
    assert trows.is_cuda and trows.device.index == 0 and tuple(trows.shape) == (len(rows), 8)
    assert trows.cpu().numpy().tobytes() == rows.tobytes() and tseq.cpu().numpy().tobytes() == seq.tobytes()
    e.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    with pytest.raises(RuntimeError, match='B200_MODE_MPILEUP'):
        e.mpileup_indels(13)
    e.close()


@pytest.mark.gpu
def test_c_abi_indel_errors(c2):
    import ctypes as C
    import torch
    from samtools_b200 import engine
    soa, _ = c2
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    rows = np.zeros(1, engine.INDEL_DTYPE); seq = np.zeros(1, np.uint8)
    fetch = lambda r, nr, s, ns: e.lib.b200_fetch_indels(e.h, r, nr, s, ns)
    assert fetch(rows.ctypes.data_as(C.c_void_p), 1, None, 0) == -1          # no compute since the stage
    assert b'no indel table' in e.lib.b200_last_error(e.h)
    n, nb = C.c_int64(0), C.c_uint64(0)
    assert e.lib.b200_mpileup_indels(e.h, 13, C.byref(n), C.byref(nb)) == 0 and n.value > 1 and nb.value > 1
    assert fetch(rows.ctypes.data_as(C.c_void_p), 1, None, 0) == -2
    assert b'allele buffer too small' in e.lib.b200_last_error(e.h)
    assert fetch(None, 0, seq.ctypes.data_as(C.c_void_p), 1) == -2
    assert b'symbol buffer too small' in e.lib.b200_last_error(e.h)
    if torch.cuda.device_count() > 1:
        t = torch.empty((n.value, 8), dtype=torch.int32, device='cuda:1')
        assert fetch(C.c_void_p(t.data_ptr()), n.value, None, 0) == -1
        assert b'is on device 1' in e.lib.b200_last_error(e.h)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    assert fetch(None, 0, None, 0) == -1                                      # a new stage drops the table
    e.close()


@pytest.mark.gpu
def test_shard_tables_concatenate(c2):
    """plan_shards windows of one contig: their tables, with col shifted by the window start, concatenate to the contig's"""
    from samtools_b200 import engine, shard
    soa, _ = c2
    L = int(soa['tid_len'])
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    rows, seq = e.mpileup_indels(13)
    whole = table_rows(rows[rows['col'] < L], seq, soa['tid_name'])
    parts = []
    for beg, end in shard.plan_shards(L, 3):
        e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, beg=beg, end=end))
        r, s = e.mpileup_indels(13)
        parts.append(table_rows(r, s, soa['tid_name'], beg))
    e.close()
    assert b''.join(parts) == whole and len(parts) == 3
