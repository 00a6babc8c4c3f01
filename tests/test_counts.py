"""Per-column base and indel counts (`b200samtools counts`, b200_mpileup_counts, Engine.mpileup_counts) against the counts a
parser takes from the oracle's `mpileup --reverse-del` text of the same options: CPU through the emulation harness, and the
CUDA path (BAQ included) under -m gpu."""
import os, re, shlex, subprocess
import numpy as np
import pytest
import golden_cases
import fuzz_sam
from conftest import ROOT

CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')
PLANES = 19
INS, DEL, REV = 7, 8, 9


# ---------------------------------------------------------------- the text -> counts parser
def entry_counts(seq, ref):
    """counts of one file's pileup sequence column, planes 0-17 (plane 18, n_plp, comes from a -Q 0 run)"""
    c = [0] * (PLANES - 1)
    ref_k = 'ACGT'.find(ref.upper()) if ref.upper() in 'ACGT' else 4
    i, last = 0, 0
    while i < len(seq):
        ch = seq[i]
        if ch == '^':                 # "^" + a mapq character, which may itself be '$', '+', '-', '.' or ','
            i += 2
        elif ch == '$':
            i += 1
        elif ch in '+-':              # "+n" / "-n" and exactly n characters; the event takes the strand of its entry
            m = re.match(r'\d+', seq[i + 1:])
            c[last + (INS if ch == '+' else DEL)] += 1
            i += 1 + len(m.group(0)) + int(m.group(0))
        else:
            rev = ch in ',#<' or ch.islower()
            last = REV if rev else 0
            if ch in '.,':
                k = ref_k
            elif ch in '*#':
                k = 5
            elif ch in '><':
                k = 6
            else:
                k = 'ACGT'.find(ch.upper())
                k = 4 if k < 0 else k
            c[last + k] += 1
            i += 1
    return c


def rows_from_text(text, text_q0):
    """the `counts` rows of mpileup's lines: chr, pos, ref, then per file the 19 planes"""
    out = []
    a, b = text.decode().split('\n')[:-1], text_q0.decode().split('\n')[:-1]
    assert len(a) == len(b)
    for la, lb in zip(a, b):
        fa, fb = la.split('\t'), lb.split('\t')
        assert fa[:3] == fb[:3]
        vals = []
        for f in range((len(fa) - 3) // 3):
            cnt, seq = int(fa[3 + 3 * f]), fa[4 + 3 * f]
            vals += (entry_counts(seq, fa[2]) if cnt else [0] * (PLANES - 1)) + [int(fb[3 + 3 * f])]
        out.append('\t'.join(fa[:3] + [str(x) for x in vals]) + '\n')
    return ''.join(out).encode()


def test_parser_on_hand_made_columns():
    assert entry_counts('^$.,+2AC-1a$*#><gN^,A', 'c') == \
        [1, 1, 0, 0, 1, 1, 1, 0, 0] + [0, 1, 1, 0, 0, 1, 1, 1, 1]


# ---------------------------------------------------------------- command lines
TEXT_ONLY_LONG = ('--output', '--no-output', '--reverse-del')


def text_only(args):
    """-s -O -M, --output-* (not --output FILE), --no-output-*, --reverse-del"""
    for t in args:
        if t.startswith('--'):
            if t.startswith(TEXT_ONLY_LONG) and t != '--output':
                return True
        elif t.startswith('-') and len(t) > 1:
            for ch in t[1:]:
                if ch in 'sOM':
                    return True
                if ch in 'frlqQCdbGo':
                    break
    return False


def split_golden(cmd):
    """(prefix, mpileup arguments) of a golden command line, without the post-processing after the mpileup's pipe"""
    m = re.search(r'\$samtools\s+mpileup\b', cmd)
    if not m:
        return None
    rest = cmd[m.end():].split('|')[0]
    return cmd[:m.start()], rest.strip()


GOLDEN = []
for _c in golden_cases.all_cases():
    if _c['table'] == 'depth.reg' or _c['skip'] or _c['kind'] != 'P':
        continue
    _s = split_golden(_c['cmd'])
    if _s and not text_only(shlex.split(_s[1])):
        GOLDEN.append(dict(id=_c['id'], cwd=_c['cwd'], prefix=_s[0], args=_s[1]))


def run_pair(tool, oracle, cwd, args, prefix='', env=None):
    """None when `tool counts <args>` prints the rows parsed from the oracle's text; 'baq' when the emulation harness
    cannot stage the case; else a description of the difference"""
    pre = re.sub(r'\$samtools\s+view', oracle + ' view', prefix).replace('$samtools', oracle)
    sh = lambda line: subprocess.run(pre + line, shell=True, cwd=cwd, capture_output=True, env=env, timeout=600)
    want = sh(f'{oracle} mpileup --reverse-del {args}')
    want0 = sh(f'{oracle} mpileup --reverse-del {args} -Q 0')
    got = sh(f'{tool} counts {args}')
    if got.returncode != 0 and b'BAQ kernel is not emulated' in got.stderr:
        return 'baq'
    exp = rows_from_text(want.stdout, want0.stdout)
    if got.returncode != 0 or got.stdout != exp:
        return (args, got.returncode, got.stderr[-300:], exp[:300], got.stdout[:300])
    return None


def run_many(tool, oracle, jobs, env=None):
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        res = list(ex.map(lambda j: run_pair(tool, oracle, *j, env=env), jobs))
    return [r for r in res if r not in (None, 'baq')], sum(r is None for r in res)


def fuzz_jobs(td, seeds, need_noBAQ):
    jobs = []
    for seed in seeds:
        sam, fa = fuzz_sam.make_sam(seed)
        d = td / f's{seed}'; d.mkdir()
        (d / 'x.sam').write_text(sam); (d / 'x.fa').write_text(fa)
        (d / 'x.bed').write_text('c0\t40\t300\nc0\t250\t600\nc1\t100\nc1\t95\t140\n')
        (d / 'rg.txt').write_text('g2\n')
        (d / 'x2.sam').write_text(fuzz_sam.make_sam(seed + 100000, n_reads=25)[0])
        for opt in fuzz_sam.MPILEUP_OPTS:
            if text_only(shlex.split(opt)) or (need_noBAQ and '-B' not in opt.split()):
                continue
            if seed % 5 == 0 and '-C' in opt.split():
                continue   # undefined upstream on SEQ '*' records
            files = 'x.sam x2.sam' if (seed % 3 == 0 and '-r' not in opt) else 'x.sam'
            ref = '-f x.fa' if seed % 4 != 1 else ''
            jobs.append((str(d), f"{opt.format(bed='x.bed', rg='rg.txt')} {ref} {files}"))
    return jobs


# ---------------------------------------------------------------- emulation harness (no GPU)
@pytest.fixture(scope='module')
def emul_bin(tmp_path_factory):
    """the CLI on the emulation harness with the count output (tests/emul/emul_counts.cpp), built here: pytest-xdist workers
    rebuild tests/emul/_build concurrently"""
    exe = str(tmp_path_factory.mktemp('emul_counts') / 'b200samtools_emul_counts')
    host = os.path.join(ROOT, 'samtools_b200', 'csrc', 'host')
    subprocess.run(['g++', '-std=c++17', '-O1', '-g', '-ffp-contract=off', '-Wall', '-Wno-unused-function', '-Wno-parentheses', '-o', exe,
                    os.path.join(host, 'cli.cpp'), os.path.join(host, 'hts_io.cpp'), os.path.join(ROOT, 'tests', 'emul', 'emul_counts.cpp'),
                    '-lz'], check=True)
    return exe


def test_engine_without_count_output_refuses(corpus):
    """the harness build without b200_mpileup_counts: `counts` stops with a message instead of printing rows"""
    subprocess.run([os.path.join(ROOT, 'tests', 'emul', 'build.sh')], check=True)
    exe = os.path.join(ROOT, 'tests', 'emul', '_build', 'b200samtools_emul')
    r = subprocess.run([exe, 'counts', 'mpileup.1.bam'], cwd=os.path.join(corpus, 'test', 'mpileup'), capture_output=True)
    assert r.returncode != 0 and r.stdout == b'' and b'no count output' in r.stderr


@pytest.mark.parametrize('case', GOLDEN, ids=[c['id'] for c in GOLDEN])
def test_golden_counts_emul(case, emul_bin, oracle_bin, corpus):
    r = run_pair(emul_bin, oracle_bin, os.path.join(corpus, case['cwd']), case['args'], case['prefix'])
    if r == 'baq':
        pytest.skip('needs the BAQ kernel (covered by -m gpu)')
    assert r is None, r


def test_golden_counts_windows_emul(emul_bin, oracle_bin, corpus):
    """97-column windows: every case crosses window edges (halo reads, -a rows, BED) and must print the same rows"""
    env = dict(os.environ, B200_WINDOW_COLS='97')
    jobs = [(os.path.join(corpus, c['cwd']), c['args'], c['prefix']) for c in GOLDEN if '>' not in c['prefix']]
    bad, ok = run_many(emul_bin, oracle_bin, jobs, env)
    assert not bad and ok > 30, bad[:2]


def test_fuzz_counts_emul(emul_bin, oracle_bin, tmp_path):
    bad, ok = run_many(emul_bin, oracle_bin, fuzz_jobs(tmp_path, range(1, 13), need_noBAQ=True))
    assert not bad and ok > 100, bad[:2]


@pytest.mark.parametrize('opt', ['-s', '-O', '-M', '--output-QNAME', '--output-extra FLAG', '--no-output-ins', '--reverse-del',
                                 '--output-BP-5', '-aBsQ0'])
def test_counts_refuses_text_options(opt, emul_bin, corpus):
    r = subprocess.run(f'{emul_bin} counts {opt} mpileup.1.bam', shell=True, cwd=os.path.join(corpus, 'test', 'mpileup'),
                       capture_output=True)
    assert r.returncode != 0 and r.stdout == b'' and b'Usage: b200samtools counts' in r.stderr


# ---------------------------------------------------------------- CUDA path
@pytest.fixture(scope='module')
def cli():
    assert os.path.exists(CLI), 'samtools_b200/bin/b200samtools missing: run python samtools_b200/build.py'
    return CLI


@pytest.mark.gpu
def test_golden_counts_gpu(cli, oracle_bin, corpus):
    """every golden mpileup case without text-only options, BAQ and multi-file lists included, plain and in 97-column windows"""
    jobs = [(os.path.join(corpus, c['cwd']), c['args'], c['prefix']) for c in GOLDEN if '>' not in c['prefix']]
    bad, ok = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == len(jobs), bad[:2]
    bad, ok = run_many(cli, oracle_bin, jobs, dict(os.environ, B200_WINDOW_COLS='97'))
    assert not bad and ok == len(jobs), bad[:2]


@pytest.mark.gpu
def test_fuzz_counts_gpu(cli, oracle_bin, tmp_path):
    bad, ok = run_many(cli, oracle_bin, fuzz_jobs(tmp_path, range(1, 7), need_noBAQ=False))
    assert not bad and ok > 100, bad[:2]


@pytest.mark.gpu
def test_long_reads_counts_gpu(cli, oracle_bin, tmp_path):
    """reads of 513 b .. 40 kb with hundreds to thousands of CIGAR ops (the cig_x lookup), one of > 65535 ops, a 70 kb deletion"""
    from test_longread import write_long_inputs
    write_long_inputs(tmp_path)
    jobs = [(str(tmp_path), a) for a in ('-B -f long.fa long.sam', '-f long.fa long.sam', '-B -Q 0 -f long.fa long.sam long2.sam',
                                          '-B -a -r chr1:90000-110000 -f long.fa long.bam', '-B -f cg.fa cg.sam', '-B -f del.fa del.sam')]
    bad, ok = run_many(cli, oracle_bin, jobs)
    assert not bad and ok == len(jobs), bad[:2]


@pytest.mark.gpu
def test_amplicon_max_depth_counts_gpu(cli, oracle_bin, tmp_path):
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


def dense_expected(oracle_bin, sam, n, *args):
    """the oracle's counts as a [1, 19, n] array over columns 0..n-1 of a single-contig file"""
    want = subprocess.run([oracle_bin, 'mpileup', '--reverse-del', *args, sam], capture_output=True, check=True).stdout
    want0 = subprocess.run([oracle_bin, 'mpileup', '--reverse-del', *args, '-Q', '0', sam], capture_output=True, check=True).stdout
    a = np.zeros((1, PLANES, n), np.uint32)
    for ln in rows_from_text(want, want0).decode().split('\n')[:-1]:
        f = ln.split('\t')
        a[0, :, int(f[1]) - 1] = [int(x) for x in f[3:]]
    return a


@pytest.fixture(scope='module')
def c2(tmp_path_factory, oracle_bin):
    """the BASELINE C2 shape at 1 Mb: 30x, 150 bp pairs, no FASTA"""
    from samtools_b200 import synth
    soa = synth.make_batch(length=1_000_000, depth=30, seed=2)
    soa = dict(soa); soa['ref'] = None
    sam = str(tmp_path_factory.mktemp('c2') / 'c2.sam')
    synth.write_sam(sam, soa)
    return soa, sam


@pytest.mark.gpu
def test_c2_counts_and_tensor_output(c2, oracle_bin):
    import torch
    from samtools_b200 import engine
    soa, sam = c2
    e = engine.Engine(0)
    st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    got = e.mpileup_counts(13)
    assert got.shape == (1, PLANES, st.n_cols) and st.n_cols >= soa['tid_len']
    assert np.array_equal(got, dense_expected(oracle_bin, sam, int(st.n_cols)))
    t = torch.full((1, PLANES, int(st.n_cols)), -1, dtype=torch.int32, device='cuda:0')
    assert e.mpileup_counts(13, out=t) is t
    assert np.array_equal(t.cpu().numpy().view(np.uint32), got)
    with pytest.raises(ValueError):
        e.mpileup_counts(13, out=torch.zeros((1, PLANES, int(st.n_cols) + 1), dtype=torch.int32, device='cuda:0'))
    e.stage(soa, engine.default_stage_conf(engine.MODE_DEPTH))
    with pytest.raises(RuntimeError, match='B200_MODE_MPILEUP'):
        e.mpileup_counts(13)
    e.close()


@pytest.mark.gpu
def test_c_abi_counts_capacity_and_compute_only(c2):
    import ctypes as C
    from samtools_b200 import engine
    soa, _ = c2
    e = engine.Engine(0)
    st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n = C.c_int64(0)
    assert e.lib.b200_mpileup_counts(e.h, 13, None, 0, C.byref(n)) == 0 and n.value == st.n_cols
    assert e.last_kernel_ms > 0
    small = np.zeros(PLANES * 16, np.uint32)
    assert e.lib.b200_mpileup_counts(e.h, 13, small.ctypes.data_as(C.c_void_p), 16, C.byref(n)) == -2
    assert b'count buffer too small' in e.lib.b200_last_error(e.h)
    e.close()


@pytest.mark.gpu
def test_shard_planes_concatenate(c2):
    """plan_shards windows of one contig: their planes, side by side, are the planes of the whole contig"""
    from samtools_b200 import engine, shard
    soa, _ = c2
    L = int(soa['tid_len'])
    e = engine.Engine(0)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    whole = e.mpileup_counts(13)
    parts = []
    for beg, end in shard.plan_shards(L, 3):
        st = e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP, beg=beg, end=end))
        assert st.n_cols == end - beg
        parts.append(e.mpileup_counts(13))
    e.close()
    assert np.array_equal(np.concatenate(parts, axis=2), whole[:, :, :L])
