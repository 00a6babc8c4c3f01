"""Many-sample cohorts through every output, against the oracle: byte for byte for text, exactly for the numbers parsed from
the oracle's text (the parsers of test_counts, test_qsums, test_psums, test_ranksums and test_indels).

Dense cohort: 37 files (not a multiple of the 4 warps per block of the column kernels, nor of 32) on a 12 289-column contig
(one past a multiple of 128: the last group and tile are partial), about 15x each with raised indel, clip and N-skip rates.
Particular files: one without records, one whose records the default filter drops, two with a stack of 480 reads on one
column (above `-d 250` and 255 usable GL bases, the rest of the cohort below), one with long reads whose D and N runs pass
512 bases, a last one with reads only in the contig's last 200 columns; every file of make_batch reads shares its QNAMEs
with the others, two of them with mates that overlap almost always, and reads of different files are never mates.  The
even-numbered files are indexed BAMs, the others SAMs.  Default windows, 997-column windows, and two window workers.

Wide cohort: 160 files of three reads each, near position 1, near 8.4 M and one ending just past 2^24, from a `-b` list on a
17 Mb contig: a window of 2^24 columns would hold 2.7e9 (column, file) pairs.  The CLI's windows hold at most 2^24 pairs,
so each command runs in bounded memory and matches the oracle.  The engine refuses a window of more than 2^31 - 1 - 1024 pairs
up front, with one message for its three per-pair tables (indels, rank sums, GL).

CPU through the emulation harness (no BAQ, no GL); the CUDA CLI and the Engine under -m gpu."""
import os, subprocess, sys
import numpy as np
import pytest
from conftest import ROOT
import test_counts
import test_indels
import test_psums
import test_qsums
import test_ranksums
from test_qsums import build_emul

CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')
CNT, QS, PS, RS = test_counts.PLANES, test_qsums.PLANES, test_psums.PLANES, test_ranksums.PLANES

N_DENSE, L_DENSE, CTG = 37, 12_289, 'coh'
EMPTY, DUPS, LONG, LAST = 3, 9, 18, N_DENSE - 1     # no records; flag 1024 only; D / N runs over 512; only the last 200 columns
STACKS = (12, 25)          # 480 reads on one column
STACK_COL = 6_050
MATES = (14, 15)           # 250 bp pairs: mates overlap, QNAMEs shared with every other make_batch file

N_WIDE, L_WIDE, WCTG = 160, 17_000_000, 'wide'
PAIRS = 1 << 24            # the CLI's (column, file) pairs per window
MAX_PAIRS = (1 << 31) - 1 - 256 * 4
GiB = 1 << 30

ENVS = {'default': {}, 'win997': {'B200_WINDOW_COLS': '997'}, 'devices00': {'B200_WINDOW_COLS': '997', 'B200_DEVICES': '0,0'}}


# ---------------------------------------------------------------- inputs
def _recs_soa(rng, ref, recs):
    from samtools_b200 import synth
    return synth._pack([synth._rec(rng, ref, p, np.array(l, np.int64), np.array(o, np.int64), flag=fl) for p, l, o, fl in recs],
                       ref, len(ref), 0, CTG)


def dense_soas(ref):
    """the 37 single-file batches of the dense cohort (None: a file without records)"""
    from samtools_b200 import synth
    L = len(ref)
    kw = dict(length=L, depth=15, ref=ref, tid_name=CTG, frac_ins=0.06, frac_del=0.06, frac_clip=0.08, frac_skip=0.01)
    out = []
    for f in range(N_DENSE):
        rng = np.random.default_rng(500 + f)
        bg = [(int(p), [100], [0], 16 * int(rng.integers(2))) for p in rng.integers(0, L - 100, 60)]
        if f == EMPTY:
            soa = None
        elif f in STACKS:
            stack = [(STACK_COL - int(rng.integers(0, 60)), [100], [0], 16 * int(rng.integers(2))) for _ in range(480)]
            soa = _recs_soa(rng, ref, bg + stack)
        elif f == LONG:
            lng = [(int(p), [200, int(rng.integers(520, 700)), 150, int(rng.integers(600, 900)), 200], [0, 2, 0, 3, 0], 16 * (k & 1))
                   for k, p in enumerate(rng.integers(0, L - 2000, 10))]
            soa = _recs_soa(rng, ref, bg + lng)
        elif f == LAST:
            soa = _recs_soa(rng, ref, [(L - 200 + int(rng.integers(0, 141)), [60], [0], 16 * int(rng.integers(2))) for _ in range(25)])
        else:
            soa = synth.make_batch(seed=1000 + f, read_len=250 if f in MATES else 150, **kw)
            if f == DUPS:
                soa = dict(soa, flag=soa['flag'] | np.uint16(1024))
        out.append(soa)
    return out


def merge(soas):
    """single-file batches of one contig (None: no records) as one multi-file batch"""
    real = [s for s in soas if s is not None]
    out, n = {}, [0 if s is None else len(s['pos']) for s in soas]
    for k in ('pos', 'flag', 'mapq', 'l_qseq', 'n_cigar', 'mtid', 'mpos', 'isize', 'rbits', 'cigar', 'seq4', 'qual', 'pair_id'):
        out[k] = np.concatenate([s[k] for s in real])
    for s in real:
        assert len(s['qual']) % 2 == 0 and len(s['seq4']) * 2 == len(s['qual'])
    ncig = np.cumsum([0] + [len(s['cigar']) for s in real])
    nq = np.cumsum([0] + [len(s['qual']) for s in real])
    nr = np.cumsum([0] + [len(s['pos']) for s in real])
    out['cigar_off'] = np.concatenate([s['cigar_off'] + np.uint64(ncig[i]) for i, s in enumerate(real)])
    out['qual_off'] = np.concatenate([s['qual_off'] + np.uint64(nq[i]) for i, s in enumerate(real)])
    out['prev_same_name'] = np.concatenate([np.where(s['prev_same_name'] >= 0, s['prev_same_name'] + nr[i], -1) for i, s in enumerate(real)])
    out['file_start'] = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    for k in ('tid', 'tid_len', 'tid_name', 'ref', 'ref_beg', 'ref_len', 'ref_full'):
        out[k] = real[0][k]
    return out


def write_file(path, soa):
    from samtools_b200 import synth
    if soa is None:
        with open(path, 'w') as f:
            f.write(f'@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:{CTG}\tLN:{L_DENSE}\n')
    elif path.endswith('.bam'):
        synth.write_bam(path, soa)
    else:
        synth.write_sam(path, soa)


@pytest.fixture(scope='module')
def emul_bin(tmp_path_factory):
    """the CLI on the emulation harness with every numeric output (emul_ranksums.cpp)"""
    return build_emul(tmp_path_factory, 'ranksums')


@pytest.fixture(scope='module')
def dense(tmp_path_factory, emul_bin):
    from samtools_b200 import synth
    d = tmp_path_factory.mktemp('dense')
    ref = synth.make_reference(L_DENSE, seed=77)
    soas = dense_soas(ref)
    names = [f'f{f:02d}.{"sam" if f % 2 or soas[f] is None else "bam"}' for f in range(N_DENSE)]
    for name, soa in zip(names, soas):
        write_file(str(d / name), soa)
        if name.endswith('.bam'):
            subprocess.run([emul_bin, 'index', name], cwd=str(d), check=True)
    synth.write_fasta(str(d / 'ref.fa'), CTG, ref)
    (d / 'cohort.bed').write_text(f'{CTG}\t0\t500\n{CTG}\t3000\t6100\n{CTG}\t9000\t9001\n{CTG}\t12000\t{L_DENSE}\n')
    return dict(dir=str(d), soas=soas, files=' '.join(names), ref=ref)


def dense_text_cmds(files):
    return [f'mpileup -B -f ref.fa {files}', f'mpileup -B -a -s -O --output-BP-5 -f ref.fa {files}', f'mpileup -B --output-QNAME {files}',
            f'mpileup -B -d 250 -f ref.fa {files}', f'mpileup -B -r {CTG}:2001-9500 -f ref.fa {files}', f'depth -a {files}',
            f'depth -s {files}', f'bedcov cohort.bed {files}']


_oracle_cache = {}


def first_diff(got, want):
    """(line number, expected line, printed line) of the first line that differs, each cut to 300 bytes"""
    g, w = got.split(b'\n'), want.split(b'\n')
    k = next((i for i in range(max(len(g), len(w))) if i >= len(g) or i >= len(w) or g[i] != w[i]), None)
    return None if k is None else (k, w[k][:300] if k < len(w) else None, g[k][:300] if k < len(g) else None)


def sh(cmd, cwd, env=None):
    r = subprocess.run(cmd, shell=True, cwd=cwd, capture_output=True, env=None if env is None else dict(os.environ, **env), timeout=1800)
    return r


def oracle(oracle_bin, cwd, args):
    key = (cwd, args)
    if key not in _oracle_cache:
        r = sh(f'{oracle_bin} {args}', cwd)
        assert r.returncode == 0, (args, r.stderr[-300:])
        _oracle_cache[key] = r.stdout
    return _oracle_cache[key]


def want_counts(oracle_bin, cwd, args):
    """the `counts --qsums --psums --ranksums <args>` rows parsed from the oracle's text"""
    o = lambda extra: oracle(oracle_bin, cwd, f'mpileup --reverse-del {extra}{args}')
    text, text_q0 = o(''), oracle(oracle_bin, cwd, f'mpileup --reverse-del {args} -Q 0')
    base = test_qsums.count_rows(o('-s '), text, text_q0)
    base = test_psums.count_rows(o('--output-BP-5 '), base, CNT + QS)
    return test_ranksums.count_rows(o('-s --output-BP-5 '), base, CNT + QS + PS, fast=True)


def want_indels(oracle_bin, cwd, args, sums):
    """the `indels [--qsums --psums] <args>` rows parsed from the oracle's text"""
    if sums:
        return test_psums.allele_rows(oracle(oracle_bin, cwd, f'mpileup --reverse-del --output-BP-5 {args}'),
                                      oracle(oracle_bin, cwd, f'mpileup --reverse-del -s {args}'))
    return test_indels.rows_from_text(oracle(oracle_bin, cwd, f'mpileup --reverse-del {args}'))


def check_dense(tool, oracle_bin, dense, env, text=True, numbers=True, gpu=False):
    cwd, files = dense['dir'], dense['files']
    bad = []
    cmds = dense_text_cmds(files) + ([f'mpileup -f ref.fa {files}', f'gl -B -f ref.fa {files}'] if gpu else [])
    for args in cmds if text else []:
        r = sh(f'{tool} {args}', cwd, env)
        want = oracle(oracle_bin, cwd, args)
        if r.returncode != 0 or r.stdout != want:
            bad.append((args, r.returncode, r.stderr[-300:], first_diff(r.stdout, want)))
        assert len(want) > 200, args
    if numbers:
        args = f'-B -f ref.fa {files}'
        r = sh(f'{tool} counts --qsums --psums --ranksums {args}', cwd, env)
        want = want_counts(oracle_bin, cwd, args)
        if r.returncode != 0 or r.stdout != want:
            bad.append(('counts', r.returncode, r.stderr[-300:], first_diff(r.stdout, want)))
        r = sh(f'{tool} indels --qsums --psums {args}', cwd, env)
        want = want_indels(oracle_bin, cwd, args, True)
        if r.returncode != 0 or r.stdout != want:
            bad.append(('indels', r.returncode, r.stderr[-300:], first_diff(r.stdout, want)))
        assert want.count(b'\n') > 500
    assert not bad, bad


# ---------------------------------------------------------------- dense cohort: the inputs are what they claim
def test_dense_cohort_shape(dense, oracle_bin):
    from samtools_b200 import synth
    soas = dense['soas']
    assert len(soas) == N_DENSE and N_DENSE % 4 and N_DENSE % 32 and L_DENSE % 128 == 1
    assert soas[EMPTY] is None and (soas[DUPS]['flag'] & 1024).all()
    for f in STACKS:
        pos, end = soas[f]['pos'], soas[f]['pos'] + synth.ref_span(soas[f])
        assert ((pos <= STACK_COL) & (end > STACK_COL)).sum() >= 400
    span, ops = synth.ref_span(soas[LONG]), soas[LONG]['cigar'] & 15
    assert span.max() > 1500 and (((ops == 2) | (ops == 3)) & ((soas[LONG]['cigar'] >> 4) > 512)).sum() >= 10
    assert soas[LAST]['pos'].min() >= L_DENSE - 200 and (soas[LAST]['pos'] + synth.ref_span(soas[LAST])).max() <= L_DENSE
    for f in MATES:     # proper pairs whose mates overlap, under the same QNAMEs as the other files'
        s = soas[f]
        first = s['prev_same_name'] < 0
        mate = s['prev_same_name'][~first]
        assert (s['pos'][~first] < s['pos'][mate] + synth.ref_span(s)[mate]).mean() > 0.9
    assert set(soas[MATES[0]]['pair_id'][:50]) & set(soas[MATES[1]]['pair_id'])
    assert sum(os.path.exists(os.path.join(dense['dir'], f'f{f:02d}.bam.bai')) for f in range(N_DENSE)) >= 18
    # the stacks go over -d 250 in their files only, and give GL more than 255 bases of -Q 13 there
    for q, least in (0, 400), (13, 256):
        deep = oracle(oracle_bin, dense['dir'], f'mpileup -B -Q {q} -r {CTG}:{STACK_COL + 1}-{STACK_COL + 1} {dense["files"]}').split(b'\t')
        n = [int(deep[3 + 3 * f]) for f in range(N_DENSE)]
        assert all(n[f] >= least for f in STACKS) and max(n[f] for f in range(N_DENSE) if f not in STACKS) < 100 and n[EMPTY] == n[DUPS] == 0


# ---------------------------------------------------------------- dense cohort: emulation harness
@pytest.mark.parametrize('env', list(ENVS), ids=list(ENVS))
def test_dense_cohort_emul(env, emul_bin, oracle_bin, dense):
    check_dense(emul_bin, oracle_bin, dense, ENVS[env], numbers=env != 'devices00')


# ---------------------------------------------------------------- dense cohort: CUDA CLI
@pytest.fixture(scope='module')
def cli():
    assert os.path.exists(CLI), 'samtools_b200/bin/b200samtools missing: run python samtools_b200/build.py'
    return CLI


@pytest.mark.gpu
@pytest.mark.parametrize('env', list(ENVS), ids=list(ENVS))
def test_dense_cohort_gpu(env, cli, oracle_bin, dense):
    """the same commands, and BAQ and GL: the stacks give two files more than 255 usable bases on one column, so GL's
    random draws run over files in the reference's order"""
    check_dense(cli, oracle_bin, dense, ENVS[env], numbers=env != 'devices00', gpu=True)


def planes_from_rows(rows, n):
    """[n_files, CNT + QS + PS + RS, n] int64 of the `counts --qsums --psums --ranksums` rows (columns without a row: 0)"""
    per = CNT + QS + PS + RS
    out = np.zeros((N_DENSE, per, n), np.int64)
    for ln in rows.decode().split('\n')[:-1]:
        v = ln.split('\t')
        out[:, :, int(v[1]) - 1] = np.array(v[3:], np.int64).reshape(N_DENSE, per)
    return out


@pytest.mark.gpu
def test_dense_cohort_engine(oracle_bin, dense):
    """the cohort staged once as 37 files: every plane output (numpy and torch out=) has shape (37, P, n) and equals the
    oracle's, and the indel table's file and column of each allele are the oracle's"""
    import torch
    from samtools_b200 import engine
    cwd, files = dense['dir'], dense['files']
    batch = merge(dense['soas'])
    assert len(batch['file_start']) == N_DENSE + 1 and batch['file_start'][EMPTY] == batch['file_start'][EMPTY + 1]
    e = engine.Engine(0)
    st = e.stage(batch, engine.default_stage_conf(engine.MODE_MPILEUP, baq=0))
    n = int(st.n_cols)
    assert n >= L_DENSE
    want = planes_from_rows(want_counts(oracle_bin, cwd, f'-B -f ref.fa {files}'), n)
    lo = 0
    for fn, p, tdt in (('mpileup_counts', CNT, torch.int32), ('mpileup_qsums', QS, torch.int32), ('mpileup_psums', PS, torch.int64),
                       ('mpileup_ranksums', RS, torch.int64)):
        got = getattr(e, fn)(13)
        assert got.shape == (N_DENSE, p, n), fn
        assert np.array_equal(got.astype(np.int64), want[:, lo:lo + p]), fn
        t = torch.full((N_DENSE, p, n), -1, dtype=tdt, device='cuda:0')
        assert getattr(e, fn)(13, out=t) is t
        assert np.array_equal(t.cpu().numpy().astype(np.int64) & (0xffffffff if tdt == torch.int32 else -1), want[:, lo:lo + p]), fn
        lo += p
    assert (want[STACKS[0], CNT - 1, STACK_COL] >= 400) and not want[EMPTY].any() and not want[DUPS].any()
    rows, seq = e.mpileup_indels(13)
    got = sorted((int(r['file']), int(r['col']), int(r['len']), bytes(seq[int(r['seq_off']):int(r['seq_off']) + max(int(r['len']), 0)]),
                  int(r['fwd']), int(r['rev'])) for r in rows)
    exp = []
    for ln in want_indels(oracle_bin, cwd, f'-B -f ref.fa {files}', False).decode().split('\n')[:-1]:
        _, pos, _, f, tok, fwd, rev = ln.split('\t')
        k = int(tok[1:].rstrip('ACGTN*'))
        exp.append((int(f), int(pos) - 1, k if tok[0] == '+' else -k, tok[1 + len(str(k)):].encode() if tok[0] == '+' else b'', int(fwd), int(rev)))
    assert got == sorted(exp) and len(got) > 500
    assert {r[0] for r in got} >= {0, LONG} and not {r[0] for r in got} & {EMPTY, DUPS}
    e.close()


# ---------------------------------------------------------------- wide cohort
def write_wide(d):
    """160 files of three reads in directory d: near position 1, near 8.4 M (every fourth with an insertion, every fourth
    with a deletion), and one ending just past 2^24; with a FASTA and a -b list"""
    import pathlib
    from samtools_b200 import synth
    d = pathlib.Path(d)
    ref = synth.make_reference(L_WIDE, seed=91)
    names = []
    for f in range(N_WIDE):
        rng = np.random.default_rng(9000 + f)
        mid = ([40, 2, 58], [0, 1, 0]) if f % 4 == 0 else ([50, 3, 50], [0, 2, 0]) if f % 4 == 1 else ([100], [0])
        recs = [(3 + f % 50, [100], [0], 16 * (f & 1)), (8_400_000 + 3 * f, *mid, 16 * (f & 1)), ((1 << 24) + 3 + f % 5 - 100, [100], [0], 0)]
        soa = synth._pack([synth._rec(rng, ref, p, np.array(l, np.int64), np.array(o, np.int64), flag=fl) for p, l, o, fl in recs],
                          ref, L_WIDE, 0, WCTG)
        names.append(f'w{f:03d}.sam')
        synth.write_sam(str(d / names[-1]), soa)
    (d / 'wide.list').write_text(''.join(n + '\n' for n in names))
    synth.write_fasta(str(d / 'wide.fa'), WCTG, ref)
    return str(d)


@pytest.fixture(scope='module')
def wide(tmp_path_factory):
    return write_wide(tmp_path_factory.mktemp('wide'))


_SPAWN = ('import os, sys\n'
          'pid = os.posix_spawn(sys.argv[2], sys.argv[2:], os.environ)\n'
          '_, st, ru = os.wait4(pid, 0)\n'
          'open(sys.argv[1], "w").write(str(ru.ru_maxrss))\n'
          'sys.exit(os.waitstatus_to_exitcode(st))\n')


def run_rss(cmd, cwd, env=None):
    """(exit code, stdout, stderr, peak RSS in bytes) of one command line, without a shell.  A small Python process starts
    it: the peak RSS Linux reports for a process counts the memory of the process it was forked from until its exec, and
    the test process may be large."""
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        rss = os.path.join(td, 'rss')
        r = subprocess.run([sys.executable, '-c', _SPAWN, rss, cmd[0] if os.path.isabs(cmd[0]) else os.path.abspath(cmd[0])] + cmd[1:],
                           cwd=cwd, capture_output=True, env=None if env is None else dict(os.environ, **env), timeout=1800)
        return r.returncode, r.stdout, r.stderr, int(open(rss).read()) * 1024


# host bytes per (column, file) pair of a window beyond the 2 GiB allowance: the count and sum planes (76 + 168 + 224 + 64 B)
# and GL's per-pair arrays, in the CLI (120 B) and in the call (120 B); 2^24 pairs of them are one file's 2^24 columns
WIDE_CMDS = {'mpileup': ('mpileup -B -f wide.fa -b wide.list', 0), 'depth': ('depth -f wide.list', 0),
             'counts': ('counts --qsums --psums --ranksums -B -f wide.fa -b wide.list', CNT * 4 + QS * 4 + PS * 8 + RS * 8),
             'indels': ('indels -B -f wide.fa -b wide.list', 0), 'gl': ('gl -B -f wide.fa -b wide.list', 240)}


def check_wide(tool, oracle_bin, wide, cmd):
    args, per_pair = WIDE_CMDS[cmd]
    rc, out, err, rss = run_rss([tool] + args.split(), wide)
    assert rc == 0, err[-400:]
    if cmd == 'counts':
        want = want_counts(oracle_bin, wide, args.split(' ', 4)[4])
    elif cmd == 'indels':
        want = want_indels(oracle_bin, wide, args.split(' ', 1)[1], False)
    else:
        want = oracle(oracle_bin, wide, args)
    assert out == want, (cmd, first_diff(out, want))
    assert want.count(b'\n') >= (3 if cmd == 'indels' else 300)
    assert rss < 2 * GiB + per_pair * PAIRS, (cmd, rss / GiB)
    return rss


@pytest.mark.parametrize('cmd', ['mpileup', 'depth', 'counts', 'indels'])
def test_wide_cohort_emul(cmd, emul_bin, oracle_bin, wide):
    check_wide(emul_bin, oracle_bin, wide, cmd)


@pytest.mark.gpu
@pytest.mark.parametrize('cmd', list(WIDE_CMDS))
def test_wide_cohort_gpu(cmd, cli, oracle_bin, wide):
    check_wide(cli, oracle_bin, wide, cmd)


@pytest.mark.gpu
def test_pair_limit_engine():
    """160 files of one read each staged over 2^24 columns: the indel, rank-sum and GL calls refuse the window with one
    message that names the limit, before they allocate (mpileup_counts is not called: its planes would take 12 GB)"""
    import ctypes as C
    from samtools_b200 import engine, synth
    rng = np.random.default_rng(3)
    ref = synth.make_reference(1 << 24, seed=5, n_frac=0)
    # the last file's read ends near column 2^24, so that GL (which visits the columns up to the last read) spans them too
    soas = [_recs_soa(rng, ref, [(1000 * f if f < N_WIDE - 1 else (1 << 24) - 200, [100], [0], 0)]) for f in range(N_WIDE)]
    batch = merge(soas)
    e = engine.Engine(0)
    st = e.stage(batch, engine.default_stage_conf(engine.MODE_MPILEUP, baq=0, end=1 << 24))
    assert st.n_cols == 1 << 24 and st.n_cols * N_WIDE > MAX_PAIRS
    msg = f'window too large: {1 << 24} columns x {N_WIDE} files exceed the limit of {MAX_PAIRS} (column, file) pairs'
    with pytest.raises(RuntimeError, match=msg.replace('(', r'\(').replace(')', r'\)')):
        e.mpileup_indels(13)
    n = C.c_int64(0)                                            # compute only: its host planes would take 171 GB
    assert e.lib.b200_mpileup_ranksums(e.h, 13, None, 0, C.byref(n)) == -1 and n.value == 1 << 24
    assert msg.encode() in e.lib.b200_last_error(e.h)
    with pytest.raises(RuntimeError, match=r'limit of \d+ \(column, file\) pairs'):
        e.glf(13, 16, n_files=N_WIDE)
    # a window under the limit is served
    e.stage(batch, engine.default_stage_conf(engine.MODE_MPILEUP, baq=0, end=1 << 14))
    e.mpileup_indels(13)
    assert e.mpileup_ranksums(13).shape == (N_WIDE, RS, 1 << 14)
    e.close()
