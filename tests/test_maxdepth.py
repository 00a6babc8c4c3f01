"""The -d max-depth rule of bam_plp_push (a read is dropped when it starts where the previous accepted read of its file
started and -d accepted reads of that file are still buffered) across column windows, through the emulation harness
against the oracle.  The rule depends on every read pushed before, so a window that continues an earlier one must see
the reads ending right at its start and must not judge its halo reads again.  Every case checks that the rule fires
(the oracle's output with -d differs from its output with -d 0), and the windowed ones that a window edge falls within a
read length of a dropped read.  The generators are shared with tests/test_gpu_maxdepth.py."""
import heapq, os, random, subprocess
import pytest
import fuzz_sam
from conftest import ROOT

EMUL = os.path.join(ROOT, 'tests', 'emul', '_build')
BASES = 'ACGT'


@pytest.fixture(scope='module')
def emul_dir():
    subprocess.run([os.path.join(ROOT, 'tests', 'emul', 'build.sh')], check=True)
    return EMUL


# ---------------------------------------------------------------------------------------------- generators
def _cigar_span(cig):
    n, span = '', 0
    for ch in cig:
        if ch.isdigit():
            n += ch
        else:
            if ch in 'MDN=X':
                span += int(n)
            n = ''
    return span


def _cigar_qlen(cig):
    n, q = '', 0
    for ch in cig:
        if ch.isdigit():
            n += ch
        else:
            if ch in 'MIS=X':
                q += int(n)
            n = ''
    return q


def write_sam(path, contig_len, recs, contig='c0'):
    """recs: dicts pos (0-based), cigar, name, flag, mpos, tlen; sorted by position (stable) and written with random
    bases and qualities.  Returns the records in file order."""
    rng = random.Random(len(recs) * 7919 + contig_len)
    recs = sorted(recs, key=lambda r: r['pos'])
    lines = ['@HD\tVN:1.6\tSO:coordinate', f'@SQ\tSN:{contig}\tLN:{contig_len}']
    for r in recs:
        q = _cigar_qlen(r['cigar'])
        seq = ''.join(rng.choice(BASES) for _ in range(q))
        qual = ''.join(chr(33 + rng.randint(5, 40)) for _ in range(q))
        paired = r.get('mpos') is not None
        lines.append('\t'.join([r['name'], str(r.get('flag', 0)), contig, str(r['pos'] + 1), '60', r['cigar'],
                                '=' if paired else '*', str(r['mpos'] + 1) if paired else '0', str(r.get('tlen', 0)), seq, qual]))
    with open(path, 'w') as f:
        f.write('\n'.join(lines) + '\n')
    return recs


def write_fasta(path, contig_len, contig='c0', seed=5):
    rng = random.Random(seed)
    seq = ''.join(rng.choice(BASES) for _ in range(contig_len))
    with open(path, 'w') as f:
        f.write(f'>{contig}\n' + ''.join(seq[i:i + 60] + '\n' for i in range(0, contig_len, 60)))


def make_stacks(seed, W, n_edges=5, origin=0, stack=(15, 35), pairs=False, spliced=False):
    """Stacks of reads sharing a start around the window edges origin + k*W: one stack ending right at the edge (its last
    column is edge-1, it is still buffered at the edge), one reaching over it, one starting on it and one a little before.
    pairs: every read gets an overlapping mate (flags 99/147).  spliced: a stack of reads whose N skip bridges the next
    edges, ending inside a stack two windows on.  The first read starts at 0, so without -r the windows start at k*W."""
    rng = random.Random(seed)
    recs = [dict(pos=0, cigar='30M', name='anchor')]
    serial = 0

    def add(pos, cig, kind):
        nonlocal serial
        serial += 1
        name = f'{kind}{serial}'
        if not pairs:
            recs.append(dict(pos=pos, cigar=cig, name=name))
            return
        span = _cigar_span(cig)
        mlen = rng.randint(30, 70)
        mpos = pos + rng.randint(max(1, span // 3), max(1, span - 5))
        tlen = max(pos + span, mpos + mlen) - pos
        recs.append(dict(pos=pos, cigar=cig, name=name, flag=99, mpos=mpos, tlen=tlen))
        recs.append(dict(pos=mpos, cigar=f'{mlen}M', name=name, flag=147, mpos=pos, tlen=-tlen))

    for k in range(1, n_edges + 1):
        e = origin + k * W
        L = rng.randint(30, 70)
        for _ in range(rng.randint(*stack)):
            add(e - L, f'{L}M', 'end')                                   # closed interval reaches the edge
        p = e - rng.randint(1, 25)
        for _ in range(rng.randint(*stack)):
            add(p, f'{rng.randint(30, 70)}M', 'halo')                    # staged again by the next window
        for _ in range(rng.randint(*stack)):
            add(e, f'{rng.randint(30, 70)}M', 'at')                      # starts on the edge
        p = e - rng.randint(30, 60)
        for _ in range(rng.randint(*stack) // 2):
            add(p, f'{rng.randint(20, 50)}M', 'near')
        if spliced and k + 2 <= n_edges:
            a, b = rng.randint(20, 40), rng.randint(30, 60)
            p = e - rng.randint(5, 15)
            q = origin + (k + 2) * W                                     # the downstream exon covers edge k+2
            n = q - (p + a) - rng.randint(1, 10)
            for _ in range(rng.randint(*stack)):
                add(p, f'{a}M{n}N{b}M', 'spl')
    contig_len = origin + (n_edges + 2) * W + 200
    return recs, contig_len


def dropped_reads(recs, maxcnt, flags_ok=lambda f: True):
    """A plain model of bam_plp_push's rule over one file's kept records (file order): [(pos, end)] of the dropped ones."""
    ends, pp, out = [], None, []
    for r in recs:
        if not flags_ok(r.get('flag', 0)):
            continue
        p, e = r['pos'], r['pos'] + _cigar_span(r['cigar'])
        if pp is not None:
            while ends and ends[0] < pp:
                heapq.heappop(ends)
            if p == pp and len(ends) + 1 > maxcnt:
                out.append((p, e))
                continue
        heapq.heappush(ends, e)
        pp = p
    return out


def edge_near_drop(drops, edges, reach=80):
    return any(p - reach <= e <= q + 1 for p, q in drops for e in edges)


def run(exe, line, d, env=None):
    return subprocess.run(f'{exe} {line}', shell=True, cwd=d, capture_output=True, env=dict(os.environ, **(env or {})))


def with_d0(line):
    """the same command line with the rule switched off"""
    t = line.split()
    for opt in ('--max-depth', '-d'):
        if opt in t:
            t[t.index(opt) + 1] = '0'
            return ' '.join(t)
    return ' '.join([t[0], '-d', '0', *t[1:]])   # the command's default -d


def check_cases(tool, oracle, d, cases, env=None):
    """every (command line, must_fire) through the oracle and the tool: outputs equal, and the rule fires where asked"""
    from concurrent.futures import ThreadPoolExecutor

    def one(c):
        line, must_fire = c
        a = run(oracle, line, d)
        if a.returncode != 0 or not a.stdout:
            return (line, 'oracle failed', a.stderr[-300:])
        if must_fire and run(oracle, with_d0(line), d).stdout == a.stdout:
            return (line, 'the rule does not fire')
        b = run(tool, line, d, env)
        if a.stdout != b.stdout or b.returncode != 0:
            return (line, env, b.returncode, b.stderr[-300:])
        return None
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        return [r for r in ex.map(one, cases) if r is not None]


# ---------------------------------------------------------------------------------------------- structured inputs
W = 97          # column window of the structured cases
DEPTH = 30


def write_structured(d, W=W, depth=DEPTH, seed=11):
    """st.sam (stacks), pe.sam (stacks of overlapping pairs), spl.sam (stacks + spliced reads), lo.sam (a shallow second
    file), rg.sam (stacks around the edges of the region -r c0:51-), x.fa; returns the dropped reads of each input and
    the window edges"""
    info = {}
    for stem, kw in (('st', {}), ('pe', {'pairs': True}), ('spl', {'spliced': True, 'n_edges': 7}), ('rg', {'origin': 50})):
        recs, L = make_stacks(seed, W, **kw)
        recs = write_sam(str(d / f'{stem}.sam'), 1000 + 8 * W + 400, recs)
        info[stem] = recs
        seed += 1
    lo, _ = make_stacks(seed, W, stack=(1, 3))
    info['lo'] = write_sam(str(d / 'lo.sam'), 1000 + 8 * W + 400, lo)
    write_fasta(str(d / 'x.fa'), 1000 + 8 * W + 400)
    (d / 'x.bed').write_text(f'c0\t0\t{3 * W + 10}\nc0\t{4 * W - 20}\t{6 * W}\n')
    return info


@pytest.fixture(scope='module')
def sdir(tmp_path_factory):
    d = tmp_path_factory.mktemp('maxdepth')
    return d, write_structured(d)


def structured_cases(depth=DEPTH, W=W):
    mp = [f'-B -d {depth}', f'-B -a -d {depth} -f x.fa', f'-B -x -O -d {depth}', f'-B -s -Q 0 -d {depth}']
    cases = []
    for stem in ('st', 'pe', 'spl'):
        cases += [f'mpileup {o} {stem}.sam' for o in mp]
    cases += [f'mpileup -B -d {depth} -x pe.sam', f'mpileup -B -d {depth} st.sam lo.sam', f'mpileup -B -d {depth} lo.sam spl.sam',
              f'mpileup -B -d {depth} -r c0:51- rg.sam', f'mpileup -B -a -d {depth} -r c0:51-{50 + 5 * W} rg.sam',
              f'coverage -d {depth} st.sam', f'coverage -d {depth} spl.sam pe.sam', f'coverage -d {depth} -r c0:51- rg.sam',
              f'coverage -d {depth} -r c0:{W // 2}-{5 * W} st.sam']
    return cases


def test_generators_put_drops_at_window_edges(sdir):
    """the plain model of the rule drops reads of every structured input within a read length of a window edge"""
    d, info = sdir
    for stem, origin in (('st', 0), ('pe', 0), ('spl', 0), ('rg', 50)):
        drops = dropped_reads(info[stem], DEPTH)
        assert len(drops) > 20, stem
        assert edge_near_drop(drops, [origin + k * W for k in range(1, 8)]), stem
    assert not dropped_reads(info['lo'], DEPTH)
    # spliced reads stay buffered across their intron: the downstream stacks lose reads to them
    spl = [r for r in info['spl'] if 'N' in r['cigar']]
    assert len(spl) > 30 and max(_cigar_span(r['cigar']) for r in spl) > 2 * W


@pytest.mark.parametrize('env', [{'B200_WINDOW_COLS': str(W)}, {'B200_WINDOW_COLS': str(W), 'B200_DEVICES': '0,0'},
                                 {'B200_WINDOW_COLS': '331'}, {}], ids=['win97', 'win97_devices00', 'win331', 'unwindowed'])
def test_structured_vs_oracle(env, sdir, emul_dir, oracle_bin):
    d, _ = sdir
    cases = [(c, True) for c in structured_cases()]
    bad = check_cases(os.path.join(emul_dir, 'b200samtools_emul'), oracle_bin, d, cases, env)
    assert not bad, f'{len(bad)} of {len(cases)}: {bad[:3]}'


def test_structured_bedcov(sdir, emul_dir, oracle_bin):
    """bedcov runs one pileup per interval, like the reference: equal by construction, kept equal"""
    d, _ = sdir
    cases = [(f'bedcov --max-depth {DEPTH} x.bed {f}', True) for f in ('st.sam', 'pe.sam', 'spl.sam lo.sam')]
    cases += [(f'bedcov -j --max-depth {DEPTH} x.bed st.sam', True)]
    bad = check_cases(os.path.join(emul_dir, 'b200samtools_emul'), oracle_bin, d, cases, {'B200_WINDOW_COLS': str(W)})
    assert not bad, bad[:3]


def test_general_path_windows(sdir, emul_dir, oracle_bin):
    """the general mpileup path (EMUL_GENERAL=1, B200_PLP_GENERAL=1 on the device) across the same windows"""
    d, _ = sdir
    cases = [(f'mpileup -B -d {DEPTH} {s}.sam', True) for s in ('st', 'pe', 'spl')]
    bad = check_cases(os.path.join(emul_dir, 'b200samtools_emul'), oracle_bin, d, cases, {'B200_WINDOW_COLS': str(W), 'EMUL_GENERAL': '1'})
    assert not bad, bad[:3]


@pytest.mark.parametrize('budget', ['1', '3000'])
def test_iterator_tier_windows(budget, sdir, emul_dir, oracle_bin):
    """plp_dump -d N [-o] with windows cut every B200_PLP_WINDOW_BYTES of bases.  A window is cut at the first read of a new
    start position once the budget is spent: with a budget of 1 byte at every new start, so every dropped read lies
    within a read length of an edge."""
    d, _ = sdir
    exe = os.path.join(emul_dir, 'plp_dump_emul')
    for files in (['st.sam'], ['pe.sam'], ['spl.sam', 'lo.sam']):
        paths = [str(d / f) for f in files]
        for ov in ([], ['-o']):
            args = [*ov, '-d', str(DEPTH), *paths]
            want = subprocess.run([oracle_bin, 'pileup-dump', *args], capture_output=True)
            off = subprocess.run([oracle_bin, 'pileup-dump', *ov, '-d', '0', *paths], capture_output=True)
            assert want.returncode == 0 and want.stdout != off.stdout, args
            got = subprocess.run([exe, *args], capture_output=True, env=dict(os.environ, B200_PLP_WINDOW_BYTES=budget))
            assert got.returncode == 0, got.stderr[-300:]
            assert got.stdout == want.stdout, (budget, args)


# ---------------------------------------------------------------------------------------------- fuzz
FUZZ_OPTS = ['-B -d 2', '-B -d 3 -x', '-B -d 2 -a', '-B -d 5 -x -O', '-B -d 3 -s -Q 0']


def fuzz_cases(d, oracle, seeds):
    """(command line, True) for every fuzz_sam seed and option set where the rule fires"""
    cases = []
    for seed in seeds:
        sam, fa = fuzz_sam.make_sam(seed)
        (d / f'f{seed}.sam').write_text(sam); (d / f'f{seed}.fa').write_text(fa)
        for o in FUZZ_OPTS:
            line = f'mpileup {o} f{seed}.sam'
            if run(oracle, line, d).stdout != run(oracle, with_d0(line), d).stdout:
                cases.append((line, True))
        line = f'coverage -d 3 f{seed}.sam'
        if run(oracle, line, d).stdout != run(oracle, with_d0(line), d).stdout:
            cases.append((line, True))
    return cases


@pytest.fixture(scope='module')
def fuzz_dir(tmp_path_factory, oracle_bin):
    d = tmp_path_factory.mktemp('mdfuzz')
    cases = fuzz_cases(d, oracle_bin, range(1, 21))
    assert len(cases) >= 80, len(cases)
    return d, cases


def edge_near_model_drop(path, line, W):
    """Does a window edge of this command line fall within a read length of a read the plain model of the rule drops?  The
    model sees the records the command keeps (not unmapped / secondary / QC-failed / duplicate; mpileup also drops
    orphans) per contig; the windows start at the contig's first record (mpileup), at 0 (mpileup -a, coverage)."""
    t = line.split()
    cmd, maxcnt = t[0], int(t[t.index('-d') + 1])
    by_contig = {}
    for l in open(path):
        if l.startswith('@'):
            continue
        f = l.split('\t')
        by_contig.setdefault(f[2], []).append(dict(pos=int(f[3]) - 1, cigar=f[5], flag=int(f[1])))
    for recs in by_contig.values():
        keep = lambda fl: not (fl & 0x704) and (cmd == 'coverage' or not (fl & 1 and not fl & 2))
        drops = dropped_reads(recs, maxcnt, keep)
        lo = 0 if cmd == 'coverage' or '-a' in t else min(r['pos'] for r in recs)
        hi = max(r['pos'] + max(1, _cigar_span(r['cigar'])) for r in recs)
        reach = max(_cigar_span(r['cigar']) for r in recs)
        if edge_near_drop(drops, range(lo + W, hi + 1, W), reach):
            return True
    return False


@pytest.mark.parametrize('env,min_near', [({'B200_WINDOW_COLS': '97'}, 0.5), ({'B200_WINDOW_COLS': '331'}, 0.5), ({'B200_WINDOW_COLS': '1000'}, 0.05),
                                          ({'B200_WINDOW_COLS': '97', 'B200_DEVICES': '0,0'}, 0.5)], ids=['win97', 'win331', 'win1000', 'win97_devices00'])
def test_fuzz_windows(env, min_near, fuzz_dir, emul_dir, oracle_bin):
    """fuzz_sam's 1500-base contigs cut into windows: the cases where an edge falls within a read length of a dropped read
    (at least half of them with 97 and 331 columns; 1000-column windows leave one edge per contig)"""
    d, cases = fuzz_dir
    W = int(env['B200_WINDOW_COLS'])
    near = [c for c in cases if edge_near_model_drop(d / c[0].split()[-1], c[0], W)]
    assert len(near) >= min_near * len(cases), (len(near), len(cases))
    bad = check_cases(os.path.join(emul_dir, 'b200samtools_emul'), oracle_bin, d, near, env)
    assert not bad, f'{len(bad)} of {len(near)}: {bad[:3]}'
