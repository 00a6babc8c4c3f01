"""Reading BAM inputs through their BAI / CSI index, and the `index` command that writes one.

With an index, `-r` (mpileup, depth, coverage) and every bedcov line inflate only the blocks that hold the region's
records; the records and their order must stay exactly those of the linear scan.  Every comparison here is byte for byte
against the same command without an index (the scan) or against the oracle.  The CPU cases run the emulation-harness CLI,
the `gpu` ones the CUDA CLI.
"""
import gzip, os, shutil, struct, subprocess
import numpy as np
import pytest
from conftest import ROOT
from samtools_b200 import synth

FIXTURES = [('test/mpileup', 'mpileup.1.bam'), ('test/mpileup', 'ce#5b.bam'), ('test/bedcov', 'bedcov.bam')]
CMDS = ['mpileup -B -r {reg} {bam}', 'depth -r {reg} {bam}', 'coverage -r {reg} {bam}']


# ---------------------------------------------------------------------------------------------------------------- helpers
def run(exe, args, cwd=None, env=None):
    return subprocess.run([exe] + args, cwd=cwd, capture_output=True, timeout=600, env={**os.environ, **(env or {})})


def out_ok(exe, args, **kw):
    r = run(exe, args, **kw)
    assert r.returncode == 0, (args, r.stderr[-400:])
    return r.stdout


def bam_refs(path):
    """(name, length) of every reference sequence in the BAM header"""
    with gzip.open(path, 'rb') as f:
        assert f.read(4) == b'BAM\1'
        (lt,) = struct.unpack('<i', f.read(4)); f.read(lt)
        (n,) = struct.unpack('<i', f.read(4))
        refs = []
        for _ in range(n):
            (ln,) = struct.unpack('<i', f.read(4))
            name = f.read(ln).rstrip(b'\0').decode()
            (lr,) = struct.unpack('<i', f.read(4))
            refs.append((name, lr))
    return refs


def sweep(refs):
    """regions over every reference sequence: whole, starts, middles, ends, past the end, 16 kb boundaries"""
    regs = []
    for name, ln in refs:
        regs += [name, f'{name}:1-1', f'{name}:1-16384', f'{name}:{max(1, ln // 2 - 500)}-{ln // 2 + 500}',
                 f'{name}:{max(1, ln - 200)}-{ln}', f'{name}:{max(1, ln - 50)}', f'{name}:16384-16385', f'{name}:{ln + 10}-{ln + 20}']
    return regs


def bed_of(refs, path):
    with open(path, 'w') as f:
        for name, ln in refs:
            for b, e in ((0, ln), (0, 1), (ln // 3, ln // 2), (max(0, ln - 100), ln), (16383, 16385), (ln // 2, ln // 2)):
                f.write(f'{name}\t{b}\t{e}\n')


def with_and_without(tmp, bam, idx=None, name='in.bam'):
    """two directories: one with the BAM and its index (`idx` copied as <name>.bai / .csi), one with the BAM alone"""
    a, b = tmp / 'indexed', tmp / 'scan'
    a.mkdir(exist_ok=True); b.mkdir(exist_ok=True)
    shutil.copy(bam, a / name); shutil.copy(bam, b / name)
    if idx:
        shutil.copy(idx, a / (name + ('.csi' if idx.endswith('.csi') else '.bai')))
    return str(a / name), str(b / name)


# ---------------------------------------------------------------------------------------------------------- synthetic BAMs
def _seq(rng, n):
    return np.frombuffer(b'ACGT', dtype=np.uint8)[rng.integers(0, 4, n)]


def _recs(rng, items):
    """(pos, cigar, flag) -> records for synth._pack (bases random: no command here takes a FASTA)"""
    out = []
    for pos, cig, flag in items:
        lens, ops = synth.parse_cigar(cig) if cig else (np.zeros(0, np.int64), np.zeros(0, np.int64))
        lq = int(lens[synth._QCONS[ops]].sum()) if len(ops) else 30
        out.append(dict(pos=int(pos), lens=lens, ops=ops, flag=int(flag), name=None, mapq=int(rng.integers(20, 61)),
                        seq=_seq(rng, lq), qual=rng.integers(10, 41, lq).astype(np.uint8)))
    return out


def _empty(tid, name, length):
    z = lambda dt: np.zeros(0, dtype=dt)
    return dict(pos=z(np.int64), flag=z(np.uint16), mapq=z(np.uint8), l_qseq=z(np.int32), n_cigar=z(np.uint32), cigar_off=z(np.uint64),
                qual_off=z(np.uint64), mtid=z(np.int32), mpos=z(np.int64), isize=z(np.int64), cigar=z(np.uint32), seq4=z(np.uint8),
                qual=z(np.uint8), pair_id=z(np.int64), tid=tid, tid_name=name, tid_len=length, read_len=None)


EDGE_LEN = 9_000_000
EDGES = [16384, 32768, 5 * 16384, 1 << 17, 3 << 17, 1 << 20, 1 << 23]   # 16 kb windows and bin boundaries of every level


def edge_contig(rng, tid, name):
    items = []
    for p in EDGES:
        items += [(p, '100M', 0), (p - 100, '100M', 0), (p - 1, '2M', 16), (p - 50, '100M', 0), (p, '10S', 0), (p, '5I', 0),
                  (p + 1, '', 4 | 1), (p, '40M70000N40M', 0), (p - 20, '20M2000D20M', 0)]
    items += [(int(p), '150M', int(f)) for p, f in zip(np.sort(rng.integers(0, EDGE_LEN - 200_000, 3000)), rng.choice([0, 16, 1024], 3000))]
    items += [(EDGE_LEN - 30, '50M', 0), (EDGE_LEN - 1, '1M', 0)]                   # reads running past the contig's end
    return synth._pack(_recs(rng, items), None, EDGE_LEN, tid, name)


def write_multi(path):
    """c0 paired 150 bp reads, c1 without reads, c2 the edge cases, c3 paired reads again"""
    rng = np.random.default_rng(11)
    soas = [synth.make_batch(length=300_000, depth=6, seed=5, tid=0, tid_name='c0'), _empty(1, 'c1', 50_000),
            edge_contig(rng, 2, 'c2'), synth.make_batch(length=120_000, depth=6, seed=6, tid=3, tid_name='c3')]
    synth.write_bam(path, soas)
    return [(s['tid_name'], int(s['tid_len'])) for s in soas]


BIG_LEN = 2_100_000_000     # BAM positions are 32-bit: this is the largest scale a BAM can hold, past BAI's 2^29


def write_large(path):
    rng = np.random.default_rng(12)
    base = [1 << 29, (1 << 29) + 16384, 1 << 30, 1_500_000_000, (1 << 31) - (1 << 26), BIG_LEN - 300]
    items = sorted([(p + d, '100M', 0) for p in base for d in (-150, -1, 0, 70)] + [((1 << 30) - 10, '50M100000N50M', 0)])
    synth.write_bam(path, [synth._pack(_recs(rng, items), None, BIG_LEN, 0, 'big')])
    return base


# ------------------------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope='module')
def emul_bin():
    subprocess.run([os.path.join(ROOT, 'tests', 'emul', 'build.sh')], check=True)
    return os.path.join(ROOT, 'tests', 'emul', '_build', 'b200samtools_emul')


@pytest.fixture(scope='module')
def cuda_cli():
    from samtools_b200 import build
    build.build_engine()
    return build.build_cli()


@pytest.fixture(scope='module')
def multi(tmp_path_factory):
    d = tmp_path_factory.mktemp('multi')
    refs = write_multi(str(d / 'multi.bam'))
    return str(d / 'multi.bam'), refs


def fixture_pair(corpus, tmp, cwd, bam):
    """the reference's BAM with its shipped .bai, and the same BAM alone"""
    src = os.path.join(corpus, cwd, bam)
    return with_and_without(tmp, src, src + '.bai', name=bam)


# -------------------------------------------------------------------------------------- the reference's indexes, read
def check_fixture(exe, oracle, corpus, tmp, cwd, bam, few=False):
    ibam, sbam = fixture_pair(corpus, tmp, cwd, bam)
    refs = bam_refs(ibam)
    n = 0
    # `few`: every CUDA CLI run creates an engine, so the GPU cases take the first and the last sequence's regions
    for reg in (sweep(refs[:1])[:4] + sweep(refs[-1:])[:4] if few else sweep(refs)):
        for cmd in CMDS:
            want = out_ok(oracle, cmd.format(reg=reg, bam=sbam).split())
            assert out_ok(exe, cmd.format(reg=reg, bam=ibam).split()) == want, (cmd, reg)
            n += len(want)
    assert n > 0
    bed = str(tmp / 'sweep.bed'); bed_of(refs, bed)
    for opts in ([], ['-c'], ['-j', '-d', '2']):
        want = out_ok(oracle, ['bedcov'] + opts + [bed, sbam])
        assert out_ok(exe, ['bedcov'] + opts + [bed, ibam]).replace(ibam.encode(), sbam.encode()) == want, opts


@pytest.mark.parametrize('cwd,bam', FIXTURES, ids=[b for _, b in FIXTURES])
def test_reference_index_emul(emul_bin, oracle_bin, corpus, tmp_path, cwd, bam):
    check_fixture(emul_bin, oracle_bin, corpus, tmp_path, cwd, bam)


@pytest.mark.gpu
@pytest.mark.parametrize('cwd,bam', FIXTURES, ids=[b for _, b in FIXTURES])
def test_reference_index_gpu(cuda_cli, oracle_bin, corpus, tmp_path, cwd, bam):
    check_fixture(cuda_cli, oracle_bin, corpus, tmp_path, cwd, bam, few=True)


# --------------------------------------------------------------------------------------- round trip through the writer
KINDS = {'bai': ['-b'], 'csi14': ['-c', '-m', '14'], 'csi12': ['-c', '-m', '12']}


def multi_regions(refs):
    regs = sweep(refs)
    for p in EDGES:   # around every edge, and over the 100 kb N skips that start there
        regs += [f'c2:{p - 5}-{p + 5}', f'c2:{p + 1}-{p + 1}', f'c2:{p}-{p + 16384}', f'c2:{p + 30_000}-{p + 30_010}']
    regs += ['c3:1-120000', 'c0:150000-170000', f'c2:{EDGE_LEN - 40}-{EDGE_LEN + 100}']
    return regs


def check_round_trip(exe, tmp, bam, refs, kind, regions, cmds, env=None):
    raw = tmp / 'raw'; raw.mkdir(exist_ok=True)
    shutil.copy(bam, raw / 'in.bam')
    ext = '.bai' if kind == 'bai' else '.csi'
    out_ok(exe, ['index'] + KINDS[kind] + [str(raw / 'in.bam'), str(raw / ('in.bam' + ext))])
    ibam, sbam = with_and_without(tmp, bam, str(raw / ('in.bam' + ext)))
    rows = 0
    for reg in regions:
        for cmd in cmds:
            want = out_ok(exe, cmd.format(reg=reg, bam=sbam).split(), env=env)
            assert out_ok(exe, cmd.format(reg=reg, bam=ibam).split(), env=env) == want, (kind, cmd, reg)
            rows += want.count(b'\n')
    assert rows > 0
    return ibam, sbam


@pytest.mark.parametrize('kind', list(KINDS))
def test_round_trip_emul(emul_bin, multi, tmp_path, kind):
    bam, refs = multi
    ibam, sbam = check_round_trip(emul_bin, tmp_path, bam, refs, kind, multi_regions(refs), CMDS)
    bed = str(tmp_path / 'multi.bed'); bed_of(refs, bed)
    with open(bed, 'a') as f:
        for p in EDGES:
            f.write(f'c2\t{p - 3}\t{p + 3}\nc2\t{p}\t{p + 100_000}\n')
    for opts in ([], ['-c', '-j']):
        want = out_ok(emul_bin, ['bedcov'] + opts + [bed, sbam])
        assert out_ok(emul_bin, ['bedcov'] + opts + [bed, ibam]).replace(ibam.encode(), sbam.encode()) == want


@pytest.mark.parametrize('kind', list(KINDS))
def test_round_trip_windows_emul(emul_bin, multi, tmp_path, kind):
    """-a / -aa rows cut into many 97-column windows, with one engine handle and with two window workers"""
    bam, refs = multi
    regs = ['c0:1000-1400', 'c1:10-300', f'c2:{(1 << 17) - 150}-{(1 << 17) + 150}', 'c3:119800-120000']
    cmds = ['mpileup -a -B -r {reg} {bam}', 'mpileup -aa -B -r {reg} {bam}', 'depth -a -r {reg} {bam}', 'depth -aa -r {reg} {bam}',
            'coverage -r {reg} {bam}']
    for env in ({'B200_WINDOW_COLS': '97'}, {'B200_WINDOW_COLS': '97', 'B200_DEVICES': '0,0'}):
        check_round_trip(emul_bin, tmp_path, bam, refs, kind, regs, cmds, env=env)


def test_large_coordinates_emul(emul_bin, tmp_path):
    bam = str(tmp_path / 'large.bam')
    base = write_large(bam)
    r = run(emul_bin, ['index', bam, str(tmp_path / 'large.bai')])
    assert r.returncode != 0 and b'-c' in r.stderr and not os.path.exists(tmp_path / 'large.bai'), r.stderr
    regs = [f'big:{p - 200}-{p + 200}' for p in base] + ['big', f'big:{(1 << 30) + 400_000}-{(1 << 30) + 400_100}', 'big:1-1000000']
    for kind in ('csi14', 'csi12'):
        d = tmp_path / kind; d.mkdir()
        check_round_trip(emul_bin, d, bam, [('big', BIG_LEN)], kind, regs, CMDS)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', list(KINDS))
def test_round_trip_gpu(cuda_cli, multi, tmp_path, kind):
    bam, refs = multi
    regs = ['c0', 'c1', 'c3:1-120000', f'c2:{(1 << 20) - 5}-{(1 << 20) + 5}', f'c2:{(1 << 17) + 30_000}-{(1 << 17) + 30_010}']
    check_round_trip(cuda_cli, tmp_path, bam, refs, kind, regs, CMDS)
    check_round_trip(cuda_cli, tmp_path, bam, refs, kind, ['c0:1000-1400', f'c2:{(1 << 17) - 150}-{(1 << 17) + 150}'],
                     ['mpileup -a -B -r {reg} {bam}', 'depth -aa -r {reg} {bam}'], env={'B200_WINDOW_COLS': '97'})


# ------------------------------------------------------------------------------------------------ the index is used
def bgzf_blocks(path):
    """[(file offset, size, uncompressed bytes)] of every BGZF block"""
    data = open(path, 'rb').read()
    out, o = [], 0
    while o < len(data):
        xlen = struct.unpack_from('<H', data, o + 10)[0]
        bsize = struct.unpack_from('<H', data, o + 16)[0] + 1
        isize = struct.unpack_from('<I', data, o + bsize - 4)[0]
        out.append((o, bsize, isize)); o += bsize
        assert xlen == 6
    return out


def first_record_of(path, tid):
    """index of the block holding the start of the first record of reference sequence `tid`"""
    blocks = bgzf_blocks(path)
    raw = gzip.open(path).read()
    starts = np.cumsum([0] + [b[2] for b in blocks])
    (lt,) = struct.unpack_from('<i', raw, 4); o = 8 + lt
    (n,) = struct.unpack_from('<i', raw, o); o += 4
    for _ in range(n):
        (ln,) = struct.unpack_from('<i', raw, o); o += 8 + ln
    while o < len(raw):
        bs, t = struct.unpack_from('<ii', raw, o)
        if t >= tid or t < 0:
            return int(np.searchsorted(starts, o, side='right') - 1)
        o += 4 + bs
    raise AssertionError('no such record')


def test_index_is_used(emul_bin, multi, tmp_path):
    """garbage in the blocks that hold only c2's records: indexed queries of c0 and c3 still succeed unchanged, the scan
    fails with a decode error"""
    bam, _ = multi
    clean = str(tmp_path / 'clean.bam'); shutil.copy(bam, clean)
    out_ok(emul_bin, ['index', clean])
    lo, hi = first_record_of(clean, 2), first_record_of(clean, 3)
    blocks = bgzf_blocks(clean)
    assert hi - lo > 3
    data = bytearray(open(clean, 'rb').read())
    rng = np.random.default_rng(3)
    for off, size, _ in blocks[lo + 1:hi]:
        data[off + 18:off + size - 8] = rng.integers(0, 256, size - 26, dtype=np.uint8).tobytes()
    bad = tmp_path / 'bad'; bad.mkdir()
    open(bad / 'in.bam', 'wb').write(bytes(data)); shutil.copy(clean + '.bai', bad / 'in.bam.bai')
    alone = tmp_path / 'alone'; alone.mkdir(); shutil.copy(bad / 'in.bam', alone / 'in.bam')
    for reg in ('c0:1000-5000', 'c3:50000-60000', 'c3'):
        for cmd in ('mpileup -B -r', 'depth -r'):
            want = out_ok(emul_bin, cmd.split() + [reg, clean])
            assert want
            assert out_ok(emul_bin, cmd.split() + [reg, str(bad / 'in.bam')]) == want, (cmd, reg)
            r = run(emul_bin, cmd.split() + [reg, str(alone / 'in.bam')])
            assert r.returncode != 0 and b'error reading' in r.stderr, (cmd, reg, r.returncode, r.stderr[-300:])


# --------------------------------------------------------------------------------------- the writer against the reference
def parse_bai(path):
    """{tid: ({bin: sorted chunks}, linear index)}, n_no_coor"""
    b = open(path, 'rb').read()
    assert b[:4] == b'BAI\1'
    (n,) = struct.unpack_from('<i', b, 4); o = 8
    refs = []
    for _ in range(n):
        (nb,) = struct.unpack_from('<i', b, o); o += 4
        bins = {}
        for _ in range(nb):
            bn, nc = struct.unpack_from('<Ii', b, o); o += 8
            bins[bn] = sorted(struct.unpack_from(f'<{2 * nc}Q', b, o)); o += 16 * nc
        (ni,) = struct.unpack_from('<i', b, o); o += 4
        refs.append((bins, list(struct.unpack_from(f'<{ni}Q', b, o)))); o += 8 * ni
    return refs, (struct.unpack_from('<Q', b, o)[0] if len(b) >= o + 8 else None)


@pytest.mark.parametrize('cwd,bam', FIXTURES, ids=[b for _, b in FIXTURES])
def test_writer_against_reference(emul_bin, corpus, tmp_path, cwd, bam, record_property):
    src = os.path.join(corpus, cwd, bam)
    mine = tmp_path / 'mine'; mine.mkdir()
    shutil.copy(src, mine / bam)
    out_ok(emul_bin, ['index', str(mine / bam)])
    theirs = tmp_path / 'theirs'; theirs.mkdir()
    shutil.copy(src, theirs / bam); shutil.copy(src + '.bai', theirs / (bam + '.bai'))
    refs = bam_refs(src)
    for reg in sweep(refs):
        for cmd in CMDS:
            want = out_ok(emul_bin, cmd.format(reg=reg, bam=str(theirs / bam)).split())
            assert out_ok(emul_bin, cmd.format(reg=reg, bam=str(mine / bam)).split()) == want, (cmd, reg)
    # a finding, not a requirement: the reference's fixtures may come from another writer
    a, b = open(mine / (bam + '.bai'), 'rb').read(), open(src + '.bai', 'rb').read()
    record_property('bytes_identical', a == b)
    record_property('same_bins_chunks_linear', parse_bai(str(mine / (bam + '.bai'))) == parse_bai(src + '.bai'))


# ------------------------------------------------------------------------------------------------------------ bad input
def test_bad_indexes(emul_bin, corpus, tmp_path):
    src = os.path.join(corpus, 'test/mpileup', 'mpileup.1.bam')
    good = open(src + '.bai', 'rb').read()
    (n_ref,) = struct.unpack_from('<i', good, 4)
    cases = {'truncated': good[:len(good) // 2], 'magic': b'BAX\1' + good[4:],
             'refs': good[:4] + struct.pack('<i', n_ref + 1) + good[8:], 'empty': b''}
    reg = bam_refs(src)[0][0] + ':100-200'
    for what, data in cases.items():
        d = tmp_path / what; d.mkdir()
        shutil.copy(src, d / 'in.bam'); open(d / 'in.bam.bai', 'wb').write(data)
        for args in (['mpileup', '-r', reg], ['depth', '-r', reg], ['coverage', '-r', reg]):
            r = run(emul_bin, args + [str(d / 'in.bam')])
            assert r.returncode != 0 and b'in.bam.bai' in r.stderr, (what, args, r.stderr)
            assert r.stdout == b'', (what, args)
        open(d / 'x.bed', 'w').write(reg.replace(':', '\t').replace('-', '\t') + '\n')
        r = run(emul_bin, ['bedcov', str(d / 'x.bed'), str(d / 'in.bam')])
        assert r.returncode != 0 and b'in.bam.bai' in r.stderr, (what, r.stderr)
        # the same broken file named by -X
        r = run(emul_bin, ['mpileup', '-X', '-r', reg, str(d / 'in.bam'), str(d / 'in.bam.bai')])
        assert r.returncode != 0 and b'in.bam.bai' in r.stderr, (what, r.stderr)
    for args in (['mpileup', '-X', '-r', reg, src], ['depth', '-X', '-r', reg, src], ['bedcov', '-X', str(tmp_path / 'refs' / 'x.bed'), src]):
        r = run(emul_bin, args)
        assert r.returncode != 0 and b'Odd number of filenames' in r.stderr, (args, r.stderr)


def test_explicit_index(emul_bin, oracle_bin, corpus, tmp_path):
    """-X pairs every data file with the index named after all data files, wherever it lives"""
    src = os.path.join(corpus, 'test/mpileup', 'mpileup.1.bam')
    (tmp_path / 'd').mkdir(); (tmp_path / 'i').mkdir()
    shutil.copy(src, tmp_path / 'd' / 'a.bam'); shutil.copy(src, tmp_path / 'd' / 'b.bam')
    shutil.copy(src + '.bai', tmp_path / 'i' / 'a.idx'); out_ok(emul_bin, ['index', '-c', str(tmp_path / 'd' / 'b.bam'), str(tmp_path / 'i' / 'b.idx')])
    a, b, ia, ib = (str(tmp_path / p) for p in ('d/a.bam', 'd/b.bam', 'i/a.idx', 'i/b.idx'))
    for reg in sweep(bam_refs(src))[:8]:
        want = out_ok(oracle_bin, ['mpileup', '-B', '-r', reg, a, b])
        assert out_ok(emul_bin, ['mpileup', '-X', '-B', '-r', reg, a, b, ia, ib]) == want, reg
        want = out_ok(oracle_bin, ['depth', '-r', reg, a, b])
        assert out_ok(emul_bin, ['depth', '-X', '-r', reg, a, b, ia, ib]) == want, reg
    bed = str(tmp_path / 'x.bed'); bed_of(bam_refs(src), bed)
    assert out_ok(emul_bin, ['bedcov', '-X', bed, a, b, ia, ib]) == out_ok(oracle_bin, ['bedcov', bed, a, b])


def test_index_refuses_unsorted(emul_bin, tmp_path):
    rng = np.random.default_rng(4)
    soa = synth._pack(_recs(rng, [(100, '50M', 0), (200, '50M', 0)]), None, 10_000, 0, 'u')
    soa['pos'] = soa['pos'][::-1].copy()
    synth.write_bam(str(tmp_path / 'u.bam'), [soa])
    r = run(emul_bin, ['index', str(tmp_path / 'u.bam')])
    assert r.returncode != 0 and b'not sorted' in r.stderr, r.stderr
    assert not os.path.exists(tmp_path / 'u.bam.bai')
