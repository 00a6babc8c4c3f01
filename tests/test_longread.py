"""Long reads (synth.make_long_set: 513 b .. 40 kb ONT-like reads, hundreds to thousands of CIGAR ops, planted edge cases)
without a GPU: the generator's own inventory, SAM vs BAM (CG:B,I long CIGARs) through the oracle, the emulation harness vs
the oracle with the no-BAQ options, the iterator tier with windows that cut through long reads, and the register-band BAQ
arithmetic.  The same inputs run through the CUDA path in tests/test_gpu_longread.py."""
import os, subprocess
import numpy as np
import pytest
import fuzz_sam
from conftest import ROOT
from test_fuzz_emul import run_all

EMUL = os.path.join(ROOT, 'tests', 'emul', '_build')


@pytest.fixture(scope='module')
def emul_dir():
    subprocess.run([os.path.join(ROOT, 'tests', 'emul', 'build.sh')], check=True)
    return EMUL


def write_long_inputs(d):
    """long.{sam,bam,fa} (two contigs), long2.sam (a second input file), cg.{sam,bam,fa} (one read of > 65535 ops),
    del.{sam,fa} (a 70 000-base deletion)"""
    from samtools_b200 import synth
    soas = synth.make_long_set()
    synth.write_sam(str(d / 'long.sam'), soas); synth.write_bam(str(d / 'long.bam'), soas)
    with open(d / 'long.fa', 'w') as f:
        for s in soas:
            f.write(f'>{s["tid_name"]}\n')
            seq = s['ref_full'].tobytes().decode()
            f.write(''.join(seq[i:i + 60] + '\n' for i in range(0, len(seq), 60)))
    synth.write_sam(str(d / 'long2.sam'), synth.make_long_set(seed=37, lengths=(200_000, 120_000), depth=3, plant=False))
    cg = synth.make_long_cigar()
    synth.write_sam(str(d / 'cg.sam'), cg); synth.write_bam(str(d / 'cg.bam'), cg); synth.write_fasta(str(d / 'cg.fa'), 'chr1', cg['ref_full'])
    dl = synth.make_long_deletion()
    synth.write_sam(str(d / 'del.sam'), dl); synth.write_fasta(str(d / 'del.fa'), 'chr1', dl['ref_full'])
    (d / 'x.bed').write_text('chr1\t0\t30000\nchr1\t99000\t101000\nchr2\t5000\t60000\n')
    return soas


@pytest.fixture(scope='module')
def long_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp('long')
    soas = write_long_inputs(d)
    return d, soas


# ---------------------------------------------------------------------------------------------- generator inventory
def test_generator_plants_edge_cases(long_dir):
    from samtools_b200 import synth
    _, soas = long_dir
    s = soas[0]
    n = len(s['pos'])
    lq = s['l_qseq'].astype(np.int64)
    rl = synth.ref_span(s)
    ops = [s['cigar'][int(s['cigar_off'][i]):int(s['cigar_off'][i]) + int(s['n_cigar'][i])] for i in range(n)]
    band = [synth.baq_band(s['pos'][i], o >> 4, o & 15, int(lq[i]), s['tid_len']) if s['qual'][int(s['qual_off'][i])] != 0xff else None
            for i, o in enumerate(ops)]
    for l in (1, 8, 9, 511, 512, 513):
        assert (lq == l).any(), l
    for l in (512, 513):                                      # band 7 on both sides of the register kernel's limit
        assert any(lq[i] == l and band[i] == 7 and s['n_cigar'][i] == 1 for i in range(n)), l
    assert (s['n_cigar'] == 8).any() and (s['n_cigar'] == 9).any() and s['n_cigar'].max() >= 1000
    for r in (511, 512, 513, 544):
        assert any(rl[i] == r and s['n_cigar'][i] == 1 for i in range(n)) and any(rl[i] == r and s['n_cigar'][i] == 3 for i in range(n)), r
    for b in (15, 16, 31, 32, 100):
        assert b in band, b
    assert sum(1 for b in band if b is not None and b >= 16) > 100         # random reads: multi-chunk bands are common
    first = lambda o, op: (int(o[0]) & 15) == op
    for clip in (65535, 65536):
        assert any(len(o) == 2 and first(o, 4) and int(o[0]) >> 4 == clip and (int(o[1]) & 15) == 0 for o in ops), clip
    assert any(((o & 15) == 5).any() for o in ops)                                        # hard clips
    dels = [int(c >> 4) for o in ops for c in o if (c & 15) == 2]
    assert max(dels) >= 1000 and sum(d >= 512 for d in dels) >= 2
    assert any(int(c >> 4) >= 2000 for o in ops for c in o if (c & 15) == 3)          # N skips of kb
    assert any(int(c >> 4) >= 2000 for o in ops for c in o if (c & 15) == 1)          # a 2-kb insertion
    q = s['qual']
    starts = s['qual_off'].astype(np.int64)
    assert any(q[starts[i]] == 0xff for i in range(n))                                    # '*' qualities
    allq = np.concatenate([q[starts[i]:starts[i] + lq[i]] for i in range(n) if q[starts[i]] != 0xff])
    assert set(range(94)) <= set(allq.tolist())
    nib = synth._nibbles(s)
    assert (nib[np.concatenate([np.arange(starts[i], starts[i] + lq[i]) for i in range(n)])] == 15).any()
    assert (s['pos'] == 0).any() and (s['pos'] + rl > s['tid_len']).any()
    # overlapping long mates: names shared by 2 and by 3 records, both name-hash parities, simple and indel-carrying mates
    ids, cnt = np.unique(s['pair_id'], return_counts=True)
    assert (cnt == 3).any() and (cnt == 2).sum() > 20
    pairs = [i for i in range(n) if s['prev_same_name'][i] >= 0]
    assert {int(s['rbits'][i]) & 2 for i in pairs} == {0, 2}
    kinds = set()
    for i in pairs:
        j = int(s['prev_same_name'][i])
        assert s['pos'][i] < s['pos'][j] + rl[j]                                          # they overlap
        kinds.add(int(s['n_cigar'][i] == 1) + int(s['n_cigar'][j] == 1))
    assert kinds >= {0, 1, 2}


def test_long_cigar_and_deletion_inputs(long_dir):
    from samtools_b200 import synth
    cg = synth.make_long_cigar()
    assert cg['n_cigar'].max() > 65535
    dl = synth.make_long_deletion()
    assert any(int(c >> 4) == 70_000 and (c & 15) == 2 for c in dl['cigar'])


def test_fixed_length_batches_unchanged(tmp_path):
    """the fixed-length generator feeds the C2 tests and bench.py: its arrays and its SAM / BAM bytes must not move; the
    variable-length writers give the same SAM text for the same records"""
    import hashlib
    from samtools_b200 import synth
    soa = synth.make_batch(length=100_000, depth=30, seed=2)
    h = hashlib.sha256()
    for k in ('pos', 'flag', 'mapq', 'cigar', 'cigar_off', 'seq4', 'qual', 'qual_off', 'prev_same_name', 'rbits'):
        h.update(soa[k].tobytes())
    synth.write_sam(str(tmp_path / 'a.sam'), soa); synth.write_bam(str(tmp_path / 'a.bam'), soa)
    h.update((tmp_path / 'a.sam').read_bytes()); h.update((tmp_path / 'a.bam').read_bytes())
    assert h.hexdigest() == '3d45a8bdc5e34959614406b659ce294c5ae68b98e9a7a816724ef0faf70cd5b6'
    var = dict(soa); var['read_len'] = None
    synth.write_sam(str(tmp_path / 'v.sam'), var)
    assert (tmp_path / 'v.sam').read_bytes() == (tmp_path / 'a.sam').read_bytes()


# ---------------------------------------------------------------------------------------------- SAM vs BAM (CG tag)
@pytest.mark.parametrize('stem', ['long', 'cg'])
def test_sam_and_bam_give_the_same_oracle_output(stem, long_dir, oracle_bin):
    d, _ = long_dir
    for cmd in (['mpileup', '-B', '-f', f'{stem}.fa'], ['mpileup', '-f', f'{stem}.fa', '-s'], ['depth', '-a', '-J'], ['coverage'], ['view']):
        a = subprocess.run([oracle_bin, *cmd, f'{stem}.sam'], cwd=d, capture_output=True, check=True).stdout
        b = subprocess.run([oracle_bin, *cmd, f'{stem}.bam'], cwd=d, capture_output=True, check=True).stdout
        assert a == b and len(a) > 100, cmd
    if stem == 'cg':   # the record behind the placeholder comes back with its real CIGAR and without the CG tag
        v = subprocess.run([oracle_bin, 'view', 'cg.bam'], cwd=d, capture_output=True, check=True).stdout
        assert b'CG:B' not in v and max(len(l.split(b'\t')[5]) for l in v.split(b'\n') if l) > 100_000


# ---------------------------------------------------------------------------------------------- emulation vs oracle
LONG_CASES = [('mpileup', '-B -f long.fa long.sam'), ('mpileup', '-B -a -f long.fa long.sam'), ('mpileup', '-B -x -Q 0 long.sam'),
              ('mpileup', '-B -s -O --output-BP-5 -f long.fa long.sam'), ('mpileup', '-B --reverse-del -f long.fa long.sam'),
              ('mpileup', '-B -d 10 -f long.fa long.sam'), ('mpileup', '-B -f long.fa long.sam long2.sam'),
              ('mpileup', '-B -f cg.fa cg.bam'), ('mpileup', '-B -f del.fa del.sam'),
              ('depth', '-a long.sam'), ('depth', '-J -q 13 long.sam'), ('depth', '-s long.sam long2.sam'), ('depth', '-a cg.bam'),
              ('coverage', 'long.sam'), ('coverage', '-m -r chr1 long.sam'), ('coverage', 'cg.bam'),
              ('bedcov', 'x.bed long.sam'), ('bedcov', '-j x.bed long.sam long2.sam')]


def run_cases(tool, oracle, d, cases, env=None):
    from concurrent.futures import ThreadPoolExecutor
    env = dict(os.environ, **(env or {}))

    def one(c):
        line = ' '.join(c)
        a = subprocess.run(f'{oracle} {line}', shell=True, cwd=d, capture_output=True)
        b = subprocess.run(f'{tool} {line}', shell=True, cwd=d, capture_output=True, env=env)
        if a.returncode != 0 or not a.stdout:
            return (line, 'oracle failed', a.stderr[-300:])
        if a.stdout != b.stdout or b.returncode != 0:
            return (line, b.returncode, b.stderr[-300:])
        return None
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        return [r for r in ex.map(one, cases) if r is not None]


@pytest.mark.parametrize('env', [{}, {'B200_WINDOW_COLS': '4099'}, {'EMUL_GENERAL': '1'}], ids=['default', 'win4099', 'general'])
def test_emulation_vs_oracle_long_reads(env, long_dir, emul_dir, oracle_bin):
    d, _ = long_dir
    bad = run_cases(os.path.join(emul_dir, 'b200samtools_emul'), oracle_bin, d, LONG_CASES, env)
    assert not bad, bad[:3]


def test_iterator_tier_windows_long_reads(long_dir, emul_dir, oracle_bin, monkeypatch):
    """B200_PLP_WINDOW_BYTES=262144: windows cut through long reads and long mate overlaps"""
    d, _ = long_dir
    monkeypatch.setenv('B200_PLP_WINDOW_BYTES', '262144')
    for files in (['long.sam'], ['long.sam', 'long2.sam'], ['cg.bam']):
        paths = [str(d / f) for f in files]
        got = subprocess.run([os.path.join(emul_dir, 'plp_dump_emul'), '-c', *paths], capture_output=True)
        want = subprocess.run([oracle_bin, 'pileup-dump', *paths], capture_output=True)
        assert got.returncode == 0, got.stderr[-300:]
        assert got.stdout == want.stdout and len(want.stdout) > 1000, files
        assert b'bad=0' in got.stderr


def test_register_band_baq_on_long_reads(long_dir, emul_dir):
    """baq_reg.h vs the oracle's sam_prob_realn on every band-7 read of <= 512 bases of the long set; the 512-base band-7
    read is taken, the 513-base one is not (it runs on the warp kernel k_baq)"""
    d, soas = long_dir
    r = subprocess.run([os.path.join(emul_dir, 'baq_host'), str(d / 'long.sam'), str(d / 'long.fa'), '-l'], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr
    taken = {int(l.split()[3]) for l in r.stdout.splitlines() if l.startswith('reg ')}
    assert 512 in taken and max(taken) == 512
    s = soas[0]
    assert any(s['l_qseq'][i] == 513 and s['n_cigar'][i] == 1 for i in range(len(s['pos'])))   # the planted band-7 513M read


# ---------------------------------------------------------------------------------------------- long fuzz flavour
def test_fuzz_long_flavour(emul_dir, oracle_bin, tmp_path):
    """fuzz_sam's long flavour (reads up to a few kb, indels up to 40, 20-kb contigs), no-BAQ option sets"""
    bad = run_all(os.path.join(emul_dir, 'b200samtools_emul'), oracle_bin, tmp_path, range(201, 209), need_noBAQ=True, long=True)
    assert not bad, f'{len(bad)} mismatches, first: {bad[0]}'
