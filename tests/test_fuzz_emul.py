"""Oracle vs engine code on random corner-case SAMs (CPU, through the emulation harness).
The same cases run through the CUDA path in tests/test_gpu_fuzz.py (including BAQ)."""
import os, subprocess
import pytest
import fuzz_sam
from conftest import ROOT


@pytest.fixture(scope='module')
def emul_bin():
    subprocess.run([os.path.join(ROOT, 'tests', 'emul', 'build.sh')], check=True)
    return os.path.join(ROOT, 'tests', 'emul', '_build', 'b200samtools_emul')


def run_all(tool, oracle, td, seeds, need_noBAQ, with_gl=False, long=False):
    """every (seed, command line): oracle output vs tool output; a few processes in flight (the cases are independent
    and read-only; on the GPU each tool process pays ~1 s of CUDA context creation)"""
    from concurrent.futures import ThreadPoolExecutor
    tasks = []
    for seed in seeds:
        sam, fa = fuzz_sam.make_sam(seed, long=long)
        d = td / f's{seed}'; d.mkdir()
        (d / 'x.sam').write_text(sam); (d / 'x.fa').write_text(fa)
        (d / 'x.bed').write_text('c0\t40\t300\nc0\t250\t600\nc1\t100\nc1\t95\t140\n')
        (d / 'rg.txt').write_text('g2\n')
        (d / 'x3.bed').write_text('#chrom\tchromStart\tchromEnd\tname\nc0\t40\t300\ta\nc1\t95\t140\tb\nc0\t250\t600\tc\nc0\t10\t10\td\nc1\t0\t2000\te\n')
        (d / 'x2.sam').write_text(fuzz_sam.make_sam(seed + 100000, n_reads=25, long=long)[0])
        cases = [('mpileup', o) for o in fuzz_sam.MPILEUP_OPTS] + [('depth', o) for o in fuzz_sam.DEPTH_OPTS] + \
                [('coverage', o) for o in fuzz_sam.COVERAGE_OPTS]
        cases += [('bedcov', o) for o in fuzz_sam.BEDCOV_OPTS]
        if with_gl:
            cases += [('gl', o) for o in fuzz_sam.GL_OPTS]
        for cmd, opt in cases:
            if need_noBAQ and cmd in ('mpileup', 'gl') and '-B' not in opt.split():
                continue
            if seed % 5 == 0 and ((cmd == 'depth' and ('-q' in opt.split() or '-J' in opt.split())) or (cmd == 'mpileup' and '-C' in opt.split())):
                continue   # undefined upstream on SEQ '*' records
            opt = opt.format(bed='x.bed', rg='rg.txt')
            files = 'x.sam x2.sam' if (seed % 3 == 0 and '-r' not in opt) else 'x.sam'
            ref = '-f x.fa' if cmd in ('mpileup', 'gl') and seed % 4 != 1 else ''
            if cmd == 'bedcov':
                files = 'x3.bed ' + files
            tasks.append((seed, f'{cmd} {opt} {ref} {files}', d))

    def one(t):
        seed, line, d = t
        a = subprocess.run(f'{oracle} {line}', shell=True, cwd=d, capture_output=True)
        b = subprocess.run(f'{tool} {line}', shell=True, cwd=d, capture_output=True)
        if a.stdout != b.stdout or (a.returncode == 0) != (b.returncode == 0):
            return (seed, line, a.stdout[:200], b.stdout[:200], b.stderr[-200:])
        return None
    with ThreadPoolExecutor(max_workers=int(os.environ.get('B200_TEST_JOBS', '6'))) as ex:
        return [r for r in ex.map(one, tasks) if r is not None]


def test_fuzz_host_and_column_code(emul_bin, oracle_bin, tmp_path):
    bad = run_all(emul_bin, oracle_bin, tmp_path, range(1, 41), need_noBAQ=True)
    assert not bad, f'{len(bad)} mismatches, first: {bad[0]}'


def test_fuzz_general_path(emul_bin, oracle_bin, tmp_path, monkeypatch):
    """Same cases through the general mpileup path (mp_line_size + mp_line_write; B200_PLP_GENERAL=1 on the device)."""
    monkeypatch.setenv('EMUL_GENERAL', '1')
    bad = run_all(emul_bin, oracle_bin, tmp_path, range(1, 13), need_noBAQ=True)
    assert not bad, f'{len(bad)} mismatches, first: {bad[0]}'
