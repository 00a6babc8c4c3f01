"""Empty -a / -aa rows of a reference sequence that has no reads, cut into column windows.  The drivers print such rows
window by window like any other; every window of the sequence (or of the region) must get its rows, not only the first.
Checked byte for byte against the oracle, through the emulation harness on the CPU and through the CUDA CLI, with one
engine handle and with two window workers."""
import os, subprocess
import pytest
from conftest import ROOT

W = 97    # B200_WINDOW_COLS: a few hundred empty rows cross several window edges

# name -> (reference sequences (name, length), first positions (1-based) of the 50-base reads per sequence)
INPUTS = {
    # an uncovered sequence after a covered one
    'tail': ([('c1', 300), ('c2', 500)], {'c1': [10, 40, 100, 180, 240]}),
    # an uncovered sequence several windows long between covered ones
    'gap': ([('c1', 300), ('c2', 1000), ('c3', 400)], {'c1': [5, 90, 96, 150, 251], 'c3': [1, 60, 200, 333, 351]}),
}
COMMANDS = {
    'tail': ['mpileup -aa -B {sam}', 'depth -aa {sam}', 'mpileup -aa -B -r c2 {sam}', 'depth -a -r c2:1-400 {sam}'],
    'gap': ['mpileup -aa -B {sam}', 'depth -aa {sam}', 'mpileup -aa -B -r c2 {sam}', 'depth -a -r c2:101-900 {sam}'],
}
ENVS = {'one_handle': {'B200_WINDOW_COLS': str(W)}, 'two_workers': {'B200_WINDOW_COLS': str(W), 'B200_DEVICES': '0,0'}}
CASES = [(inp, cmd, env) for inp in INPUTS for cmd in COMMANDS[inp] for env in ENVS]
IDS = [f'{inp}-{cmd.split()[0]}-{"region" if " -r " in cmd else "all"}-{env}' for inp, cmd, env in CASES]


def write_sam(path, contigs, reads):
    bases = 'ACGTTGCAAGCTTCGA' * 4
    with open(path, 'w') as f:
        f.write('@HD\tVN:1.6\tSO:coordinate\n')
        for name, length in contigs:
            f.write(f'@SQ\tSN:{name}\tLN:{length}\n')
        k = 0
        for name, _ in contigs:
            for pos in reads.get(name, []):
                seq = bases[k % 7:k % 7 + 50]
                f.write(f'r{k}\t{16 if k % 3 == 1 else 0}\t{name}\t{pos}\t60\t50M\t*\t0\t0\t{seq}\t{"I" * 50}\n')
                k += 1


@pytest.fixture(scope='module')
def sams(tmp_path_factory):
    d = tmp_path_factory.mktemp('cliwin')
    out = {}
    for inp, (contigs, reads) in INPUTS.items():
        out[inp] = str(d / f'{inp}.sam')
        write_sam(out[inp], contigs, reads)
    return out


def check(exe, oracle_bin, sams, inp, cmd, env):
    args = cmd.format(sam=sams[inp]).split()
    want = subprocess.run([oracle_bin] + args, capture_output=True, check=True).stdout
    got = subprocess.run([exe] + args, capture_output=True, env={**os.environ, **ENVS[env]}, timeout=300)
    assert got.returncode == 0, got.stderr[-300:]
    assert want.count(b'\n') > 3 * W
    assert got.stdout == want, f'{len(got.stdout.splitlines())} rows, the oracle prints {len(want.splitlines())}'


@pytest.fixture(scope='module')
def emul_bin():
    subprocess.run([os.path.join(ROOT, 'tests', 'emul', 'build.sh')], check=True)
    return os.path.join(ROOT, 'tests', 'emul', '_build', 'b200samtools_emul')


@pytest.fixture(scope='module')
def cuda_cli():
    from samtools_b200 import build
    build.build_engine()
    return build.build_cli()


@pytest.mark.parametrize('inp,cmd,env', CASES, ids=IDS)
def test_uncovered_rows_emul(emul_bin, oracle_bin, sams, inp, cmd, env):
    check(emul_bin, oracle_bin, sams, inp, cmd, env)


@pytest.mark.gpu
@pytest.mark.parametrize('inp,cmd,env', CASES, ids=IDS)
def test_uncovered_rows_gpu(cuda_cli, oracle_bin, sams, inp, cmd, env):
    check(cuda_cli, oracle_bin, sams, inp, cmd, env)
