"""Oracle vs CUDA path on random corner-case SAMs (all option sets of tests/fuzz_sam.py, BAQ included)."""
import os
import pytest
from conftest import ROOT
from test_fuzz_emul import run_all

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')


@pytest.mark.parametrize('lo', [1, 5])
def test_fuzz_cuda_path(lo, oracle_bin, tmp_path):
    # 2 x 4 seeds (~500 CLI runs, each paying a CUDA context, 6 in flight), GL included
    bad = run_all(CLI, oracle_bin, tmp_path, range(lo, lo + 4), need_noBAQ=False, with_gl=True)
    assert not bad, f'{len(bad)} mismatches, first: {bad[0]}'


def test_fuzz_cuda_path_long(oracle_bin, tmp_path):
    """the long flavour (reads up to a few kb, indels up to 40: BAQ bands over several 32-cell chunks), BAQ included"""
    bad = run_all(CLI, oracle_bin, tmp_path, range(301, 303), need_noBAQ=False, with_gl=True, long=True)
    assert not bad, f'{len(bad)} mismatches, first: {bad[0]}'
