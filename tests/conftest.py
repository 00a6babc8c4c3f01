import os, subprocess, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100, sm_90a)')


@pytest.fixture(scope='session')
def oracle_bin():
    """Build (if needed) and return the CPU oracle CLI.  Test infrastructure only."""
    subprocess.run(['make', '-s', '-C', os.path.join(ROOT, 'oracle')], check=True)
    return os.path.join(ROOT, 'oracle', '_build', 'plp_oracle')


@pytest.fixture(scope='session')
def corpus(tmp_path_factory):
    import golden_cases
    return golden_cases.prepare(tmp_path_factory.mktemp('golden'))
