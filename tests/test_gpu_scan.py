"""The engine's single-pass scans (samtools_b200/csrc/scan.cuh, k_scan), each instantiation against numpy.

Every other test reaches the scans only through text outputs; here each one runs on inputs that sit at its edges:
  sizes     1 item, one block's items minus one, exactly and plus one, and a few thousand blocks (so the look-back walks
            back over many rounds of 32 predecessors);
  max8      prefix max of read ends: runs of INT32_MIN (the empty value) and negative values;
  sum4      coverage difference array, mod 2^32: partial sums that go negative, and values that wrap;
  sum1_*    exclusive offsets with the total: block sums below 2^32 whose running total passes 2^32 (u64 output; the
            int32 output is the same sum mod 2^32)."""
import os
import subprocess
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, 'tests', 'gpu', '_build', 'scan_check')
BLOCK = {'max8': 256 * 8, 'sum4': 256 * 4, 'sum1_u64': 256, 'sum1_i32': 256}


def _sizes(b):
    return [1, b - 1, b, b + 1, 3000 * b + 17]


def _inputs(kind, n, rng):
    if kind == 'max8':
        x = rng.integers(-2**31, 2**31, size=n, dtype=np.int64)
        x[rng.random(n) < 0.5] = -2**31
        if n > 5000:
            x[: n // 3] = rng.integers(-2**31, 0, size=n // 3)       # a negative stretch over many blocks ...
            x[: n // 3: 2] = -2**31
            x[:5000] = -2**31                                        # ... after two blocks and more of the empty value alone
        return x.astype(np.int32)
    if kind == 'sum4':
        x = rng.integers(-1, 2, size=n).astype(np.int32)             # +1 / -1 / 0: partial sums go negative
        if n > 4000:
            x[::997] = rng.integers(-2**31, 2**31, size=x[::997].size, dtype=np.int64).astype(np.int32)   # wrap mod 2^32
        return x
    return rng.integers(0, 2**24, size=n, dtype=np.int64).astype(np.uint32)   # a block sum stays below 2^32, the total passes it


def _expected(kind, x):
    if kind == 'max8':
        return np.maximum.accumulate(x)
    if kind == 'sum4':
        return np.cumsum(x.astype(np.int64)).astype(np.uint64).astype(np.uint32).view(np.int32)
    c = np.concatenate([np.zeros(1, np.uint64), np.cumsum(x.astype(np.uint64))])
    return c if kind == 'sum1_u64' else c.astype(np.uint32).view(np.int32)


@pytest.mark.parametrize('kind', sorted(BLOCK))
def test_scan_against_numpy(kind, tmp_path):
    assert os.path.exists(EXE), 'tests/gpu/_build/scan_check missing: run python samtools_b200/build.py'
    rng = np.random.default_rng(7)
    cases, argv = [], [EXE]
    for n in _sizes(BLOCK[kind]):
        x = _inputs(kind, n, rng)
        fi, fo = tmp_path / f'{n}.in', tmp_path / f'{n}.out'
        x.tofile(fi)
        cases.append((n, x, fo))
        argv += [kind, str(fi), str(fo)]
    subprocess.run(argv, check=True)
    dt = {'max8': np.int32, 'sum4': np.int32, 'sum1_u64': np.uint64, 'sum1_i32': np.int32}[kind]
    for n, x, fo in cases:
        got, want = np.fromfile(fo, dtype=dt), _expected(kind, x)
        assert got.shape == want.shape, (n, got.shape, want.shape)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f'n={n}: first difference at {bad[0]}: got {got[bad[0]]}, want {want[bad[0]]}'
    if kind == 'sum1_u64':
        assert cases[-1][1].astype(np.uint64).sum() > 2**32          # the large case did pass 2^32
