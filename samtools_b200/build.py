"""Build recipe for the native pieces (nvcc cross-compiles sm_90a; no GPU is needed to build).

  samtools_b200/lib/libb200pileup.so   CUDA engine + C ABI (include/b200_pileup.h)
  samtools_b200/bin/b200samtools       host CLI (C++), linked against the engine
  tests/*/_build/*                     test clients (compat tier, scan check)
  oracle/_build/*                      CPU oracle (test infrastructure, built by its own Makefile)

Everything is built in-tree, so the package runs from the source tree without an install step.
"""
import os, shutil, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'samtools_b200', 'csrc')
LIB = os.path.join(ROOT, 'samtools_b200', 'lib', 'libb200pileup.so')
BIN = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-fmad=false',            # BAQ must not contract a*b+c (bit-exact with the reference's non-FMA x86 build)
              '-Xcompiler', '-fPIC', '-shared']


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _sources(d, exts):
    out = []
    for r, _, fs in os.walk(d):
        out += [os.path.join(r, f) for f in fs if f.endswith(exts)]
    return out


def build_engine(force=False, verbose=False):
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    srcs = _sources(CSRC, ('.cu', '.cuh', '.h')) + [os.path.join(ROOT, 'include', 'b200_pileup.h'), os.path.join(ROOT, 'include', 'b200_htslib_compat.h'),
                                                    os.path.join(CSRC, 'host', 'plp_compat.cpp'), os.path.join(CSRC, 'host', 'hts_read_ops.cpp')]
    if force or _newer(LIB, srcs):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-o', LIB, os.path.join(CSRC, 'engine.cu'),
                                                                                os.path.join(CSRC, 'host', 'plp_compat.cpp'), os.path.join(CSRC, 'host', 'hts_read_ops.cpp')]
        subprocess.run(cmd, check=True)
    return LIB


def build_cli(force=False):
    host = os.path.join(CSRC, 'host')
    srcs = _sources(host, ('.cpp', '.hpp')) + [LIB]
    if force or _newer(BIN, srcs):
        os.makedirs(os.path.dirname(BIN), exist_ok=True)
        cmd = ['g++', '-std=c++17', '-O2', '-g', '-Wall', '-o', BIN, os.path.join(host, 'cli.cpp'), os.path.join(host, 'hts_io.cpp'),
               '-L' + os.path.dirname(LIB), '-lb200pileup', '-Wl,-rpath,$ORIGIN/../lib', '-lz']
        subprocess.run(cmd, check=True)
    return BIN


def build_compat_client(force=False):
    """tests/compat/plp_dump: a client of the htslib-compatible iterator tier (include/b200_htslib_compat.h)."""
    src = os.path.join(ROOT, 'tests', 'compat', 'plp_dump.cpp')
    exe = os.path.join(ROOT, 'tests', 'compat', '_build', 'plp_dump')
    if force or _newer(exe, [src, LIB, os.path.join(ROOT, 'include', 'b200_htslib_compat.h')]):
        os.makedirs(os.path.dirname(exe), exist_ok=True)
        subprocess.run(['g++', '-std=c++17', '-O2', '-g', '-Wall', '-I', os.path.join(ROOT, 'include'), '-o', exe, src,
                        os.path.join(CSRC, 'host', 'hts_io.cpp'), '-L' + os.path.dirname(LIB), '-lb200pileup',
                        '-Wl,-rpath,$ORIGIN/../../../samtools_b200/lib', '-lz'], check=True)
    return exe


def build_read_ops_client(force=False):
    """tests/compat/read_ops_check: a client of the per-read / per-column htslib entry points (sam_prob_realn, sam_cap_mapq,
    errmod_cal, bcf_call_glfgen) that compares every result with the oracle's restatement in-process (links liboracle.so:
    test infrastructure; the product library does not)."""
    src = os.path.join(ROOT, 'tests', 'compat', 'read_ops_check.cpp')
    exe = os.path.join(ROOT, 'tests', 'compat', '_build', 'read_ops_check')
    ora = os.path.join(ROOT, 'oracle', '_build')
    if force or _newer(exe, [src, LIB, os.path.join(ora, 'liboracle.so'), os.path.join(ROOT, 'include', 'b200_htslib_compat.h')]):
        os.makedirs(os.path.dirname(exe), exist_ok=True)
        subprocess.run(['g++', '-std=c++17', '-O2', '-g', '-Wall', '-I', os.path.join(ROOT, 'include'), '-o', exe, src,
                        '-L' + os.path.dirname(LIB), '-lb200pileup', '-L' + ora, '-loracle',
                        '-Wl,-rpath,$ORIGIN/../../../samtools_b200/lib', '-Wl,-rpath,$ORIGIN/../../../oracle/_build', '-lz', '-lm'], check=True)
    return exe


def build_scan_check(force=False):
    """tests/gpu/scan_check: runs the engine's single-pass scans (csrc/scan.cuh) on inputs the GPU test writes."""
    src = os.path.join(ROOT, 'tests', 'gpu', 'scan_check.cu')
    exe = os.path.join(ROOT, 'tests', 'gpu', '_build', 'scan_check')
    if force or _newer(exe, [src, os.path.join(CSRC, 'scan.cuh')]):
        os.makedirs(os.path.dirname(exe), exist_ok=True)
        nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
        subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-o', exe, src], check=True)
    return exe


def build_oracle():
    subprocess.run(['make', '-s', '-C', os.path.join(ROOT, 'oracle')], check=True)
    subprocess.run(['make', '-s', '-C', os.path.join(ROOT, 'oracle'), 'ref'], check=True)
    return os.path.join(ROOT, 'oracle', '_build', 'plp_oracle')


def build_all(force=False, verbose=False):
    build_engine(force, verbose)
    build_cli(force)
    build_compat_client(force)
    build_scan_check(force)
    build_oracle()
    build_read_ops_client(force)


if __name__ == '__main__':
    build_all(force='--force' in sys.argv, verbose='-v' in sys.argv)
    print('built', LIB, BIN)
