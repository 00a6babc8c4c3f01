"""samtools_b200 -- CUDA (sm_90a) mpileup / depth / coverage engine.

The product is the CUDA library samtools_b200/lib/libb200pileup.so (C ABI in
include/b200_pileup.h) and the CLI samtools_b200/bin/b200samtools.  This Python
package only binds the C ABI (engine.py), generates the seeded synthetic
workloads (synth.py) and builds the native pieces (build.py).
"""
from . import engine, synth  # noqa: F401

__all__ = ['engine', 'synth']
