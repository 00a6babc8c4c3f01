#!/usr/bin/env python3
"""Bundle the reference's own pileup test corpus into tests/golden/ref_corpus.tar.gz.

The reference tree does not travel with this repository, so the golden inputs (small
SAM/BAM/FASTA/BED fixtures) and the expected outputs that pin the hot path
(SURVEY.md section 8c) are packed here, once, by this script:

  test/mpileup/*            (fixtures; CRAM variants dropped - out of scope)
  test/mpileup/expected/*   (159 golden outputs of mpileup.reg / depth.reg)
  test/mpileup/{mpileup,depth}.reg  (the regression tables themselves)
  test/dat/{mpileup.*,sample.sam,view.001.*}   (test.pl mpileup/coverage cases)
  test/coverage/*.expected, test/large_pos/{longref.sam,test.bed,depth*.out}
  test/bedcov/*, examples/{ex1.fa,ex1.sam.gz,toy.*}

Nothing here is reference SOURCE code; these are data files of the
reference's test-suite.  Run:  python tests/golden/make_golden.py <samtools source tree>
"""
import os, tarfile, io, sys, glob

if len(sys.argv) != 2:
    sys.exit('usage: make_golden.py <samtools source tree>')
REF = sys.argv[1]
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'ref_corpus.tar.gz')

def want(path):
    b = os.path.basename(path)
    if b.endswith(('.cram', '.crai')) or b in ('md5', 'cram-size.reg'):
        return False
    return os.path.isfile(path)

files = []
for pat in ['test/mpileup/*', 'test/mpileup/expected/*', 'test/dat/mpileup.*', 'test/dat/sample.sam',
            'test/dat/view.001.*', 'test/coverage/*', 'test/large_pos/longref.sam', 'test/large_pos/test.bed',
            'test/large_pos/depth*.out', 'test/bedcov/*', 'examples/ex1.fa', 'examples/ex1.sam.gz', 'examples/toy.*']:
    files += [p for p in sorted(glob.glob(os.path.join(REF, pat))) if want(p)]

with tarfile.open(OUT, 'w:gz', compresslevel=9) as tf:
    for p in files:
        ti = tf.gettarinfo(p, arcname=os.path.relpath(p, REF))
        ti.mtime = 0; ti.uid = ti.gid = 0; ti.uname = ti.gname = ''; ti.mode = 0o644
        with open(p, 'rb') as fh:
            tf.addfile(ti, fh)
print(f'{len(files)} files -> {OUT} ({os.path.getsize(OUT)/1e6:.2f} MB)')
