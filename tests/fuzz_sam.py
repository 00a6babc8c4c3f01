"""Random small SAM files full of corner cases, for oracle-vs-engine fuzzing.

SEQ '*' records appear only in seeds divisible by 5; for those seeds the option sets that make the reference
read qualities/bases of a record that has none (depth -q/-J, mpileup -C: undefined behaviour upstream) are skipped.

Reads get arbitrary valid CIGARs (S/H clips, I/D/N/P runs, leading insertions, =/X), duplicate names
(pairs, triplets, supplementary), odd flags, '*' sequences / qualities, mates on other contigs, zero
MAPQ, and start positions that repeat (max-depth rule).  Everything is seeded."""
import random

OPS_REF = 'MDN=X'


def rand_cigar(rng, max_len=40, indel_max=6, n_ops_choices=(1, 1, 1, 2, 3, 4, 6)):
    n_ops = rng.choice(n_ops_choices)
    ops = []
    if rng.random() < 0.15:
        ops.append((rng.randint(1, 5), 'H'))
    if rng.random() < 0.25:
        ops.append((rng.randint(1, 6), 'S'))
    if rng.random() < 0.08:
        ops.append((rng.randint(1, 3), 'I'))          # leading insertion (never reported by the iterator)
    core = []
    for k in range(n_ops):
        if k % 2 == 0:
            core.append((rng.randint(1, max_len), rng.choice('MMMM=X')))
        else:
            op = rng.choice('IDDNPI')
            ln = rng.randint(1, indel_max) if op != 'N' else rng.randint(1, 700)
            core.append((ln, op))
            if rng.random() < 0.2:                    # compound: D after I, P after I, D after D ...
                core.append((rng.randint(1, 3), rng.choice('IDP')))
    if core[-1][1] in 'IDNP' and rng.random() < 0.8:
        core.append((rng.randint(1, 20), 'M'))
    ops += core
    if rng.random() < 0.25:
        ops.append((rng.randint(1, 6), 'S'))
    if rng.random() < 0.1:
        ops.append((rng.randint(1, 5), 'H'))
    if not any(o in 'M=X' for _, o in ops):
        ops.append((rng.randint(1, 10), 'M'))
    return ops


def make_sam(seed, n_reads=60, n_contigs=2, contig_len=1500, with_ref=True, long=False):
    """long: the long-read flavour -- reads up to ~3 kb with many ops and indels up to 40 bases (BAQ bands over several
    32-cell chunks), on 20-kb contigs"""
    rng = random.Random(seed)
    if long:
        contig_len = 20_000
    names = [f'c{i}' for i in range(n_contigs)]
    refs = [''.join(rng.choice('ACGTACGTACGTN' if rng.random() < 0.3 else 'ACGT') for _ in range(contig_len)) for _ in names]
    recs = []
    for i in range(n_reads):
        tid = rng.randrange(n_contigs)
        pos = rng.choice([rng.randint(1, contig_len - 50), rng.randint(1, 60), 100, 100, 101])
        cig = rand_cigar(rng, 400, 40, (3, 5, 9, 13)) if long else rand_cigar(rng)
        qlen = sum(l for l, o in cig if o in 'MIS=X')
        rlen = sum(l for l, o in cig if o in 'MDN=X')
        flag = rng.choice([0, 16, 99, 147, 83, 163, 65, 129, 73, 1, 1024, 256, 512, 2048 + 16, 4, 99, 147])
        name = rng.choice([f'r{i}', f'p{i // 2}', f'p{i // 2}', f't{i // 3}'])
        mapq = rng.choice([0, 1, 20, 30, 60, 60, 60, 255])
        star_seq = seed % 5 == 0 and rng.random() < 0.06
        seq = '*' if star_seq else ''.join(rng.choice('ACGTN' if rng.random() < 0.05 else 'ACGT') for _ in range(qlen))
        if not star_seq and with_ref and rng.random() < 0.7:   # mostly agree with the reference
            s, q, r = list(seq), 0, pos - 1
            for l, o in cig:
                if o in 'M=X':
                    for k in range(l):
                        if r + k < contig_len and rng.random() < 0.9:
                            s[q + k] = refs[tid][r + k]
                    q += l; r += l
                elif o in 'IS':
                    q += l
                elif o in 'DN':
                    r += l
            seq = ''.join(s)
        if star_seq or rng.random() < 0.05:
            qual = '*'
        else:
            qual = ''.join(chr(33 + rng.choice([0, 2, 12, 13, 14, 20, 30, 37, 40, 41, 60, 93])) for _ in range(qlen))
        mate = rng.choice(['=', '=', '=', '*', names[(tid + 1) % n_contigs]])
        mpos = 0 if mate == '*' else rng.choice([pos, max(1, pos + rng.randint(-40, 80)), rng.randint(1, contig_len)])
        tlen = rng.choice([0, rlen, rng.randint(-300, 300)])
        tags = []
        if rng.random() < 0.3:
            tags.append('RG:Z:' + rng.choice(['g1', 'g2']))
        if rng.random() < 0.2:
            tags.append(f'NM:i:{rng.randint(0, 5)}')
        recs.append((tid, pos, i, '\t'.join([name, str(flag), names[tid], str(pos), str(mapq),
                                             ''.join(f'{l}{o}' for l, o in cig), mate, str(mpos), str(tlen), seq, qual] + tags)))
    recs.sort(key=lambda r: (r[0], r[1], r[2]))
    hdr = ['@HD\tVN:1.6\tSO:coordinate'] + [f'@SQ\tSN:{n}\tLN:{contig_len}' for n in names] + ['@RG\tID:g1\tSM:s1', '@RG\tID:g2\tSM:s2']
    sam = '\n'.join(hdr + [r[3] for r in recs]) + '\n'
    fa = ''.join(f'>{n}\n' + '\n'.join(r[i:i + 60] for i in range(0, len(r), 60)) + '\n' for n, r in zip(names, refs))
    return sam, fa


MPILEUP_OPTS = [
    '-B', '-B -x', '-B -Q 0', '-B -Q 0 -x -A', '-B -a', '-B -aa -Q 0', '-B -q 20 -Q 14', '-B -d 3 -x', '-B -d 2', '-B -s -O --output-BP-5 -Q 0',
    '-B --reverse-del --no-output-ends -Q 0', '-B --no-output-ins --no-output-del', '-B --no-output-ins --no-output-ins --no-output-del --no-output-del',
    '-B --rf 0x10', '-B --ff 0x400 -A', '-B -r c0:50-400', '-B -aa -r c1:90-130', '-B -a -r c0:100-101', '-B -6 -Q 0', '-B -l {bed}', '-B -a -l {bed}',
    '-B -G {rg}', '-B -R', '-B -C 50', '', '-E', '-x', '-a -Q 0', '-6 -A', '-r c1:1-200 -A -Q 5',
    '-B --output-QNAME -a', "-B -s -O --output-extra FLAG,QNAME,RG,NM,POS,MAPQ,RNEXT,PNEXT,RLEN,RNAME --output-sep ';' --output-empty -",
]
DEPTH_OPTS = ['', '-a', '-aa', '-J', '-q 13', '-Q 20 -l 10', '-s', '-s -J -q 14', '-g 0x400', '-G 16', '--incl-flags 0x40', '--require-flags 0x3',
              '-r c0:50-400', '-a -r c1:1-100', '-b {bed}', '-aa -b {bed}', '-H']
COVERAGE_OPTS = ['', '-q 20', '-Q 13', '--min-depth 2', '-l 20', '--ff 0', '--rf 0x10', '-r c0:50-400', '-r c1', '-H']
# bedcov over x.bed (bedcov.c): -j / -d / -c / flag filters / header
BEDCOV_OPTS = ['', '-j', '-d 2', '-c', '-H -d 1 -c', '-Q 20', '-g 0x400 -G 0x10', '-j -d 0']
# genotype likelihoods (bcf_call_glfgen + errmod_cal per column and file); CUDA path only: the emulation harness has no GL
GL_OPTS = ['-B', '-B -Q 0', '-B -x -A', '-B -q 20', '-B -r c0:50-400', '-B -6 -Q 0', '']
