"""Device time of the per-column indel alleles (b200_mpileup_indels) next to the per-column counts (k_mp_counts,
b200_mpileup_counts) on the same staged batch: the benchmark's synthetic window (8 Mb, 30x, 150 bp pairs, 1.5 % of the reads
with an insertion and 1.5 % with a deletion, no FASTA, -Q13), restaged every step with b200_restage so that both calls see a
fresh read stage.  Then one deep column, timed once: --deep reads over one column, each with a random insertion of 1 to 40
symbols (distinct but for the shortest ones).  Prints one JSON line.
  python tools/indels_probe.py [--region-mb 8] [--steps 20] [--warmup 3] [--deep 20000]"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import ctypes as C
from samtools_b200 import engine, synth


def gpu_name_and_power():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().split('\n')[0]
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def deep_column_soa(n, seed=5, L=150):
    """n unpaired reads at position 100, CIGAR 60M <k>I <90-k>M with k = 1 + i % 40 and random symbols: one column (159)
    whose insertions are distinct but for the shortest ones"""
    rng = np.random.default_rng(seed)
    k = 1 + np.arange(n) % 40
    cigar = np.zeros(3 * n, np.uint32)
    cigar[0::3] = (60 << 4) | 0
    cigar[1::3] = (k.astype(np.uint32) << 4) | 1
    cigar[2::3] = ((L - 60 - k).astype(np.uint32) << 4) | 0
    code = rng.choice(np.array([1, 2, 4, 8], np.uint8), size=(n, L))
    seq4 = ((code[:, 0::2] << 4) | code[:, 1::2]).reshape(-1)
    return dict(file_start=np.array([0, n], np.int64), pos=np.full(n, 100, np.int64), flag=np.where(np.arange(n) % 3 == 0, 16, 0).astype(np.uint16),
                mapq=np.full(n, 60, np.uint8), l_qseq=np.full(n, L, np.int32), n_cigar=np.full(n, 3, np.uint32),
                cigar_off=np.arange(0, 3 * n, 3, dtype=np.uint64), qual_off=np.arange(n, dtype=np.uint64) * np.uint64(L),
                mtid=np.full(n, -1, np.int32), mpos=np.full(n, -1, np.int64), isize=np.zeros(n, np.int64), prev_same_name=np.full(n, -1, np.int64),
                rbits=np.zeros(n, np.uint8), cigar=cigar, seq4=np.ascontiguousarray(seq4), qual=np.full(n * L, 40, np.uint8),
                tid=0, tid_len=1000, tid_name='deep', ref=None, ref_beg=0, ref_len=1000)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--region-mb', type=float, default=8.0)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--deep', type=int, default=20000)
    args = ap.parse_args()
    ncols = int(args.region_mb * 1e6)
    soa = synth.make_region(ncols, seed=2, with_ref=True)
    soa = dict(soa); soa['ref'] = None
    e = engine.Engine(0)
    e.set_keep_raw(True)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n, na, nb = C.c_int64(0), C.c_int64(0), C.c_uint64(0)
    ind_ms, cnt_ms = [], []
    for k in range(args.warmup + args.steps):
        e.restage()
        if e.lib.b200_mpileup_indels(e.h, 13, C.byref(na), C.byref(nb)) != 0:
            e._err('b200_mpileup_indels')
        i_ms = e.last_kernel_ms
        if e.lib.b200_mpileup_counts(e.h, 13, None, 0, C.byref(n)) != 0:
            e._err('b200_mpileup_counts')
        if k >= args.warmup:
            ind_ms.append(i_ms); cnt_ms.append(e.last_kernel_ms)
    rows, _ = e.mpileup_indels(13)
    n_events = int(rows['fwd'].sum() + rows['rev'].sum())
    deep = deep_column_soa(args.deep)
    e.set_keep_raw(False)
    e.stage(deep, engine.default_stage_conf(engine.MODE_MPILEUP, max_depth=10 ** 6))
    e.mpileup_indels(13)                     # buffers grown for this shape
    drows, _ = e.mpileup_indels(13)
    deep_ms = e.last_kernel_ms
    e.mpileup_counts(13)                     # the same column through k_mp_counts, for scale
    deep_cnt_ms = e.last_kernel_ms
    e.close()
    print(json.dumps({
        'what': 'b200_mpileup_indels device time (CUDA events, median) vs k_mp_counts (b200_mpileup_counts) on the same batch, -Q13',
        'gpu': gpu_name_and_power(), 'region_mb': args.region_mb, 'steps': args.steps, 'n_cols': n.value,
        'n_alleles': na.value, 'n_events': n_events, 'symbol_bytes': nb.value,
        'indels_ms': round(float(np.median(ind_ms)), 4), 'counts_ms': round(float(np.median(cnt_ms)), 4),
        'deep_column_reads': args.deep, 'deep_column_alleles': int(len(drows)), 'deep_column_ms_once': round(deep_ms, 4),
        'deep_column_counts_ms_once': round(deep_cnt_ms, 4),
    }))


if __name__ == '__main__':
    main()
