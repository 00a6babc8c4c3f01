"""Device time of the per-column quality sums (k_mp_qsums, b200_mpileup_qsums) and of the indel allele sums (k_ind_qsums,
b200_indel_qsums) next to the per-column counts (k_mp_counts, b200_mpileup_counts) on the same staged batch: the benchmark's
synthetic window (8 Mb, 30x, 150 bp pairs, no FASTA, -Q13), restaged every step with b200_restage so that every call sees a
fresh read stage.  Compute only: the planes and rows stay in HBM.  Prints one JSON line with the card and its power limit.
  python tools/qsums_probe.py [--region-mb 8] [--steps 20] [--warmup 3]"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import ctypes as C
from samtools_b200 import engine, synth

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet (700 W)


def gpu_name_and_power():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().split('\n')[0]
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--region-mb', type=float, default=8.0)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    ncols = int(args.region_mb * 1e6)
    soa = synth.make_region(ncols, seed=2, with_ref=True)
    soa = dict(soa); soa['ref'] = None
    e = engine.Engine(0)
    e.set_keep_raw(True)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n, na, nb = C.c_int64(0), C.c_int64(0), C.c_uint64(0)
    cnt_ms, qs_ms, iqs_ms = [], [], []
    for k in range(args.warmup + args.steps):
        e.restage()
        if e.lib.b200_mpileup_counts(e.h, 13, None, 0, C.byref(n)) != 0:
            e._err('b200_mpileup_counts')
        c_ms = e.last_kernel_ms
        if e.lib.b200_mpileup_qsums(e.h, 13, None, 0, C.byref(n)) != 0:
            e._err('b200_mpileup_qsums')
        q_ms = e.last_kernel_ms
        if e.lib.b200_mpileup_indels(e.h, 13, C.byref(na), C.byref(nb)) != 0:
            e._err('b200_mpileup_indels')
        if e.lib.b200_indel_qsums(e.h, None, 0) != 0:
            e._err('b200_indel_qsums')
        if k >= args.warmup:
            cnt_ms.append(c_ms); qs_ms.append(q_ms); iqs_ms.append(e.last_kernel_ms)
    rows, _ = e.mpileup_indels(13)
    n_events = int(rows['fwd'].sum() + rows['rev'].sum())
    e.close()
    ms, cms = float(np.median(qs_ms)), float(np.median(cnt_ms))
    n_files = 1
    bytes_in = synth.algorithmic_bytes_in(soa, overlap=True)
    bytes_alg = bytes_in + 4 * engine.QSUM_PLANES * n_files * n.value
    print(json.dumps({
        'what': 'b200_mpileup_qsums and b200_indel_qsums device time (CUDA events, median, compute only) vs k_mp_counts '
                '(b200_mpileup_counts) on the same batch, -Q13',
        'gpu': gpu_name_and_power(), 'region_mb': args.region_mb, 'steps': args.steps, 'n_cols': n.value,
        'qsums_ms': round(ms, 4), 'counts_ms': round(cms, 4), 'qsums_over_counts': round(ms / cms, 3),
        'qsums_columns_per_s': n.value / (ms * 1e-3), 'qsums_algorithmic_bytes': bytes_alg,
        'qsums_fraction_of_3.35TBps': bytes_alg / (ms * 1e-3) / HBM_BYTES_PER_S,
        'n_alleles': na.value, 'n_events': n_events, 'indel_qsums_ms': round(float(np.median(iqs_ms)), 4),
    }))


if __name__ == '__main__':
    main()
