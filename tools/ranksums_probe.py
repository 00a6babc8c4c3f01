"""Device time of the per-column rank sums (b200_mpileup_ranksums: k_rank_counts, the scan and list of active pairs,
k_rank_hist) next to the per-column counts (k_mp_counts, b200_mpileup_counts) on the same staged batch: the benchmark's
synthetic window (8 Mb, 30x, 150 bp pairs, -Q13), restaged every step with b200_restage so that every call sees a fresh read
stage.  The window keeps its reference: without one no base is of the ref class and no (file, column) pair would be
active.  Compute only, then one call into host memory for the fraction of active pairs.  Prints one JSON line with the card
and its power limit.
  python tools/ranksums_probe.py [--region-mb 8] [--steps 20] [--warmup 3]"""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import ctypes as C
from samtools_b200 import engine, synth
from qsums_probe import HBM_BYTES_PER_S, gpu_name_and_power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--region-mb', type=float, default=8.0)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    ncols = int(args.region_mb * 1e6)
    soa = synth.make_region(ncols, seed=2, with_ref=True)
    e = engine.Engine(0)
    e.set_keep_raw(True)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n = C.c_int64(0)
    cnt_ms, rs_ms = [], []
    for k in range(args.warmup + args.steps):
        e.restage()
        if e.lib.b200_mpileup_counts(e.h, 13, None, 0, C.byref(n)) != 0:
            e._err('b200_mpileup_counts')
        c_ms = e.last_kernel_ms
        if e.lib.b200_mpileup_ranksums(e.h, 13, None, 0, C.byref(n)) != 0:
            e._err('b200_mpileup_ranksums')
        if k >= args.warmup:
            cnt_ms.append(c_ms); rs_ms.append(e.last_kernel_ms)
    planes = e.mpileup_ranksums(13)
    e.close()
    active = float(((planes[:, 0] > 0) & (planes[:, 1] > 0)).mean())
    ms, cms = float(np.median(rs_ms)), float(np.median(cnt_ms))
    bytes_alg = synth.algorithmic_bytes_in(soa, overlap=True) + 8 * engine.RANK_PLANES * n.value
    print(json.dumps({
        'what': 'b200_mpileup_ranksums device time (CUDA events, median, compute only) vs k_mp_counts (b200_mpileup_counts) '
                'on the same batch, -Q13, with the reference',
        'gpu': gpu_name_and_power(), 'region_mb': args.region_mb, 'steps': args.steps, 'n_cols': n.value,
        'ranksums_ms': round(ms, 4), 'ranksums_ms_min_max': [round(min(rs_ms), 4), round(max(rs_ms), 4)],
        'counts_ms': round(cms, 4), 'ranksums_over_counts': round(ms / cms, 3), 'active_fraction': round(active, 4),
        'ranksums_columns_per_s': n.value / (ms * 1e-3), 'ranksums_algorithmic_bytes': bytes_alg,
        'ranksums_fraction_of_3.35TBps': bytes_alg / (ms * 1e-3) / HBM_BYTES_PER_S,
    }))


if __name__ == '__main__':
    main()
