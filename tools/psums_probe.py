"""Device time of the per-column read-position sums (k_mp_psums, b200_mpileup_psums) and of the indel allele position sums
(k_ind_psums, b200_indel_psums) next to the per-column counts (k_mp_counts, b200_mpileup_counts) on the same staged batch:
the benchmark's synthetic window (8 Mb, 30x, 150 bp pairs, no FASTA, -Q13), restaged every step with b200_restage so that
every call sees a fresh read stage.  Compute only: the planes and rows stay in HBM.  Prints one JSON line with the card and
its power limit.
  python tools/psums_probe.py [--region-mb 8] [--steps 20] [--warmup 3]"""
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
    soa = dict(soa); soa['ref'] = None
    e = engine.Engine(0)
    e.set_keep_raw(True)
    e.stage(soa, engine.default_stage_conf(engine.MODE_MPILEUP))
    n, na, nb = C.c_int64(0), C.c_int64(0), C.c_uint64(0)
    cnt_ms, ps_ms, ips_ms = [], [], []
    for k in range(args.warmup + args.steps):
        e.restage()
        if e.lib.b200_mpileup_counts(e.h, 13, None, 0, C.byref(n)) != 0:
            e._err('b200_mpileup_counts')
        c_ms = e.last_kernel_ms
        if e.lib.b200_mpileup_psums(e.h, 13, None, 0, C.byref(n)) != 0:
            e._err('b200_mpileup_psums')
        p_ms = e.last_kernel_ms
        if e.lib.b200_mpileup_indels(e.h, 13, C.byref(na), C.byref(nb)) != 0:
            e._err('b200_mpileup_indels')
        if e.lib.b200_indel_psums(e.h, None, 0) != 0:
            e._err('b200_indel_psums')
        if k >= args.warmup:
            cnt_ms.append(c_ms); ps_ms.append(p_ms); ips_ms.append(e.last_kernel_ms)
    rows, _ = e.mpileup_indels(13)
    n_events = int(rows['fwd'].sum() + rows['rev'].sum())
    e.close()
    ms, cms = float(np.median(ps_ms)), float(np.median(cnt_ms))
    n_files = 1
    bytes_in = synth.algorithmic_bytes_in(soa, overlap=True)
    bytes_alg = bytes_in + 8 * engine.PSUM_PLANES * n_files * n.value
    print(json.dumps({
        'what': 'b200_mpileup_psums and b200_indel_psums device time (CUDA events, median, compute only) vs k_mp_counts '
                '(b200_mpileup_counts) on the same batch, -Q13',
        'gpu': gpu_name_and_power(), 'region_mb': args.region_mb, 'steps': args.steps, 'n_cols': n.value,
        'psums_ms': round(ms, 4), 'counts_ms': round(cms, 4), 'psums_over_counts': round(ms / cms, 3),
        'psums_columns_per_s': n.value / (ms * 1e-3), 'psums_algorithmic_bytes': bytes_alg,
        'psums_fraction_of_3.35TBps': bytes_alg / (ms * 1e-3) / HBM_BYTES_PER_S,
        'n_alleles': na.value, 'n_events': n_events, 'indel_psums_ms': round(float(np.median(ips_ms)), 4),
    }))


if __name__ == '__main__':
    main()
