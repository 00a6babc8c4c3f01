"""Device time of the per-column counts (b200_mpileup_counts) next to the pileup text's column stage (b200_mpileup_text) on
the same staged batch: the benchmark's synthetic window (8 Mb, 30x, 150 bp pairs, no FASTA, -Q13), restaged every step with
b200_restage so that both calls see a fresh read stage.  Prints one JSON line.
  python tools/counts_probe.py [--region-mb 8] [--steps 20] [--warmup 3]"""
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
    n = C.c_int64(0)
    cnt_ms, txt_ms = [], []
    for k in range(args.warmup + args.steps):
        e.restage()
        if e.lib.b200_mpileup_counts(e.h, 13, None, 0, C.byref(n)) != 0:
            e._err('b200_mpileup_counts')
        c_ms = e.last_kernel_ms
        e.mpileup_text(all=1, fetch=False)
        if k >= args.warmup:
            cnt_ms.append(c_ms); txt_ms.append(e.last_kernel_ms)
    e.close()
    ms, text_ms = float(np.median(cnt_ms)), float(np.median(txt_ms))
    n_files = 1
    bytes_alg = synth.algorithmic_bytes_in(soa, overlap=True) + 4 * engine.COUNT_PLANES * n_files * n.value
    print(json.dumps({
        'what': 'b200_mpileup_counts device time (CUDA events, median), -Q13, vs the b200_mpileup_text column stage (-a) on the same batch',
        'gpu': gpu_name_and_power(), 'region_mb': args.region_mb, 'steps': args.steps, 'n_cols': n.value,
        'counts_ms': round(ms, 4), 'text_column_stage_ms': round(text_ms, 4),
        'counts_columns_per_s': n.value / (ms * 1e-3), 'algorithmic_bytes': bytes_alg,
        'counts_bytes_per_s': bytes_alg / (ms * 1e-3), 'fraction_of_3.35TBps': bytes_alg / (ms * 1e-3) / HBM_BYTES_PER_S,
    }))


if __name__ == '__main__':
    main()
