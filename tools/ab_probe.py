"""A/B timing of engine variants in ONE process launch per variant (development aid; keeps GPU runs short).

  python tools/ab_probe.py [--mb 8] [--reps 5] label[:ENV=V[,ENV=V...]] ...
  e.g.  python tools/ab_probe.py default general:B200_PLP_GENERAL=1 vec:B200_PLP_TMA=0

Each variant runs in its own subprocess (the engine reads its environment at creation) on the bench workload
(synthetic region, 30x, 150 bp, `mpileup -a`, no FASTA) and reports CUDA-event times of the read stage (device
part), the size pass, the tile scan, the write kernel, and a digest of the output so that a variant that changes
the bytes is caught immediately."""
import argparse, hashlib, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child(mb, reps):
    sys.path.insert(0, ROOT)
    import numpy as np
    from samtools_b200 import engine, synth
    soa = synth.make_region(int(mb * 1e6), seed=2)
    soa['ref'] = None
    eng = engine.Engine(0)
    eng.set_keep_raw(True)
    sconf = engine.default_stage_conf(engine.MODE_MPILEUP)
    eng.stage(soa, sconf); eng.stage(soa, sconf)
    text = eng.mpileup_text(all=1)
    st, parts, tot = [], [], []
    for _ in range(reps):
        eng.restage(); st.append(eng.last_stage_device_ms)
        eng.mpileup_text(engine.mpileup_conf(all=1), fetch=False)
        parts.append(eng.last_mpileup_parts_ms); tot.append(eng.last_kernel_ms)
    p = np.median(np.array(parts), axis=0)
    print(json.dumps({'stage_ms': float(np.median(st)), 'size_ms': float(p[0]), 'scan_ms': float(p[1]), 'write_ms': float(p[2]),
                      'column_ms': float(np.median(tot)), 'bytes': len(text), 'sha': hashlib.sha256(text).hexdigest()[:16]}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--mb', type=float, default=8.0)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--child', action='store_true')
    ap.add_argument('specs', nargs='*')
    a = ap.parse_args()
    if a.child:
        return child(a.mb, a.reps)
    rows = []
    for spec in a.specs or ['default']:
        label, _, envs = spec.partition(':')
        env = dict(os.environ)
        for kv in filter(None, envs.split(',')):
            k, _, v = kv.partition('=')
            env[k] = v
        r = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', '--mb', str(a.mb), '--reps', str(a.reps)],
                           env=env, capture_output=True, text=True)
        if r.returncode != 0:
            print(f'{label:24s} FAILED: {r.stderr.strip().splitlines()[-1] if r.stderr.strip() else r.returncode}')
            continue
        j = json.loads(r.stdout.strip().splitlines()[-1])
        rows.append((label, j))
        print(f"{label:24s} stage {j['stage_ms']:6.3f}  size {j['size_ms']:6.3f}  scan {j['scan_ms']:6.3f}  write {j['write_ms']:6.3f}  "
              f"column {j['column_ms']:6.3f} ms   total {j['stage_ms'] + j['column_ms']:6.3f} ms   {a.mb * 1e3 / (j['stage_ms'] + j['column_ms']):8.1f} Mcol/s   sha {j['sha']}",
              flush=True)
    if len({j['sha'] for _, j in rows}) > 1:
        print('WARNING: variants disagree on the output bytes')


if __name__ == '__main__':
    main()
