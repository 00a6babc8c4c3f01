"""A/B timing of engine variants in ONE process launch per variant (development aid; keeps GPU runs short).

  python tools/ab_probe.py [--mb 8] [--reps 5] [--profile] label[:ENV=V[,ENV=V...]] ...
  e.g.  python tools/ab_probe.py default general:B200_PLP_GENERAL=1 direct:B200_PLP_SMEM_TEXT=1024

Each variant runs in its own subprocess (the engine reads its environment at creation) on the bench workload
(synthetic region, 30x, 150 bp, `mpileup -a`, no FASTA) and reports CUDA-event times of the read stage (device
part), the size pass, the tile scan, the write kernel, and a digest of the output so that a variant that changes
the bytes is caught immediately.

--profile  runs one more child per variant under torch.profiler (CUDA activities only) and prints the device time
           of every kernel, memset and copy of one restage + `mpileup_text` step (the median over --reps traced steps),
           so that the parts above can be split by kernel.  Tracing adds host overhead between launches; the per-kernel
           device times are what it is for, not the step total."""
import argparse, hashlib, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def setup(mb):
    sys.path.insert(0, ROOT)
    from samtools_b200 import engine, synth
    soa = synth.make_region(int(mb * 1e6), seed=2)
    soa['ref'] = None
    eng = engine.Engine(0)
    eng.set_keep_raw(True)
    sconf = engine.default_stage_conf(engine.MODE_MPILEUP)
    eng.stage(soa, sconf); eng.stage(soa, sconf)
    return engine, eng


def profile_child(mb, reps):
    """device time per kernel name of one restage + mpileup_text step, median over `reps` traced steps"""
    import numpy as np
    import torch
    from torch.profiler import profile, ProfilerActivity
    engine, eng = setup(mb)
    conf = engine.mpileup_conf(all=1)
    torch.cuda.init()
    for _ in range(2):                                    # warm: module load, first-touch allocations
        eng.restage(); eng.mpileup_text(conf, fetch=False)
    per_step = {}
    for s in range(reps):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.restage(); eng.mpileup_text(conf, fetch=False)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            us = getattr(ev, 'device_time_total', None)
            if us is None:
                us = ev.cuda_time_total
            if us > 0:
                per_step.setdefault(ev.key, [0.0] * reps)[s] += us * 1e-3
    rows = sorted(((k, float(np.median(v))) for k, v in per_step.items()), key=lambda kv: -kv[1])
    print(json.dumps({'kernels_ms': rows}))


def child(mb, reps):
    import numpy as np
    engine, eng = setup(mb)
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
    ap.add_argument('--profile', action='store_true', help='also print the device time per kernel of one step (torch.profiler)')
    ap.add_argument('--child', choices=['time', 'profile'])
    ap.add_argument('specs', nargs='*')
    a = ap.parse_args()
    if a.child == 'time':
        return child(a.mb, a.reps)
    if a.child == 'profile':
        return profile_child(a.mb, a.reps)
    rows = []
    for spec in a.specs or ['default']:
        label, _, envs = spec.partition(':')
        env = dict(os.environ)
        for kv in filter(None, envs.split(',')):
            k, _, v = kv.partition('=')
            env[k] = v
        for kind in ['time'] + (['profile'] if a.profile else []):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', kind, '--mb', str(a.mb), '--reps', str(a.reps)],
                               env=env, capture_output=True, text=True)
            if r.returncode != 0:
                print(f'{label:24s} FAILED: {r.stderr.strip().splitlines()[-1] if r.stderr.strip() else r.returncode}')
                break
            j = json.loads(r.stdout.strip().splitlines()[-1])
            if kind == 'profile':
                for name, ms in j['kernels_ms']:
                    print(f"{'':24s} {ms:7.3f} ms  {name[:100]}")
                continue
            rows.append((label, j))
            print(f"{label:24s} stage {j['stage_ms']:6.3f}  size {j['size_ms']:6.3f}  scan {j['scan_ms']:6.3f}  write {j['write_ms']:6.3f}  "
                  f"column {j['column_ms']:6.3f} ms   total {j['stage_ms'] + j['column_ms']:6.3f} ms   {a.mb * 1e3 / (j['stage_ms'] + j['column_ms']):8.1f} Mcol/s   sha {j['sha']}",
                  flush=True)
    if len({j['sha'] for _, j in rows}) > 1:
        print('WARNING: variants disagree on the output bytes')


if __name__ == '__main__':
    main()
