"""Region reads with and without a BAI: `mpileup -a -B -r <region>` and `bedcov` of many intervals through the CUDA CLI
on an indexed multi-contig synthetic BAM of a few GB.  With the index only the blocks holding the region's records are
inflated, so that time should follow the region; without it the reader decodes the whole file.  Both outputs of each
command are checked to be identical.  Prints one JSON line (the card and its power limit included).

  python tools/index_timing.py [--contigs 4] [--contig-mb 12] [--depth 30] [--region-mb 1] [--intervals 1000] [--out f.json]

The BAM and its index go to a temporary directory that is removed at the end."""
import argparse, hashlib, json, os, struct, subprocess, sys, tempfile, time, zlib
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from samtools_b200 import synth


class BgzfWriter:
    def __init__(self, path, level=1):
        self.f, self.level, self.buf = open(path, 'wb'), level, bytearray()

    def write(self, data):
        self.buf += data
        while len(self.buf) >= 0xff00:
            self._block(bytes(self.buf[:0xff00])); del self.buf[:0xff00]

    def _block(self, chunk):
        c = zlib.compressobj(self.level, zlib.DEFLATED, -15)
        comp = c.compress(chunk) + c.flush()
        self.f.write(b'\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0' + struct.pack('<H', len(comp) + 25) + comp +
                     struct.pack('<II', zlib.crc32(chunk) & 0xffffffff, len(chunk)))

    def close(self):
        if self.buf:
            self._block(bytes(self.buf))
        self.f.write(bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000'))
        self.f.close()


def records_of(soa, td):
    """the BAM records of one contig, as synth.write_bam encodes them (its header stripped)"""
    p = os.path.join(td, 'one.bam')
    synth.write_bam(p, soa)
    import gzip
    raw = gzip.open(p).read()
    os.remove(p)
    (lt,) = struct.unpack_from('<i', raw, 4); o = 8 + lt
    (n,) = struct.unpack_from('<i', raw, o); o += 4
    for _ in range(n):
        (ln,) = struct.unpack_from('<i', raw, o); o += 8 + ln
    return raw[o:]


def write_multi(path, td, n_contigs, length, depth):
    names = [f'chr{i + 1}' for i in range(n_contigs)]
    text = ('@HD\tVN:1.6\tSO:coordinate\n' + ''.join(f'@SQ\tSN:{n}\tLN:{length}\n' for n in names)).encode()
    w = BgzfWriter(path)
    w.write(b'BAM\1' + struct.pack('<i', len(text)) + text + struct.pack('<i', n_contigs) +
            b''.join(struct.pack('<i', len(n) + 1) + n.encode() + b'\0' + struct.pack('<i', length) for n in names))
    n_reads = 0
    for t, n in enumerate(names):
        soa = synth.make_region(length, depth=depth, seed=7 + t, tid_name=n)
        soa['tid'] = t
        soa['mtid'] = np.full(len(soa['pos']), t, dtype=np.int32)
        n_reads += len(soa['pos'])
        w.write(records_of(soa, td))
    w.close()
    return names, n_reads


def timed(args, out_path):
    t0 = time.perf_counter()
    with open(out_path, 'wb') as f:
        subprocess.run(args, stdout=f, check=True)
    dt = time.perf_counter() - t0
    return dt, hashlib.sha256(open(out_path, 'rb').read()).hexdigest(), os.path.getsize(out_path)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, check=True).stdout.strip()
        return q
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--contigs', type=int, default=4)
    ap.add_argument('--contig-mb', type=float, default=12)
    ap.add_argument('--depth', type=int, default=30)
    ap.add_argument('--region-mb', type=float, default=1)
    ap.add_argument('--intervals', type=int, default=1000)
    ap.add_argument('--out')
    a = ap.parse_args()
    cli = os.environ.get('B200_TEST_CLI') or os.path.join(ROOT, 'samtools_b200', 'bin', 'b200samtools')
    length = int(a.contig_mb * 1e6)
    res = {'card': card(), 'contigs': a.contigs, 'contig_bp': length, 'depth': a.depth}
    with tempfile.TemporaryDirectory() as td:
        idx_dir, scan_dir = os.path.join(td, 'indexed'), os.path.join(td, 'scan')
        os.makedirs(idx_dir); os.makedirs(scan_dir)
        bam = os.path.join(idx_dir, 'big.bam')
        t0 = time.perf_counter()
        names, n_reads = write_multi(bam, td, a.contigs, length, a.depth)
        res.update(reads=n_reads, bam_bytes=os.path.getsize(bam), generate_s=time.perf_counter() - t0)
        os.symlink(bam, os.path.join(scan_dir, 'big.bam'))          # the same file without an index next to it
        t0 = time.perf_counter()
        subprocess.run([cli, 'index', bam], check=True)
        res['index_s'] = time.perf_counter() - t0
        mid = names[len(names) // 2]
        beg = length // 2
        reg = f'{mid}:{beg + 1}-{beg + int(a.region_mb * 1e6)}'
        rng = np.random.default_rng(1)
        bed = os.path.join(td, 'x.bed')
        with open(bed, 'w') as f:
            for _ in range(a.intervals):
                s = int(rng.integers(0, length - 1000))
                f.write(f'{names[int(rng.integers(0, len(names)))]}\t{s}\t{s + 1000}\n')
        for name, cmd in (('mpileup', ['mpileup', '-a', '-B', '-r', reg]), ('bedcov', ['bedcov', bed])):
            t_i, h_i, n_i = timed([cli] + cmd + [bam], os.path.join(td, 'o1'))
            t_s, h_s, n_s = timed([cli] + cmd + [os.path.join(scan_dir, 'big.bam')], os.path.join(td, 'o2'))
            if h_i != h_s:
                raise SystemExit(f'{name}: the indexed and the scanned outputs differ')
            res[name] = {'args': ' '.join(cmd[:-1] + ([reg] if name == 'mpileup' else [f'<{a.intervals} x 1 kb>'])),
                         'indexed_s': t_i, 'scan_s': t_s, 'speedup': t_s / t_i, 'output_bytes': n_i}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
