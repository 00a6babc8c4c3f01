"""ctypes binding of the C ABI in include/b200_pileup.h (the CUDA engine).

This is the reference-side binding a maintainer would add around the batch
tier (see INTEGRATION.md).  It mirrors the C structs field by field; numpy
arrays are passed as plain pointers.  There is no fallback of any kind: if the
shared library is missing or no CUDA device is present the call raises.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libb200pileup.so')

MODE_MPILEUP, MODE_DEPTH, MODE_COVERAGE = 0, 1, 2
RB_HOST_SKIP, RB_NAME_ODD, RB_BAQ_DONE = 1, 2, 4
POS_MAX = (0x7fffffff << 32) | 0xffffffff

EXPORTS = ['b200_engine_create', 'b200_engine_destroy', 'b200_last_error', 'b200_version', 'b200_stage',
           'b200_mpileup_text', 'b200_depth_text', 'b200_coverage', 'b200_coverage_hist', 'b200_glf', 'b200_fetch_qual',
           'b200_fetch_mapq_keep', 'b200_pileup_entries', 'b200_last_kernel_ms', 'b200_last_stage_ms', 'b200_set_keep_raw', 'b200_restage', 'b200_last_stage_device_ms',
           'b200_launch_count', 'b200_last_mpileup_parts_ms', 'b200_gl_rng_draws', 'b200_last_baq_ms',
           'b200_errmod_cal', 'b200_glfgen', 'b200_cap_mapq', 'b200_mpileup_text_bound', 'b200_depth_text_bound', 'b200_bedcov',
           'b200_mpileup_counts', 'b200_mpileup_indels', 'b200_fetch_indels', 'b200_mpileup_qsums', 'b200_indel_qsums',
           'b200_mpileup_psums', 'b200_indel_psums', 'b200_mpileup_ranksums']
COUNT_PLANES = 19   # b200_mpileup_counts: per file A C G T N del skip +ins -del, forward then reverse strand, then n_plp
QSUM_PLANES = 42    # b200_mpileup_qsums: per file BQ sums, MQ sums, MQ0 counts, each of A C G T N del skip, forward then reverse
# b200_indel_qsum_t, one row of b200_indel_qsums beside the row of b200_mpileup_indels
INDEL_QSUM_FIELDS = ('bq_fwd', 'bq_rev', 'mq_fwd', 'mq_rev', 'mq0_fwd', 'mq0_rev')
PSUM_PLANES = 28    # b200_mpileup_psums: per file BP-5 sums, sums of BP-5 squared, each of A C G T N del skip, forward then reverse
RANK_PLANES = 8     # b200_mpileup_ranksums: per file n_ref, n_alt, then U2 and T of BQ, of MQ and of BP-5 (capped at 1024)


class IndelPsum(C.Structure):
    """b200_indel_psum_t, one row of b200_indel_psums beside the row of b200_mpileup_indels"""
    _fields_ = [('bp5_fwd', C.c_int64), ('bp5_rev', C.c_int64), ('bp5sq_fwd', C.c_int64), ('bp5sq_rev', C.c_int64)]


INDEL_PSUM_FIELDS = tuple(f for f, _ in IndelPsum._fields_)
# b200_indel_t, one row of b200_mpileup_indels: len >= 0 an insertion of len symbols at seq[seq_off:], < 0 a deletion of -len
INDEL_DTYPE = np.dtype([('col', '<i4'), ('file', '<i4'), ('len', '<i4'), ('fwd', '<u4'), ('rev', '<u4'), ('pad', '<u4'),
                        ('seq_off', '<u8')])


class Batch(C.Structure):
    _fields_ = [('n_files', C.c_int32), ('n_reads', C.c_int64), ('file_start', C.c_void_p),
                ('pos', C.c_void_p), ('flag', C.c_void_p), ('mapq', C.c_void_p), ('l_qseq', C.c_void_p),
                ('n_cigar', C.c_void_p), ('cigar_off', C.c_void_p), ('qual_off', C.c_void_p), ('mtid', C.c_void_p),
                ('mpos', C.c_void_p), ('isize', C.c_void_p), ('prev_same_name', C.c_void_p), ('rbits', C.c_void_p), ('depth_clip', C.c_void_p),
                ('cigar', C.c_void_p), ('n_cigar_total', C.c_uint64), ('seq4', C.c_void_p), ('qual', C.c_void_p),
                ('qual_bytes', C.c_uint64), ('tid', C.c_int32), ('tid_len', C.c_int64), ('tid_name', C.c_char_p),
                ('ref', C.c_void_p), ('ref_beg', C.c_int64), ('ref_n', C.c_int64), ('ref_len', C.c_int64)]


class StageConf(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ('mode', 'rflag_require', 'rflag_filter', 'min_mq', 'no_orphan', 'illumina13', 'baq',
                                          'capq_thres', 'overlaps', 'max_depth', 'd_flag_excl', 'd_flag_incl', 'd_flag_require',
                                          'd_min_mapq', 'd_min_len', 'd_remove_overlaps', 'c_min_len')] + \
               [('beg', C.c_int64), ('end', C.c_int64)]


class StageStats(C.Structure):
    _fields_ = [('n_kept', C.c_int64), ('n_kept_in_window', C.c_int64), ('out_bound', C.c_uint64), ('n_cols', C.c_int64),
                ('n_reads', C.c_uint64), ('n_selected_reads', C.c_uint64), ('summed_mapq', C.c_uint64)]


class MpileupConf(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ('min_baseQ', 'all', 'rev_del', 'no_ins', 'no_del', 'no_ends', 'out_mapq', 'out_qpos',
                                          'out_qpos5', 'n_star_cols')] + \
               [('bed_beg', C.c_void_p), ('bed_end', C.c_void_p), ('n_bed', C.c_int32), ('bed_active', C.c_int32)] + \
               [('n_x', C.c_int32), ('x_off', C.c_void_p), ('x_dat', C.c_void_p), ('x_bytes', C.c_uint64), ('x_sep', C.c_char * 16)]


class DepthConf(C.Structure):
    _fields_ = [('min_qual', C.c_int32), ('count_del', C.c_int32), ('all', C.c_int32),
                ('bed_beg', C.c_void_p), ('bed_end', C.c_void_p), ('n_bed', C.c_int32), ('bed_active', C.c_int32)]


class CoverageConf(C.Structure):
    _fields_ = [('min_baseQ', C.c_int32), ('min_depth', C.c_int32)]


class CoverageSums(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ('n_covered_bases', 'summed_coverage', 'summed_baseQ', 'quality_bases', 'missing_qual')]


class Pileup1(C.Structure):
    _fields_ = [('read', C.c_int64), ('qpos', C.c_int32), ('indel', C.c_int32), ('cigar_ind', C.c_int32), ('bits', C.c_uint32)]


_lib = None


def load_library():
    """Load libb200pileup.so; raises (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f'{LIB_PATH} is missing: build it with `python samtools_b200/build.py` '
                               '(there is no CPU fallback for the pileup engine)')
        lib = C.CDLL(LIB_PATH)
        lib.b200_engine_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        lib.b200_engine_destroy.argtypes = [C.c_void_p]
        lib.b200_last_error.argtypes = [C.c_void_p]; lib.b200_last_error.restype = C.c_char_p
        lib.b200_version.restype = C.c_char_p
        lib.b200_stage.argtypes = [C.c_void_p, C.POINTER(Batch), C.POINTER(StageConf), C.POINTER(StageStats)]
        lib.b200_mpileup_text.argtypes = [C.c_void_p, C.POINTER(MpileupConf), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        lib.b200_depth_text.argtypes = [C.c_void_p, C.POINTER(DepthConf), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        lib.b200_coverage.argtypes = [C.c_void_p, C.POINTER(CoverageConf), C.POINTER(CoverageSums)]
        lib.b200_glf.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int64), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        lib.b200_mpileup_counts.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64)]
        lib.b200_mpileup_indels.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]
        lib.b200_fetch_indels.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        lib.b200_mpileup_qsums.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64)]
        lib.b200_indel_qsums.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        lib.b200_mpileup_psums.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64)]
        lib.b200_indel_psums.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        lib.b200_mpileup_ranksums.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64)]
        lib.b200_fetch_qual.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        lib.b200_fetch_mapq_keep.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        lib.b200_pileup_entries.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        lib.b200_last_kernel_ms.argtypes = [C.c_void_p]; lib.b200_last_kernel_ms.restype = C.c_double
        lib.b200_last_stage_ms.argtypes = [C.c_void_p]; lib.b200_last_stage_ms.restype = C.c_double
        lib.b200_last_stage_device_ms.argtypes = [C.c_void_p]; lib.b200_last_stage_device_ms.restype = C.c_double
        lib.b200_set_keep_raw.argtypes = [C.c_void_p, C.c_int]; lib.b200_set_keep_raw.restype = C.c_int
        lib.b200_restage.argtypes = [C.c_void_p, C.c_void_p]; lib.b200_restage.restype = C.c_int
        lib.b200_launch_count.argtypes = [C.c_void_p]; lib.b200_launch_count.restype = C.c_int64
        lib.b200_last_mpileup_parts_ms.argtypes = [C.c_void_p, C.POINTER(C.c_double * 3)]
        lib.b200_last_baq_ms.argtypes = [C.c_void_p]; lib.b200_last_baq_ms.restype = C.c_double
        lib.b200_gl_rng_draws.argtypes = [C.c_void_p]; lib.b200_gl_rng_draws.restype = C.c_uint64
        _lib = lib
    return _lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def default_stage_conf(mode=MODE_MPILEUP, **kw):
    """Defaults of the reference CLIs (bam_plcmd.c:1083-1093, bam2depth.c:740-754, coverage.c:311-330)."""
    c = StageConf()
    c.mode = mode
    c.rflag_filter = 4 | 256 | 512 | 1024
    c.no_orphan = 1
    c.overlaps = 1
    c.baq = 1
    c.max_depth = 8000 if mode == MODE_MPILEUP else 1000000
    c.d_flag_excl = 4 | 256 | 1024 | 512
    c.beg, c.end = 0, POS_MAX
    for k, v in kw.items():
        if not hasattr(c, k):
            raise AttributeError(k)
        setattr(c, k, v)
    return c


def ranksum_z(planes):
    """z-scores of the rank-sum planes of Engine.mpileup_ranksums (numpy or torch int64, [..., 8, n]): float64 [..., 3, n]
    for BQ, MQ and the BP-5, of the same kind and on the same device.  With n1 = n_ref, n2 = n_alt, N = n1 + n2 and per
    value U = U2 / 2, mu = n1 n2 / 2 and sigma^2 = n1 n2 / 12 ((N + 1) - T / (N (N - 1))) (the tie-corrected normal
    approximation, no continuity correction), z = (U - mu) / sigma: positive where the non-reference bases have the larger
    values.  NaN where a class is empty or sigma = 0 (every entry of the column has the same value)."""
    import sys
    torch = sys.modules.get('torch')
    is_t = torch is not None and isinstance(planes, torch.Tensor)
    f64 = (lambda a: a.to(torch.float64)) if is_t else (lambda a: np.asarray(a).astype(np.float64))
    n1, n2 = planes[..., 0:1, :], planes[..., 1:2, :]
    u2, t = planes[..., 2::2, :], planes[..., 3::2, :]
    n = n1 + n2
    num = (n + 1) * n * (n - 1) - t                # 12 N (N - 1) sigma^2 / (n1 n2), exact in int64
    ok = (n1 > 0) & (n2 > 0) & (num > 0)
    with np.errstate(divide='ignore', invalid='ignore'):
        var = f64(n1) * f64(n2) * f64(num) / (12.0 * f64(n) * f64(n - 1))
        z = (f64(u2) / 2 - f64(n1) * f64(n2) / 2) / (var.sqrt() if is_t else np.sqrt(var))
    return z.masked_fill(~ok, float('nan')) if is_t else np.where(ok, z, np.nan)


class Engine:
    """One engine handle = one CUDA device + stream (not thread-safe)."""

    def __init__(self, device=0):
        self.lib = load_library()
        h = C.c_void_p()
        if self.lib.b200_engine_create(device, C.byref(h)) != 0:
            raise RuntimeError('b200_engine_create failed: no usable CUDA device (the engine has no CPU fallback)')
        self.h = h
        self.device = device
        self._keep = None
        self._n_files = self._n_cols = 0
        self._n_alleles = 0   # rows of the last mpileup_indels on the staged batch

    def close(self):
        if self.h:
            self.lib.b200_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self, what):
        raise RuntimeError(f'{what}: {self.lib.b200_last_error(self.h).decode()}')

    def stage(self, soa, conf):
        """soa: dict of numpy arrays with the b200_batch_t fields (see synth.make_batch)."""
        b = Batch()
        b.n_files = len(soa['file_start']) - 1
        b.n_reads = len(soa['pos'])
        for k in ('file_start', 'pos', 'flag', 'mapq', 'l_qseq', 'n_cigar', 'cigar_off', 'qual_off', 'mtid', 'mpos', 'isize',
                  'prev_same_name', 'rbits', 'depth_clip', 'cigar', 'seq4', 'qual'):
            setattr(b, k, _ptr(soa.get(k)))
        b.n_cigar_total = len(soa['cigar'])
        b.qual_bytes = len(soa['qual'])
        b.tid = int(soa.get('tid', 0)); b.tid_len = int(soa['tid_len'])
        name = soa['tid_name'].encode()
        b.tid_name = name
        ref = soa.get('ref')
        b.ref = _ptr(ref); b.ref_beg = int(soa.get('ref_beg', 0)); b.ref_n = 0 if ref is None else len(ref)
        b.ref_len = 0 if ref is None else int(soa.get('ref_len', len(ref)))
        st = StageStats()
        self._keep = (soa, name)
        self._n_files = b.n_files
        self._n_alleles = 0
        if self.lib.b200_stage(self.h, C.byref(b), C.byref(conf), C.byref(st)) != 0:
            self._err('b200_stage')
        self._n_cols = st.n_cols
        return st

    def set_keep_raw(self, on=True):
        """keep pristine qualities / mapq resident so that restage() can repeat the device side of the read stage"""
        if self.lib.b200_set_keep_raw(self.h, 1 if on else 0) != 0:
            self._err('b200_set_keep_raw')

    def restage(self):
        st = StageStats()
        self._n_alleles = 0
        if self.lib.b200_restage(self.h, C.byref(st)) != 0:
            self._err('b200_restage')
        self._n_cols = st.n_cols
        return st

    def _text(self, fn, conf, out=None, fetch=True):
        n = C.c_size_t(0)
        if not fetch:
            if fn(self.h, C.byref(conf), None, 0, C.byref(n)) != 0:
                self._err('column stage')
            return n.value
        if out is None:
            if fn(self.h, C.byref(conf), None, 0, C.byref(n)) != 0:
                self._err('column stage')
            out = np.empty(n.value + 1, dtype=np.uint8)
        if fn(self.h, C.byref(conf), _ptr(out), out.nbytes, C.byref(n)) != 0:
            self._err('column stage')
        return out[:n.value].tobytes()

    def mpileup_text(self, conf=None, out=None, fetch=True, **kw):
        conf = conf or mpileup_conf(**kw)
        return self._text(self.lib.b200_mpileup_text, conf, out, fetch)

    def depth_text(self, conf=None, out=None, fetch=True, **kw):
        if conf is None:
            conf = DepthConf()
            for k, v in kw.items():
                setattr(conf, k, v)
        return self._text(self.lib.b200_depth_text, conf, out, fetch)

    def coverage(self, min_baseQ=0, min_depth=1):
        c = CoverageConf(min_baseQ, min_depth); s = CoverageSums()
        if self.lib.b200_coverage(self.h, C.byref(c), C.byref(s)) != 0:
            self._err('b200_coverage')
        return {k: getattr(s, k) for k, _ in CoverageSums._fields_}

    def glf(self, min_baseQ, cap_cols, n_files=1, fetch=True):
        n = C.c_int64(0)
        if not fetch:     # compute only; the likelihoods stay in HBM
            if self.lib.b200_glf(self.h, min_baseQ, C.byref(n), None, None, None, None, 0) != 0:
                self._err('b200_glf')
            return n.value
        pos = np.zeros(cap_cols, np.int64); nb = np.zeros(cap_cols * n_files, np.int32)
        qs = np.zeros(cap_cols * n_files * 4, np.float32); p25 = np.zeros(cap_cols * n_files * 25, np.float32)
        if self.lib.b200_glf(self.h, min_baseQ, C.byref(n), _ptr(pos), _ptr(nb), _ptr(qs), _ptr(p25), cap_cols) != 0:
            self._err('b200_glf')
        k = n.value
        return pos[:k], nb[:k * n_files].reshape(k, n_files), qs[:k * n_files * 4].reshape(k, n_files, 4), p25[:k * n_files * 25].reshape(k, n_files, 25)

    def _planes(self, fn, planes, min_baseQ, out, np_dtype=np.uint32, torch_dtype='int32'):
        n = C.c_int64(0)
        shape = (self._n_files, planes, self._n_cols)     # the stage's n_cols are the columns of the planes
        if out is None:
            a = np.zeros(shape, np_dtype)
            if getattr(self.lib, fn)(self.h, min_baseQ, _ptr(a), shape[2], C.byref(n)) != 0:
                self._err(fn)
            return a
        import torch
        if out.dtype != getattr(torch, torch_dtype) or not out.is_cuda or not out.is_contiguous() or out.device.index != self.device:
            raise ValueError(f'out must be a contiguous torch.{torch_dtype} tensor on cuda:{self.device}')
        if tuple(out.shape) != shape:
            raise ValueError(f'out must have shape {list(shape)}')
        torch.cuda.current_stream(out.device).synchronize()   # the engine writes on its own stream
        if getattr(self.lib, fn)(self.h, min_baseQ, C.c_void_p(out.data_ptr()), shape[2], C.byref(n)) != 0:
            self._err(fn)
        return out

    def mpileup_counts(self, min_baseQ=13, out=None):
        """Per-column strand-split base and indel counts of the staged window (b200_mpileup_counts): a numpy uint32
        [n_files, 19, n] array, or, given `out`, a contiguous torch.int32 CUDA tensor of that shape on the handle's device,
        filled in place on the device (and returned)."""
        return self._planes('b200_mpileup_counts', COUNT_PLANES, min_baseQ, out)

    def mpileup_qsums(self, min_baseQ=13, out=None):
        """Per-column quality sums of the staged window (b200_mpileup_qsums): a numpy uint32 [n_files, 42, n] array of BQ
        sums, MQ sums and MQ0 counts (plane s * 14 + strand * 7 + kind), or, given `out`, a contiguous torch.int32 CUDA
        tensor of that shape on the handle's device, filled in place on the device (and returned)."""
        return self._planes('b200_mpileup_qsums', QSUM_PLANES, min_baseQ, out)

    def mpileup_psums(self, min_baseQ=13, out=None):
        """Per-column read-position sums of the staged window (b200_mpileup_psums): a numpy int64 [n_files, 28, n] array of
        BP-5 sums and sums of BP-5 squared (plane s * 14 + strand * 7 + kind), or, given `out`, a contiguous torch.int64 CUDA
        tensor of that shape on the handle's device, filled in place on the device (and returned)."""
        return self._planes('b200_mpileup_psums', PSUM_PLANES, min_baseQ, out, np.int64, 'int64')

    def mpileup_ranksums(self, min_baseQ=13, out=None):
        """Per-column rank-sum bias statistics of the staged window (b200_mpileup_ranksums): a numpy int64 [n_files, 8, n]
        array of n_ref, n_alt and, for BQ, MQ and the BP-5 (capped at 1024) in turn, U2 (twice the Mann-Whitney U of the
        non-reference bases) and the tie term T; or, given `out`, a contiguous torch.int64 CUDA tensor of that shape on the
        handle's device, filled in place on the device (and returned).  ranksum_z turns the planes into z-scores."""
        return self._planes('b200_mpileup_ranksums', RANK_PLANES, min_baseQ, out, np.int64, 'int64')

    def mpileup_indels(self, min_baseQ=13, device=False):
        """Per-column indel alleles of the staged window (b200_mpileup_indels): (rows, symbols).  By default a numpy structured
        array of INDEL_DTYPE and the insertion symbols as uint8 bytes; with device=True an int32 [n, 8] CUDA tensor (the
        same 32-byte rows) and a uint8 CUDA tensor on the handle's device, filled on the device."""
        n, nb = C.c_int64(0), C.c_uint64(0)
        self._n_alleles = 0
        if self.lib.b200_mpileup_indels(self.h, min_baseQ, C.byref(n), C.byref(nb)) != 0:
            self._err('b200_mpileup_indels')
        self._n_alleles = n.value
        if not device:
            rows, seq = np.zeros(n.value, INDEL_DTYPE), np.zeros(nb.value, np.uint8)
            if self.lib.b200_fetch_indels(self.h, _ptr(rows) if n.value else None, n.value,
                                          _ptr(seq) if nb.value else None, nb.value) != 0:
                self._err('b200_fetch_indels')
            return rows, seq
        import torch
        dev = torch.device('cuda', self.device)
        rows = torch.empty((n.value, INDEL_DTYPE.itemsize // 4), dtype=torch.int32, device=dev)
        seq = torch.empty(nb.value, dtype=torch.uint8, device=dev)
        torch.cuda.current_stream(dev).synchronize()   # the engine writes on its own stream
        if self.lib.b200_fetch_indels(self.h, C.c_void_p(rows.data_ptr()) if n.value else None, n.value,
                                      C.c_void_p(seq.data_ptr()) if nb.value else None, nb.value) != 0:
            self._err('b200_fetch_indels')
        return rows, seq

    def _allele_rows(self, fn, width, np_dtype, torch_dtype, device):
        n = self._n_alleles
        if not device:
            a = np.zeros((n, width), np_dtype)
            if getattr(self.lib, fn)(self.h, _ptr(a) if n else None, n) != 0:
                self._err(fn)
            return a
        import torch
        dev = torch.device('cuda', self.device)
        t = torch.empty((n, width), dtype=getattr(torch, torch_dtype), device=dev)
        torch.cuda.current_stream(dev).synchronize()   # the engine writes on its own stream
        if getattr(self.lib, fn)(self.h, C.c_void_p(t.data_ptr()) if n else None, n) != 0:
            self._err(fn)
        return t

    def indel_qsums(self, device=False):
        """Quality sums of the rows of the last mpileup_indels on the staged batch (b200_indel_qsums), one row per allele in
        the table's order, columns INDEL_QSUM_FIELDS: a numpy uint32 [n, 6] array, or with device=True an int32 [n, 6] CUDA
        tensor on the handle's device, filled on the device."""
        return self._allele_rows('b200_indel_qsums', len(INDEL_QSUM_FIELDS), np.uint32, 'int32', device)

    def indel_psums(self, device=False):
        """Read-position sums of the rows of the last mpileup_indels on the staged batch (b200_indel_psums), one row per
        allele in the table's order, columns INDEL_PSUM_FIELDS (the IndelPsum row): a numpy int64 [n, 4] array, or with
        device=True an int64 [n, 4] CUDA tensor on the handle's device, filled on the device."""
        return self._allele_rows('b200_indel_psums', len(INDEL_PSUM_FIELDS), np.int64, 'int64', device)

    def fetch_qual(self, nbytes):
        q = np.zeros(nbytes, np.uint8)
        if self.lib.b200_fetch_qual(self.h, _ptr(q), nbytes) != 0:
            self._err('b200_fetch_qual')
        return q

    def pileup_entries(self, file, beg, end, cap):
        ncol = end - beg
        col_n = np.zeros(max(ncol, 1), np.uint32)
        ents = np.zeros(cap, dtype=np.dtype([('read', '<i8'), ('qpos', '<i4'), ('indel', '<i4'), ('cigar_ind', '<i4'), ('bits', '<u4')]))
        n = C.c_size_t(0)
        if self.lib.b200_pileup_entries(self.h, file, beg, end, _ptr(col_n), _ptr(ents), cap, C.byref(n)) != 0:
            self._err('b200_pileup_entries')
        return col_n, ents[:n.value]

    @property
    def last_kernel_ms(self):
        return self.lib.b200_last_kernel_ms(self.h)

    @property
    def last_stage_ms(self):
        return self.lib.b200_last_stage_ms(self.h)

    @property
    def last_stage_device_ms(self):
        return self.lib.b200_last_stage_device_ms(self.h)

    @property
    def last_baq_ms(self):
        return self.lib.b200_last_baq_ms(self.h)

    @property
    def last_mpileup_parts_ms(self):
        a = (C.c_double * 3)()
        self.lib.b200_last_mpileup_parts_ms(self.h, C.byref(a))
        return list(a)

    @property
    def gl_rng_draws(self):
        """hts_drand48 draws consumed so far by errmod_cal's ks_shuffle (columns with more than 255 usable bases)"""
        return self.lib.b200_gl_rng_draws(self.h)

    @property
    def launches(self):
        return self.lib.b200_launch_count(self.h)


def mpileup_conf(**kw):
    c = MpileupConf()
    c.min_baseQ = 13
    for k, v in kw.items():
        if not hasattr(c, k):
            raise AttributeError(k)
        setattr(c, k, v)
    return c
