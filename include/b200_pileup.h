/*
 * b200_pileup.h -- C ABI of the CUDA (sm_90a) pileup engine (tier T2, batch API).
 *
 * Drop-in boundary for the mpileup / depth / coverage hot path of samtools
 * 1.23.1 (SURVEY.md section 8b).  The reference reaches this path through htslib's
 * per-column pull iterators; a GPU cannot be fed one column at a time, so the
 * engine takes a BATCH of pre-decoded alignment records as structure-of-arrays
 * (the fields of htslib's bam1_core_t plus the packed cigar/seq/qual blocks),
 * runs the whole column loop on the device and hands back the finished
 * output (pileup text, depth rows, coverage sums, genotype likelihoods).
 *
 * What each entry point replaces in the reference:
 *   b200_stage()          mplp_func read filters          bam_plcmd.c:400-461
 *                         fastdepth_core read filters     bam2depth.c:552-570
 *                         read_bam filters + read stats   coverage.c:178-198
 *                         sam_prob_realn (BAQ) call       bam_plcmd.c:451
 *                         sam_cap_mapq call               bam_plcmd.c:453
 *                         bam_plp_push + overlap_push     (htslib sam.c; enabled bam_plcmd.c:586)
 *   b200_mpileup_text()   bam_mplp64_auto column loop     bam_plcmd.c:607-868
 *                         pileup_seq                      bam_plcmd.c:54-169
 *                         print_empty_pileup / -a gaps    bam_plcmd.c:372-398, :610-660, :880-910
 *   b200_depth_text()     add_depth + flush rows          bam2depth.c:209-477, zero_region :88-118
 *   b200_coverage()       column reducers                 coverage.c:589-661
 *   b200_coverage_hist()  per-bin counters of -m / -D     coverage.c:609-660
 *   b200_bedcov()         per-interval column reducers    bedcov.c:303-331
 *   b200_glf()            bcf_call_glfgen + errmod_cal    bam2bcf.c:65-123 (+ htslib errmod.c)
 *   b200_pileup_entries() bam_plp64_next/resolve_cigar2   (htslib sam.c) -> arrays of bam_pileup1_t fields
 *
 * Conventions: plain C, caller-owned host buffers, int return codes (0 ok,
 * <0 error; b200_last_error() gives the text).  A handle is bound to one CUDA
 * device and one stream and is NOT thread-safe (same as the htslib handles it
 * replaces).  All positions are 0-based; text output is byte-identical to the
 * reference's.  There is no CPU fallback: every call fails if no CUDA device.
 */
#ifndef B200_PILEUP_H
#define B200_PILEUP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200_engine b200_engine_t;

/* ---- batch of pre-decoded records, structure-of-arrays ------------------ */
/* Reads of ONE reference sequence (tid), grouped by input file; inside a file
 * they keep file (= coordinate) order.  This is the SoA image of bam1_t. */
typedef struct {
    int32_t n_files;
    int64_t n_reads;             /* total over all files */
    const int64_t *file_start;   /* [n_files+1] first read index of each file */
    /* bam1_core_t fields */
    const int64_t *pos;          /* [n_reads] leftmost coordinate, 0-based */
    const uint16_t *flag;        /* [n_reads] */
    const uint8_t *mapq;         /* [n_reads] */
    const int32_t *l_qseq;       /* [n_reads] */
    const uint32_t *n_cigar;     /* [n_reads] */
    const uint64_t *cigar_off;   /* [n_reads] index of first op in cigar[] */
    const uint64_t *qual_off;    /* [n_reads] byte offset into qual[]; MUST be even.
                                    The read's bases are nibbles qual_off.. of seq4
                                    (high nibble first), i.e. byte qual_off/2 */
    const int32_t *mtid;         /* [n_reads] mate tid (-1 none)          */
    const int64_t *mpos;         /* [n_reads] mate pos                    */
    const int64_t *isize;        /* [n_reads] template length             */
    /* name linkage, per file: index (into this batch) of the previous record
     * carrying the same QNAME in the same file, or -1.  Replaces the qname
     * string hash of overlap_push (htslib) / olap_hash (bam2depth.c:483). */
    const int64_t *prev_same_name; /* [n_reads], may be NULL if unused */
    /* per read host bits, see B200_RB_* */
    const uint8_t *rbits;        /* [n_reads], may be NULL (= all zero) */
    /* depth -s only: absolute clip coordinate of each read (0 = none), when the caller has replayed the
     * reference's name hash itself (bam2depth.c:598-623 keeps ONE hash per file across reference sequences, so a
     * name seen on an earlier contig can clip a read here); NULL = the device derives it from prev_same_name */
    const int64_t *depth_clip;   /* [n_reads], may be NULL */
    /* packed payload */
    const uint32_t *cigar;  uint64_t n_cigar_total;   /* BAM encoding len<<4|op */
    const uint8_t *seq4;    /* 4-bit bases, (qual_bytes+1)/2 bytes */
    const uint8_t *qual;    uint64_t qual_bytes;      /* raw phred, 0xff.. when absent */
    /* this reference sequence */
    int32_t tid;
    int64_t tid_len;             /* sam_hdr_tid2len */
    const char *tid_name;        /* sam_hdr_tid2name */
    /* reference bases (optional): ref[0..ref_n) are contig positions
     * ref_beg..ref_beg+ref_n; ref_len = contig length in the FASTA (0: none) */
    const char *ref; int64_t ref_beg, ref_n, ref_len;
} b200_batch_t;

#define B200_RB_HOST_SKIP 1   /* dropped by a host-side string filter (BED -l per read, RG -G) */
#define B200_RB_NAME_ODD  2   /* __ac_Wang_hash(__ac_X31_hash_string(qname)) & 1: which mate keeps the evidence */
#define B200_RB_BAQ_DONE  4   /* BAQ already applied from a stored BQ:Z tag (integer path) */
#define B200_RB_HALO      8   /* the read starts before this window and was already staged with the previous one (a driver that
                                 cuts a reference sequence into column windows stages every read overlapping a window: the -r
                                 rule, bam_plcmd.c:550-554,609): leave it out of the coverage read statistics (coverage.c:185-193) */
/* The max-depth rule of bam_plp_push depends on every read pushed before: a driver that cuts a reference sequence into
 * windows stages the reads that reach a window from the left again and hands over the verdicts the previous window made
 * (B200_RB_MAXDEPTH_OF below).  A SEEN read is not judged again: kept, it counts as buffered and as the
 * previous read; dropped, it takes no part.  Only reads without SEEN are judged. */
#define B200_RB_MAXDEPTH_SEEN 16   /* the read's max-depth verdict was made in an earlier window */
#define B200_RB_MAXDEPTH_DROP 32   /* ... and that verdict was a drop */
#define B200_KEEP_KEPT    2        /* b200_fetch_mapq_keep state: the read reaches the pileup */
#define B200_KEEP_MAXDROP 3        /* ... the max-depth rule dropped it (lower states: a filter did, before the rule) */
/* the carry bits of a b200_fetch_mapq_keep state: 0 for a read the max-depth rule never judged */
#define B200_RB_MAXDEPTH_OF(keep) ((keep) == B200_KEEP_KEPT ? B200_RB_MAXDEPTH_SEEN : \
                                   (keep) == B200_KEEP_MAXDROP ? (B200_RB_MAXDEPTH_SEEN | B200_RB_MAXDEPTH_DROP) : 0)

/* ---- read-level configuration (what happens before a read is pushed) ---- */
typedef enum { B200_MODE_MPILEUP = 0, B200_MODE_DEPTH = 1, B200_MODE_COVERAGE = 2 } b200_mode_t;

typedef struct {
    int32_t mode;            /* b200_mode_t: which command's read filters apply */
    /* mpileup (bam_plcmd.c:413-458) / coverage (coverage.c:187-190) */
    int32_t rflag_require;   /* --rf: keep only reads with ANY of these bits (0: off) */
    int32_t rflag_filter;    /* --ff: drop reads with ANY of these bits */
    int32_t min_mq;          /* -q */
    int32_t no_orphan;       /* 1 unless -A */
    int32_t illumina13;      /* -6 */
    int32_t baq;             /* 0 off, 1 = sam_prob_realn flag 3, 2 = flag 7 (-E), 3 = flag 1 (APPLY without EXTEND: calmd -A); needs ref */
    int32_t capq_thres;      /* -C */
    int32_t overlaps;        /* read-pair overlap detection (off with -x) */
    int32_t max_depth;       /* -d (bam_mplp_set_maxcnt) */
    /* depth (bam2depth.c:552-570) */
    int32_t d_flag_excl, d_flag_incl, d_flag_require, d_min_mapq, d_min_len, d_remove_overlaps;
    /* coverage: min read length (-l, bam_cigar2qlen) */
    int32_t c_min_len;
    /* output window: columns [beg,end) of this tid may be reported */
    int64_t beg, end;
} b200_stage_conf_t;

typedef struct {
    int64_t n_kept;          /* reads that reach the pileup */
    int64_t n_kept_in_window;/* kept reads overlapping [beg,end) with a non-empty reference span */
    uint64_t out_bound;      /* upper bound of the text bytes any mode can emit for this batch */
    int64_t n_cols;          /* candidate output columns of this batch (covered span or -a span) */
    /* coverage read statistics (coverage.c:185-193) */
    uint64_t n_reads, n_selected_reads, summed_mapq;
} b200_stage_stats_t;

/* ---- mpileup column configuration --------------------------------------- */
typedef struct {
    int32_t min_baseQ;       /* -Q */
    int32_t all;             /* 0, 1 (-a), 2 (-aa): emit zero-depth rows inside [beg,end) */
    int32_t rev_del;         /* --reverse-del */
    int32_t no_ins, no_del;  /* --no-output-ins / --no-output-del (0,1,2) */
    int32_t no_ends;         /* --no-output-ends */
    int32_t out_mapq;        /* -s */
    int32_t out_qpos;        /* -O */
    int32_t out_qpos5;       /* --output-BP-5 */
    int32_t n_star_cols;     /* further optional columns the host will NOT get from the device
                                (QNAME/extras): only their "\t*" placeholders on empty rows */
    /* per-column BED filter (-l): sorted, non-overlapping-start intervals of this tid */
    const int64_t *bed_beg, *bed_end; int32_t n_bed; int32_t bed_active;
    /* host columns ON the device (--output-QNAME, --output-extra fields and tags; bam_plcmd.c:727-855): the caller renders,
     * per read of the staged batch, the string each column prints for it (a decimal FLAG, the QNAME, a tag value or the
     * --output-empty character ...) and the device gathers them per pileup column, in file order, for the reads that pass
     * -Q, joined by x_sep[k].  n_x (<= 16) must equal n_star_cols; column k of read i is
     * x_dat[x_off[k * (n_reads + 1) + i] .. x_off[k * (n_reads + 1) + i + 1]).  n_x = 0: place holders only. */
    int32_t n_x; const uint32_t *x_off; const char *x_dat; uint64_t x_bytes; char x_sep[16];
} b200_mpileup_conf_t;

typedef struct {
    int32_t min_qual;        /* -q */
    int32_t count_del;       /* -J */
    int32_t all;             /* -a / -aa */
    const int64_t *bed_beg, *bed_end; int32_t n_bed; int32_t bed_active;
} b200_depth_conf_t;

typedef struct {
    int32_t min_baseQ;       /* -Q */
    int32_t min_depth;       /* --min-depth */
} b200_coverage_conf_t;

typedef struct {             /* coverage.c:58-70 column sums for one tid */
    uint64_t n_covered_bases, summed_coverage, summed_baseQ, quality_bases;
    uint64_t missing_qual;   /* print_value_warning */
} b200_coverage_sums_t;

/* one (read, column) entry: the fields of htslib's bam_pileup1_t */
typedef struct {
    int64_t read;            /* index into the staged batch */
    int32_t qpos;
    int32_t indel;
    int32_t cigar_ind;
    uint32_t is_del:1, is_head:1, is_tail:1, is_refskip:1;
} b200_pileup1_t;

/* ---- engine ------------------------------------------------------------- */
int  b200_engine_create(int device, b200_engine_t **out);
void b200_engine_destroy(b200_engine_t *e);
const char *b200_last_error(const b200_engine_t *e);   /* never NULL */
const char *b200_version(void);

/* Host -> HBM staging (pinned cudaMemcpyAsync) + the per-read stage: filters,
 * BAQ, mapq cap, pair-overlap quality tweak, max-depth rule, read descriptors. */
int b200_stage(b200_engine_t *e, const b200_batch_t *batch, const b200_stage_conf_t *conf,
               b200_stage_stats_t *stats);

/* Column stage over the staged batch.  out may be NULL to keep the result in
 * HBM (device-only timing); *out_len always receives the byte count. */
int b200_mpileup_text(b200_engine_t *e, const b200_mpileup_conf_t *conf, char *out, size_t out_cap, size_t *out_len);
int b200_depth_text(b200_engine_t *e, const b200_depth_conf_t *conf, char *out, size_t out_cap, size_t *out_len);
/* upper bounds of what the text calls can write for the staged batch with these options (a few per cent above the real size): a
 * caller sizes its host buffer once and gets the text in ONE call instead of asking for the length first */
uint64_t b200_mpileup_text_bound(const b200_engine_t *e, const b200_mpileup_conf_t *conf);
uint64_t b200_depth_text_bound(const b200_engine_t *e);
int b200_coverage(b200_engine_t *e, const b200_coverage_conf_t *conf, b200_coverage_sums_t *sums);
/* the per-bin counters behind `coverage -m / -D` (coverage.c:609-660): column `pos` of the staged window adds to bin
 * (pos - beg) / bin_width (bins >= n_bins are dropped) either 1 when the column counts as covered (plot_depth == 0: breadth)
 * or its filtered depth summed over the files (plot_depth != 0).  hist[n_bins] is ADDED to (32-bit wrap, like the
 * reference's uint32_t counters), so the windows of one reference sequence accumulate. */
int b200_coverage_hist(b200_engine_t *e, const b200_coverage_conf_t *conf, int64_t beg, int64_t bin_width, int32_t n_bins,
                       int32_t plot_depth, uint32_t *hist);
/* bedcov reducers (bedcov.c:316-331) over the staged window [beg,end): per input file the sum of the per-column depth --
 * without deletions and reference skips when skip_del_refskip or min_depth >= 0, as the reference does -- and, for
 * min_depth >= 0, the number of columns whose depth reaches it (pcov may be NULL).  Stage with B200_MODE_COVERAGE
 * (rflag_filter = the -g/-G flag set, min_mq = -Q). */
int b200_bedcov(b200_engine_t *e, int32_t skip_del_refskip, int32_t min_depth, uint64_t *cnt, uint64_t *pcov);
/* genotype likelihoods per covered column and file: n, qsum[4], p[25].  col_pos == NULL: compute only, results stay in
 * HBM (device-only timing, like out == NULL of the text calls); *n_cols is then the number of candidate columns */
int b200_glf(b200_engine_t *e, int32_t min_baseQ, int64_t *n_cols, int64_t *col_pos, int32_t *n_bases,
             float *qsum, float *p25, size_t cap_cols);
/* htslib's per-column / per-read entry points on the device (tier T1 support; one column or one small batch per call):
 *   b200_errmod_cal   errmod_cal(em, n, m, bases, q) of htslib errmod.c (callers bam2bcf.c:121, phase.c:754, cut_target.c:84):
 *                     `bases` (q<<5|strand<<4|allele) is left sorted like the reference leaves it, q[m*m] receives the
 *                     phred-scaled genotype likelihoods; depcorr = the errmod_init argument; n > 255 consumes n-1 draws of
 *                     the handle's drand48 stream (b200_gl_rng_draws)
 *   b200_glfgen       bcf_call_glfgen (bam2bcf.c:65-123) for one column: per read the base quality at qpos (0 past the
 *                     read's end), mapq, 4-bit base (0xff past the end) and fl (bit 0: is_del | is_refskip | unmapped,
 *                     bit 1: reverse strand); returns n like the reference (-1 when n_reads <= 0)
 *   b200_cap_mapq     sam_cap_mapq (htslib realn.c; call bam_plcmd.c:453) of every read of the staged batch */
int b200_errmod_cal(b200_engine_t *e, double depcorr, int32_t n, int32_t m, uint16_t *bases, float *q);
int b200_glfgen(b200_engine_t *e, double depcorr, int32_t n_reads, const uint8_t *q, const uint8_t *mapq, const uint8_t *base4, const uint8_t *fl,
                int32_t ref_base, int32_t min_baseQ, int32_t capQ, float *qsum, float *p25);
int b200_cap_mapq(b200_engine_t *e, int32_t thres, int32_t *out, size_t n);
/* qualities after the read stage (BAQ / overlap tweak), for inspection and the iterator tier */
int b200_fetch_qual(b200_engine_t *e, uint8_t *qual, size_t cap);
int b200_fetch_mapq_keep(b200_engine_t *e, uint8_t *mapq, uint8_t *keep, size_t n);
/* column-major pileup entries (tier T1 support): col_n[c-beg] entries per column */
int b200_pileup_entries(b200_engine_t *e, int32_t file, int64_t beg, int64_t end, uint32_t *col_n,
                        b200_pileup1_t *entries, size_t cap_entries, size_t *n_entries);

/* device timing of the last column-stage call (CUDA events on the engine stream), milliseconds */
/* Benchmark support: repeat the device side of the read stage (everything b200_stage does after its host->device
 * copies: filters, -6, BAQ, -C, descriptors, read slices, max-depth rule, overlap tweak) on the batch already resident in
 * device memory.  The read stage edits qualities / mapq in place, so a pristine copy has to stay resident:
 * call b200_set_keep_raw(e, 1) before b200_stage().  Replaces nothing in the reference; lets a device-resident
 * measurement cover the whole hot path (bam_plcmd.c:400-461 + the column loop) without the PCIe copies. */
int b200_set_keep_raw(b200_engine_t *e, int on);
int b200_restage(b200_engine_t *e, b200_stage_stats_t *stats);
double b200_last_stage_device_ms(const b200_engine_t *e);   /* device part of the last b200_stage / b200_restage */
double b200_last_baq_ms(const b200_engine_t *e);            /* of which: the BAQ kernels (sam_prob_realn), 0 when BAQ did not run */
double b200_last_kernel_ms(const b200_engine_t *e);
double b200_last_stage_ms(const b200_engine_t *e);
int64_t b200_launch_count(const b200_engine_t *e);   /* kernels launched by this handle so far */
/* hts_drand48 draws consumed so far by b200_glf (errmod_cal shuffles a column's bases when it holds more than 255; the
 * reference draws from ONE process-wide stream, so a region shard continues from its predecessor's count) */
uint64_t b200_gl_rng_draws(const b200_engine_t *e);
/* last b200_mpileup_text(): device time of its three launches -- sizing kernel, tile-offset scan, write kernel */
void b200_last_mpileup_parts_ms(const b200_engine_t *e, double *ms3);

#ifdef __cplusplus
}
#endif
#endif
