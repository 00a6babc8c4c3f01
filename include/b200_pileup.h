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
 *   b200_mpileup_counts() pileup_seq, as numbers           bam_plcmd.c:54-169 -> per-column strand-split base / indel counts
 *   b200_mpileup_indels() pileup_seq's +n / -n tokens      bam_plcmd.c:54-169 -> per-column indel alleles, strand-split support
 *   b200_mpileup_qsums()  the qual and -s columns          bam_plcmd.c:674-688, :728-748 -> per-column BQ / MQ sums, MQ0
 *   b200_indel_qsums()    (the same, per indel allele)     -> BQ / MQ sums and MQ0 counts of each allele's entries
 *   b200_mpileup_psums()  the --output-BP-5 column         bam_plcmd.c:753-759 -> per-column BP-5 sums and sums of squares
 *   b200_indel_psums()    (the same, per indel allele)     -> BP-5 sums and sums of squares of each allele's entries
 *   b200_mpileup_ranksums() the -s, qual and BP-5 columns  -> per-column Mann-Whitney U of BQ / MQ / BP-5, ref vs alt bases
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
/* per-column base and indel counts of the mpileup column stage: what a parser of the `mpileup --reverse-del` text of the
 * staged window counts, without the text.  Per file 19 uint32 planes of n_cols columns, planar: out[(f * 19 + k) * n + c]
 * for column c = position - window start, c in [0, n) (the columns b200_mpileup_text() formats with all = 1; empty ones are
 * zero).  Planes k = 0..8 count forward-strand entries, 9..17 reverse-strand ones, each as
 *   0-3 A C G T (a '.' / ',' counts as the column's reference base)   4 any other base (also '.' / ',' without an A/C/G/T
 *   reference)   5 deletion ('*' / '#')   6 reference skip ('>' / '<')   7 a "+n" insertion follows   8 a "-n" deletion follows
 * counting only entries that pass -Q (min_baseQ, as in the text); plane 18 is n_plp, the reads over the column before -Q.
 * out == NULL: compute only, the planes stay in HBM (device-only timing, like out == NULL of the text calls).  Otherwise out
 * is host or device memory (a device buffer must be on the handle's device) of at least n_files * 19 * cap_cols words;
 * cap_cols < n returns -2.  *n_cols always receives n.  Needs a batch staged in B200_MODE_MPILEUP. */
#define B200_COUNT_PLANES 19
int b200_mpileup_counts(b200_engine_t *e, int32_t min_baseQ, uint32_t *out, size_t cap_cols, int64_t *n_cols);
/* per-column indel alleles of the mpileup column stage: the distinct "+n..." / "-n" tokens that the `mpileup` text of the
 * staged window prints after the entries passing -Q (min_baseQ), one row per (column, file, allele), ordered by column
 * c = position - window start, then file, then first appearance in the line (file order of the reads; a read's insertion
 * before its deletion).  len >= 0: an insertion of len symbols, seq[seq_off, seq_off + len) -- the read's upper-case IUPAC
 * bases, 'N' past the read's sequence, '*' for a pad; len < 0: a deletion of -len reference bases (named by its length:
 * the bases are the reference's at c+1 .. c-len).  fwd / rev: the entries on each strand that carry the token.  Per
 * (column, file) the fwd sums over insertions and deletions are planes 7 and 8 of b200_mpileup_counts, the rev sums 16 and
 * 17.  32 bytes per row (an int32 [n, 8] view).
 *   b200_mpileup_indels  computes the table and keeps it in HBM; *n_alleles and *n_seq_bytes receive its size.  Needs a batch
 *                        staged in B200_MODE_MPILEUP.  b200_last_kernel_ms() covers it.
 *   b200_fetch_indels    copies the table of the last b200_mpileup_indels since the batch was staged to host or device memory
 *                        (a device buffer must be on the handle's device); either pointer may be NULL to skip its part.
 *                        cap_alleles < n_alleles or cap_seq < n_seq_bytes returns -2. */
typedef struct {
    int32_t col, file, len;
    uint32_t fwd, rev, pad;
    uint64_t seq_off;
} b200_indel_t;
int b200_mpileup_indels(b200_engine_t *e, int32_t min_baseQ, int64_t *n_alleles, uint64_t *n_seq_bytes);
int b200_fetch_indels(b200_engine_t *e, b200_indel_t *alleles, size_t cap_alleles, char *seq, size_t cap_seq);
/* per-column quality sums of the mpileup column stage, beside the counts: what a parser of the `mpileup --reverse-del -s`
 * text adds up over the entries that pass -Q (min_baseQ).  An entry's BQ is its quality character minus 33 (the quality
 * after BAQ, -6 and the overlap tweak, clamped at 93 as the text prints '~'), its MQ its -s character minus 33 (the mapq
 * after -C, clamped at 93), its MQ0 1 where that character is '!' (mapq 0).  Per file 42 uint32 planes, laid out, sized and
 * delivered exactly as those of b200_mpileup_counts: out[(f * 42 + k) * n + c], zero where a column is empty; out == NULL
 * computes only; host or device memory; cap_cols < n returns -2; needs a batch staged in B200_MODE_MPILEUP.  Plane
 *   k = s * 14 + r * 7 + kind,   s: 0 BQ sum, 1 MQ sum, 2 MQ0 count;  r: 0 forward, 1 reverse strand;
 *                                kind: 0-6 A C G T N deletion skip, as planes r * 9 + kind of b200_mpileup_counts
 * Sums are exact while a column has at most 46182444 reads (93 times that fits in 32 bits); the call fails on a deeper one
 * (possible only without a max-depth limit) instead of wrapping.  b200_last_kernel_ms() covers it. */
#define B200_QSUM_PLANES 42
int b200_mpileup_qsums(b200_engine_t *e, int32_t min_baseQ, uint32_t *out, size_t cap_cols, int64_t *n_cols);
/* quality sums beside the indel table: row j holds, per strand, the BQ and MQ sums and the MQ0 count (as above) of the
 * entries that carry allele j of the last b200_mpileup_indels since the batch was staged (with that call's -Q), so fwd and
 * rev of row j are the counts they are taken over.  Refused without such a table, as b200_fetch_indels is.  out == NULL
 * computes only; otherwise host or device memory (a device buffer must be on the handle's device); cap_rows below the row
 * count returns -2.  b200_last_kernel_ms() covers it.  24 bytes per row (a uint32 [n, 6] view). */
typedef struct {
    uint32_t bq_fwd, bq_rev, mq_fwd, mq_rev, mq0_fwd, mq0_rev;
} b200_indel_qsum_t;
int b200_indel_qsums(b200_engine_t *e, b200_indel_qsum_t *out, size_t cap_rows);
/* per-column read-position sums of the mpileup column stage, beside the counts: what a parser of the
 * `mpileup --reverse-del --output-BP-5` text adds up over the entries that pass -Q (min_baseQ).  An entry's BP-5 is the
 * 5'-based position of its base in the read, the sequencing cycle: qpos + 1 on the forward strand, l_qseq - qpos + is_del
 * on the reverse strand (signed: <= 0 for a reverse-strand entry of a read without SEQ at -Q 0, as the text prints it).
 * Per file 28 int64 planes, laid out, sized and delivered exactly as those of b200_mpileup_counts:
 * out[(f * 28 + k) * n + c], zero where a column is empty; out == NULL computes only; host or device memory;
 * cap_cols < n returns -2; needs a batch staged in B200_MODE_MPILEUP.  Plane
 *   k = s * 14 + r * 7 + kind,   s: 0 BP-5 sum, 1 sum of BP-5 squared;  r: 0 forward, 1 reverse strand;
 *                                kind: 0-6 A C G T N deletion skip, as planes r * 9 + kind of b200_mpileup_counts
 * so with the count planes they give the mean and the variance of the position.  The BP-5 sums cannot overflow; the call
 * fails instead of wrapping where a sum of squares would exceed 2^63 - 1.  b200_last_kernel_ms() covers it. */
#define B200_PSUM_PLANES 28
int b200_mpileup_psums(b200_engine_t *e, int32_t min_baseQ, int64_t *out, size_t cap_cols, int64_t *n_cols);
/* read-position sums beside the indel table: row j holds, per strand, the BP-5 sum and the sum of its squares (as above)
 * of the entries that carry allele j of the last b200_mpileup_indels since the batch was staged (with that call's -Q); an
 * indel token takes the BP-5 of the entry it follows.  Refusals, destinations and caps as b200_indel_qsums; the call fails
 * where a sum of squares would exceed 2^63 - 1.  b200_last_kernel_ms() covers it.  32 bytes per row (an int64 [n, 4]
 * view). */
typedef struct {
    int64_t bp5_fwd, bp5_rev, bp5sq_fwd, bp5sq_rev;
} b200_indel_psum_t;
int b200_indel_psums(b200_engine_t *e, b200_indel_psum_t *out, size_t cap_rows);
/* per-column rank-sum bias statistics of the mpileup column stage, beside the counts: the Mann-Whitney U test of base
 * quality, mapping quality and read position, reference against non-reference bases, as a parser of the
 * `mpileup --reverse-del -s --output-BP-5` text would compute it over the entries that pass -Q (min_baseQ).  A class entry
 * is an A, C, G or T entry (count planes r * 9 + 0..3): of the ref class where the text prints '.' / ',', of the alt class
 * where it prints a letter (all non-reference bases pooled); deletions, skips and N / IUPAC bases take no part.  Its values
 * are BQ and MQ as in b200_mpileup_qsums (0..93) and its BP-5 as in b200_mpileup_psums (>= 1), with a BP-5 above 1024
 * ranked as 1024 (the cap is part of the definition: it keeps the work per column independent of the read length).
 * Per file 8 int64 planes, laid out, sized and delivered exactly as those of b200_mpileup_counts:
 * out[(f * 8 + k) * n + c]; out == NULL computes only; host or device memory; cap_cols < n returns -2; needs a batch staged
 * in B200_MODE_MPILEUP.  Planes
 *   0 n_ref,  1 n_alt,  2 / 3 U2 / T of BQ,  4 / 5 U2 / T of MQ,  6 / 7 U2 / T of BP-5
 *   U2 = sum over (alt a, ref r) of 2 [a > r] + [a == r]    (twice the U of the alt sample)
 *   T  = sum over values v of t_v^3 - t_v                    (t_v: ref and alt entries of value v; the tie term)
 * planes 2-7 are 0 where a class is empty; n_ref + n_alt is the sum of count planes A C G T of both strands.  With
 * N = n_ref + n_alt, U = U2 / 2 has mean n_ref n_alt / 2 and variance n_ref n_alt / 12 ((N + 1) - T / (N (N - 1))).  The
 * planes are exact for N <= 2097151 (2^21 - 1); the call fails instead of wrapping on a deeper column.
 * b200_last_kernel_ms() covers it. */
#define B200_RANK_PLANES 8
int b200_mpileup_ranksums(b200_engine_t *e, int32_t min_baseQ, int64_t *out, size_t cap_cols, int64_t *n_cols);
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
/* last b200_mpileup_text(): device time of its three parts.  Default path (one input file, no -O columns): entry pass
 * (k_mp_entries), line sizes + tile offsets (k_mp_place), gather (k_mp_gather).  General path: sizing kernel, tile-offset
 * scan, write kernel. */
void b200_last_mpileup_parts_ms(const b200_engine_t *e, double *ms3);

#ifdef __cplusplus
}
#endif
#endif
