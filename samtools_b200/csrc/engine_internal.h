// engine_internal.h -- the engine handle: grow-only HBM buffers + batch state.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "../../include/b200_pileup.h"
#include "plp_stage.h"

#define DBUF(type, name) type *name = nullptr; size_t cap_##name = 0

// What b200_restage has to undo in the staged qualities (e->qual) before it repeats the read stage: everything (a full
// copy from qual0), the mates of the pairs the last overlap tweak listed (k_qual_restore), or nothing.  The device
// writers of e->qual, each of which must be accounted for here:
//   stage_prep1 (plp_stage.h)                -6 (cf.illumina13)                       -> QUAL_DIRTY
//   k_baq / k_baq_reg (baq.cuh, baq_reg.h)   BAQ                                      -> QUAL_DIRTY
//   k_overlap_tweak (overlap.cuh)            mates of the pairs in ov_pairs           -> QUAL_PAIRS
// QUAL_PAIRS holds only while ov_pairs, its count d_misc[MISC_OVERLAP] and the descriptors are those of the stage that
// ran the tweak: nothing but launch_overlap writes the first two, and only a stage of the same batch (same n, so no
// buffer moves) has run since.
enum QualState : int {
    QUAL_DIRTY,      // unknown or widely edited: the first stage after an upload, BAQ, -6, a stage that stopped early
    QUAL_PAIRS,      // only k_overlap_tweak wrote, to the mates ov_pairs lists
    QUAL_PRISTINE,   // equal to qual0
};

struct b200_engine {
    int device = 0, n_sm = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evA = nullptr, evB = nullptr, evB0 = nullptr, evB1 = nullptr;
    bool baq_ran = false; double last_baq_ms = 0;
    double last_parts_ms[3] = {0, 0, 0};
    char err[512];
    int64_t launches = 0;
    double last_kernel_ms = 0, last_stage_ms = 0, last_stage_device_ms = 0;
    bool keep_raw = false, uploaded = false, has_host_clip = false;
    size_t qual_bytes = 0, n_cigar_total = 0;
    uint32_t smem_text = 24 * 1024;
    void *d_gfmt = nullptr;      // device copy of the gather's parameter block (cold paths)
    bool baq_attr_set = false;   // k_baq_reg's dynamic shared-memory attribute has been raised on this handle's device
    int general = 0;
    int baq_reg = 1;             // 0: every BAQ read on the warp kernel k_baq (B200_BAQ_REG, cross-check of k_baq_reg)

    // raw SoA image of the staged records
    DBUF(int64_t, pos); DBUF(uint16_t, flag); DBUF(uint8_t, mapq); DBUF(int32_t, l_qseq); DBUF(uint32_t, n_cigar);
    DBUF(uint64_t, cigar_off); DBUF(uint64_t, qual_off); DBUF(int32_t, mtid); DBUF(int64_t, mpos); DBUF(int64_t, isize);
    DBUF(int64_t, prev); DBUF(uint8_t, rbits);
    DBUF(uint32_t, cigar); DBUF(uint8_t, seq4); DBUF(uint8_t, qual); DBUF(char, ref); DBUF(char, dname);
    DBUF(int64_t, file_start);
    DBUF(uint8_t, qual0); DBUF(uint8_t, mapq0);   // pristine copies for b200_restage (b200_set_keep_raw)
    QualState qual_state = QUAL_DIRTY;            // of qual against qual0 (keep_raw only)
    // derived
    DBUF(uint8_t, state); DBUF(int32_t, rlen); DBUF(plp::ReadDesc, desc); DBUF(int32_t, endv); DBUF(int32_t, pmax);
    DBUF(int32_t, glo); DBUF(int32_t, ghi); DBUF(uint64_t, status); DBUF(char, out);   // status: look-back state of the scans (scan.cuh)
    DBUF(int64_t, bed_beg); DBUF(int64_t, bed_end);
    DBUF(uint32_t, col_n); DBUF(uint64_t, col_off); DBUF(uint64_t, col_state); DBUF(uint32_t, tile_total);
    DBUF(uint32_t, ovf_cnt); DBUF(int32_t, ovf_off); DBUF(int32_t, ovf_idx);
    DBUF(int32_t, ss_diff); DBUF(int32_t, ss_nplp); DBUF(uint32_t, ss_fail); DBUF(uint32_t, ss_extra); DBUF(b200_pileup1_t, ents);
    DBUF(int32_t, clip); DBUF(int64_t, next); DBUF(int32_t, cig_x); DBUF(int32_t, cig_y);
    DBUF(double, baq_f); DBUF(int32_t, baq_idx); DBUF(uint8_t, ref_codes); DBUF(uint16_t, ent); DBUF(uint16_t, ent2); DBUF(uint32_t, x_off); DBUF(char, x_dat); DBUF(int32_t, ov_pairs);
    DBUF(float, gl_out); DBUF(int32_t, gl_n); DBUF(uint32_t, gl_flag); DBUF(uint32_t, cnt);   // cnt: planes of b200_mpileup_counts / _qsums / _psums / _ranksums bound for host memory
    // b200_mpileup_indels (mpileup_indel.cuh): per (column, file) event counts and offsets; per event the record (IndelEv),
    // symbol count, symbol offset, key, table slot, first-appearance flag and allele bytes, allele index and allele symbol
    // offset; 2 hash slots per event and their strand counts; the symbols of the events, then the table and its symbols
    DBUF(uint32_t, ind_cnt); DBUF(uint32_t, ind_off); DBUF(uint8_t, ind_ev); DBUF(uint32_t, ind_len); DBUF(uint64_t, ind_soff);
    DBUF(uint64_t, ind_key); DBUF(uint32_t, ind_slot); DBUF(uint32_t, ind_first); DBUF(uint32_t, ind_bytes); DBUF(uint32_t, ind_aidx);
    DBUF(uint64_t, ind_aseq); DBUF(int32_t, ind_tbl); DBUF(uint32_t, ind_tcnt); DBUF(char, ind_sym); DBUF(b200_indel_t, ind_tab); DBUF(char, ind_seq);
    DBUF(b200_indel_qsum_t, ind_qs);   // b200_indel_qsums: the rows of the table's quality sums
    DBUF(b200_indel_psum_t, ind_ps);   // b200_indel_psums: the rows of the table's read-position sums
    // b200_mpileup_ranksums (mpileup_rank.cuh): per (file, column) the active flag and its exclusive scan, then the active list
    DBUF(uint32_t, rk_act); DBUF(uint32_t, rk_off); DBUF(int32_t, rk_list);
    bool ind_ready = false; int64_t ind_n = 0; uint64_t ind_nseq = 0; uint32_t ind_nev = 0;   // the table of the staged batch: rows, symbol bytes, events
    void *d_acc = nullptr;
    unsigned long long *d_misc = nullptr;   // 64 words of small device results; slots MISC_* below, each zeroed by its writer's caller
    double *d_beta = nullptr, *d_fk = nullptr, *d_lhet = nullptr;   // errmod tables
    double fk_depcorr = 0;                                             // dependency coefficient d_fk was built for
    double *d_q2p = nullptr, *d_qthr = nullptr;                      // BAQ tables

    // batch state
    bool staged = false, has_ref = false, has_prev = false, has_rbits = false, has_clip = false, maxdrop_applied = false;
    int64_t n = 0; int32_t n_files = 0, tid = 0; int64_t tid_len = 0;
    std::string name;
    b200_stage_conf_t sconf;
    int64_t win_base = 0, ref_beg = 0, ref_n = 0, ref_len = 0;
    plp::ColDomain cols = {0, 0}; int32_t ncols_max = 0, n_groups = 0;
    int64_t acc_n_kept = 0; int32_t max_rend = 0;
    unsigned long long sum_rlen = 0, sum_indel_text = 0, sum_rlen_gen = 0;
    size_t last_out_len = 0;
    uint64_t gl_rng_draws = 0;   // hts_drand48 draws consumed so far by errmod's ks_shuffle
    std::vector<int64_t> h_file_start;
    std::vector<int32_t> h_rlen_tmp, h_clip_tmp;

    plp::TextTotals totals(int64_t ncols) const { return {sum_rlen, sum_indel_text, n, ncols, (uint64_t)name.size(), n_files}; }
    void free_all()
    {
        void *ps[] = { qual0, mapq0, pos, flag, mapq, l_qseq, n_cigar, cigar_off, qual_off, mtid, mpos, isize, prev, rbits, cigar, seq4, qual,
                       ref, dname, file_start, state, rlen, desc, endv, pmax, glo, ghi, status, out, bed_beg, bed_end, col_n,
                       col_off, col_state, tile_total, ovf_cnt, ovf_off, ovf_idx, ss_diff, ss_nplp, ss_fail, ss_extra, ents, clip, next, cig_x, cig_y, baq_f, baq_idx, ref_codes, ent, ent2, x_off, x_dat, ov_pairs, gl_out, gl_n, gl_flag, cnt,
                       ind_cnt, ind_off, ind_ev, ind_len, ind_soff, ind_key, ind_slot, ind_first, ind_bytes, ind_aidx, ind_aseq, ind_tbl, ind_tcnt,
                       ind_sym, ind_tab, ind_seq, ind_qs, ind_ps, rk_act, rk_off, rk_list, d_beta, d_fk, d_lhet, d_q2p, d_qthr };
        for (void *p : ps) if (p) cudaFree(p);
    }
};

// Slots (64-bit words) of b200_engine::d_misc
enum : int {
    MISC_RANGE_MAX = 1,    // k_ranges (low half: widest read slice), k_ovf_max (high half: longest far-reaching list); read by build_ranges
    MISC_MAX_BUFFERED = 2, // k_max_i32: most reads of one file buffered at a position; read by max_buffered_reads
    MISC_ENT2_CURSOR = 3,  // k_mp_entries: cursor of the second entry array
    MISC_COVERAGE = 8,     // 5 words: k_coverage's sums; read by b200_coverage
    MISC_BAQ = 16,         // 16 words: k_baq_plan's counters (first 5, read by launch_baq) and k_baq's work counter (word 11)
    MISC_OVERLAP = 40,     // k_overlap: number of pairs to tweak; read by k_overlap_tweak and, at the next restage, k_qual_restore
    MISC_QSUM_DEEP = 41,   // k_mp_qsums / k_ind_qsums: a column or allele too deep for 32-bit sums; read by their calls
    MISC_PSUM_OVF = 42,    // k_mp_psums / k_ind_psums: a sum of squared read positions past INT64_MAX; read by their calls
    MISC_RANK_DEEP = 43,   // k_rank_counts: a column with more class entries than exact rank sums allow; read by b200_mpileup_ranksums
};

using plp::RawSoA;
int build_ranges(b200_engine *e, int *max_range);
int launch_baq(b200_engine *e, const RawSoA &r, const b200_stage_conf_t &cf);
int launch_overlap(b200_engine *e, const RawSoA &r);
int launch_qual_restore(b200_engine *e, const RawSoA &r);
int launch_depth_clip(b200_engine *e, const RawSoA &r);
