// baq_host.cpp -- TEST HARNESS (not shipped, not linked into the product): runs the register-band BAQ arithmetic of
// samtools_b200/csrc/baq_reg.h on the CPU, read by read, and compares the rewritten qualities with the oracle's
// restatement of sam_prob_realn (oracle/baq.c, flag 3 = APPLY|EXTEND).  The device kernel executes the same
// __host__ __device__ functions; only the memory policy differs.
//   baq_host in.sam ref.fa [-l]   -> "checked N reads (M on the register path), K mismatches"
//   -l also lists the reads the register path takes ("reg <qname> <pos> <l_qseq>", one per line)
// build: tests/emul/build.sh (g++ -ffp-contract=off, links oracle/_build/liboracle.so)
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../samtools_b200/csrc/baq_reg.h"
extern "C" {
#include "../../oracle/plp.h"
}

struct HostMem {
    const char *ref; int64_t ref_len, xb;
    std::vector<double> fm, fi, iv; std::vector<int32_t> w;
    int ref_code(int p) const
    {
        const int64_t a = xb + p;
        const char ch = (a >= 0 && a < ref_len) ? ref[a] : 'N';
        return plp::nt16_int_of(plp::nt16_of((unsigned char)ch));
    }
    uint64_t ref8(int p) const { uint64_t w = 0; for (int k = 0; k < 8; ++k) w |= (uint64_t)ref_code(p + k) << (8 * k); return w; }
    void put_row(int i, const double (&M)[baqr::NB], const double (&I)[baqr::NB], double inv)
    {
        for (int j = 0; j < baqr::NB; ++j) { fm[(size_t)i * baqr::NB + j] = M[j]; fi[(size_t)i * baqr::NB + j] = I[j]; }
        iv[i] = inv;
    }
    void fence() {}
    void fetch(int) {}
    void wait(int) {}
    void get(int i, int j, double &a, double &b) const { a = fm[(size_t)i * baqr::NB + j]; b = fi[(size_t)i * baqr::NB + j]; }
    double inv(int i) const { return iv[i]; }
    void put_word(int j, int32_t x) { w[j] = x; }
    int32_t get_word(int j) const { return w[j]; }
};

// longest read k_baq_plan sends to the register kernel (BAQR_MAX_LQ in baq.cuh); longer band-7 reads run on k_baq
constexpr int kMaxRegLq = 512;

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: baq_host in.sam ref.fa [-l]\n"); return 2; }
    const bool list = argc > 3 && strcmp(argv[3], "-l") == 0;
    reader_t *rd = reader_open(argv[1], NULL);
    fasta_t *fa = fasta_load(argv[2]);
    if (!rd || !fa) { fprintf(stderr, "cannot open inputs\n"); return 2; }
    hdr_t *h = reader_hdr(rd);
    double q2p[256], q2pf[256], qthr[102];
    baqr::host_tables(q2p, qthr);
    for (int i = 0; i < 256; ++i) q2pf[i] = (double)(float)q2p[i];
    rec_t r; rec_init(&r);
    long n = 0, n_fast = 0, bad = 0;
    while (reader_next(rd, &r) >= 0) {
        if (r.tid < 0 || (r.flag & F_UNMAP)) continue;
        const int fi = fasta_find(fa, h->name[r.tid]);
        if (fi < 0) continue;
        const char *ref = fa->seq[fi]; const int64_t ref_len = fa->len[fi];
        if (rec_aux_get(&r, "BQ") || rec_aux_get(&r, "ZQ")) continue;
        rec_t want; rec_init(&want); rec_copy(&want, &r);
        baq_realn(&want, ref, ref_len, 3);
        ++n;
        // the plan of k_baq_plan (sam_prob_realn prologue)
        const int lq = r.l_qseq;
        bool fast = lq > 0 && r.qual[0] != 0xff;
        int64_t x = r.pos, xb = -1, xe = -1; int y = 0, yb = -1, ye = -1;
        for (uint32_t k = 0; fast && k < r.n_cigar; ++k) {
            const int op = r.cigar[k] & 0xf, l = (int)(r.cigar[k] >> 4);
            if (plp::is_mop(op)) { if (yb < 0) yb = y; if (xb < 0) xb = x; ye = y + l; xe = x + l; x += l; y += l; }
            else if (op == plp::OP_S || op == plp::OP_I) y += l;
            else if (op == plp::OP_D) x += l;
            else if (op == plp::OP_N) fast = false;
        }
        if (xb == -1) fast = false;
        int64_t l_ref = 0; int b2 = 0;
        if (fast) {
            int bw = 7;
            int64_t dd = (xe - xb) - (ye - yb); if (dd < 0) dd = -dd;
            if (dd > bw) bw = (int)dd + 3;
            const int cbw = bw;
            xb -= yb + bw / 2; if (xb < 0) xb = 0;
            xe += lq - ye + bw / 2;
            if (xe - xb - lq > bw) { xb += (xe - xb - lq - bw) / 2; xe -= (xe - xb - lq - bw) / 2; }
            if (xe > ref_len) xe = ref_len;
            l_ref = xe - xb;
            if (l_ref <= 0) fast = false;
            b2 = (int)(l_ref > lq ? l_ref : lq); if (b2 > cbw) b2 = cbw;
            int64_t d2 = l_ref - lq; if (d2 < 0) d2 = -d2;
            if (b2 < d2) b2 = (int)d2;
            if (b2 != baqr::BW) fast = false;
            if (lq > kMaxRegLq) fast = false;
        }
        if (fast) {
            ++n_fast;
            if (list) printf("reg %s %lld %d\n", r.qname, (long long)r.pos, lq);
            HostMem mem; mem.ref = ref; mem.ref_len = ref_len; mem.xb = xb;
            mem.fm.assign((size_t)(lq + 2) * baqr::NB, 0.); mem.fi = mem.fm; mem.iv.assign(lq + 2, 0.); mem.w.assign(lq + 1, 0);
            std::vector<uint8_t> q(r.qual, r.qual + lq);
            q.resize((size_t)lq + 16, 0);                                  // ld8 slack (the staged device arrays carry it too)
            std::vector<uint8_t> sq(r.seq, r.seq + (lq + 1) / 2);
            sq.resize(sq.size() + 16, 0);
            baqr::baq_read(mem, q.data(), sq.data(), 0u, lq, (int)l_ref, r.pos, xb, r.cigar, (int)r.n_cigar, q2pf, qthr);
            if (memcmp(q.data(), want.qual, lq) != 0) {
                if (++bad <= 5) {
                    fprintf(stderr, "MISMATCH read %s pos %lld lq %d l_ref %lld\n", r.qname, (long long)r.pos, lq, (long long)l_ref);
                    for (int j = 0; j < lq; ++j) if (q[j] != want.qual[j]) { fprintf(stderr, "  base %d: got %d want %d (orig %d)\n", j, q[j], want.qual[j], r.qual[j]); break; }
                }
            }
        }
        rec_free(&want);
    }
    printf("checked %ld reads (%ld on the register path), %ld mismatches\n", n, n_fast, bad);
    return bad ? 1 : 0;
}
