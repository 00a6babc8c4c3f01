// cli.cpp -- `b200samtools mpileup|depth|coverage|bedcov|gl`: the reference's CLI surface
// for the pileup hot path, driving the CUDA engine through its C ABI.
//
// Option surfaces follow bam_plcmd.c:1096-1223 (mpileup), bam2depth.c:757-882
// (depth) and coverage.c:343-424 (coverage), SURVEY.md Appendix B.  What stays
// on the host is what the reference also does outside the column loop: option
// parsing, file decode, per-contig sequencing of -a/-aa output
// (bam_plcmd.c:610-660, :880-910; bam2depth.c:215-287; coverage.c:591-688) and
// the final %g formatting of coverage rows (coverage.c:200-221).  Every read
// filter, BAQ, overlap handling, the column loop and all text formatting run on
// the GPU; there is no CPU fallback (engine creation fails without a device).
//
// Not offered on the device path yet (SURVEY 8f rank 3): -M/--output-mods,
// (none here any more: host string columns and the coverage histogram views are served from device results too).
#include "hts_io.hpp"
#include "packer.hpp"
#include <getopt.h>
#include <sys/ioctl.h>
#include <math.h>
#include <zlib.h>
#include <cctype>
#include <cstdarg>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cerrno>
#include <algorithm>
#include <thread>
#include <queue>
#include <set>
#include <unordered_map>

using namespace b200;

namespace {

// One input file, decoded ONE REFERENCE SEQUENCE AT A TIME: the drivers walk the reference sequences in header order and
// ask for the records of the sequence they are about to process (load_tid); the records of the sequences already handled
// are released, so the resident set is one sequence per file, not the whole input.
struct FileData {
    std::unique_ptr<AlnReader> rd;
    std::vector<std::vector<Record>> by_tid;   // decoded records per reference sequence, file order (only the current one is populated)
    Record pending; bool have_pending = false, eof = false;
    int last_tid = -1;                          // reference sequence of the last mapped record seen (sortedness check)
    bool keep_all = false;                      // bedcov: BED lines address the sequences in any order, keep everything
    int64_t n_no_tid = 0;
};

bool load_file(const std::string &fn, const std::string &fai, const char *reg, FileData &fd, int &rtid, int64_t &rbeg, int64_t &rend,
               const char *cmd)
{
    fd.rd = AlnReader::open(fn, fai);
    if (!fd.rd) { fprintf(stderr, "[%s] failed to open %s: %s\n", cmd, fn.c_str(), strerror(errno)); return false; }
    if (reg && !fd.rd->set_region(reg, rtid, rbeg, rend)) {
        fprintf(stderr, "[E::%s] fail to parse region '%s' with %s\n", cmd, reg, fn.c_str());
        return false;
    }
    fd.by_tid.resize((size_t)fd.rd->header().n_ref());
    return true;
}

// records of reference sequence `tid` -> fd.by_tid[tid]; everything decoded for earlier sequences is dropped.
// Returns false on a read error or when the file's reference sequences are out of order.
bool load_tid(FileData &fd, int tid, const char *cmd)
{
    if (tid < 0 || tid >= (int)fd.by_tid.size()) return true;
    if (!fd.keep_all) for (int t = 0; t < tid; ++t) if (!fd.by_tid[(size_t)t].empty()) std::vector<Record>().swap(fd.by_tid[(size_t)t]);
    std::vector<Record> &dst = fd.by_tid[(size_t)tid];
    for (;;) {
        if (!fd.have_pending) {
            if (fd.eof) break;
            const int ret = fd.rd->next(fd.pending);
            if (ret == -1) { fd.eof = true; break; }
            if (ret < -1) { fprintf(stderr, "samtools %s: error reading from input file\n", cmd); return false; }
            fd.have_pending = true;
        }
        Record &r = fd.pending;
        if (r.tid < 0 || r.tid >= (int)fd.by_tid.size()) { ++fd.n_no_tid; fd.have_pending = false; continue; }
        if (!(r.flag & F_UNMAP)) {
            // records are handed out per reference sequence, which would silently repair a file whose chromosomes are
            // out of order; htslib's bam_plp_push refuses it (order within a sequence is checked by the engine's read stage)
            if (r.tid < fd.last_tid) { fprintf(stderr, "[%s] The input is not sorted (chromosomes out of order)\n", cmd); return false; }
            fd.last_tid = r.tid;
        }
        if (r.tid > tid) break;                       // belongs to a later sequence: stays pending
        if (r.tid == tid) dst.push_back(std::move(r));
        fd.have_pending = false;                      // (an unmapped straggler of an earlier sequence is dropped)
    }
    return true;
}

struct Engine {
    b200_engine_t *e = nullptr;
    ~Engine() { if (e) b200_engine_destroy(e); }
    bool init(int dev = -1)
    {
        if (dev < 0) { dev = 0; if (const char *s = getenv("B200_DEVICE")) dev = atoi(s); }
        if (b200_engine_create(dev, &e) != 0) { fprintf(stderr, "b200samtools: cannot create the CUDA pileup engine (an H100/sm_90a device is required)\n"); return false; }
        return true;
    }
};
// Devices for the window workers of a driver: B200_DEVICES="0,1,2,3" (one handle each), times B200_HANDLES handles per
// device (default 1).  The column windows of a reference sequence are independent (each stages its own halo), so they are
// handed round-robin to the workers -- region sharding across GPUs (SURVEY 8e) below the Python layer, and, with several
// handles on one device, H2D / kernels / D2H of consecutive windows overlapping.  Unset: one handle on B200_DEVICE.
std::vector<int> worker_devices()
{
    std::vector<int> d;
    if (const char *s = getenv("B200_DEVICES")) {
        for (const char *p = s; *p;) { if (isdigit((unsigned char)*p)) { d.push_back(atoi(p)); while (isdigit((unsigned char)*p)) ++p; } else ++p; }
    }
    int per = 1;
    if (const char *s = getenv("B200_HANDLES")) per = std::max(1, atoi(s));
    if (d.empty() && per > 1) { int dev = 0; if (const char *s = getenv("B200_DEVICE")) dev = atoi(s); d.push_back(dev); }
    std::vector<int> out;
    for (int k = 0; k < per; ++k) for (int dev : d) out.push_back(dev);
    return out;
}
// One engine handle of a driver: its packer, record cursors (one per file) and the output of the window it last ran.
struct WinWorker {
    Engine eng; PackedBatch pb; std::vector<char> out; std::vector<size_t> sel, cursor; size_t need = 0; int rc = 0; std::string err;
    void rewind() { std::fill(cursor.begin(), cursor.end(), 0); }
    int fail(const char *tool) { rc = -1; err = std::string("samtools ") + tool + ": " + b200_last_error(eng.e); return -1; }
};
using Workers = std::vector<std::unique_ptr<WinWorker>>;
// The handles of a driver, never none: one per entry of worker_devices() where that lists several and the driver can use
// them (`several`), else one on B200_DEVICE.
bool make_workers(Workers &workers, int n_files, bool several)
{
    std::vector<int> wd = several ? worker_devices() : std::vector<int>();
    if (wd.size() < 2) wd.assign(1, -1);
    for (int dev : wd) { workers.emplace_back(new WinWorker()); if (!workers.back()->eng.init(dev)) return false; workers.back()->cursor.assign((size_t)n_files, 0); }
    return true;
}
// printf onto the end of a worker's output
__attribute__((format(printf, 2, 3))) void appendf(WinWorker &w, const char *fmt, ...)
{
    for (;;) {
        va_list ap;
        va_start(ap, fmt);
        const int k = vsnprintf(w.out.data() + w.need, w.out.size() - w.need, fmt, ap);
        va_end(ap);
        if (k < 0) return;
        if (w.need + (size_t)k < w.out.size()) { w.need += (size_t)k; return; }
        w.out.resize(std::max(2 * w.out.size(), w.need + (size_t)k + 1));
    }
}

using Windows = std::vector<std::pair<int64_t, int64_t>>;
// Rounds of one window per worker over the first k workers: job(worker, wb, we) stages its window concurrently with the
// others (a round of one window runs on the calling thread) and leaves its text in out[0, need) (or sets rc / err); then
// the texts are written in window order.
template <class Job>
int run_window_rounds(Workers &workers, const Windows &wins, size_t k, FILE *fp, Job job)
{
    for (auto &w : workers) w->rewind();
    k = std::min(k, workers.size());
    for (size_t base = 0; base < wins.size(); base += k) {
        const size_t m = std::min(k, wins.size() - base);
        auto run = [&](size_t t) { WinWorker &w = *workers[t]; w.rc = 0; w.need = 0; job(w, wins[base + t].first, wins[base + t].second); };
        if (m == 1) run(0);
        else {
            std::vector<std::thread> th;
            for (size_t t = 0; t < m; ++t) th.emplace_back(run, t);
            for (auto &t : th) t.join();
        }
        for (size_t t = 0; t < m; ++t) {
            const WinWorker &w = *workers[t];
            if (w.rc != 0) { fprintf(stderr, "%s\n", w.err.c_str()); return -1; }
            if (w.need) fwrite(w.out.data(), 1, w.need, fp);
        }
    }
    return 0;
}

// ---- column windows ------------------------------------------------------------------------------------------------
// The engine addresses columns as 32-bit offsets from the window start and takes < 4 GiB of read payload per staged
// batch, so the drivers cut a reference sequence into windows of at most window_cols() columns.  A window [wb,we)
// stages every record that overlaps it -- pos < we && endpos > wb, the rule a `-r` run applies (bam_plcmd.c:550-554,609)
// -- so a read reaching in from the left is staged again ("halo"); the engine reports only columns inside the window.
// Per-read work (filters, BAQ) is simply repeated for halo reads; a mate pair whose overlap lies in the window has both
// mates staged, so the overlap tweak sees what an unsplit run sees.  The -d max-depth rule of bam_plp_push counts a read
// as buffered over the closed interval [pos, endpos], so a window that continues an earlier one also stages the reads
// ending right at its start (endpos == wb: they cover none of its columns), and the halo reads carry the verdicts the
// earlier window made (B200_RB_MAXDEPTH_*; see MaxDepthCarry).
int64_t window_cols()
{
    static int64_t w = 0;
    if (!w) { const char *s = getenv("B200_WINDOW_COLS"); w = s ? atoll(s) : (1LL << 24); if (w < 1) w = 1; if (w > (1LL << 30)) w = 1LL << 30; }
    return w;
}
// records of v (sorted by pos) overlapping [wb,we) -- with `closed`, also those ending at wb; `lo` is a cursor that only
// moves forward across successive windows
void window_records(const std::vector<Record> &v, size_t &lo, int64_t wb, int64_t we, std::vector<size_t> &out, bool closed = false)
{
    out.clear();
    const int64_t lim = closed && wb > INT64_MIN ? wb - 1 : wb;
    while (lo < v.size() && v[lo].endpos() <= lim) ++lo;
    for (size_t j = lo; j < v.size() && v[j].pos < we; ++j) if (v[j].endpos() > lim) out.push_back(j);
}
// Largest number of records of one file (before any filter) whose closed intervals [pos, endpos] share a position: no
// column of the contig can make the max-depth rule fire while this is <= -d, and then its windows are independent.
int64_t max_stacked_records(const std::vector<FileData> &fd, int tid)
{
    int64_t best = 0;
    for (const FileData &f : fd) {
        if (tid >= (int)f.by_tid.size()) continue;
        std::priority_queue<int64_t, std::vector<int64_t>, std::greater<int64_t>> ends;
        int64_t last = INT64_MIN;
        for (const Record &r : f.by_tid[(size_t)tid]) {
            if (r.pos < last) return INT64_MAX;   // unsorted: the engine refuses it; no bound
            last = r.pos;
            while (!ends.empty() && ends.top() < r.pos) ends.pop();
            ends.push(r.endpos());
            if ((int64_t)ends.size() > best) best = (int64_t)ends.size();
        }
    }
    return best;
}
// The max-depth verdicts of one contig's records, handed from each window to the next: after a window is staged, every
// record the engine kept or dropped (B200_KEEP_*) remembers it, and a later window that stages the record again passes it on.
struct MaxDepthCarry {
    bool on = false;
    std::vector<std::vector<uint8_t>> bits;   // per file, per record of the contig: B200_RB_MAXDEPTH_* or 0
    std::vector<std::pair<int, size_t>> staged;   // (file, record) of each read of the staged batch
    std::vector<uint8_t> keep;
    void reset(const std::vector<FileData> &fd, int tid, bool enable)
    {
        on = enable; bits.assign(fd.size(), {}); staged.clear();
        if (on) for (size_t i = 0; i < fd.size(); ++i) bits[i].assign(tid < (int)fd[i].by_tid.size() ? fd[i].by_tid[(size_t)tid].size() : 0, 0);
    }
    uint8_t add(int file, size_t j) { if (!on) return 0; staged.emplace_back(file, j); return bits[(size_t)file][j]; }
    int collect(b200_engine_t *e)
    {
        if (!on) return 0;
        keep.resize(staged.size());
        if (!staged.empty() && b200_fetch_mapq_keep(e, nullptr, keep.data(), keep.size()) != 0) return -1;
        for (size_t k = 0; k < staged.size(); ++k)
            if (const uint8_t b = B200_RB_MAXDEPTH_OF(keep[k])) bits[(size_t)staged[k].first][staged[k].second] = b;
        staged.clear();
        return 0;
    }
};
// first / one-past-last reference position touched by the records of a contig (over all files)
bool records_extent(const std::vector<FileData> &fd, int tid, int64_t &first, int64_t &last)
{
    bool any = false; first = POS_MAX; last = 0;
    for (const FileData &f : fd) {
        if (tid >= (int)f.by_tid.size()) continue;
        for (const Record &r : f.by_tid[(size_t)tid]) { any = true; if (r.pos < first) first = r.pos; const int64_t e = r.endpos(); if (e > last) last = e; }
    }
    return any;
}
// Columns [lo,hi) whose rows mpileup / depth print for contig tid: the region [rb,re), cut down to the span of the records
// unless empty rows are wanted (`all`), and in that case extended to records running past the contig's end.  Without
// reads, the region within the contig.  False when the contig's records leave no column to visit.
bool column_range(const std::vector<FileData> &fd, int tid, int64_t tid_len, int64_t rb, int64_t re, bool all, bool with_reads,
                  int64_t &lo, int64_t &hi)
{
    lo = rb; hi = std::min(re, tid_len);
    if (!with_reads) return true;
    int64_t first = 0, last = 0;
    if (!records_extent(fd, tid, first, last)) return false;
    if (!all) { lo = std::max(rb, first); hi = std::min(re, last); } else hi = std::max(hi, std::min(re, last));
    return lo < hi;
}
// [lo,hi) cut into windows of window_cols() columns; an empty range is still one (empty) window
Windows column_windows(int64_t lo, int64_t hi)
{
    Windows wins;
    for (int64_t wb = lo; wb < hi || wb == lo; wb += window_cols()) wins.emplace_back(wb, std::max(std::min(wb + window_cols(), hi), wb));
    return wins;
}
// Stages window [wb,we) of contig tid on worker w: add(i) packs into w.pb the records file i contributes (w.cursor[i] and
// w.sel are its to use), and `md`, if given, then takes the engine's max-depth verdicts.  A coverage window without records
// has nothing to count and is not staged (returns 1).  Returns -1 with w.err set on an error.
template <class Add>
int stage_window(WinWorker &w, const Header &h, int tid, const std::string *ref, const b200_stage_conf_t &sc, int64_t wb, int64_t we,
                 MaxDepthCarry *md, const char *tool, b200_stage_stats_t &st, Add add)
{
    w.pb.clear();
    for (int i = 0; i < (int)w.cursor.size(); ++i) { w.pb.begin_file(); add(i); }
    w.pb.finish();
    if (sc.mode == B200_MODE_COVERAGE && w.pb.pos.empty()) return 1;
    b200_batch_t batch = w.pb.view(tid, h.lens[(size_t)tid], h.names[(size_t)tid], ref);
    b200_stage_conf_t wsc = sc; wsc.beg = wb; wsc.end = we;
    if (b200_stage(w.eng.e, &batch, &wsc, &st) != 0 || (md && md->collect(w.eng.e) != 0)) return w.fail(tool);
    return 0;
}

// ----------------------------------------------------------------------------- mpileup
struct MpOpts {
    int min_mq = 0, min_baseQ = 13, capQ = 0, max_depth = 8000, all = 0, rev_del = 0;
    int rf = 0, ff = F_UNMAP | F_SECONDARY | F_QCFAIL | F_DUP;
    bool no_orphan = true, realn = true, redo_baq = false, illumina13 = false, ignore_rg = false, overlaps = true;
    int no_ins = 0, no_del = 0, no_ends = 0, out_mapq = 0, out_qpos = 0, out_qpos5 = 0;
    const char *reg = nullptr, *fa_fn = nullptr, *out_fn = nullptr;
    std::unique_ptr<Fasta> fa; std::unique_ptr<Bed> bed;
    std::set<std::string> rg_excl; bool have_rg = false;
    bool gl = false;
    // host columns (bam_plcmd.c:727-855): record fields in the order of the MPLP_PRINT_* bits, then aux tags in the order given
    std::vector<std::string> xcols;      // "QNAME" "FLAG" "RNAME" "POS" "MAPQ" "RNEXT" "PNEXT" "RLEN" or a two-letter tag
    int n_xfields = 0;                   // how many of them are record fields (joined with ','; tags use x_sep)
    char x_sep = ',', x_empty = '*';
};

int count_samples(const std::vector<std::string> &fn, const std::vector<FileData> &fd, bool ignore_rg)
{
    // bam_smpl_add (sample.c:79-121): distinct @RG SM values, else the file name
    std::set<std::string> smpl;
    for (size_t i = 0; i < fn.size(); ++i) {
        int n = 0;
        if (!ignore_rg) {
            const std::string &t = fd[i].rd->header().text;
            size_t p = 0;
            while ((p = t.find("@RG", p)) != std::string::npos) {
                p += 3;
                size_t id = t.find("\tID:", p), sm = t.find("\tSM:", p);
                if (id == std::string::npos || sm == std::string::npos) break;
                sm += 4;
                size_t e = t.find_first_of("\t\n", sm);
                smpl.insert(t.substr(sm, e == std::string::npos ? std::string::npos : e - sm));
                p = std::max(id + 4, sm);
                ++n;
            }
        }
        if (n == 0) smpl.insert(fn[i]);
    }
    return (int)smpl.size();
}

// host bits of one record for mpileup: string filters and the stored-BAQ-tag integer path
uint8_t mp_host_bits(const MpOpts &o, const Header &h, Record &r, bool has_ref)
{
    uint8_t rb = 0;
    if (o.bed && o.all == 0 && !o.bed->overlap(h.names[(size_t)r.tid], r.pos, r.endpos())) rb |= B200_RB_HOST_SKIP;
    if (o.have_rg) {
        const uint8_t *rg = r.aux_get("RG");
        if (rg && o.rg_excl.count((const char *)rg + 1)) rb |= B200_RB_HOST_SKIP;
    }
    if (has_ref && o.realn && !(rb & B200_RB_HOST_SKIP) && !(r.flag & F_UNMAP) && r.l_qseq > 0 && r.qual[0] != 0xff) {
        // sam_prob_realn with existing tags (htslib realn.c; SURVEY 8a a2): BQ:Z present and not -E -> integer adjust
        const uint8_t *bq = r.aux_get("BQ"), *zq = r.aux_get("ZQ");
        if (bq && *bq != 'Z') bq = nullptr;
        if (zq && *zq != 'Z') zq = nullptr;
        if (bq && o.redo_baq) bq = nullptr;        // -E: the tag is deleted, HMM recomputed on the device
        else if (bq && zq) zq = nullptr;
        if (bq) {
            if (o.illumina13) for (auto &q : r.qual) q = q > 31 ? q - 31 : 0;   // -6 precedes BAQ (bam_plcmd.c:428-433)
            const uint8_t *b = bq + 1;
            for (int32_t i = 0; i < r.l_qseq; ++i) r.qual[(size_t)i] = r.qual[(size_t)i] + 64 < b[i] ? 0 : (uint8_t)(r.qual[(size_t)i] - ((int)b[i] - 64));
            rb |= B200_RB_BAQ_DONE;
        } else if (zq && !(o.redo_baq && false)) {
            if (o.illumina13) for (auto &q : r.qual) q = q > 31 ? q - 31 : 0;
            rb |= B200_RB_BAQ_DONE;               // ZQ present with APPLY: left untouched
        }
    }
    return rb;
}

int run_mpileup(MpOpts &o, const std::vector<std::string> &fn)
{
    const int nfn = (int)fn.size();
    if (nfn == 0) { fprintf(stderr, "[mpileup] no input file/data given\n"); return 1; }
    std::vector<FileData> fd((size_t)nfn);
    int tid0 = 0; int64_t beg0 = 0, end0 = POS_MAX;
    const std::string fai = o.fa_fn ? std::string(o.fa_fn) + ".fai" : "";
    for (int i = 0; i < nfn; ++i) {
        int t = 0; int64_t b = 0, e = POS_MAX;
        if (!load_file(fn[(size_t)i], fai, o.reg, fd[(size_t)i], t, b, e, "mpileup")) return 1;
        if (i == 0) { tid0 = t; beg0 = b; end0 = e; }
    }
    const Header &h = fd[0].rd->header();
    fprintf(stderr, "[mpileup] %d samples in %d input files\n", count_samples(fn, fd, o.ignore_rg), nfn);
    FILE *fp = o.out_fn ? fopen(o.out_fn, "w") : stdout;
    if (!fp) { fprintf(stderr, "[mpileup] failed to write to %s: %s\n", o.out_fn, strerror(errno)); return 1; }
    int max_depth = o.max_depth;
    if (!max_depth) { max_depth = INT_MAX; fprintf(stderr, "[mpileup] Max depth set to maximum value (%d)\n", INT_MAX); }
    else if ((long long)max_depth * nfn > 1 << 20) fprintf(stderr, "[mpileup] Combined max depth is above 1M. Potential memory hog!\n");

    // window workers (worker_devices()): the text path without host columns can be spread over several handles
    Workers workers;
    if (!make_workers(workers, nfn, !o.gl && o.xcols.empty())) return 1;
    b200_stage_conf_t sc; memset(&sc, 0, sizeof sc);
    sc.mode = B200_MODE_MPILEUP; sc.rflag_require = o.rf; sc.rflag_filter = o.ff; sc.min_mq = o.min_mq; sc.no_orphan = o.no_orphan;
    sc.illumina13 = o.illumina13; sc.baq = o.realn ? (o.redo_baq ? 2 : 1) : 0; sc.capq_thres = o.capQ; sc.overlaps = o.overlaps;
    sc.max_depth = max_depth;
    b200_mpileup_conf_t mc; memset(&mc, 0, sizeof mc);
    mc.min_baseQ = o.min_baseQ; mc.all = o.all; mc.rev_del = o.rev_del; mc.no_ins = o.no_ins; mc.no_del = o.no_del; mc.no_ends = o.no_ends;
    mc.out_mapq = o.out_mapq; mc.out_qpos = o.out_qpos; mc.out_qpos5 = o.out_qpos5;

    std::vector<int64_t> bb, be;
    const int nref = h.n_ref();
    std::vector<std::vector<uint8_t>> hbits((size_t)nfn);   // host bits of the contig's records, decided ONCE (the BQ:Z path edits the record)
    std::vector<const Record *> staged;                     // records of the staged window, batch order (host columns)
    std::vector<uint32_t> x_off; std::string x_dat; std::vector<uint8_t> x_mapq;
    // per-read strings of the host columns (--output-QNAME / --output-extra, bam_plcmd.c:727-855) for the staged window
    auto render_host_columns = [&](WinWorker &w) -> int {
        const size_t nr = staged.size(), nx = o.xcols.size();
        x_off.assign(nx * (nr + 1), 0); x_dat.clear();
        bool need_mapq = false;
        for (const std::string &cname : o.xcols) if (cname == "MAPQ") need_mapq = true;
        if (need_mapq && nr) { x_mapq.resize(nr); if (b200_fetch_mapq_keep(w.eng.e, x_mapq.data(), nullptr, nr) != 0) return -1; }   // after -C
        char tmp[64];
        for (size_t k = 0; k < nx; ++k) {
            const std::string &cname = o.xcols[k];
            const bool is_tag = (int)k >= o.n_xfields;
            for (size_t i = 0; i < nr; ++i) {
                const Record &r = *staged[i];
                x_off[k * (nr + 1) + i] = (uint32_t)x_dat.size();
                if (!is_tag) {
                    if (cname == "QNAME") x_dat += r.qname;
                    else if (cname == "FLAG") { snprintf(tmp, sizeof tmp, "%d", (int)r.flag); x_dat += tmp; }
                    else if (cname == "RNAME") x_dat += r.tid >= 0 ? h.names[(size_t)r.tid] : std::string("*");
                    else if (cname == "POS") { snprintf(tmp, sizeof tmp, "%lld", (long long)r.pos + 1); x_dat += tmp; }
                    else if (cname == "MAPQ") { snprintf(tmp, sizeof tmp, "%d", (int)x_mapq[i]); x_dat += tmp; }
                    else if (cname == "RNEXT") x_dat += (r.mtid >= 0 && r.mtid < h.n_ref()) ? h.names[(size_t)r.mtid] : std::string("*");
                    else if (cname == "PNEXT") { snprintf(tmp, sizeof tmp, "%lld", (long long)r.mpos + 1); x_dat += tmp; }
                    else if (cname == "RLEN") { snprintf(tmp, sizeof tmp, "%d", (int)r.l_qseq); x_dat += tmp; }
                } else {
                    const uint8_t *t = r.aux_get(cname.c_str());
                    if (!t) x_dat += o.x_empty;
                    else switch (*t) {
                        case 'Z': case 'H': x_dat += (const char *)t + 1; break;
                        case 'c': snprintf(tmp, sizeof tmp, "%d", (int)(int8_t)t[1]); x_dat += tmp; break;
                        case 'C': snprintf(tmp, sizeof tmp, "%d", (int)t[1]); x_dat += tmp; break;
                        case 's': { int16_t v; memcpy(&v, t + 1, 2); snprintf(tmp, sizeof tmp, "%d", (int)v); x_dat += tmp; break; }
                        case 'S': { uint16_t v; memcpy(&v, t + 1, 2); snprintf(tmp, sizeof tmp, "%d", (int)v); x_dat += tmp; break; }
                        case 'i': { int32_t v; memcpy(&v, t + 1, 4); snprintf(tmp, sizeof tmp, "%d", v); x_dat += tmp; break; }
                        case 'I': { uint32_t v; memcpy(&v, t + 1, 4); snprintf(tmp, sizeof tmp, "%u", v); x_dat += tmp; break; }
                        case 'f': { float v; memcpy(&v, t + 1, 4); snprintf(tmp, sizeof tmp, "%g", (double)v); x_dat += tmp; break; }
                        case 'd': { double v; memcpy(&v, t + 1, 8); snprintf(tmp, sizeof tmp, "%g", v); x_dat += tmp; break; }
                        case 'A': x_dat += (char)t[1]; break;
                        default: x_dat += '*'; break;
                    }
                }
            }
            x_off[k * (nr + 1) + nr] = (uint32_t)x_dat.size();
        }
        mc.n_x = (int32_t)nx; mc.n_star_cols = (int32_t)nx; mc.x_off = x_off.data(); mc.x_dat = x_dat.data(); mc.x_bytes = x_dat.size();
        for (size_t k = 0; k < nx; ++k) mc.x_sep[k] = (int)k < o.n_xfields ? ',' : o.x_sep;
        return 0;
    };
    MaxDepthCarry md;
    auto process_tid = [&](int tid, bool with_reads) -> int {
        // returns 1 when rows were requested and produced, 0 when the contig has no pileup column, <0 on error
        const std::string &name = h.names[(size_t)tid];
        const std::string *ref = nullptr;
        if (o.fa) { int fi = o.fa->find(name); if (fi >= 0) ref = &o.fa->seqs[(size_t)fi]; }
        if (o.bed) { o.bed->merged(name, bb, be); mc.bed_beg = bb.data(); mc.bed_end = be.data(); mc.n_bed = (int)bb.size(); mc.bed_active = 1; }
        int64_t lo = 0, hi = 0;
        if (!column_range(fd, tid, h.lens[(size_t)tid], beg0, end0, o.all, with_reads, lo, hi)) return 0;
        for (int i = 0; i < nfn; ++i) {
            hbits[(size_t)i].clear();
            if (with_reads && tid < (int)fd[(size_t)i].by_tid.size())
                for (Record &r : fd[(size_t)i].by_tid[(size_t)tid]) hbits[(size_t)i].push_back(mp_host_bits(o, h, r, ref != nullptr));
        }
        const Windows wins = column_windows(lo, hi);
        // a window that continues an earlier one also takes the records ending at its start (the -d rule's closed intervals)
        auto stage = [&](WinWorker &w, int64_t wb, int64_t we, b200_stage_stats_t &st) {
            if (!o.xcols.empty()) staged.clear();
            return stage_window(w, h, tid, ref, sc, wb, we, &md, "mpileup", st, [&](int i) {
                if (!with_reads || tid >= (int)fd[(size_t)i].by_tid.size()) return;
                std::vector<Record> &v = fd[(size_t)i].by_tid[(size_t)tid];
                window_records(v, w.cursor[(size_t)i], wb, we, w.sel, wb > lo);
                for (size_t j : w.sel) { w.pb.add(v[j], (uint8_t)(hbits[(size_t)i][j] | md.add(i, j)), o.overlaps); if (!o.xcols.empty()) staged.push_back(&v[j]); }
            });
        };
        // the first window with a pileup column decides whether the contig is reported at all (its empty -a rows before that
        // column included), so find it before anything is written
        md.reset(fd, tid, false);
        if (with_reads) {
            WinWorker &w = *workers[0];
            w.rewind();
            bool hit = false;
            for (size_t k = 0; k < wins.size() && !hit; ++k) {
                b200_stage_stats_t st;
                if (stage(w, wins[k].first, wins[k].second, st) != 0) { fprintf(stderr, "%s\n", w.err.c_str()); return -1; }
                hit = st.n_kept_in_window > 0;
            }
            if (!hit) return 0;
        }
        // a contig split into several windows where the max-depth rule may fire runs them in order on worker 0, each handing
        // its verdicts to the next; so do the empty rows of a contig without reads (GL and host columns have one worker).
        // Elsewhere the windows are independent.
        const bool carry = with_reads && wins.size() > 1 && max_stacked_records(fd, tid) > (int64_t)max_depth;
        md.reset(fd, tid, carry);
        const int rc = run_window_rounds(workers, wins, carry || !with_reads ? 1 : workers.size(), fp, [&](WinWorker &w, int64_t wb, int64_t we) {
            b200_stage_stats_t st;
            if (stage(w, wb, we, st) != 0) return;
            if (with_reads && !o.all && st.n_kept_in_window == 0) return;
            if (o.gl) {
                int64_t ncols = 0; const size_t cap = (size_t)st.n_cols + 16;
                std::vector<int64_t> cpos(cap); std::vector<int32_t> nb(cap * (size_t)nfn); std::vector<float> qs(cap * (size_t)nfn * 4), p25(cap * (size_t)nfn * 25);
                if (b200_glf(w.eng.e, o.min_baseQ, &ncols, cpos.data(), nb.data(), qs.data(), p25.data(), cap) != 0) { w.fail("gl"); return; }
                for (int64_t k = 0; k < ncols; ++k) {
                    const int64_t p = cpos[(size_t)k];
                    if (o.bed && !o.bed->overlap(name, p, p + 1)) continue;
                    appendf(w, "%s\t%lld\t%c", name.c_str(), (long long)p + 1, (ref && p < (int64_t)ref->size()) ? (*ref)[(size_t)p] : 'N');
                    for (int f = 0; f < nfn; ++f) {
                        const size_t d = (size_t)k * (size_t)nfn + (size_t)f;
                        appendf(w, "\t%d", nb[d] < 0 ? 0 : nb[d]);
                        for (int j = 0; j < 4; ++j) appendf(w, "\t%.9g", qs[d * 4 + (size_t)j]);
                        for (int j = 0; j < 25; ++j) appendf(w, "\t%.9g", p25[d * 25 + (size_t)j]);
                    }
                    appendf(w, "\n");
                }
                return;
            }
            if (!o.xcols.empty() && render_host_columns(w) != 0) { w.fail("mpileup"); return; }
            const size_t bound = (size_t)b200_mpileup_text_bound(w.eng.e, &mc);
            if (w.out.size() < bound + 64) w.out.resize(bound + 64);
            if (b200_mpileup_text(w.eng.e, &mc, w.out.data(), w.out.size(), &w.need) != 0) w.fail("mpileup");   // format and fetch in one call
        });
        return rc != 0 ? -1 : 1;
    };

    // contigs that yield at least one pileup column inside the region, in order (bam_plcmd.c:607-609)
    bool any = false;
    if (o.all < 2 || o.reg) {
        for (int tid = 0; tid < nref; ++tid) {
            if (o.reg && tid != tid0) continue;
            bool has = false;
            for (int i = 0; i < nfn; ++i) { if (!load_tid(fd[(size_t)i], tid, "mpileup")) return 1; if (tid < (int)fd[(size_t)i].by_tid.size() && !fd[(size_t)i].by_tid[(size_t)tid].empty()) has = true; }
            if (!has) continue;
            int rc = process_tid(tid, true);
            if (rc < 0) return 1;
            if (rc > 0) any = true;
        }
        // -aa with a region but no column at all: the region's empty rows (bam_plcmd.c:882-885)
        if (!any && o.all > 1 && o.reg && !o.gl) { if (process_tid(tid0, false) < 0) return 1; }
    } else {
        // -aa without a region: every contig, covered or not (bam_plcmd.c:612-636, :886-909)
        for (int tid = 0; tid < nref; ++tid) {
            bool has = false;
            for (int i = 0; i < nfn; ++i) { if (!load_tid(fd[(size_t)i], tid, "mpileup")) return 1; if (tid < (int)fd[(size_t)i].by_tid.size() && !fd[(size_t)i].by_tid[(size_t)tid].empty()) has = true; }
            int rc = has ? process_tid(tid, true) : 0;
            if (rc < 0) return 1;
            if (rc == 0 && !o.gl) { if (process_tid(tid, false) < 0) return 1; }
        }
    }
    if (o.out_fn) fclose(fp); else fflush(fp);
    return 0;
}

int main_mpileup(int argc, char **argv, bool gl)
{
    MpOpts o; o.gl = gl;
    const char *file_list = nullptr; bool use_orphan = false, has_index_file = false;
    int want_fields = 0; std::vector<std::string> want_tags;
    static const struct option lo[] = {
        {"rf", 1, 0, 1}, {"ff", 1, 0, 2}, {"incl-flags", 1, 0, 1}, {"excl-flags", 1, 0, 2}, {"output", 1, 0, 3},
        {"output-QNAME", 0, 0, 5}, {"output-qname", 0, 0, 5}, {"illumina1.3+", 0, 0, '6'}, {"count-orphans", 0, 0, 'A'},
        {"bam-list", 1, 0, 'b'}, {"no-BAQ", 0, 0, 'B'}, {"no-baq", 0, 0, 'B'}, {"adjust-MQ", 1, 0, 'C'}, {"adjust-mq", 1, 0, 'C'},
        {"max-depth", 1, 0, 'd'}, {"redo-BAQ", 0, 0, 'E'}, {"redo-baq", 0, 0, 'E'}, {"fasta-ref", 1, 0, 'f'}, {"reference", 1, 0, 'f'},
        {"exclude-RG", 1, 0, 'G'}, {"exclude-rg", 1, 0, 'G'}, {"positions", 1, 0, 'l'}, {"region", 1, 0, 'r'},
        {"ignore-RG", 0, 0, 'R'}, {"ignore-rg", 0, 0, 'R'}, {"min-MQ", 1, 0, 'q'}, {"min-mq", 1, 0, 'q'}, {"min-BQ", 1, 0, 'Q'},
        {"min-bq", 1, 0, 'Q'}, {"ignore-overlaps-removal", 0, 0, 'x'}, {"disable-overlap-removal", 0, 0, 'x'},
        {"output-mods", 0, 0, 'M'}, {"output-BP", 0, 0, 'O'}, {"output-bp", 0, 0, 'O'}, {"output-BP-5", 0, 0, 14}, {"output-bp-5", 0, 0, 14},
        {"output-MQ", 0, 0, 's'}, {"output-mq", 0, 0, 's'}, {"customized-index", 0, 0, 'X'}, {"reverse-del", 0, 0, 6},
        {"output-extra", 1, 0, 7}, {"output-sep", 1, 0, 8}, {"output-empty", 1, 0, 9}, {"no-output-ins", 0, 0, 10},
        {"no-output-ins-mods", 0, 0, 11}, {"no-output-del", 0, 0, 12}, {"no-output-ends", 0, 0, 13}, {0, 0, 0, 0} };
    int c;
    optind = 1;
    while ((c = getopt_long(argc, argv, "Af:r:l:q:Q:RC:Bd:b:o:EG:6OsxXaM", lo, nullptr)) >= 0) {
        switch (c) {
        case 'x': o.overlaps = false; break;
        case 1: o.rf = parse_flag(optarg); if (o.rf < 0) { fprintf(stderr, "Could not parse --rf %s\n", optarg); return 1; } break;
        case 2: o.ff = parse_flag(optarg); if (o.ff < 0) { fprintf(stderr, "Could not parse --ff %s\n", optarg); return 1; } break;
        case 3: case 'o': o.out_fn = optarg; break;
        case 'M':
            fprintf(stderr, "b200samtools mpileup: --output-mods is not available on the device path yet\n");
            return 1;
        case 5: want_fields |= 1 << 0; break;                      // --output-QNAME
        case 7: {                                                  // --output-extra FLAG,QNAME,TAG,...   (bam_plcmd.c:1013-1067)
            static const char *names[] = { "QNAME", "FLAG", "RNAME", "POS", "MAPQ", "RNEXT", "PNEXT", "RLEN" };
            std::string a = optarg; size_t st = 0;
            while (st <= a.size()) {
                size_t e2 = a.find(',', st); if (e2 == std::string::npos) e2 = a.size();
                const std::string t = a.substr(st, e2 - st);
                int fld = -1;
                for (int k = 0; k < 8; ++k) if (t == names[k]) fld = k;
                if (fld >= 0) want_fields |= 1 << fld;
                else if (t.size() == 2) { if (std::find(want_tags.begin(), want_tags.end(), t) == want_tags.end()) want_tags.push_back(t); }
                else if (t == "MAPQ" || t.empty()) {}
                else { fprintf(stderr, "[mpileup] unknown field or bad tag name in --output-extra: \"%s\"\n", t.c_str()); return 1; }
                st = e2 + 1;
            }
            break;
        }
        case 6: o.rev_del = 1; break;
        case 8: o.x_sep = optarg[0]; break;                      // --output-sep
        case 9: o.x_empty = optarg[0]; break;                    // --output-empty
        case 11: break;
        case 10: o.no_ins++; break;
        case 12: o.no_del++; break;
        case 13: o.no_ends = 1; break;
        case 14: o.out_qpos5 = 1; break;
        case 'f': o.fa = Fasta::load(optarg); if (!o.fa) { fprintf(stderr, "[E::fai_load] failed to open %s\n", optarg); return 1; } o.fa_fn = optarg; break;
        case 'd': o.max_depth = atoi(optarg); break;
        case 'r': o.reg = optarg; break;
        case 'l': o.bed = Bed::load(optarg); if (!o.bed) { fprintf(stderr, "samtools mpileup: Could not read file \"%s\"\n", optarg); return 1; } break;
        case 'B': o.realn = false; break;
        case 'X': has_index_file = true; break;
        case 'E': o.redo_baq = true; break;
        case '6': o.illumina13 = true; break;
        case 'R': o.ignore_rg = true; break;
        case 's': o.out_mapq = 1; break;
        case 'O': o.out_qpos = 1; break;
        case 'C': o.capQ = atoi(optarg); break;
        case 'q': o.min_mq = atoi(optarg); break;
        case 'Q': o.min_baseQ = atoi(optarg); break;
        case 'b': file_list = optarg; break;
        case 'A': use_orphan = true; break;
        case 'G': {
            o.have_rg = true;
            if (FILE *f = fopen(optarg, "r")) { char b[1024]; while (fscanf(f, "%1023s", b) > 0) o.rg_excl.insert(b); fclose(f); }
            else fprintf(stderr, "[bam_mpileup] Fail to open file %s. Continue anyway.\n", optarg);
            break;
        }
        case 'a': o.all++; break;
        default: fprintf(stderr, "\nUsage: samtools mpileup [options] in1.bam [in2.bam [...]]\n"); return 1;
        }
    }
    if (!o.realn && o.redo_baq) { fprintf(stderr, "Error: The -B option cannot be combined with -E\n"); return 1; }
    if (use_orphan) o.no_orphan = false;
    {   // record fields print in the order of the MPLP_PRINT_* bits (bam_plcmd.c:185-196,728-795), tags after them in the order given
        static const char *names[] = { "QNAME", "FLAG", "RNAME", "POS", "MAPQ", "RNEXT", "PNEXT", "RLEN" };
        for (int k = 0; k < 8; ++k) if (want_fields & (1 << k)) o.xcols.push_back(names[k]);
        o.n_xfields = (int)o.xcols.size();
        for (const std::string &t : want_tags) o.xcols.push_back(t);
        if (o.xcols.size() > 16) { fprintf(stderr, "b200samtools mpileup: at most 16 --output-extra columns\n"); return 1; }
        if (o.n_xfields && o.out_qpos5) { fprintf(stderr, "b200samtools mpileup: --output-BP-5 together with --output-QNAME/--output-extra fields is not available on the device path\n"); return 1; }
    }
    if (argc == 1) { fprintf(stderr, "\nUsage: samtools mpileup [options] in1.bam [in2.bam [...]]\n"); return 1; }
    std::vector<std::string> fn;
    if (file_list) {
        if (has_index_file) { fprintf(stderr, "Error: The -b option cannot be combined with -X\n"); return 1; }
        if (!read_file_list(file_list, fn)) return 1;
    } else {
        int n = argc - optind;
        if (has_index_file) { if (n % 2) { fprintf(stderr, "Odd number of filenames detected! Each BAM file should have an index file\n"); return 1; } n /= 2; }
        for (int i = 0; i < n; ++i) fn.push_back(argv[optind + i]);
    }
    return run_mpileup(o, fn);
}

// ----------------------------------------------------------------------------- depth
int main_depth(int argc, char **argv)
{
    int flag = F_UNMAP | F_SECONDARY | F_DUP | F_QCFAIL, incl = 0, require = 0, min_qual = 0, min_mqual = 0, min_len = 0;
    int skip_del = 1, header = 0, all_pos = 0, remove_overlaps = 0, tmp;
    const char *reg = nullptr, *file_list = nullptr, *out_fn = nullptr;
    std::unique_ptr<Bed> bed;
    static const struct option lo[] = { {"min-MQ", 1, 0, 'Q'}, {"min-mq", 1, 0, 'Q'}, {"min-BQ", 1, 0, 'q'}, {"min-bq", 1, 0, 'q'},
        {"excl-flags", 1, 0, 'G'}, {"incl-flags", 1, 0, 1}, {"require-flags", 1, 0, 2}, {"threads", 1, 0, '@'}, {0, 0, 0, 0} };
    int c;
    optind = 1;
    while ((c = getopt_long(argc, argv, "@:q:Q:JHd:m:l:g:G:o:ar:Xf:b:s", lo, nullptr)) >= 0) {
        switch (c) {
        case 'a': all_pos++; break;
        case 'b': bed = Bed::load(optarg); if (!bed) { fprintf(stderr, "samtools depth: Could not read file \"%s\"\n", optarg); return 1; } break;
        case 'f': file_list = optarg; break;
        case 'd': case 'm': case '@': case 'X': break;
        case 'g': tmp = parse_flag(optarg); if (tmp < 0) { fprintf(stderr, "samtools depth: Unknown flag '%s'\n", optarg); return 1; } flag &= ~tmp; break;
        case 'G': tmp = parse_flag(optarg); if (tmp < 0) { fprintf(stderr, "samtools depth: Unknown flag '%s'\n", optarg); return 1; } flag |= tmp; break;
        case 1: tmp = parse_flag(optarg); if (tmp < 0) { fprintf(stderr, "samtools depth: Unknown flag '%s'\n", optarg); return 1; } incl |= tmp; break;
        case 2: tmp = parse_flag(optarg); if (tmp < 0) { fprintf(stderr, "samtools depth: Unknown flag '%s'\n", optarg); return 1; } require |= tmp; break;
        case 'l': min_len = atoi(optarg); break;
        case 'H': header = 1; break;
        case 'q': min_qual = atoi(optarg); break;
        case 'Q': min_mqual = atoi(optarg); break;
        case 'J': skip_del = 0; break;
        case 'o': out_fn = optarg; break;
        case 'r': reg = optarg; break;
        case 's': remove_overlaps = 1; break;
        default: fprintf(stderr, "Usage: samtools depth [options] in.bam [in.bam ...]\n"); return 1;
        }
    }
    std::vector<std::string> fn;
    if (file_list) { if (!read_file_list(file_list, fn)) return 1; }
    else for (int i = optind; i < argc; ++i) fn.push_back(argv[i]);
    if (fn.empty()) { fprintf(stderr, "Usage: samtools depth [options] in.bam [in.bam ...]\n"); return 1; }
    const int nfn = (int)fn.size();
    std::vector<FileData> fd((size_t)nfn);
    int tid0 = 0; int64_t beg0 = 0, end0 = POS_MAX;
    for (int i = 0; i < nfn; ++i) {
        int t = 0; int64_t b = 0, e = POS_MAX;
        fd[(size_t)i].rd = nullptr;
        if (!load_file(fn[(size_t)i], "", reg, fd[(size_t)i], t, b, e, "depth")) return 1;
        if (i == 0) { tid0 = t; beg0 = b; end0 = e; }
    }
    const Header &h = fd[0].rd->header();
    FILE *fp = out_fn ? fopen(out_fn, "w") : stdout;
    if (!fp) { fprintf(stderr, "samtools depth: Cannot open \"%s\" for writing.\n", out_fn); return 1; }
    if (header) { fprintf(fp, "#CHROM\tPOS"); for (auto &f : fn) fprintf(fp, "\t%s", f.c_str()); fputc('\n', fp); }
    Workers workers;      // window workers (worker_devices())
    if (!make_workers(workers, nfn, true)) return 1;
    b200_stage_conf_t sc; memset(&sc, 0, sizeof sc);
    sc.mode = B200_MODE_DEPTH; sc.d_flag_excl = flag; sc.d_flag_incl = incl; sc.d_flag_require = require; sc.d_min_mapq = min_mqual;
    sc.d_min_len = min_len; sc.d_remove_overlaps = remove_overlaps;
    b200_depth_conf_t dc; memset(&dc, 0, sizeof dc);
    dc.min_qual = min_qual; dc.count_del = !skip_del; dc.all = all_pos;
    std::vector<int64_t> bb, be;
    // depth -s: the reference keeps one qname -> end-position hash PER FILE for the whole run (bam2depth.c:598-623),
    // i.e. across reference sequences, and only records that pass the read filters take part.  It is replayed here
    // in file order (name hashing is host work anyway) and handed to the engine as one clip coordinate per record.
    std::vector<std::vector<std::vector<int64_t>>> clips((size_t)nfn);
    std::vector<std::unordered_map<std::string, int64_t>> seen((size_t)nfn);   // the per-file name hash, alive across reference sequences
    auto qlen_used = [](const Record &r) -> int64_t {
        int64_t l;
        const int n = (int)r.cigar.size();
        if (r.l_qseq) {
            l = r.l_qseq; int kl, kr;
            for (kl = 0; kl < n; kl++) { if ((r.cigar[(size_t)kl] & 0xf) == 4) l -= r.cigar[(size_t)kl] >> 4; else break; }
            for (kr = n - 1; kr > kl; kr--) { if ((r.cigar[(size_t)kr] & 0xf) == 4) l -= r.cigar[(size_t)kr] >> 4; else break; }
        } else { l = 0; for (uint32_t c : r.cigar) { int op = c & 0xf; if (op == 0 || op == 1 || op == 7 || op == 8) l += c >> 4; } }
        return l;
    };
    // records of reference sequence tid of file i are in: replay the hash over them (file order = the order the reference sees them)
    auto replay_clips = [&](int i, int tid) {
        if (!remove_overlaps || tid >= (int)fd[(size_t)i].by_tid.size()) return;
        clips[(size_t)i].resize(fd[(size_t)i].by_tid.size());
        for (int t = 0; t < tid; ++t) std::vector<int64_t>().swap(clips[(size_t)i][(size_t)t]);
        auto &cv = clips[(size_t)i][(size_t)tid];
        cv.clear();
        for (const Record &r : fd[(size_t)i].by_tid[(size_t)tid]) {
            int64_t clip = 0;
            const bool pass = !(r.flag & flag) && !(incl && (r.flag & incl) == 0) && (r.flag & require) == require &&
                              r.mapq >= min_mqual && !(min_len && qlen_used(r) < min_len);
            if (pass && (r.flag & F_PAIRED) && !(r.flag & F_MUNMAP)) {
                auto it = seen[(size_t)i].find(r.qname);
                if (it == seen[(size_t)i].end()) { const int64_t e = r.endpos(); if (r.mpos == -1 || (r.tid == r.mtid && r.mpos <= e)) seen[(size_t)i].emplace(r.qname, e); }
                else { clip = it->second; seen[(size_t)i].erase(it); }
            }
            cv.push_back(clip);
        }
    };
    auto process_tid = [&](int tid, bool with_reads) -> int {
        const std::string &name = h.names[(size_t)tid];
        if (bed) { bed->merged(name, bb, be); dc.bed_beg = bb.data(); dc.bed_end = be.data(); dc.n_bed = (int)bb.size(); dc.bed_active = 1; }
        int64_t lo = 0, hi = 0;
        if (!column_range(fd, tid, h.lens[(size_t)tid], beg0, end0, all_pos, with_reads, lo, hi)) return 0;
        const Windows wins = column_windows(lo, hi);
        auto stage = [&](WinWorker &w, int64_t wb, int64_t we, b200_stage_stats_t &st) {
            return stage_window(w, h, tid, nullptr, sc, wb, we, nullptr, "depth", st, [&](int i) {
                if (!with_reads || tid >= (int)fd[(size_t)i].by_tid.size()) return;
                std::vector<Record> &v = fd[(size_t)i].by_tid[(size_t)tid];
                window_records(v, w.cursor[(size_t)i], wb, we, w.sel);
                for (size_t j : w.sel) {
                    w.pb.add(v[j], 0, false);
                    if (remove_overlaps) w.pb.depth_clip.push_back(clips[(size_t)i][(size_t)tid][j]);
                }
            });
        };
        if (with_reads) {   // a contig no record of which survives the filters is never "seen" (bam2depth.c:255-263): decide before writing
            WinWorker &w = *workers[0];
            w.rewind();
            bool seen = false;
            for (size_t k = 0; k < wins.size() && !seen; ++k) {
                b200_stage_stats_t st;
                if (stage(w, wins[k].first, wins[k].second, st) != 0) { fprintf(stderr, "%s\n", w.err.c_str()); return -1; }
                seen = st.n_kept > 0;
            }
            if (!seen) return 0;
        }
        // the empty rows of a contig without reads run on worker 0 alone
        const int rc = run_window_rounds(workers, wins, with_reads ? workers.size() : 1, fp, [&](WinWorker &w, int64_t wb, int64_t we) {
            b200_stage_stats_t st;
            if (stage(w, wb, we, st) != 0) return;
            const size_t bound = (size_t)b200_depth_text_bound(w.eng.e);
            if (w.out.size() < bound + 64) w.out.resize(bound + 64);
            if (b200_depth_text(w.eng.e, &dc, w.out.data(), w.out.size(), &w.need) != 0) w.fail("depth");
        });
        return rc != 0 ? -1 : 1;
    };
    const int nref = h.n_ref();
    bool any = false;
    for (int tid = 0; tid < nref; ++tid) {
        if (reg && tid != tid0) continue;
        bool has = false;
        for (int i = 0; i < nfn; ++i) {
            if (!load_tid(fd[(size_t)i], tid, "depth")) return 1;
            replay_clips(i, tid);
            if (tid < (int)fd[(size_t)i].by_tid.size() && !fd[(size_t)i].by_tid[(size_t)tid].empty()) has = true;
        }
        int rc = has ? process_tid(tid, true) : 0;
        if (rc < 0) return 1;
        if (rc > 0) any = true;
        else if (all_pos > 1 && !reg) { if (process_tid(tid, false) < 0) return 1; }   // -aa: unused references (bam2depth.c:255-263)
    }
    if (!any && all_pos && reg) { if (process_tid(tid0, false) < 0) return 1; }            // bam2depth.c:267-270
    if (out_fn) fclose(fp); else fflush(fp);
    return 0;
}

// ----------------------------------------------------------------------------- coverage
int main_coverage(int argc, char **argv)
{
    int max_depth = 1000000, min_baseQ = 0, min_mapQ = 0, min_len = 0, mindepth = 1;
    int fail_flags = F_UNMAP | F_SECONDARY | F_QCFAIL | F_DUP, required_flags = 0;
    const char *reg = nullptr, *file_list = nullptr, *out_fn = nullptr;
    bool print_header = true;
    // histogram views (coverage.c:391-402): -m, -A (ASCII glyphs), -D (depth instead of breadth), -w bins
    bool want_hist = false, utf = true, plot_depth = false, full_width = true;
    int n_bins_opt = 50;
    static const struct option lo[] = { {"rf", 1, 0, 1}, {"ff", 1, 0, 2}, {"incl-flags", 1, 0, 1}, {"excl-flags", 1, 0, 2},
        {"bam-list", 1, 0, 'b'}, {"min-read-len", 1, 0, 'l'}, {"min-MQ", 1, 0, 'q'}, {"min-mq", 1, 0, 'q'}, {"min-BQ", 1, 0, 'Q'},
        {"min-bq", 1, 0, 'Q'}, {"histogram", 0, 0, 'm'}, {"ascii", 0, 0, 'A'}, {"plot-depth", 0, 0, 'D'}, {"output", 1, 0, 'o'},
        {"no-header", 0, 0, 'H'}, {"n-bins", 1, 0, 'w'}, {"region", 1, 0, 'r'}, {"help", 0, 0, 'h'}, {"depth", 1, 0, 'd'},
        {"min-depth", 1, 0, 3}, {0, 0, 0, 0} };
    int c, i;
    optind = 1; opterr = 0;
    while ((c = getopt_long(argc, argv, "Ao:l:q:Q:hHw:r:b:md:D", lo, nullptr)) != -1) {
        switch (c) {
        case 1: if ((required_flags = parse_flag(optarg)) < 0) { fprintf(stderr, "Could not parse --rf %s\n", optarg); return 1; } break;
        case 2: if ((fail_flags = parse_flag(optarg)) < 0) { fprintf(stderr, "Could not parse --ff %s\n", optarg); return 1; } break;
        case 3: if ((i = atoi(optarg)) > 0) mindepth = i; break;
        case 'o': out_fn = optarg; full_width = false; break;
        case 'l': min_len = atoi(optarg); break;
        case 'q': min_mapQ = atoi(optarg); break;
        case 'Q': min_baseQ = atoi(optarg); break;
        case 'd': max_depth = atoi(optarg); break;
        case 'r': reg = optarg; break;
        case 'b': file_list = optarg; break;
        case 'H': print_header = false; break;
        case 'm': want_hist = true; break;
        case 'A': utf = false; want_hist = true; break;
        case 'D': plot_depth = true; want_hist = true; break;
        case 'w': n_bins_opt = atoi(optarg); full_width = false; want_hist = true; break;
        default: fprintf(stderr, "Usage: samtools coverage [options] in1.bam [in2.bam [...]]\n"); return 1;
        }
    }
    if (n_bins_opt <= 0 || full_width) {     // terminal width - 40, at least 40 (coverage.c:437-461)
        int columns = 0;
        if (const char *ec = getenv("COLUMNS")) columns = atoi(ec);
        else { struct winsize ws; if (ioctl(2, TIOCGWINSZ, &ws) == 0) columns = ws.ws_col; }
        n_bins_opt = columns > 60 ? columns - 40 : 40;
    }
    std::vector<std::string> fn;
    if (file_list) { if (!read_file_list(file_list, fn)) return 1; }
    else for (i = optind; i < argc; ++i) fn.push_back(argv[i]);
    if (fn.empty()) { fprintf(stderr, "Usage: samtools coverage [options] in1.bam [in2.bam [...]]\n"); return 1; }
    const int nfn = (int)fn.size();
    std::vector<FileData> fd((size_t)nfn);
    int tid0 = -1; int64_t beg0 = 0, end0 = POS_MAX;
    for (i = 0; i < nfn; ++i) {
        int t = 0; int64_t b = 0, e = POS_MAX;
        if (!load_file(fn[(size_t)i], "", reg, fd[(size_t)i], t, b, e, "coverage")) return 1;
        if (i == 0 && reg) { tid0 = t; beg0 = b; end0 = e; }
    }
    const Header &h = fd[0].rd->header();
    FILE *fp = (out_fn && strcmp(out_fn, "-")) ? fopen(out_fn, "w") : stdout;
    if (!fp) { fprintf(stderr, "samtools coverage: Cannot open \"%s\" for writing.\n", out_fn); return 1; }
    Workers workers;
    if (!make_workers(workers, nfn, false)) return 1;
    const int nref = h.n_ref();
    struct Row { b200_coverage_sums_t s; uint64_t n_sel = 0, sum_mq = 0, n_reads = 0; bool covered = false; int64_t beg = 0, end = 0, bin_width = 1; int n_bins = 0; std::vector<uint32_t> hist; };
    std::vector<Row> rows((size_t)nref);
    b200_stage_conf_t sc; memset(&sc, 0, sizeof sc);
    sc.mode = B200_MODE_COVERAGE; sc.rflag_filter = fail_flags; sc.rflag_require = required_flags; sc.min_mq = min_mapQ; sc.c_min_len = min_len;
    sc.max_depth = max_depth > 0 ? max_depth : (max_depth == 0 ? INT_MAX : 8000);
    b200_coverage_conf_t cc; cc.min_baseQ = min_baseQ; cc.min_depth = mindepth;
    bool warn = false;
    std::vector<int> order;   // contigs in the order their first column appears
    MaxDepthCarry md;
    for (int tid = 0; tid < nref; ++tid) {
        Row &rw = rows[(size_t)tid];
        memset(&rw.s, 0, sizeof rw.s);
        rw.beg = 0; rw.end = h.lens[(size_t)tid];
        if (reg && tid == tid0) { rw.beg = beg0; rw.end = end0 == POS_MAX ? h.lens[(size_t)tid] : end0; }
        if (want_hist) {      // bins of this reference sequence (coverage.c:552-563, :609-610)
            const int64_t span = rw.end - rw.beg;
            int64_t nb = (int64_t)n_bins_opt > span ? span : (int64_t)n_bins_opt;
            rw.n_bins = (int)nb; rw.bin_width = span / (nb > 0 ? nb : 1);
            rw.hist.assign((size_t)(nb > 0 ? nb : 0), 0u);
        }
        bool has = false;
        for (i = 0; i < nfn; ++i) { if (!load_tid(fd[(size_t)i], tid, "coverage")) return 1; if (tid < (int)fd[(size_t)i].by_tid.size() && !fd[(size_t)i].by_tid[(size_t)tid].empty()) has = true; }
        if (!has) continue;
        // column windows of [rw.beg, rw.end): the sums add up.  Every record is counted once in the read statistics
        // (coverage.c:185-193): a read that reaches in from the previous window is staged again as halo (B200_RB_HALO);
        // the first / last window also take the records that lie before / beyond the region.
        // A window that continues an earlier one also stages the records ending right at its start (the closed intervals
        // of the -d rule; they cover none of its columns), and where the rule may fire the windows hand their verdicts on.
        const Windows wins = column_windows(rw.beg, rw.end);
        md.reset(fd, tid, wins.size() > 1 && max_stacked_records(fd, tid) > (int64_t)sc.max_depth);
        const int rc = run_window_rounds(workers, wins, 1, fp, [&](WinWorker &w, int64_t wb, int64_t we) {
            const bool first_w = wb == rw.beg, last_w = we >= rw.end;
            b200_stage_stats_t st;
            if (stage_window(w, h, tid, nullptr, sc, wb, we, &md, "coverage", st, [&](int i) {
                    if (tid >= (int)fd[(size_t)i].by_tid.size()) return;
                    std::vector<Record> &v = fd[(size_t)i].by_tid[(size_t)tid];
                    window_records(v, w.cursor[(size_t)i], first_w ? INT64_MIN : wb, last_w ? POS_MAX : we, w.sel, !first_w);
                    for (size_t j : w.sel) w.pb.add(v[j], (uint8_t)(((!first_w && v[j].pos < wb) ? B200_RB_HALO : 0) | md.add(i, j)), false);
                }) != 0) return;
            rw.n_sel += st.n_selected_reads; rw.sum_mq += st.summed_mapq; rw.n_reads += st.n_reads;
            // a column exists as soon as one kept read has a non-empty reference span (before the region test)
            if (st.n_kept > 0) {
                b200_coverage_sums_t ws;
                if (b200_coverage(w.eng.e, &cc, &ws) != 0) { w.fail("coverage"); return; }
                rw.s.n_covered_bases += ws.n_covered_bases; rw.s.summed_coverage += ws.summed_coverage; rw.s.summed_baseQ += ws.summed_baseQ;
                rw.s.quality_bases += ws.quality_bases; rw.s.missing_qual += ws.missing_qual;
                if (!rw.covered) { rw.covered = true; order.push_back(tid); }   // refined: zero-span-only contigs are vanishingly rare
                if (ws.missing_qual) warn = true;
                if (want_hist && rw.n_bins > 0 && rw.bin_width > 0 &&
                    b200_coverage_hist(w.eng.e, &cc, rw.beg, rw.bin_width, rw.n_bins, plot_depth ? 1 : 0, rw.hist.data()) != 0) w.fail("coverage");
            }
        });
        if (rc != 0) return 1;
    }
    auto print_row = [&](int tid) {
        const Row &r = rows[(size_t)tid];
        if (print_header) { fputs("#rname\tstartpos\tendpos\tnumreads\tcovbases\tcoverage\tmeandepth\tmeanbaseq\tmeanmapq\n", fp); print_header = false; }
        fputs(h.names[(size_t)tid].c_str(), fp);
        double region_len = (double)r.end - r.beg;
        fprintf(fp, "\t%lld\t%lld\t%u\t%llu\t%g\t%g\t%.3g\t%.3g\n", (long long)r.beg + 1, (long long)r.end, (unsigned)r.n_sel,
                (unsigned long long)r.s.n_covered_bases, 100.0 * r.s.n_covered_bases / region_len, r.s.summed_coverage / region_len,
                r.s.quality_bases > 0 ? r.s.summed_baseQ / (double)r.s.quality_bases : 0,
                r.n_sel > 0 ? r.sum_mq / (double)r.n_sel : 0);
    };
    // ---- histogram view (coverage.c:223-304): ten rows of block glyphs over the bins, the row's statistic to the right
    auto fmt_bp = [](double bp, char *buf) -> char * {
        static const char *unit[] = {"", "K", "M", "G", "T"};
        int u = 0;
        for (; bp >= 1000 && u < 4; ++u) bp /= 1000;
        snprintf(buf, 48, "%.*f%s", u, bp, unit[u]);
        return buf;
    };
    auto centred = [](const char *t, char *buf, int width) -> char * {
        const int len = (int)strlen(t), pad = (width - len) / 2, odd = (width - len) % 2;
        if (pad >= 1) snprintf(buf, 96, " %*s%*s", len + pad, t, pad - 1 + odd, " ");
        else snprintf(buf, 96, "%s", t);
        return buf;
    };
    auto print_hist = [&](int tid) {
        static const char *const g8[8] = {"\xE2\x96\x81", "\xE2\x96\x82", "\xE2\x96\x83", "\xE2\x96\x84", "\xE2\x96\x85", "\xE2\x96\x86", "\xE2\x96\x87", "\xE2\x96\x88"};
        static const char *const g2[2] = {".", ":"};
        const Row &r = rows[(size_t)tid];
        const int n_rows = 10, steps = utf ? 8 : 2, nb = r.n_bins;
        const char *const *glyph = utf ? g8 : g2;
        const char *bar = utf ? "\xE2\x94\x82" : "|";
        const double region_len = (double)(r.end - r.beg);
        std::vector<double> val((size_t)std::max(nb, 1), 0.0);
        double top = 0.0;
        for (int k = 0; k < nb; ++k) {
            val[(size_t)k] = (uint32_t)((plot_depth ? 1u : 100u) * r.hist[(size_t)k]) / (double)r.bin_width;   // 32-bit product, like the reference
            top = std::max(top, val[(size_t)k]);
        }
        char b1[64], b2[128];
        fprintf(fp, "%s (%sbp)\n", h.names[(size_t)tid].c_str(), fmt_bp((double)h.lens[(size_t)tid], b1));
        const double step = top / n_rows;
        for (int row = n_rows - 1; row >= 0; --row) {
            const double base = step * row;
            if (plot_depth) fprintf(fp, ">%8.1f ", row * step); else fprintf(fp, ">%7.2f%% ", base);
            fputs(bar, fp);
            for (int k = 0; k < nb; ++k) {
                int g = steps - 1;                      // all-zero histogram: the reference divides 0 by 0; its x86-64 build prints the full block
                if (step != 0.0) { g = (int)round(steps * (val[(size_t)k] - base) / step) - 1; if (g >= steps) g = steps - 1; }
                if (g < 0) fputc(' ', fp); else fputs(glyph[g], fp);
            }
            fputs(bar, fp); fputc(' ', fp);
            const unsigned n_sel = (unsigned)r.n_sel, n_all = (unsigned)r.n_reads;
            switch (row) {
            case 9: fprintf(fp, "Number of reads: %u", n_sel); break;
            case 8: if (n_all - n_sel > 0) fprintf(fp, "    (%i filtered)", (int)(n_all - n_sel)); break;
            case 7: fprintf(fp, "Covered bases:   %sbp", fmt_bp((double)r.s.n_covered_bases, b1)); break;
            case 6: fprintf(fp, "Percent covered: %.4g%%", 100.0 * r.s.n_covered_bases / region_len); break;
            case 5: fprintf(fp, "Mean coverage:   %.3gx", r.s.summed_coverage / region_len); break;
            case 4: fprintf(fp, "Mean baseQ:      %.3g", r.s.quality_bases > 0 ? r.s.summed_baseQ / (double)r.s.quality_bases : 0); break;
            case 3: fprintf(fp, "Mean mapQ:       %.3g", r.sum_mq / (double)r.n_sel); break;
            case 1: fprintf(fp, "Histo bin width: %sbp", fmt_bp((double)r.bin_width, b1)); break;
            case 0: if (plot_depth) fprintf(fp, "Histo max cov:   %.5g", top); else fprintf(fp, "Histo max bin:   %.5g%%", top); break;
            default: break;
            }
            fputc('\n', fp);
        }
        fprintf(fp, "     %s", centred(fmt_bp((double)(r.beg + 1), b1), b2, 10));
        for (int k = 10; k < 10 * (nb / 10); k += 10) fprintf(fp, "%s", centred(fmt_bp((double)(r.beg + r.bin_width * k), b1), b2, 10));
        fprintf(fp, "%*s%s", nb % 10, " ", centred(fmt_bp((double)r.end, b1), b2, 10));
        fputc('\n', fp);
    };
    if (want_hist) {     // one block per reference sequence that has columns, blank line between blocks (coverage.c:592-597, :672-675)
        for (size_t k = 0; k < order.size(); ++k) { if (k) fputc('\n', fp); print_hist(order[k]); }
        if (order.empty() && reg && *reg != '*' && tid0 >= 0) print_hist(tid0);
    } else {
        for (int tid : order) print_row(tid);
        if (order.empty() && reg && *reg != '*' && tid0 >= 0) print_row(tid0);
        if (!reg) for (int tid = 0; tid < nref; ++tid) if (!rows[(size_t)tid].covered) print_row(tid);
    }
    if (warn) fprintf(stderr, "samtools coverage: Warning:  Missing quality values in alignments.  Mean base quality calculated only on available values.\n");
    if (fp != stdout) fclose(fp); else fflush(fp);
    return 0;
}

// ----------------------------------------------------------------------------- bedcov
// `samtools bedcov` (bedcov.c): for every BED line the reference opens an index query over [beg,end) and runs the
// multi-file pileup iterator with the column reducers of bedcov.c:316-331.  Here every line stages the records that
// overlap its interval (B200_MODE_COVERAGE read filters: the -g/-G flag set and -Q) and b200_bedcov() reduces the window
// on the device.  BED lines may name the reference sequences in any order, so the inputs are decoded completely up front
// (the reference has random access through the BAI; this driver has no index reader).
int main_bedcov(int argc, char **argv)
{
    int c, min_mapQ = 0, skip_DN = 0, do_rcount = 0, min_depth = -1, max_depth = INT_MAX, print_header = 0, hdr = 0, status = 0, tflags;
    int flags = F_UNMAP | F_SECONDARY | F_QCFAIL | F_DUP;
    static const struct option lo[] = { {"min-MQ", 1, 0, 'Q'}, {"min-mq", 1, 0, 'Q'}, {"max-depth", 1, 0, 1000}, {0, 0, 0, 0} };
    optind = 1;
    while ((c = getopt_long(argc, argv, "Q:Xg:G:jd:Hc", lo, nullptr)) >= 0) {
        switch (c) {
        case 'Q': min_mapQ = atoi(optarg); break;
        case 'X': break;
        case 'c': do_rcount = 1; break;
        case 'H': print_header = 1; break;
        case 'g': tflags = parse_flag(optarg); if (tflags < 0 || tflags > 4095) { fprintf(stderr, "[bedcov] Flag value \"%s\" is not supported\n", optarg); return 1; } flags &= ~tflags; break;
        case 'G': tflags = parse_flag(optarg); if (tflags < 0 || tflags > 4095) { fprintf(stderr, "[bedcov] Flag value \"%s\" is not supported\n", optarg); return 1; } flags |= tflags; break;
        case 'j': skip_DN = 1; break;
        case 'd': min_depth = atoi(optarg); break;
        case 1000: max_depth = atoi(optarg); break;
        default: fprintf(stderr, "Usage: samtools bedcov [options] <in.bed> <in1.bam> [...]\n"); return 1;
        }
    }
    if (optind + 2 > argc) { fprintf(stderr, "Usage: samtools bedcov [options] <in.bed> <in1.bam> [...]\n"); return 1; }
    const int n = argc - optind - 1;
    char **fn = argv + optind + 1;
    if (!print_header) hdr = 1;
    std::vector<FileData> fd((size_t)n);
    for (int i = 0; i < n; ++i) {
        int t = 0; int64_t b = 0, e = POS_MAX;
        if (!load_file(fn[i], "", nullptr, fd[(size_t)i], t, b, e, "bedcov")) { fprintf(stderr, "ERROR: fail to open index BAM file '%s'\n", fn[i]); return 2; }
        fd[(size_t)i].keep_all = true;
        for (int tid = 0; tid < fd[(size_t)i].rd->header().n_ref(); ++tid) if (!load_tid(fd[(size_t)i], tid, "bedcov")) return 2;
    }
    const Header &h = fd[0].rd->header();
    // per file and reference sequence: running maximum of the record ends, so that the first record that can reach an
    // interval is found by binary search
    std::vector<std::vector<std::vector<int64_t>>> runmax((size_t)n);
    for (int i = 0; i < n; ++i) {
        runmax[(size_t)i].resize(fd[(size_t)i].by_tid.size());
        for (size_t t = 0; t < fd[(size_t)i].by_tid.size(); ++t) {
            int64_t m = INT64_MIN;
            for (const Record &r : fd[(size_t)i].by_tid[t]) { m = std::max(m, r.endpos()); runmax[(size_t)i][t].push_back(m); }
        }
    }
    gzFile fp = gzopen(argv[optind], "rb");
    if (!fp) { fprintf(stderr, "[bedcov] can't open BED file '%s': %s\n", argv[optind], strerror(errno)); return 2; }
    Engine eng;
    if (!eng.init()) return 1;
    b200_stage_conf_t sc; memset(&sc, 0, sizeof sc);
    sc.mode = B200_MODE_COVERAGE; sc.rflag_filter = flags; sc.min_mq = min_mapQ; sc.max_depth = min_depth > max_depth ? min_depth : max_depth;
    auto output_header = [&](const char *hline, int fields) {
        static const char *bedcols[] = { "chrom", "chromStart", "chromEnd", "name", "score", "strand", "thickStart", "thickEnd", "itemRgb", "blockCount", "blockSizes", "blockStarts" };
        if (hline) fputs(hline, stdout);
        else for (int i = 0; i < fields; ++i) printf("%s%s", i ? "\t" : "#", i < 12 ? bedcols[i] : ".");
        for (int i = 0; i < n; ++i) printf("\t%s_cov", fn[i]);
        if (min_depth >= 0) for (int i = 0; i < n; ++i) printf("\t%s_depth", fn[i]);
        if (do_rcount) for (int i = 0; i < n; ++i) printf("\t%s_count", fn[i]);
        putchar('\n');
    };
    PackedBatch pb;
    std::vector<uint64_t> cnt((size_t)n), pcov((size_t)n), rcnt((size_t)n);
    std::vector<uint8_t> keep;
    std::vector<char> line(1 << 16);
    while (gzgets(fp, line.data(), (int)line.size())) {
        size_t l = strlen(line.data());
        while (l && (line[l - 1] == '\n' || line[l - 1] == '\r')) line[--l] = 0;
        if (l == 0) continue;
        if (line[0] == '#') { if (!hdr && !strncmp(line.data(), "#chrom", 6)) { output_header(line.data(), -1); hdr = 1; } continue; }
        if (!strncmp(line.data(), "track ", 6) || !strncmp(line.data(), "browser ", 8)) continue;
        if (!hdr) { int fields = 0; for (const char *t = line.data(); *t; ++t) if (*t == '\t') fields++; output_header(nullptr, fields + 1); hdr = 1; }
        char *p = line.data();
        while (*p && !isspace((unsigned char)*p)) ++p;
        long long beg = 0, end = 0; int tid = -1;
        bool ok = *p != 0;
        if (ok) { const char sv = *p; *p = 0; tid = h.name2tid(line.data()); *p = sv; ok = tid >= 0; }
        if (ok) ok = sscanf(p + 1, "%lld %lld", &beg, &end) >= 2 && end >= beg;
        if (!ok) { fprintf(stderr, "Errors in BED line '%s'\n", line.data()); status = 2; continue; }
        std::fill(cnt.begin(), cnt.end(), 0); std::fill(pcov.begin(), pcov.end(), 0); std::fill(rcnt.begin(), rcnt.end(), 0);
        if (end > beg) {
            pb.clear();
            for (int i = 0; i < n; ++i) {
                pb.begin_file();
                if (tid >= (int)fd[(size_t)i].by_tid.size()) continue;
                const std::vector<Record> &v = fd[(size_t)i].by_tid[(size_t)tid];
                const std::vector<int64_t> &rm = runmax[(size_t)i][(size_t)tid];
                size_t j = (size_t)(std::upper_bound(rm.begin(), rm.end(), (int64_t)beg) - rm.begin());   // first record whose running max end exceeds beg
                for (; j < v.size() && v[j].pos < end; ++j) if (v[j].endpos() > beg) pb.add(v[j], 0, false);
            }
            pb.finish();
            if (!pb.pos.empty()) {
                b200_batch_t batch = pb.view(tid, h.lens[(size_t)tid], h.names[(size_t)tid], nullptr);
                sc.beg = beg; sc.end = end;
                b200_stage_stats_t st;
                if (b200_stage(eng.e, &batch, &sc, &st) != 0) { fprintf(stderr, "samtools bedcov: %s\n", b200_last_error(eng.e)); return 2; }
                if (b200_bedcov(eng.e, skip_DN, min_depth, cnt.data(), pcov.data()) != 0) { fprintf(stderr, "samtools bedcov: %s\n", b200_last_error(eng.e)); return 2; }
                if (do_rcount) {   // reads the iterator buffered (its constructor hook, bedcov.c:72-76): the kept reads of each file
                    keep.resize(pb.pos.size());
                    if (b200_fetch_mapq_keep(eng.e, nullptr, keep.data(), keep.size()) != 0) return 2;
                    for (int i = 0; i < n; ++i) for (int64_t k = pb.file_start[(size_t)i]; k < pb.file_start[(size_t)i + 1]; ++k) if (keep[(size_t)k] == 2) rcnt[(size_t)i]++;
                }
            }
        }
        fputs(line.data(), stdout);
        for (int i = 0; i < n; ++i) printf("\t%llu", (unsigned long long)cnt[(size_t)i]);
        if (min_depth >= 0) for (int i = 0; i < n; ++i) printf("\t%llu", (unsigned long long)pcov[(size_t)i]);
        if (do_rcount) for (int i = 0; i < n; ++i) printf("\t%llu", (unsigned long long)rcnt[(size_t)i]);
        putchar('\n');
    }
    gzclose(fp);
    fflush(stdout);
    return status;
}

}  // namespace

int main(int argc, char **argv)
{
    if (argc < 2) { fprintf(stderr, "Usage: b200samtools <mpileup|depth|coverage|bedcov|gl> [options]\n"); return 1; }
    std::string cmd = argv[1];
    if (cmd == "mpileup") return main_mpileup(argc - 1, argv + 1, false);
    if (cmd == "gl") return main_mpileup(argc - 1, argv + 1, true);
    if (cmd == "depth") return main_depth(argc - 1, argv + 1);
    if (cmd == "coverage") return main_coverage(argc - 1, argv + 1);
    if (cmd == "bedcov") return main_bedcov(argc - 1, argv + 1);
    fprintf(stderr, "b200samtools: unrecognized command '%s'\n", argv[1]);
    return 1;
}
