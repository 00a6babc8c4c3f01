// hts_io.hpp -- host-side record I/O for the pileup drivers (C++17, zlib only).
//
// Plays the role of the htslib calls the reference's drivers make around the
// hot path (SURVEY.md section 2b "record I/O"): sam_open/sam_hdr_read/sam_read1,
// bgzf_read/bgzf_seek, sam_index_load/sam_itr_querys/sam_itr_next, the index
// writer of `samtools index`, fai_load/faidx_fetch_seq64, plus bedidx.c's BED
// reader and bam_str2flag.  Formats per hts-specs SAMv1 (SURVEY.md Appendix C).
// This is decode/plumbing, not the accelerated path; CRAM is out of scope.
#pragma once
#include <cstdint>
#include <string>
#include <vector>
#include <map>
#include <memory>
#include <unordered_map>

namespace b200 {

constexpr int64_t POS_MAX = ((int64_t)INT32_MAX << 32) | UINT32_MAX;

enum : uint16_t { F_PAIRED = 1, F_PROPER = 2, F_UNMAP = 4, F_MUNMAP = 8, F_REVERSE = 16, F_MREVERSE = 32, F_READ1 = 64,
                  F_READ2 = 128, F_SECONDARY = 256, F_QCFAIL = 512, F_DUP = 1024, F_SUPP = 2048 };

struct Record {
    int64_t pos = 0, mpos = 0, isize = 0;
    int32_t tid = -1, mtid = -1, l_qseq = 0;
    uint16_t flag = 0;
    uint8_t mapq = 0;
    std::string qname;
    std::vector<uint32_t> cigar;   // BAM encoding len<<4|op
    std::vector<uint8_t> seq4;     // 4-bit packed, high nibble first
    std::vector<uint8_t> qual;     // l_qseq bytes (0xff.. when absent)
    std::vector<uint8_t> aux;      // BAM-encoded tags

    int64_t rlen() const;          // bam_cigar2rlen
    int64_t endpos() const;        // bam_endpos
    const uint8_t *aux_get(const char tag[2]) const;   // -> type byte, or nullptr
};

struct Header {
    std::vector<std::string> names;
    std::vector<int64_t> lens;
    std::string text;
    int name2tid(const std::string &n) const;
    int n_ref() const { return (int)names.size(); }
};

// region string "name[:beg[-end]]" -> tid, [beg,end) 0-based; false on failure
bool parse_region(const Header &h, const std::string &reg, int &tid, int64_t &beg, int64_t &end);
int parse_flag(const std::string &s);   // bam_str2flag; -1 on failure

// Decompressed byte stream of one input (SAMv1 4.1).  A BGZF file is read block by block: each block's gzip header and
// BC subfield are parsed, its raw DEFLATE payload is inflated and checked against ISIZE and CRC32, and positions are
// virtual offsets (block file offset << 16 | offset inside the block) that seek() returns to.  Any other input -- plain
// gzip (one or several members) or uncompressed text -- is read sequentially.  "-" is stdin (sequential only).
// A malformed block is an error (read() < 0, failed() true), never a read past the block.
class InStream {
public:
    static std::unique_ptr<InStream> open(const std::string &path);
    ~InStream();
    bool bgzf() const { return mode_ == BGZF; }
    bool failed() const { return err_; }
    int64_t read(void *dst, size_t n);        // bytes read (fewer than n only at the end of the input), -1 on an error
    size_t peek(void *dst, size_t n);         // up to n bytes of the current block without consuming them
    bool getline(std::string &s);             // one line without its "\n" / "\r\n"; false at the end or on an error
    uint64_t tell() const;                    // virtual offset of the next byte (BGZF)
    bool seek(uint64_t voff);                 // BGZF on a seekable file
private:
    enum Mode { BGZF, GZIP, PLAIN };
    InStream() = default;
    bool fill(size_t need);                   // at least `need` raw bytes buffered unless the file ends first
    bool refill();                            // next decompressed block into out_; false at the end or on an error
    bool load_bgzf_block();
    int fd_ = -1; Mode mode_ = PLAIN; bool err_ = false, eof_raw_ = false, z_end_ = false, z_done_ = false;
    std::vector<uint8_t> raw_, out_;
    size_t rpos_ = 0, rlen_ = 0, opos_ = 0, olen_ = 0;
    int64_t raw_off_ = 0;                     // file offset of raw_[0]
    int64_t block_addr_ = 0, next_addr_ = 0;  // file offsets of the current and the next BGZF block
    void *z_ = nullptr;                       // z_stream
};

// BAI / CSI index (SAMv1 5, CSIv1): per reference sequence the chunks [beg, end) of virtual offsets of every bin, the
// linear index (BAI, one offset per 2^min_shift bases) or each bin's loffset (CSI).  BAI is CSI's (14, 5) scheme.
struct HtsIndex {
    struct Chunk { uint64_t beg, end; };
    struct Bin { uint64_t loff = 0; std::vector<Chunk> chunks; };
    struct Ref { std::map<uint32_t, Bin> bins; std::vector<uint64_t> lin; uint64_t meta[4] = {0, 0, 0, 0}; bool has_meta = false; };
    bool csi = false;
    int min_shift = 14, depth = 5;
    std::vector<Ref> refs;
    uint64_t n_no_coor = 0; bool has_no_coor = false;
    uint32_t pseudo_bin() const { return (uint32_t)(((1ull << 3 * (depth + 1)) - 1) / 7 + 1); }
    int64_t max_pos() const { return (int64_t)1 << (min_shift + 3 * depth); }
    // n_ref: reference sequences of the data file's header; err names the file and the fault
    static std::unique_ptr<HtsIndex> load(const std::string &path, int n_ref, std::string &err);
    bool save(const std::string &path, std::string &err) const;
    // chunks to read for [beg, end) of tid: sorted, merged, those ending before the region's minimum offset dropped
    std::vector<Chunk> query(int tid, int64_t beg, int64_t end) const;
};
uint32_t reg2bin(int64_t beg, int64_t end, int min_shift, int depth);                    // end exclusive
void reg2bins(int64_t beg, int64_t end, int min_shift, int depth, std::vector<uint32_t> &out);
// `index`: a BAI (csi false; min_shift 14) or a CSI of the coordinate-sorted BAM `in`; 0 ok, else err says why
int build_index(const std::string &in, const std::string &out, bool csi, int min_shift, std::string &err);

class AlnReader {
public:
    // fai: optional "<ref>.fai" used as contig list for headerless SAM
    static std::unique_ptr<AlnReader> open(const std::string &path, const std::string &fai = "");
    ~AlnReader();
    const Header &header() const { return hdr_; }
    bool is_bam() const { return is_bam_; }
    bool bgzf() const { return in_ && in_->bgzf(); }
    // The index of a BAM input: `explicit_fn` if given, else <fn>.bai, <stem>.bai or <fn>.csi next to it.  True with no
    // index found (the reader then scans); false with error() set when the index is unreadable or inconsistent.
    bool open_index(const std::string &explicit_fn = "");
    bool has_index() const { return (bool)idx_; }
    const std::string &error() const { return err_; }
    bool set_region(const std::string &reg, int &tid, int64_t &beg, int64_t &end);
    // the records of tid overlapping [beg, end), through the index (has_index() must hold); a later call starts anew
    void query(int tid, int64_t beg, int64_t end);
    int next(Record &r);   // 0 ok, -1 EOF, < -1 error
    uint64_t tell() const; // virtual offset of the next record (BAM)
private:
    AlnReader() = default;
    int next_raw(Record &r);
    int next_indexed(Record &r);
    int parse_sam(char *line, Record &r);
    int read_bam(Record &r);
    std::unique_ptr<InStream> in_;
    std::string path_, err_;
    bool is_bam_ = false, has_reg_ = false, have_pending_ = false;
    int rtid_ = -1; int64_t rbeg_ = 0, rend_ = 0;
    std::unique_ptr<HtsIndex> idx_;
    std::vector<HtsIndex::Chunk> chunks_; size_t ck_ = 0; bool in_chunk_ = false;
    uint64_t reached_ = 0;                    // furthest virtual offset read by the current query
    std::string pending_, line_;
    Header hdr_;
};

struct Fasta {
    std::vector<std::string> names, seqs;
    static std::unique_ptr<Fasta> load(const std::string &path);
    int find(const std::string &n) const;
};

// BED / "chr pos" list with bedidx.c semantics
struct Bed {
    struct Chr { std::vector<std::pair<int64_t, int64_t>> iv; std::vector<int> idx; int64_t max_idx = 0; };
    std::unordered_map<std::string, Chr> chr;
    static std::unique_ptr<Bed> load(const std::string &path);
    bool overlap(const std::string &name, int64_t beg, int64_t end) const;   // bed_overlap
    // per-contig intervals merged into a disjoint sorted union (same point-overlap predicate)
    void merged(const std::string &name, std::vector<int64_t> &b, std::vector<int64_t> &e) const;
};

bool read_file_list(const std::string &path, std::vector<std::string> &out);   // bam_plcmd.c:944-998
uint32_t qname_hash_bit(const std::string &qname);   // __ac_Wang_hash(__ac_X31_hash_string(name)) & 1

}  // namespace b200
