// hts_io.hpp -- host-side record I/O for the pileup drivers (C++17, zlib only).
//
// Plays the role of the htslib calls the reference's drivers make around the
// hot path (SURVEY.md section 2b "record I/O"): sam_open/sam_hdr_read/sam_read1,
// sam_itr_querys/sam_itr_next, fai_load/faidx_fetch_seq64, plus bedidx.c's BED
// reader and bam_str2flag.  Formats per hts-specs SAMv1 (SURVEY.md Appendix C).
// This is decode/plumbing, not the accelerated path; CRAM is out of scope.
#pragma once
#include <cstdint>
#include <string>
#include <vector>
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

class AlnReader {
public:
    // fai: optional "<ref>.fai" used as contig list for headerless SAM
    static std::unique_ptr<AlnReader> open(const std::string &path, const std::string &fai = "");
    ~AlnReader();
    const Header &header() const { return hdr_; }
    bool set_region(const std::string &reg, int &tid, int64_t &beg, int64_t &end);
    int next(Record &r);   // 0 ok, -1 EOF, < -1 error
private:
    AlnReader() = default;
    int next_raw(Record &r);
    int parse_sam(char *line, Record &r);
    int read_bam(Record &r);
    bool getline(std::string &s);
    void *gz_ = nullptr;
    bool is_bam_ = false, has_reg_ = false, have_pending_ = false;
    int rtid_ = -1; int64_t rbeg_ = 0, rend_ = 0;
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
