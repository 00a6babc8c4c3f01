// hts_io.cpp -- see hts_io.hpp.
#include "hts_io.hpp"
#include <zlib.h>
#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cerrno>
#include <cstdlib>
#include <cstring>
#include <strings.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

namespace b200 {

static const char kOps[] = "MIDNSHP=XB";

static uint8_t nt16(unsigned char c)
{
    switch (c | 0x20) {
    case 'a': return 1; case 'c': return 2; case 'm': return 3; case 'g': return 4; case 'r': return 5; case 's': return 6;
    case 'v': return 7; case 't': return 8; case 'w': return 9; case 'y': return 10; case 'h': return 11; case 'k': return 12;
    case 'd': return 13; case 'b': return 14; case 'n': return 15;
    default: break;
    }
    if (c == '=') return 0;
    if (c >= '0' && c <= '3') return (uint8_t)(1 << (c - '0'));
    return 15;
}

int64_t Record::rlen() const
{
    int64_t l = 0;
    for (uint32_t c : cigar) { int op = c & 0xf; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) l += c >> 4; }
    return l;
}
int64_t Record::endpos() const
{
    int64_t rl = 1;
    if (!(flag & F_UNMAP) && !cigar.empty()) { rl = rlen(); if (rl == 0) rl = 1; }
    return pos + rl;
}
static int aux_size(int t)
{
    switch (t) { case 'A': case 'c': case 'C': return 1; case 's': case 'S': return 2; case 'i': case 'I': case 'f': return 4; case 'd': return 8; default: return 0; }
}
static const uint8_t *aux_skip(const uint8_t *s, const uint8_t *end)
{
    int t = *s++;
    if (int sz = aux_size(t)) return s + sz <= end ? s + sz : nullptr;
    if (t == 'Z' || t == 'H') { while (s < end && *s) ++s; return s < end ? s + 1 : nullptr; }
    if (t == 'B') {
        if (s + 5 > end) return nullptr;
        int esz = aux_size(*s); uint32_t n; memcpy(&n, s + 1, 4);
        s += 5 + (size_t)esz * n;
        return (esz && s <= end) ? s : nullptr;
    }
    return nullptr;
}
const uint8_t *Record::aux_get(const char tag[2]) const
{
    const uint8_t *s = aux.data(), *end = s + aux.size();
    while (s && s + 3 <= end) {
        if (s[0] == (uint8_t)tag[0] && s[1] == (uint8_t)tag[1]) return s + 2;
        s = aux_skip(s + 2, end);
    }
    return nullptr;
}

int Header::name2tid(const std::string &n) const
{
    for (size_t i = 0; i < names.size(); ++i) if (names[i] == n) return (int)i;
    return -1;
}

bool parse_region(const Header &h, const std::string &reg, int &tid, int64_t &beg, int64_t &end)
{
    beg = 0; end = POS_MAX;
    int t = h.name2tid(reg);
    if (t >= 0) { tid = t; return true; }
    size_t colon = reg.rfind(':');
    if (colon == std::string::npos) return false;
    t = h.name2tid(reg.substr(0, colon));
    if (t < 0) return false;
    std::string a, b; bool dash = false;
    for (size_t i = colon + 1; i < reg.size(); ++i) {
        char c = reg[i];
        if (c == ',') continue;
        if (c == '-' && !dash) { dash = true; continue; }
        (dash ? b : a).push_back(c);
    }
    long long lb = a.empty() ? 0 : atoll(a.c_str());
    beg = lb > 0 ? lb - 1 : 0;
    end = (dash && !b.empty()) ? atoll(b.c_str()) : POS_MAX;
    if (beg >= end) return false;
    tid = t;
    return true;
}

int parse_flag(const std::string &s)
{
    char *e; long v = strtol(s.c_str(), &e, 0);
    if (e != s.c_str() && *e == 0) return v < 0 ? -1 : (int)v;
    static const struct { const char *n; int f; } names[] = {
        {"PAIRED", 1}, {"PROPER_PAIR", 2}, {"UNMAP", 4}, {"MUNMAP", 8}, {"REVERSE", 16}, {"MREVERSE", 32},
        {"READ1", 64}, {"READ2", 128}, {"SECONDARY", 256}, {"QCFAIL", 512}, {"DUP", 1024}, {"SUPPLEMENTARY", 2048} };
    int flag = 0; size_t p = 0;
    while (p < s.size()) {
        size_t q = s.find(',', p); if (q == std::string::npos) q = s.size();
        std::string tok = s.substr(p, q - p); bool ok = false;
        for (auto &n : names) if (strcasecmp(tok.c_str(), n.n) == 0) { flag |= n.f; ok = true; break; }
        if (!ok) return -1;
        p = q + 1;
    }
    return flag;
}

uint32_t qname_hash_bit(const std::string &q)
{
    const char *s = q.c_str();
    uint32_t h = (uint32_t)*s;
    if (h) for (++s; *s; ++s) h = (h << 5) - h + (uint32_t)*s;
    h += ~(h << 15); h ^= (h >> 10); h += (h << 3); h ^= (h >> 6); h += ~(h << 11); h ^= (h >> 16);
    return h & 1;
}

// ------------------------------------------------------------------ byte stream (BGZF, SAMv1 4.1)
static constexpr size_t kRawBuf = 1 << 20;

// size of the BGZF block at p (BSIZE + 1), 0 when p[0, n) is not the header of one; n covers the gzip extra field
static long bgzf_block_size(const uint8_t *p, size_t n)
{
    if (n < 12 || p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || !(p[3] & 4)) return 0;
    const size_t xend = 12 + (p[10] | (size_t)p[11] << 8);
    if (n < xend) return 0;
    for (size_t k = 12; k + 4 <= xend;) {
        const size_t slen = p[k + 2] | (size_t)p[k + 3] << 8;
        if (p[k] == 'B' && p[k + 1] == 'C' && slen == 2 && k + 6 <= xend) return (long)(p[k + 4] | (size_t)p[k + 5] << 8) + 1;
        k += 4 + slen;
    }
    return 0;
}

InStream::~InStream()
{
    if (z_) { inflateEnd((z_stream *)z_); delete (z_stream *)z_; }
    if (fd_ > 0) ::close(fd_);
}

std::unique_ptr<InStream> InStream::open(const std::string &path)
{
    const int fd = path == "-" ? 0 : ::open(path.c_str(), O_RDONLY);
    if (fd < 0) return nullptr;
    std::unique_ptr<InStream> s(new InStream());
    s->fd_ = fd;
    s->raw_.resize(kRawBuf);
    s->out_.resize(1 << 16);
    s->fill(18);
    if (s->err_) return nullptr;
    if (s->rlen_ >= 2 && s->raw_[0] == 0x1f && s->raw_[1] == 0x8b) {
        if (s->rlen_ >= 12) s->fill(12 + (s->raw_[10] | (size_t)s->raw_[11] << 8));
        s->mode_ = bgzf_block_size(s->raw_.data(), s->rlen_) > 0 ? BGZF : GZIP;
        z_stream *z = new z_stream();
        if (inflateInit2(z, s->mode_ == BGZF ? -15 : 15 + 16) != Z_OK) { delete z; return nullptr; }
        s->z_ = z;
    }
    return s;
}

bool InStream::fill(size_t need)
{
    if (rlen_ - rpos_ >= need) return true;
    if (rpos_) { memmove(raw_.data(), raw_.data() + rpos_, rlen_ - rpos_); raw_off_ += (int64_t)rpos_; rlen_ -= rpos_; rpos_ = 0; }
    if (need > raw_.size()) raw_.resize(need);
    while (rlen_ < need && !eof_raw_) {
        const ssize_t k = ::read(fd_, raw_.data() + rlen_, raw_.size() - rlen_);
        if (k < 0) { if (errno == EINTR) continue; err_ = true; return false; }
        if (k == 0) eof_raw_ = true;
        rlen_ += (size_t)k;
    }
    return rlen_ >= need;
}

bool InStream::load_bgzf_block()
{
    block_addr_ = raw_off_ + (int64_t)rpos_;
    if (!fill(12)) { if (rlen_ != rpos_) err_ = true; return false; }   // no byte left: the end of the file
    if (!fill(12 + (raw_[rpos_ + 10] | (size_t)raw_[rpos_ + 11] << 8))) { err_ = true; return false; }
    const long bs = bgzf_block_size(&raw_[rpos_], rlen_ - rpos_);
    const size_t xend = 12 + (raw_[rpos_ + 10] | (size_t)raw_[rpos_ + 11] << 8);
    if (bs < (long)xend + 8 || !fill((size_t)bs)) { err_ = true; return false; }
    const uint8_t *p = &raw_[rpos_];
    uint32_t crc, isize;
    memcpy(&crc, p + bs - 8, 4); memcpy(&isize, p + bs - 4, 4);
    if (isize > out_.size()) { err_ = true; return false; }
    z_stream *z = (z_stream *)z_;
    inflateReset(z);
    z->next_in = (Bytef *)(p + xend); z->avail_in = (uInt)((size_t)bs - xend - 8);
    z->next_out = out_.data(); z->avail_out = (uInt)out_.size();
    if (inflate(z, Z_FINISH) != Z_STREAM_END || z->total_out != isize || z->avail_in != 0 ||
        crc32(crc32(0L, Z_NULL, 0), out_.data(), isize) != crc) { err_ = true; return false; }
    rpos_ += (size_t)bs;
    next_addr_ = block_addr_ + bs;
    opos_ = 0; olen_ = isize;
    return true;
}

bool InStream::refill()
{
    if (err_) return false;
    if (mode_ == BGZF) {
        do { if (!load_bgzf_block()) return false; } while (olen_ == 0);   // an empty block (the EOF marker) carries no data
        return true;
    }
    opos_ = olen_ = 0;
    if (mode_ == PLAIN) {
        if (!fill(1)) return false;
        olen_ = std::min(rlen_ - rpos_, out_.size());
        memcpy(out_.data(), &raw_[rpos_], olen_); rpos_ += olen_;
        return true;
    }
    // gzip: members back to back; what follows the last one, if not another member, is ignored (as gzread does)
    z_stream *z = (z_stream *)z_;
    while (olen_ == 0) {
        if (z_done_) return false;
        if (z_end_) {
            if (!fill(2) || raw_[rpos_] != 0x1f || raw_[rpos_ + 1] != 0x8b) { z_done_ = true; return false; }
            inflateReset(z); z_end_ = false;
        }
        if (!fill(1)) { err_ = true; return false; }   // the member is cut short
        z->next_in = &raw_[rpos_]; z->avail_in = (uInt)(rlen_ - rpos_);
        z->next_out = out_.data(); z->avail_out = (uInt)out_.size();
        const int ret = inflate(z, Z_NO_FLUSH);
        rpos_ = rlen_ - z->avail_in;
        olen_ = out_.size() - z->avail_out;
        if (ret == Z_STREAM_END) z_end_ = true;
        else if (ret != Z_OK && ret != Z_BUF_ERROR) { err_ = true; return false; }
    }
    return true;
}

int64_t InStream::read(void *dst, size_t n)
{
    uint8_t *d = (uint8_t *)dst;
    size_t got = 0;
    while (got < n) {
        if (opos_ == olen_ && !refill()) { if (err_) return -1; break; }
        const size_t k = std::min(n - got, olen_ - opos_);
        memcpy(d + got, &out_[opos_], k); opos_ += k; got += k;
    }
    return (int64_t)got;
}

size_t InStream::peek(void *dst, size_t n)
{
    if (opos_ == olen_ && !refill()) return 0;
    const size_t k = std::min(n, olen_ - opos_);
    memcpy(dst, &out_[opos_], k);
    return k;
}

bool InStream::getline(std::string &s)
{
    s.clear();
    bool got = false;
    for (;;) {
        if (opos_ == olen_ && !refill()) break;
        got = true;
        const uint8_t *b = &out_[opos_], *nl = (const uint8_t *)memchr(b, '\n', olen_ - opos_);
        if (nl) {
            s.append((const char *)b, (size_t)(nl - b)); opos_ += (size_t)(nl - b) + 1;
            if (!s.empty() && s.back() == '\r') s.pop_back();
            return true;
        }
        s.append((const char *)b, olen_ - opos_); opos_ = olen_;
    }
    return got && !err_;
}

uint64_t InStream::tell() const
{
    // at the end of a block the next record starts in the next one
    return opos_ == olen_ ? (uint64_t)next_addr_ << 16 : (uint64_t)block_addr_ << 16 | opos_;
}

bool InStream::seek(uint64_t voff)
{
    if (mode_ != BGZF || err_) return false;
    const int64_t coff = (int64_t)(voff >> 16);
    const size_t uoff = (size_t)(voff & 0xffff);
    if (!(coff == block_addr_ && next_addr_ > block_addr_)) {   // not the block already inflated
        if (coff >= raw_off_ && coff <= raw_off_ + (int64_t)rlen_) rpos_ = (size_t)(coff - raw_off_);
        else {
            if (lseek(fd_, (off_t)coff, SEEK_SET) != (off_t)coff) { err_ = true; return false; }
            raw_off_ = coff; rpos_ = rlen_ = 0; eof_raw_ = false;
        }
        if (!load_bgzf_block()) { err_ = true; return false; }
    }
    if (uoff > olen_) { err_ = true; return false; }
    opos_ = uoff;
    return true;
}

// ------------------------------------------------------------------ reader
AlnReader::~AlnReader() = default;

std::unique_ptr<AlnReader> AlnReader::open(const std::string &path, const std::string &fai)
{
    std::unique_ptr<AlnReader> rd(new AlnReader());
    rd->in_ = InStream::open(path);
    if (!rd->in_) return nullptr;
    rd->path_ = path;
    InStream &in = *rd->in_;
    auto add_ref = [&](const std::string &n, int64_t l) { rd->hdr_.names.push_back(n); rd->hdr_.lens.push_back(l); };
    char magic[4];
    const size_t got = in.peek(magic, 4);
    if (in.failed()) return nullptr;
    if (got == 0) return rd;
    if (got == 4 && memcmp(magic, "BAM\1", 4) == 0) {
        int32_t l_text, n_ref;
        if (in.read(magic, 4) != 4 || in.read(&l_text, 4) != 4 || l_text < 0) return nullptr;
        rd->is_bam_ = true;
        rd->hdr_.text.resize((size_t)l_text);
        if (l_text && in.read(&rd->hdr_.text[0], (size_t)l_text) != l_text) return nullptr;
        while (!rd->hdr_.text.empty() && rd->hdr_.text.back() == '\0') rd->hdr_.text.pop_back();
        if (in.read(&n_ref, 4) != 4 || n_ref < 0) return nullptr;
        for (int i = 0; i < n_ref; ++i) {
            int32_t ln, lr;
            if (in.read(&ln, 4) != 4 || ln < 0) return nullptr;
            std::string nm((size_t)ln, '\0');
            if (in.read(&nm[0], (size_t)ln) != ln || in.read(&lr, 4) != 4) return nullptr;
            nm.resize(strlen(nm.c_str()));
            add_ref(nm, lr);
        }
        return rd;
    }
    std::string ln;
    while (in.getline(ln)) {
        if (!ln.empty() && ln[0] == '@') {
            rd->hdr_.text += ln; rd->hdr_.text += '\n';
            if (ln.compare(0, 3, "@SQ") == 0) {
                std::string sn; int64_t len = 0; size_t p = 0;
                while (p < ln.size()) {
                    size_t q = ln.find('\t', p); if (q == std::string::npos) q = ln.size();
                    if (ln.compare(p, 3, "SN:") == 0) sn = ln.substr(p + 3, q - p - 3);
                    else if (ln.compare(p, 3, "LN:") == 0) len = atoll(ln.c_str() + p + 3);
                    p = q + 1;
                }
                if (!sn.empty()) add_ref(sn, len);
            }
        } else { rd->pending_ = ln; rd->have_pending_ = true; break; }
    }
    if (rd->hdr_.names.empty() && !fai.empty()) {
        if (FILE *f = fopen(fai.c_str(), "r")) {
            char buf[4096], nm[1024]; long long l;
            while (fgets(buf, sizeof buf, f)) if (sscanf(buf, "%1023s %lld", nm, &l) == 2) add_ref(nm, l);
            fclose(f);
        }
    }
    return rd;
}

bool AlnReader::open_index(const std::string &fn)
{
    const bool seekable = is_bam_ && in_->bgzf() && path_ != "-";
    std::string p = fn;
    if (p.empty()) {
        if (!seekable) return true;
        std::vector<std::string> cand = { path_ + ".bai" };
        if (path_.size() > 4 && path_.compare(path_.size() - 4, 4, ".bam") == 0) cand.push_back(path_.substr(0, path_.size() - 4) + ".bai");
        cand.push_back(path_ + ".csi");
        for (const std::string &c : cand) { struct stat sb; if (stat(c.c_str(), &sb) == 0) { p = c; break; } }
        if (p.empty()) return true;
    } else if (!seekable) {
        err_ = "cannot use the index \"" + fn + "\": \"" + path_ + "\" is not a BGZF-compressed BAM file";
        return false;
    }
    idx_ = HtsIndex::load(p, hdr_.n_ref(), err_);
    return (bool)idx_;
}

bool AlnReader::set_region(const std::string &reg, int &tid, int64_t &beg, int64_t &end)
{
    if (!parse_region(hdr_, reg, rtid_, rbeg_, rend_)) return false;
    has_reg_ = true;
    if (idx_) query(rtid_, rbeg_, rend_);
    tid = rtid_; beg = rbeg_; end = rend_;
    return true;
}

void AlnReader::query(int tid, int64_t beg, int64_t end)
{
    has_reg_ = true; rtid_ = tid; rbeg_ = beg; rend_ = end;
    chunks_ = idx_->query(tid, beg, end);
    ck_ = 0; in_chunk_ = false; reached_ = 0;
}

uint64_t AlnReader::tell() const { return in_ ? in_->tell() : 0; }

static void aux_put(std::vector<uint8_t> &a, const char *tag, char type, const void *d, size_t n)
{
    a.push_back((uint8_t)tag[0]); a.push_back((uint8_t)tag[1]); a.push_back((uint8_t)type);
    const uint8_t *p = (const uint8_t *)d; a.insert(a.end(), p, p + n);
}
static void aux_put_int(std::vector<uint8_t> &a, const char *tag, long long v)
{
    if (v < 0) {
        if (v >= -128) { int8_t x = (int8_t)v; aux_put(a, tag, 'c', &x, 1); }
        else if (v >= -32768) { int16_t x = (int16_t)v; aux_put(a, tag, 's', &x, 2); }
        else { int32_t x = (int32_t)v; aux_put(a, tag, 'i', &x, 4); }
    } else {
        if (v < 256) { uint8_t x = (uint8_t)v; aux_put(a, tag, 'C', &x, 1); }
        else if (v < 65536) { uint16_t x = (uint16_t)v; aux_put(a, tag, 'S', &x, 2); }
        else { uint32_t x = (uint32_t)v; aux_put(a, tag, 'I', &x, 4); }
    }
}

int AlnReader::parse_sam(char *line, Record &r)
{
    char *f[11]; int nf = 0; char *p = line;
    while (nf < 11) {
        f[nf++] = p;
        char *t = strchr(p, '\t');
        if (!t) { p = nullptr; break; }
        *t = 0; p = t + 1;
    }
    if (nf < 11) return -2;
    r = Record();
    r.qname = f[0];
    r.flag = (uint16_t)strtol(f[1], nullptr, 10);
    r.tid = strcmp(f[2], "*") ? hdr_.name2tid(f[2]) : -1;
    r.pos = atoll(f[3]) - 1;
    r.mapq = (uint8_t)strtol(f[4], nullptr, 10);
    if (strcmp(f[5], "*")) {
        const char *c = f[5];
        while (*c) {
            char *e; unsigned long l = strtoul(c, &e, 10);
            const char *o = *e ? strchr(kOps, *e) : nullptr;
            if (!o || o - kOps > 8) return -2;                            // 'B' (and anything else) is not an alignment op
            r.cigar.push_back((uint32_t)l << 4 | (uint32_t)(o - kOps));
            c = e + 1;
        }
    }
    if (!strcmp(f[6], "=")) r.mtid = r.tid; else r.mtid = strcmp(f[6], "*") ? hdr_.name2tid(f[6]) : -1;
    r.mpos = atoll(f[7]) - 1;
    r.isize = atoll(f[8]);
    if (strcmp(f[9], "*")) {
        size_t l = strlen(f[9]);
        r.l_qseq = (int32_t)l;
        r.seq4.assign((l + 1) / 2, 0);
        for (size_t i = 0; i < l; ++i) r.seq4[i >> 1] |= (uint8_t)(nt16((unsigned char)f[9][i]) << ((~i & 1) << 2));
        r.qual.resize(l);
        if (!strcmp(f[10], "*")) std::fill(r.qual.begin(), r.qual.end(), 0xff);
        else for (size_t i = 0; i < l; ++i) r.qual[i] = (uint8_t)(f[10][i] - 33);
    }
    while (p && *p) {
        char *t = strchr(p, '\t');
        if (t) *t = 0;
        size_t L = strlen(p);
        if (L >= 5 && p[2] == ':' && p[4] == ':') {
            char type = p[3]; const char *v = p + 5;
            if (type == 'A') aux_put(r.aux, p, 'A', v, 1);
            else if (type == 'i') aux_put_int(r.aux, p, atoll(v));
            else if (type == 'f') { float x = strtof(v, nullptr); aux_put(r.aux, p, 'f', &x, 4); }
            else if (type == 'Z' || type == 'H') aux_put(r.aux, p, type, v, strlen(v) + 1);
            else if (type == 'B') {
                char st = v[0]; int esz = aux_size(st); uint32_t n = 0;
                for (const char *q = v + 1; *q; ++q) if (*q == ',') ++n;
                std::vector<uint8_t> buf(5 + (size_t)esz * n);
                buf[0] = (uint8_t)st; memcpy(&buf[1], &n, 4);
                uint8_t *o = buf.data() + 5; const char *q = v + 1;
                while (*q == ',') {
                    char *e; ++q;
                    if (st == 'f') { float x = strtof(q, &e); memcpy(o, &x, 4); }
                    else { long long x = strtoll(q, &e, 10); memcpy(o, &x, (size_t)esz); }
                    o += esz; q = e;
                }
                aux_put(r.aux, p, 'B', buf.data(), buf.size());
            }
        }
        p = t ? t + 1 : nullptr;
    }
    return 0;
}

int AlnReader::read_bam(Record &r)
{
    int32_t bs;
    const int64_t n = in_->read(&bs, 4);
    if (n == 0) return -1;
    if (n != 4 || bs < 32) return -2;
    std::vector<uint8_t> d((size_t)bs);
    if (in_->read(d.data(), (size_t)bs) != bs) return -2;
    r = Record();
    int32_t i32; uint16_t u16;
    memcpy(&r.tid, &d[0], 4);
    memcpy(&i32, &d[4], 4); r.pos = i32;
    int l_name = d[8]; r.mapq = d[9];
    memcpy(&u16, &d[12], 2); uint32_t ncig = u16;
    memcpy(&r.flag, &d[14], 2);
    memcpy(&r.l_qseq, &d[16], 4);
    memcpy(&r.mtid, &d[20], 4);
    memcpy(&i32, &d[24], 4); r.mpos = i32;
    memcpy(&i32, &d[28], 4); r.isize = i32;
    // the variable part must fit the block (a truncated / corrupt record must not be read past its end)
    if (r.l_qseq < 0 || l_name < 1 ||
        32ull + (uint64_t)l_name + 4ull * ncig + ((uint64_t)r.l_qseq + 1) / 2 + (uint64_t)r.l_qseq > (uint64_t)bs) return -2;
    const uint8_t *p = d.data() + 32;
    r.qname.assign((const char *)p, strnlen((const char *)p, (size_t)l_name)); p += l_name;
    r.cigar.resize(ncig); if (ncig) memcpy(r.cigar.data(), p, 4 * (size_t)ncig); p += 4 * (size_t)ncig;
    r.seq4.assign(p, p + (r.l_qseq + 1) / 2); p += (r.l_qseq + 1) / 2;
    r.qual.assign(p, p + r.l_qseq); p += r.l_qseq;
    r.aux.assign(p, (const uint8_t *)d.data() + bs);
    for (uint32_t c : r.cigar) if ((c & 0xf) > 8) return -2;          // only MIDNSHP=X are defined for alignments
    // long CIGARs (> 65535 ops) live in the CG:B,I tag behind a <l_qseq>S<rlen>N placeholder (SAMv1 4.2.2; htslib bam_tag2cigar)
    if (r.cigar.size() == 2 && (r.cigar[0] & 0xf) == 4 && (int32_t)(r.cigar[0] >> 4) == r.l_qseq && (r.cigar[1] & 0xf) == 3) {
        const uint8_t *cg = r.aux_get("CG");
        if (cg && cg[0] == 'B' && cg[1] == 'I') {
            uint32_t n; memcpy(&n, cg + 2, 4);
            const size_t off = (size_t)(cg - r.aux.data());
            if (n > 0 && off + 6 + 4ull * n <= r.aux.size()) {
                std::vector<uint32_t> real(n);
                memcpy(real.data(), cg + 6, 4ull * n);
                for (uint32_t c : real) if ((c & 0xf) > 8) return -2;
                r.cigar.swap(real);
                r.aux.erase(r.aux.begin() + (long)off - 2, r.aux.begin() + (long)(off + 6 + 4ull * n));   // drop the tag like htslib does
            }
        }
    }
    return 0;
}

int AlnReader::next_raw(Record &r)
{
    if (!in_) return -1;
    if (is_bam_) return read_bam(r);
    for (;;) {
        if (have_pending_) { line_ = pending_; have_pending_ = false; }
        else if (!in_->getline(line_)) return in_->failed() ? -2 : -1;
        if (line_.empty()) continue;
        std::vector<char> buf(line_.begin(), line_.end()); buf.push_back(0);
        return parse_sam(buf.data(), r);
    }
}

// The chunks of the current query, in file order.  The index only decides which blocks are inflated: next() keeps the
// linear scan's predicate, so the records and their order are the scan's.
int AlnReader::next_indexed(Record &r)
{
    for (;;) {
        if (ck_ >= chunks_.size()) return -1;
        const HtsIndex::Chunk &c = chunks_[ck_];
        if (!in_chunk_) {
            const uint64_t from = std::max(c.beg, reached_);   // never read a record twice, whatever the chunks say
            if (from >= c.end) { ++ck_; continue; }
            if (from != in_->tell() && !in_->seek(from)) { err_ = "cannot seek in \"" + path_ + "\": corrupt data or index"; return -2; }
            in_chunk_ = true;
        }
        if (in_->tell() >= c.end) { ++ck_; in_chunk_ = false; continue; }
        const int ret = read_bam(r);
        if (ret == -1) { ck_ = chunks_.size(); return -1; }
        if (ret < -1) return ret;
        reached_ = in_->tell();
        // sorted input: the first record of another sequence or past the region ends the query
        if (r.tid != rtid_ || r.pos >= rend_) { ck_ = chunks_.size(); return -1; }
        return 0;
    }
}

int AlnReader::next(Record &r)
{
    for (;;) {
        const int ret = idx_ && has_reg_ ? next_indexed(r) : next_raw(r);
        if (ret < 0) return ret;
        if (has_reg_) {
            if (r.tid != rtid_) continue;
            if (!(r.pos < rend_ && r.endpos() > rbeg_)) continue;
        }
        return 0;
    }
}

// ------------------------------------------------------------------ BAI / CSI (SAMv1 5.3, CSIv1)
static int64_t level_first_bin(int l) { return ((1ll << 3 * l) - 1) / 7; }

uint32_t reg2bin(int64_t beg, int64_t end, int min_shift, int depth)
{
    --end;
    int s = min_shift;
    int64_t t = level_first_bin(depth);
    for (int l = depth; l > 0; --l, s += 3, t -= 1ll << 3 * l)
        if (beg >> s == end >> s) return (uint32_t)(t + (beg >> s));
    return 0;
}

void reg2bins(int64_t beg, int64_t end, int min_shift, int depth, std::vector<uint32_t> &out)
{
    out.clear();
    if (beg >= end) return;
    --end;
    int64_t t = 0;
    for (int l = 0, s = min_shift + 3 * depth; l <= depth; s -= 3, t += 1ll << 3 * l, ++l)
        for (int64_t b = t + (beg >> s); b <= t + (end >> s); ++b) out.push_back((uint32_t)b);
}

namespace {
struct ByteCursor {   // bounds-checked reads of an index held in memory
    const uint8_t *p, *e;
    bool bad = false;
    size_t left() const { return (size_t)(e - p); }
    template <class T> bool take(T &v) { return take_n(&v, sizeof v); }
    bool take_n(void *d, size_t n) { if (bad || left() < n) { bad = true; return false; } memcpy(d, p, n); p += n; return true; }
};
}

std::unique_ptr<HtsIndex> HtsIndex::load(const std::string &path, int n_ref, std::string &err)
{
    auto fail = [&](const std::string &why) { err = "invalid index file \"" + path + "\": " + why; return nullptr; };
    std::unique_ptr<InStream> in = InStream::open(path);   // BAI is stored plain, CSI in BGZF
    if (!in) { err = "cannot open index file \"" + path + "\": " + strerror(errno); return nullptr; }
    std::vector<uint8_t> buf;
    for (;;) {
        const size_t o = buf.size(), step = 1 << 20;
        buf.resize(o + step);
        const int64_t k = in->read(buf.data() + o, step);
        if (k < 0) return fail("corrupt compressed data");
        buf.resize(o + (size_t)k);
        if ((size_t)k < step) break;
    }
    ByteCursor c{buf.data(), buf.data() + buf.size()};
    std::unique_ptr<HtsIndex> x(new HtsIndex());
    char magic[4];
    if (!c.take_n(magic, 4)) return fail("truncated");
    if (memcmp(magic, "CSI\1", 4) == 0) {
        int32_t ms, d, l_aux;
        if (!c.take(ms) || !c.take(d) || !c.take(l_aux)) return fail("truncated");
        if (ms < 1 || d < 0 || d > 9 || ms + 3 * d > 62) return fail("min_shift " + std::to_string(ms) + " / depth " + std::to_string(d) + " out of range");
        if (l_aux < 0 || (size_t)l_aux > c.left()) return fail("truncated");
        c.p += l_aux;
        x->csi = true; x->min_shift = ms; x->depth = d;
    } else if (memcmp(magic, "BAI\1", 4) != 0) return fail("not a BAI or CSI index (bad magic)");
    int32_t nr;
    if (!c.take(nr)) return fail("truncated");
    if (nr < 0) return fail("negative reference count");
    if (nr > n_ref)
        return fail("it lists " + std::to_string(nr) + " reference sequences, the data file's header " + std::to_string(n_ref));
    x->refs.resize((size_t)nr);
    const uint32_t pseudo = x->pseudo_bin();
    for (Ref &R : x->refs) {
        int32_t nb;
        if (!c.take(nb)) return fail("truncated");
        if (nb < 0 || (size_t)nb > c.left() / 8) return fail(nb < 0 ? "negative bin count" : "truncated");
        for (int32_t j = 0; j < nb; ++j) {
            uint32_t bin; uint64_t loff = 0; int32_t nc;
            if (!c.take(bin) || (x->csi && !c.take(loff)) || !c.take(nc)) return fail("truncated");
            if (nc < 0 || (size_t)nc > c.left() / 16) return fail(nc < 0 ? "negative chunk count" : "truncated");
            if (bin > pseudo) return fail("bin " + std::to_string(bin) + " out of range");
            if (R.bins.count(bin) || (bin == pseudo && R.has_meta)) return fail("bin " + std::to_string(bin) + " listed twice");
            if (bin == pseudo) {
                if (nc != 2) return fail("malformed pseudo-bin");
                for (uint64_t &m : R.meta) c.take(m);
                R.has_meta = true;
                continue;
            }
            Bin &B = R.bins[bin];
            B.loff = loff;
            B.chunks.resize((size_t)nc);
            for (Chunk &k : B.chunks) {
                if (!c.take(k.beg) || !c.take(k.end)) return fail("truncated");
                if (k.beg > k.end) return fail("a chunk ends before it begins");
            }
        }
        if (!x->csi) {
            int32_t ni;
            if (!c.take(ni)) return fail("truncated");
            if (ni < 0 || (size_t)ni > c.left() / 8) return fail(ni < 0 ? "negative linear index size" : "truncated");
            R.lin.resize((size_t)ni);
            if (ni) c.take_n(R.lin.data(), 8 * (size_t)ni);
        }
    }
    if (c.left() >= 8) { c.take(x->n_no_coor); x->has_no_coor = true; }
    else if (c.left()) return fail("truncated");
    if (c.bad) return fail("truncated");
    return x;
}

std::vector<HtsIndex::Chunk> HtsIndex::query(int tid, int64_t beg, int64_t end) const
{
    std::vector<Chunk> out;
    if (tid < 0 || tid >= (int)refs.size()) return out;   // a sequence the index does not list has no records
    const Ref &R = refs[(size_t)tid];
    if (beg < 0) beg = 0;
    end = std::min(end, max_pos());
    if (beg >= end) return out;
    // no record overlapping [beg, ...) starts before min_off: the linear index (BAI), the loffset of the smallest listed
    // bin containing beg (CSI)
    uint64_t min_off = 0;
    if (!csi) {
        if (!R.lin.empty()) min_off = R.lin[std::min((size_t)(beg >> min_shift), R.lin.size() - 1)];
    } else {
        for (int64_t b = level_first_bin(depth) + (beg >> min_shift);; b = (b - 1) >> 3) {
            auto it = R.bins.find((uint32_t)b);
            if (it != R.bins.end()) { min_off = it->second.loff; break; }
            if (b == 0) break;
        }
    }
    std::vector<uint32_t> bins;
    reg2bins(beg, end, min_shift, depth, bins);
    for (uint32_t b : bins) {
        auto it = R.bins.find(b);
        if (it == R.bins.end()) continue;
        for (const Chunk &k : it->second.chunks) if (k.end > min_off) out.push_back(k);
    }
    std::sort(out.begin(), out.end(), [](const Chunk &a, const Chunk &b) { return a.beg < b.beg; });
    size_t m = 0;
    for (const Chunk &k : out) {
        if (m && k.beg <= out[m - 1].end) out[m - 1].end = std::max(out[m - 1].end, k.end);
        else out[m++] = k;
    }
    out.resize(m);
    return out;
}

// data as BGZF blocks of at most 0xff00 input bytes, then the empty EOF block
static bool write_bgzf(FILE *f, const std::string &data)
{
    std::vector<uint8_t> blk(1 << 17);
    for (size_t o = 0; o < data.size(); o += 0xff00) {
        const size_t n = std::min((size_t)0xff00, data.size() - o);
        z_stream z = z_stream();
        if (deflateInit2(&z, Z_DEFAULT_COMPRESSION, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) return false;
        z.next_in = (Bytef *)data.data() + o; z.avail_in = (uInt)n;
        z.next_out = blk.data() + 18; z.avail_out = (uInt)(blk.size() - 26);
        const int ret = deflate(&z, Z_FINISH);
        const size_t cl = z.total_out;
        deflateEnd(&z);
        if (ret != Z_STREAM_END || cl + 26 > 65536) return false;
        static const uint8_t head[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
        memcpy(blk.data(), head, 16);
        blk[16] = (uint8_t)((cl + 25) & 0xff); blk[17] = (uint8_t)((cl + 25) >> 8);
        const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), (const Bytef *)data.data() + o, (uInt)n), isize = (uint32_t)n;
        memcpy(blk.data() + 18 + cl, &crc, 4); memcpy(blk.data() + 22 + cl, &isize, 4);
        if (fwrite(blk.data(), 1, cl + 26, f) != cl + 26) return false;
    }
    static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    return fwrite(eof, 1, sizeof eof, f) == sizeof eof;
}

bool HtsIndex::save(const std::string &path, std::string &err) const
{
    std::string b;
    auto put = [&](const void *p, size_t n) { b.append((const char *)p, n); };
    auto i32 = [&](int32_t v) { put(&v, 4); };
    auto u64 = [&](uint64_t v) { put(&v, 8); };
    put(csi ? "CSI\1" : "BAI\1", 4);
    if (csi) { i32(min_shift); i32(depth); i32(0); }
    i32((int32_t)refs.size());
    for (const Ref &R : refs) {
        i32((int32_t)(R.bins.size() + (R.has_meta ? 1 : 0)));
        for (const auto &kv : R.bins) {
            put(&kv.first, 4);
            if (csi) u64(kv.second.loff);
            i32((int32_t)kv.second.chunks.size());
            for (const Chunk &k : kv.second.chunks) { u64(k.beg); u64(k.end); }
        }
        if (R.has_meta) {   // pseudo-bin: the sequence's first and end offsets, its mapped and unmapped record counts
            const uint32_t pb = pseudo_bin();
            put(&pb, 4);
            if (csi) u64(0);
            i32(2);
            for (uint64_t m : R.meta) u64(m);
        }
        if (!csi) { i32((int32_t)R.lin.size()); put(R.lin.data(), 8 * R.lin.size()); }
    }
    if (has_no_coor) u64(n_no_coor);
    FILE *f = fopen(path.c_str(), "wb");
    if (!f) { err = "cannot create \"" + path + "\": " + strerror(errno); return false; }
    bool ok = csi ? write_bgzf(f, b) : fwrite(b.data(), 1, b.size(), f) == b.size();
    ok = (fclose(f) == 0) && ok;
    if (!ok) { err = "error writing \"" + path + "\""; remove(path.c_str()); }
    return ok;
}

int build_index(const std::string &in, const std::string &out, bool csi, int min_shift, std::string &err)
{
    std::unique_ptr<AlnReader> rd = AlnReader::open(in);
    if (!rd) { err = "failed to open \"" + in + "\": " + strerror(errno); return 1; }
    if (!rd->is_bam() || !rd->bgzf() || in == "-") { err = "\"" + in + "\" is not a BGZF-compressed BAM file"; return 1; }
    const Header &h = rd->header();
    HtsIndex x;
    x.csi = csi;
    x.min_shift = csi ? min_shift : 14;
    if (csi) {   // enough levels for the longest sequence and reads running up to 1 Mb past its end
        int64_t max_len = 0;
        for (int64_t l : h.lens) max_len = std::max(max_len, l);
        for (x.depth = 0; x.max_pos() < max_len + (1 << 20); ++x.depth) {}
    }
    x.refs.resize((size_t)h.n_ref());
    x.has_no_coor = true;
    const int ms = x.min_shift;
    const uint64_t unset = UINT64_MAX;
    int last_tid = -2; int64_t last_pos = 0;
    Record r;
    for (;;) {
        const uint64_t ob = rd->tell();
        const int ret = rd->next(r);
        if (ret == -1) break;
        if (ret < -1) { err = "error reading \"" + in + "\""; return 1; }
        const uint64_t oe = rd->tell();
        if (r.tid < -1 || r.tid >= h.n_ref()) { err = "\"" + in + "\": a record names reference sequence #" + std::to_string(r.tid); return 1; }
        auto where = [&](int t, int64_t p) { return t < 0 ? std::string("*") : h.names[(size_t)t] + ":" + std::to_string(p + 1); };
        if ((last_tid == -1 && r.tid != -1) || (r.tid >= 0 && r.tid < last_tid) || (r.tid >= 0 && r.tid == last_tid && r.pos < last_pos)) {
            err = "\"" + in + "\" is not sorted by coordinate: " + where(r.tid, r.pos) + " follows " + where(last_tid, last_pos);
            return 1;
        }
        last_tid = r.tid; last_pos = r.pos;
        if (r.tid < 0) { ++x.n_no_coor; continue; }
        const int64_t beg = std::max<int64_t>(r.pos, 0), end = std::max(r.endpos(), beg + 1);   // unmapped placed reads: one base
        if (end > x.max_pos()) {
            err = "\"" + in + "\": " + where(r.tid, end - 1) + " lies beyond the " + std::to_string(x.max_pos()) + " positions a " +
                  (csi ? "CSI of these parameters" : "BAI") + " can address" + (csi ? "" : "; use -c for a CSI index");
            return 1;
        }
        HtsIndex::Ref &R = x.refs[(size_t)r.tid];
        if (!R.has_meta) { R.has_meta = true; R.meta[0] = ob; }
        R.meta[1] = oe;
        ++R.meta[(r.flag & F_UNMAP) ? 3 : 2];
        HtsIndex::Bin &B = R.bins[reg2bin(beg, end, ms, x.depth)];
        if (!B.chunks.empty() && B.chunks.back().end == ob) B.chunks.back().end = oe;
        else B.chunks.push_back({ob, oe});
        // linear index: the first record overlapping a window has the smallest offset of all that do
        const size_t w0 = (size_t)(beg >> ms), w1 = (size_t)((end - 1) >> ms);
        if (R.lin.size() <= w1) R.lin.resize(w1 + 1, unset);
        for (size_t w = w0; w <= w1; ++w) if (R.lin[w] == unset) R.lin[w] = ob;
    }
    for (HtsIndex::Ref &R : x.refs) {
        uint64_t prev = 0;
        for (uint64_t &v : R.lin) { if (v == unset) v = prev; else prev = v; }   // forward fill: an empty window takes the one before
        if (!csi) continue;
        // CSI: a bin's loffset is the linear offset of its first window (no record overlapping the bin starts before it)
        for (auto &kv : R.bins) {
            int l = 0;
            while (l < x.depth && (int64_t)kv.first >= level_first_bin(l + 1)) ++l;
            const size_t w = (size_t)(((int64_t)kv.first - level_first_bin(l)) << 3 * (x.depth - l));
            kv.second.loff = R.lin.empty() ? 0 : R.lin[std::min(w, R.lin.size() - 1)];
        }
        std::vector<uint64_t>().swap(R.lin);
    }
    return x.save(out, err) ? 0 : 1;
}

// ------------------------------------------------------------------ FASTA
std::unique_ptr<Fasta> Fasta::load(const std::string &path)
{
    gzFile fp = gzopen(path.c_str(), "rb");
    if (!fp) return nullptr;
    gzbuffer(fp, 1 << 18);
    std::unique_ptr<Fasta> fa(new Fasta());
    char buf[1 << 16];
    bool in_name = false;
    while (gzgets(fp, buf, sizeof buf)) {
        size_t n = strlen(buf);
        bool eol = n && buf[n - 1] == '\n';
        if (in_name) { in_name = !eol; continue; }   // tail of a very long header line
        if (buf[0] == '>') {
            char *e = buf + 1;
            while (*e && !isspace((unsigned char)*e)) ++e;
            fa->names.emplace_back(buf + 1, e);
            fa->seqs.emplace_back();
            in_name = !eol;
        } else if (!fa->seqs.empty()) {
            std::string &s = fa->seqs.back();
            for (size_t i = 0; i < n; ++i) if (isgraph((unsigned char)buf[i])) s.push_back(buf[i]);
        }
    }
    gzclose(fp);
    return fa;
}
int Fasta::find(const std::string &n) const
{
    for (size_t i = 0; i < names.size(); ++i) if (names[i] == n) return (int)i;
    return -1;
}

// ------------------------------------------------------------------ BED (bedidx.c:102-191, :258-360)
static constexpr int kBedShift = 13;

std::unique_ptr<Bed> Bed::load(const std::string &path)
{
    gzFile fp = gzopen(path.c_str(), "rb");
    if (!fp) return nullptr;
    std::unique_ptr<Bed> bed(new Bed());
    char buf[1 << 16];
    while (gzgets(fp, buf, sizeof buf)) {
        char *ref = buf;
        while (*ref && isspace((unsigned char)*ref)) ++ref;
        if (!*ref || *ref == '#') continue;
        char *re = ref;
        while (*re && !isspace((unsigned char)*re)) ++re;
        unsigned long long b = 0, e = 0; int num = 0;
        if (*re) { *re = 0; num = sscanf(re + 1, "%llu %llu", &b, &e); }
        if (num == 1) e = b--;
        if (num < 1 || e < b) {
            if (!strcmp(ref, "browser") || !strcmp(ref, "track")) continue;
            fprintf(stderr, "[bed_read] Parse error reading \"%s\"\n", path.c_str());
            gzclose(fp);
            return nullptr;
        }
        bed->chr[ref].iv.emplace_back((int64_t)b, (int64_t)e);
    }
    gzclose(fp);
    for (auto &kv : bed->chr) {
        Chr &c = kv.second;
        std::stable_sort(c.iv.begin(), c.iv.end(), [](const std::pair<int64_t, int64_t> &x, const std::pair<int64_t, int64_t> &y) { return x.first < y.first; });
        int64_t last_end = 0;
        for (size_t i = 0; i < c.iv.size(); ++i) {
            int64_t bb = c.iv[i].first >= 0 ? c.iv[i].first >> kBedShift : 0, ee = c.iv[i].second >= 0 ? c.iv[i].second >> kBedShift : 0;
            if (ee < last_end) continue;
            if ((size_t)ee + 1 > c.idx.size()) c.idx.resize((size_t)ee + 1, 0);
            int64_t j;
            for (j = last_end; j < bb; ++j) c.idx[(size_t)j] = i > 0 ? (int)i - 1 : 0;
            for (; j <= ee; ++j) c.idx[(size_t)j] = (int)i;
            last_end = ee + 1;
        }
        c.max_idx = last_end;
    }
    return bed;
}

bool Bed::overlap(const std::string &name, int64_t beg, int64_t end) const
{
    auto it = chr.find(name);
    if (it == chr.end() || it->second.iv.empty()) return false;
    const Chr &c = it->second;
    size_t off = 0;
    if (!c.idx.empty() && c.max_idx > 0 && beg >= 0)
        off = (size_t)((beg >> kBedShift) >= c.max_idx ? c.idx[(size_t)c.max_idx - 1] : c.idx[(size_t)(beg >> kBedShift)]);
    for (size_t i = off; i < c.iv.size(); ++i) {
        if (c.iv[i].first >= end) break;
        if (c.iv[i].second > beg && c.iv[i].first < end) return true;
    }
    return false;
}

void Bed::merged(const std::string &name, std::vector<int64_t> &b, std::vector<int64_t> &e) const
{
    b.clear(); e.clear();
    auto it = chr.find(name);
    if (it == chr.end()) return;
    for (auto &iv : it->second.iv) {   // already sorted by start
        if (iv.second <= iv.first) continue;   // empty interval never contains a position
        if (!b.empty() && iv.first <= e.back()) { if (iv.second > e.back()) e.back() = iv.second; }
        else { b.push_back(iv.first); e.push_back(iv.second); }
    }
}

bool read_file_list(const std::string &path, std::vector<std::string> &out)
{
    FILE *f = fopen(path.c_str(), "r");
    if (!f) { fprintf(stderr, "%s: %s\n", path.c_str(), strerror(errno)); return false; }
    char buf[1024];
    while (fgets(buf, sizeof buf, f)) {
        size_t l = strlen(buf);
        while (l && isspace((unsigned char)buf[l - 1])) --l;
        if (!l) continue;
        buf[l] = 0;
        std::string s = buf;
        struct stat sb;
        bool url = s.compare(0, 7, "file://") == 0;
        if (url) s = s.substr(7);
        if (stat(s.c_str(), &sb) != 0) {
            fprintf(stderr, "The file list \"%s\" appears broken, could not locate: %s\n", path.c_str(), buf);
            fclose(f);
            return false;
        }
        out.push_back(s);
    }
    fclose(f);
    if (out.empty()) { fprintf(stderr, "No files read from %s\n", path.c_str()); return false; }
    return true;
}

}  // namespace b200
