/*
 * oracle/io.c -- TEST INFRASTRUCTURE ONLY (CPU oracle).
 *
 * File-format substrate for the oracle: SAM text / BAM (BGZF through zlib's
 * multi-member gzread) record reader, FASTA loader, BED reader, region and
 * flag parsing.  These play the role of the htslib calls listed in SURVEY.md
 * section 2b (sam_open/sam_hdr_read/sam_read1/sam_itr_*, fai_load/
 * faidx_fetch_seq64) and of bedidx.c; formats follow hts-specs SAMv1.
 */
#include "hl.h"
#include <ctype.h>
#include <errno.h>
#include <zlib.h>

const unsigned char nt16_table[256] = {
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
     1, 2, 4, 8, 15,15,15,15, 15,15,15,15, 15, 0,15,15,
    15, 1,14, 2, 13,15,15, 4, 11,15,15,12, 15, 3,15,15,
    15,15, 5, 6,  8,15, 7, 9, 15,10,15,15, 15,15,15,15,
    15, 1,14, 2, 13,15,15, 4, 11,15,15,12, 15, 3,15,15,
    15,15, 5, 6,  8,15, 7, 9, 15,10,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15,
    15,15,15,15, 15,15,15,15, 15,15,15,15, 15,15,15,15
};
const char nt16_str[] = "=ACMGRSVTWYHKDBN";
const int nt16_int[] = { 4, 0, 1, 4, 2, 4, 4, 4, 3, 4, 4, 4, 4, 4, 4, 4 };

/* ---------- str_t ---------- */
static void s_need(str_t *s, size_t extra)
{
    if (s->l + extra + 1 > s->m) {
        size_t m = s->m ? s->m : 256;
        while (m < s->l + extra + 1) m <<= 1;
        s->s = realloc(s->s, m);
        s->m = m;
    }
}
void s_putc(str_t *s, int c) { s_need(s, 1); s->s[s->l++] = (char)c; s->s[s->l] = 0; }
void s_putn(str_t *s, const char *p, size_t n) { s_need(s, n); memcpy(s->s + s->l, p, n); s->l += n; s->s[s->l] = 0; }
void s_puts(str_t *s, const char *p) { s_putn(s, p, strlen(p)); }
void s_putll(str_t *s, long long v)
{
    char b[32]; int n = 0; unsigned long long u = v < 0 ? 0ULL - (unsigned long long)v : (unsigned long long)v;
    do { b[n++] = (char)('0' + u % 10); u /= 10; } while (u);
    if (v < 0) b[n++] = '-';
    s_need(s, (size_t)n);
    while (n) s->s[s->l++] = b[--n];
    s->s[s->l] = 0;
}

/* ---------- records ---------- */
void rec_init(rec_t *r) { memset(r, 0, sizeof(*r)); r->tid = r->mtid = -1; }
void rec_free(rec_t *r)
{
    free(r->qname); free(r->cigar); free(r->seq); free(r->qual); free(r->aux);
    memset(r, 0, sizeof(*r));
}
static void *dupmem(const void *p, size_t n) { void *q = malloc(n ? n : 1); if (n) memcpy(q, p, n); return q; }
void rec_copy(rec_t *d, const rec_t *s)
{
    rec_free(d);
    *d = *s;
    d->qname = dupmem(s->qname, strlen(s->qname) + 1);
    d->cigar = dupmem(s->cigar, 4 * (size_t)s->n_cigar);
    d->seq = dupmem(s->seq, (size_t)(s->l_qseq + 1) / 2);
    d->qual = dupmem(s->qual, (size_t)s->l_qseq);
    d->aux = dupmem(s->aux, (size_t)s->l_aux);
}
hpos_t rec_rlen(const rec_t *r)
{
    hpos_t l = 0; uint32_t k;
    for (k = 0; k < r->n_cigar; k++) {
        int op = cop(r->cigar[k]);
        if (op == C_M || op == C_D || op == C_N || op == C_EQ || op == C_X) l += cln(r->cigar[k]);
    }
    return l;
}
hpos_t rec_qlen(const rec_t *r)
{
    hpos_t l = 0; uint32_t k;
    for (k = 0; k < r->n_cigar; k++) {
        int op = cop(r->cigar[k]);
        if (op == C_M || op == C_I || op == C_S || op == C_EQ || op == C_X) l += cln(r->cigar[k]);
    }
    return l;
}
hpos_t rec_endpos(const rec_t *r)
{
    hpos_t rl = 1;
    if (!(r->flag & F_UNMAP) && r->n_cigar > 0) { rl = rec_rlen(r); if (rl == 0) rl = 1; }
    return r->pos + rl;
}

static int aux_type_size(int t)
{
    switch (t) {
    case 'A': case 'c': case 'C': return 1;
    case 's': case 'S': return 2;
    case 'i': case 'I': case 'f': return 4;
    case 'd': return 8;
    default: return 0;
    }
}
/* skip one aux value starting at type byte s; returns pointer past it, or NULL */
static const uint8_t *aux_skip(const uint8_t *s, const uint8_t *end)
{
    int t = *s++;
    int sz = aux_type_size(t);
    if (sz) return s + sz <= end ? s + sz : NULL;
    if (t == 'Z' || t == 'H') { while (s < end && *s) s++; return s < end ? s + 1 : NULL; }
    if (t == 'B') {
        if (s + 5 > end) return NULL;
        int esz = aux_type_size(*s); uint32_t n; memcpy(&n, s + 1, 4);
        s += 5 + (size_t)esz * n;
        return (esz && s <= end) ? s : NULL;
    }
    return NULL;
}
const uint8_t *rec_aux_get(const rec_t *r, const char tag[2])
{
    const uint8_t *s = r->aux, *end = r->aux + r->l_aux;
    while (s && s + 3 <= end) {
        if (s[0] == (uint8_t)tag[0] && s[1] == (uint8_t)tag[1]) return s + 2;
        s = aux_skip(s + 2, end);
    }
    return NULL;
}
int rec_aux_del(rec_t *r, const uint8_t *s)
{
    uint8_t *end = r->aux + r->l_aux;
    const uint8_t *nx = aux_skip(s, end);
    if (!nx) return -1;
    uint8_t *from = (uint8_t *)s - 2;
    memmove(from, nx, (size_t)(end - nx));
    r->l_aux -= (int)(nx - from);
    return 0;
}
void rec_aux_append(rec_t *r, const char tag[2], char type, int len, const uint8_t *data)
{
    r->aux = realloc(r->aux, (size_t)r->l_aux + 3 + (size_t)len);
    r->aux[r->l_aux] = (uint8_t)tag[0]; r->aux[r->l_aux + 1] = (uint8_t)tag[1]; r->aux[r->l_aux + 2] = (uint8_t)type;
    memcpy(r->aux + r->l_aux + 3, data, (size_t)len);
    r->l_aux += 3 + len;
}

/* ---------- header ---------- */
int hdr_name2tid(const hdr_t *h, const char *name)
{
    int i;
    for (i = 0; i < h->n_ref; i++) if (strcmp(h->name[i], name) == 0) return i;
    return -1;
}
void hdr_free(hdr_t *h)
{
    int i;
    if (!h) return;
    for (i = 0; i < h->n_ref; i++) free(h->name[i]);
    free(h->name); free(h->len); free(h->text); free(h);
}
static void hdr_add_ref(hdr_t *h, const char *name, hpos_t len)
{
    h->name = realloc(h->name, sizeof(char *) * (size_t)(h->n_ref + 1));
    h->len = realloc(h->len, sizeof(hpos_t) * (size_t)(h->n_ref + 1));
    h->name[h->n_ref] = strdup(name);
    h->len[h->n_ref] = len;
    h->n_ref++;
}
/* parse @SQ lines out of header text */
static void hdr_parse_sq(hdr_t *h)
{
    const char *p = h->text;
    while (p && *p) {
        const char *e = strchr(p, '\n');
        size_t n = e ? (size_t)(e - p) : strlen(p);
        if (n > 3 && strncmp(p, "@SQ", 3) == 0) {
            char *line = strndup(p, n), *sn = NULL, *save = NULL, *tok;
            hpos_t ln = 0;
            for (tok = strtok_r(line, "\t", &save); tok; tok = strtok_r(NULL, "\t", &save)) {
                if (strncmp(tok, "SN:", 3) == 0) sn = tok + 3;
                else if (strncmp(tok, "LN:", 3) == 0) ln = strtoll(tok + 3, NULL, 10);
            }
            if (sn) hdr_add_ref(h, sn, ln);
            free(line);
        }
        p = e ? e + 1 : NULL;
    }
}

/* ---------- reader ---------- */
struct reader_t {
    gzFile fp;
    int is_bam;
    hdr_t *h;
    char *pending;           /* first SAM record line read while scanning header */
    int has_reg, rtid; hpos_t rbeg, rend;
    str_t line;
};

static int gz_getline(gzFile fp, str_t *s)
{
    char buf[65536];
    s->l = 0; if (s->s) s->s[0] = 0;
    int got = 0;
    while (gzgets(fp, buf, sizeof buf)) {
        size_t n = strlen(buf);
        got = 1;
        if (n && buf[n - 1] == '\n') { s_putn(s, buf, n - 1); if (s->l && s->s[s->l - 1] == '\r') s->s[--s->l] = 0; return 1; }
        s_putn(s, buf, n);
    }
    return got;
}

static int rd_i32(gzFile fp, int32_t *v) { return gzread(fp, v, 4) == 4 ? 0 : -1; }

reader_t *reader_open(const char *fn, const char *fai)
{
    reader_t *rd = calloc(1, sizeof(*rd));
    rd->fp = strcmp(fn, "-") ? gzopen(fn, "rb") : gzdopen(0, "rb");
    if (!rd->fp) { free(rd); return NULL; }
    gzbuffer(rd->fp, 1 << 18);
    rd->h = calloc(1, sizeof(hdr_t));
    int c0 = gzgetc(rd->fp);
    if (c0 < 0) { rd->h->text = strdup(""); return rd; } /* empty input */
    gzungetc(c0, rd->fp);
    int is_bam = 0;
    if (c0 == 'B') {   /* "BAM\1" magic, or a SAM record whose name starts with B: look at four bytes */
        char magic[4]; int got = gzread(rd->fp, magic, 4), j;
        if (got == 4 && memcmp(magic, "BAM\1", 4) == 0) is_bam = 1;
        else for (j = got - 1; j >= 0; j--) gzungetc((unsigned char)magic[j], rd->fp);
    }
    if (is_bam) {
        rd->is_bam = 1;
        int32_t l_text, n_ref, i;
        if (rd_i32(rd->fp, &l_text)) goto fail;
        rd->h->text = calloc((size_t)l_text + 1, 1);
        if (gzread(rd->fp, rd->h->text, (unsigned)l_text) != l_text) goto fail;
        if (rd_i32(rd->fp, &n_ref)) goto fail;
        for (i = 0; i < n_ref; i++) {
            int32_t l_name, l_ref;
            if (rd_i32(rd->fp, &l_name)) goto fail;
            char *nm = malloc((size_t)l_name + 1);
            if (gzread(rd->fp, nm, (unsigned)l_name) != l_name) goto fail;
            nm[l_name] = 0;
            if (rd_i32(rd->fp, &l_ref)) goto fail;
            hdr_add_ref(rd->h, nm, l_ref);
            free(nm);
        }
        return rd;
    }
    /* SAM text: slurp header lines */
    str_t text = {0, 0, NULL};
    for (;;) {
        if (!gz_getline(rd->fp, &rd->line)) break;
        if (rd->line.l && rd->line.s[0] == '@') { s_puts(&text, rd->line.s); s_putc(&text, '\n'); }
        else { rd->pending = strdup(rd->line.s ? rd->line.s : ""); break; }
    }
    rd->h->text = text.s ? text.s : strdup("");
    hdr_parse_sq(rd->h);
    if (rd->h->n_ref == 0 && fai) { /* headerless SAM: contigs from a .fai */
        FILE *f = fopen(fai, "r");
        if (f) {
            char nm[1024]; long long ln;
            char ln_buf[4096];
            while (fgets(ln_buf, sizeof ln_buf, f))
                if (sscanf(ln_buf, "%1023s %lld", nm, &ln) == 2) hdr_add_ref(rd->h, nm, ln);
            fclose(f);
        }
    }
    return rd;
fail:
    reader_close(rd);
    return NULL;
}
hdr_t *reader_hdr(reader_t *rd) { return rd->h; }
void reader_close(reader_t *rd)
{
    if (!rd) return;
    if (rd->fp) gzclose(rd->fp);
    hdr_free(rd->h); free(rd->pending); free(rd->line.s); free(rd);
}

int parse_region(const hdr_t *h, const char *reg, int *tid, hpos_t *beg, hpos_t *end)
{
    *beg = 0; *end = HPOS_MAX;
    int t = hdr_name2tid(h, reg);
    if (t >= 0) { *tid = t; return 0; }
    const char *colon = strrchr(reg, ':');
    if (!colon) return -1;
    char *name = strndup(reg, (size_t)(colon - reg));
    t = hdr_name2tid(h, name);
    free(name);
    if (t < 0) return -1;
    /* numbers with optional thousands commas: beg[-end], 1-based inclusive */
    char num[64]; int n = 0; const char *p = colon + 1;
    long long b = 0, e = -1; int have_dash = 0;
    for (; *p && *p != '-'; p++) if (*p != ',') { if (n < 62) num[n++] = *p; }
    num[n] = 0; if (n) b = strtoll(num, NULL, 10);
    if (*p == '-') {
        have_dash = 1; p++; n = 0;
        for (; *p; p++) if (*p != ',') { if (n < 62) num[n++] = *p; }
        num[n] = 0; if (n) e = strtoll(num, NULL, 10);
    }
    *beg = b > 0 ? b - 1 : 0;
    *end = (have_dash && e >= 0) ? e : HPOS_MAX;
    if (*beg >= *end) return -1;
    *tid = t;
    return 0;
}
int reader_set_region(reader_t *rd, const char *reg, int *tid, hpos_t *beg, hpos_t *end)
{
    if (parse_region(rd->h, reg, &rd->rtid, &rd->rbeg, &rd->rend) < 0) return -1;
    rd->has_reg = 1;
    *tid = rd->rtid; *beg = rd->rbeg; *end = rd->rend;
    return 0;
}

static void put_aux_int(rec_t *r, const char tag[2], long long v)
{
    uint8_t b[4];
    if (v < 0) {
        if (v >= -128) { int8_t x = (int8_t)v; rec_aux_append(r, tag, 'c', 1, (uint8_t *)&x); }
        else if (v >= -32768) { int16_t x = (int16_t)v; memcpy(b, &x, 2); rec_aux_append(r, tag, 's', 2, b); }
        else { int32_t x = (int32_t)v; memcpy(b, &x, 4); rec_aux_append(r, tag, 'i', 4, b); }
    } else {
        if (v < 256) { uint8_t x = (uint8_t)v; rec_aux_append(r, tag, 'C', 1, &x); }
        else if (v < 65536) { uint16_t x = (uint16_t)v; memcpy(b, &x, 2); rec_aux_append(r, tag, 'S', 2, b); }
        else { uint32_t x = (uint32_t)v; memcpy(b, &x, 4); rec_aux_append(r, tag, 'I', 4, b); }
    }
}

static int parse_sam_line(const hdr_t *h, char *line, rec_t *r)
{
    char *f[12], *p = line; int nf = 0;
    rec_free(r); rec_init(r);
    while (nf < 11) {
        f[nf++] = p;
        char *t = strchr(p, '\t');
        if (!t) { p = NULL; break; }
        *t = 0; p = t + 1;
    }
    if (nf < 11) return -2;
    char *aux = p; /* may be NULL */
    r->qname = strdup(f[0]);
    r->flag = (uint16_t)strtol(f[1], NULL, 10);
    r->tid = strcmp(f[2], "*") ? hdr_name2tid(h, f[2]) : -1;
    r->pos = strtoll(f[3], NULL, 10) - 1;
    r->mapq = (uint8_t)strtol(f[4], NULL, 10);
    if (strcmp(f[5], "*")) {
        const char *c = f[5]; uint32_t n = 0, cap = 8;
        r->cigar = malloc(4 * cap);
        while (*c) {
            char *e; unsigned long l = strtoul(c, &e, 10);
            static const char ops[] = "MIDNSHP=XB";
            const char *o = strchr(ops, *e);
            if (!o || !*e) return -2;
            if (n == cap) { cap <<= 1; r->cigar = realloc(r->cigar, 4 * cap); }
            r->cigar[n++] = (uint32_t)l << 4 | (uint32_t)(o - ops);
            c = e + 1;
        }
        r->n_cigar = n;
    } else r->cigar = malloc(4);
    if (strcmp(f[6], "=") == 0) r->mtid = r->tid;
    else r->mtid = strcmp(f[6], "*") ? hdr_name2tid(h, f[6]) : -1;
    r->mpos = strtoll(f[7], NULL, 10) - 1;
    r->isize = strtoll(f[8], NULL, 10);
    if (strcmp(f[9], "*")) {
        int l = (int)strlen(f[9]), i;
        r->l_qseq = l;
        r->seq = calloc((size_t)(l + 1) / 2 + 1, 1);
        for (i = 0; i < l; i++) r->seq[i >> 1] |= (uint8_t)(nt16_table[(uint8_t)f[9][i]] << ((~i & 1) << 2));
        r->qual = malloc((size_t)l + 1);
        if (strcmp(f[10], "*") == 0) memset(r->qual, 0xff, (size_t)l);
        else for (i = 0; i < l; i++) r->qual[i] = (uint8_t)(f[10][i] - 33);
    } else { r->l_qseq = 0; r->seq = calloc(1, 1); r->qual = calloc(1, 1); }
    r->aux = malloc(1); r->l_aux = 0;
    while (aux && *aux) {
        char *t = strchr(aux, '\t');
        if (t) *t = 0;
        size_t L = strlen(aux);
        if (L >= 5 && aux[2] == ':' && aux[4] == ':') {
            char type = aux[3]; const char *v = aux + 5;
            if (type == 'A') rec_aux_append(r, aux, 'A', 1, (const uint8_t *)v);
            else if (type == 'i') put_aux_int(r, aux, strtoll(v, NULL, 10));
            else if (type == 'f') { float x = strtof(v, NULL); rec_aux_append(r, aux, 'f', 4, (uint8_t *)&x); }
            else if (type == 'Z' || type == 'H') rec_aux_append(r, aux, type, (int)strlen(v) + 1, (const uint8_t *)v);
            else if (type == 'B') {
                char st = v[0]; int esz = aux_type_size(st); uint32_t n = 0; const char *q;
                for (q = v + 1; *q; q++) if (*q == ',') n++;
                uint8_t *buf = malloc(5 + (size_t)esz * n + 8); buf[0] = (uint8_t)st; memcpy(buf + 1, &n, 4);
                uint8_t *o = buf + 5; q = v + 1;
                while (*q == ',') {
                    char *e; q++;
                    if (st == 'f') { float x = strtof(q, &e); memcpy(o, &x, 4); }
                    else { long long x = strtoll(q, &e, 10); memcpy(o, &x, (size_t)esz); }
                    o += esz; q = e;
                }
                rec_aux_append(r, aux, 'B', (int)(o - buf), buf);
                free(buf);
            }
        }
        aux = t ? t + 1 : NULL;
    }
    return 0;
}

static int read_bam_rec(reader_t *rd, rec_t *r)
{
    int32_t bs;
    int n = gzread(rd->fp, &bs, 4);
    if (n == 0) return -1;
    if (n != 4 || bs < 32) return -2;
    uint8_t *d = malloc((size_t)bs);
    if (gzread(rd->fp, d, (unsigned)bs) != bs) { free(d); return -2; }
    rec_free(r); rec_init(r);
    int32_t i32; uint16_t u16;
    memcpy(&r->tid, d, 4);
    memcpy(&i32, d + 4, 4); r->pos = i32;
    int l_name = d[8]; r->mapq = d[9];
    memcpy(&u16, d + 12, 2); r->n_cigar = u16;
    memcpy(&r->flag, d + 14, 2);
    memcpy(&r->l_qseq, d + 16, 4);
    memcpy(&r->mtid, d + 20, 4);
    memcpy(&i32, d + 24, 4); r->mpos = i32;
    memcpy(&i32, d + 28, 4); r->isize = i32;
    uint8_t *p = d + 32;
    r->qname = strndup((char *)p, (size_t)l_name); p += l_name;
    r->cigar = dupmem(p, 4 * (size_t)r->n_cigar); p += 4 * (size_t)r->n_cigar;
    r->seq = dupmem(p, (size_t)(r->l_qseq + 1) / 2); p += (r->l_qseq + 1) / 2;
    r->qual = dupmem(p, (size_t)r->l_qseq); p += r->l_qseq;
    r->l_aux = (int)(d + bs - p);
    r->aux = dupmem(p, (size_t)r->l_aux);
    free(d);
    /* SAMv1 4.2.2: a CIGAR of more than 65535 ops is stored in a CG:B,I tag; the record's own CIGAR is then the
       placeholder <l_qseq>S <rlen>N.  The tag's ops become the CIGAR and the tag is dropped. */
    if (r->n_cigar == 2 && (r->cigar[0] & 0xf) == 4 && (int32_t)(r->cigar[0] >> 4) == r->l_qseq && (r->cigar[1] & 0xf) == 3) {
        const uint8_t *cg = rec_aux_get(r, "CG");
        if (cg && cg[0] == 'B' && cg[1] == 'I') {
            uint32_t nc; memcpy(&nc, cg + 2, 4);
            if (nc > 0 && cg + 6 + 4 * (size_t)nc <= r->aux + r->l_aux) {
                uint32_t *ops = malloc(4 * (size_t)nc);
                memcpy(ops, cg + 6, 4 * (size_t)nc);
                free(r->cigar); r->cigar = ops; r->n_cigar = nc;
                rec_aux_del(r, cg);
            }
        }
    }
    return 0;
}

int reader_next(reader_t *rd, rec_t *r)
{
    for (;;) {
        int ret;
        if (rd->is_bam) ret = read_bam_rec(rd, r);
        else {
            char *ln;
            if (rd->pending) { ln = rd->pending; rd->pending = NULL; ret = *ln ? parse_sam_line(rd->h, ln, r) : 1; free(ln); }
            else if (gz_getline(rd->fp, &rd->line)) ret = rd->line.l ? parse_sam_line(rd->h, rd->line.s, r) : 1;
            else ret = -1;
            if (ret == 1) continue; /* blank line */
        }
        if (ret < 0) return ret;
        if (rd->has_reg) {
            if (r->tid != rd->rtid) continue;
            if (!(r->pos < rd->rend && rec_endpos(r) > rd->rbeg)) continue;
        }
        return 0;
    }
}

/* ---------- FASTA ---------- */
fasta_t *fasta_load(const char *fn)
{
    gzFile fp = gzopen(fn, "rb");
    if (!fp) return NULL;
    gzbuffer(fp, 1 << 18);
    fasta_t *fa = calloc(1, sizeof(*fa));
    str_t line = {0, 0, NULL}, seq = {0, 0, NULL};
    int cur = -1;
    while (gz_getline(fp, &line)) {
        if (line.l && line.s[0] == '>') {
            if (cur >= 0) { fa->seq[cur] = seq.s ? seq.s : strdup(""); fa->len[cur] = (hpos_t)seq.l; seq.s = NULL; seq.l = seq.m = 0; }
            char *nm = line.s + 1, *e = nm;
            while (*e && !isspace((unsigned char)*e)) e++;
            *e = 0;
            cur = fa->n++;
            fa->name = realloc(fa->name, sizeof(char *) * (size_t)fa->n);
            fa->seq = realloc(fa->seq, sizeof(char *) * (size_t)fa->n);
            fa->len = realloc(fa->len, sizeof(hpos_t) * (size_t)fa->n);
            fa->name[cur] = strdup(nm); fa->seq[cur] = NULL; fa->len[cur] = 0;
        } else if (cur >= 0) {
            size_t i;
            for (i = 0; i < line.l; i++) if (isgraph((unsigned char)line.s[i])) s_putc(&seq, line.s[i]);
        }
    }
    if (cur >= 0) { fa->seq[cur] = seq.s ? seq.s : strdup(""); fa->len[cur] = (hpos_t)seq.l; }
    free(line.s);
    gzclose(fp);
    return fa;
}
int fasta_find(const fasta_t *fa, const char *name)
{
    int i;
    for (i = 0; i < fa->n; i++) if (strcmp(fa->name[i], name) == 0) return i;
    return -1;
}
void fasta_free(fasta_t *fa)
{
    int i;
    if (!fa) return;
    for (i = 0; i < fa->n; i++) { free(fa->name[i]); free(fa->seq[i]); }
    free(fa->name); free(fa->seq); free(fa->len); free(fa);
}

/* ---------- BED (follows bedidx.c:102-191 index+overlap, :258-360 reader) ---------- */
typedef struct { hpos_t beg, end; } ival_t;
typedef struct { char *chr; int n, m; ival_t *a; int *idx; hpos_t max_idx; } bedchr_t;
struct bed_t { int n; bedchr_t *c; };
#define BED_SHIFT 13

static int ival_cmp(const void *a, const void *b)
{
    hpos_t x = ((const ival_t *)a)->beg, y = ((const ival_t *)b)->beg;
    return x < y ? -1 : x > y;
}
static void bed_index_chr(bedchr_t *p)
{
    int i; size_t cap = 0; hpos_t last_end = 0;
    qsort(p->a, (size_t)p->n, sizeof(ival_t), ival_cmp);
    for (i = 0; i < p->n; i++) {
        hpos_t beg = p->a[i].beg >= 0 ? p->a[i].beg >> BED_SHIFT : 0;
        hpos_t end = p->a[i].end >= 0 ? p->a[i].end >> BED_SHIFT : 0, j;
        if (end < last_end) continue;
        if ((size_t)end + 1 > cap) { cap = ((size_t)end + 1) * 2; p->idx = realloc(p->idx, cap * sizeof(int)); }
        for (j = last_end; j < beg; j++) p->idx[j] = i > 0 ? i - 1 : 0;
        for (; j <= end; j++) p->idx[j] = i;
        last_end = end + 1;
    }
    p->max_idx = last_end;
}
bed_t *bed_load(const char *fn)
{
    gzFile fp = gzopen(fn, "rb");
    if (!fp) return NULL;
    bed_t *b = calloc(1, sizeof(*b));
    str_t line = {0, 0, NULL};
    while (gz_getline(fp, &line)) {
        char *ref = line.s, *re;
        unsigned long long beg = 0, end = 0; int num = 0, i;
        if (!line.l) continue;
        while (*ref && isspace((unsigned char)*ref)) ref++;
        if (!*ref || *ref == '#') continue;
        re = ref;
        while (*re && !isspace((unsigned char)*re)) re++;
        if (*re) { *re = 0; num = sscanf(re + 1, "%llu %llu", &beg, &end); }
        if (num == 1) end = beg--;
        if (num < 1 || end < beg) {
            if (!strcmp(ref, "browser") || !strcmp(ref, "track")) continue;
            fprintf(stderr, "[bed_read] Parse error reading \"%s\"\n", fn);
            bed_free(b); gzclose(fp); free(line.s);
            return NULL;
        }
        bedchr_t *p = NULL;
        for (i = 0; i < b->n; i++) if (!strcmp(b->c[i].chr, ref)) { p = &b->c[i]; break; }
        if (!p) {
            b->c = realloc(b->c, sizeof(bedchr_t) * (size_t)(b->n + 1));
            p = &b->c[b->n++]; memset(p, 0, sizeof(*p)); p->chr = strdup(ref);
        }
        if (p->n == p->m) { p->m = p->m ? p->m << 1 : 4; p->a = realloc(p->a, sizeof(ival_t) * (size_t)p->m); }
        p->a[p->n].beg = (hpos_t)beg; p->a[p->n++].end = (hpos_t)end;
    }
    free(line.s);
    gzclose(fp);
    int i;
    for (i = 0; i < b->n; i++) bed_index_chr(&b->c[i]);
    return b;
}
int bed_hit(const bed_t *b, const char *chr, hpos_t beg, hpos_t end)
{
    int i, min_off = 0;
    const bedchr_t *p = NULL;
    if (!b) return 0;
    for (i = 0; i < b->n; i++) if (!strcmp(b->c[i].chr, chr)) { p = &b->c[i]; break; }
    if (!p || p->n == 0) return 0;
    if (p->idx && p->max_idx > 0 && beg >= 0)
        min_off = (beg >> BED_SHIFT) >= p->max_idx ? p->idx[p->max_idx - 1] : p->idx[beg >> BED_SHIFT];
    for (i = min_off; i < p->n; i++) {
        if (p->a[i].beg >= end) break;
        if (p->a[i].end > beg && p->a[i].beg < end) return 1;
    }
    return 0;
}
void bed_free(bed_t *b)
{
    int i;
    if (!b) return;
    for (i = 0; i < b->n; i++) { free(b->c[i].chr); free(b->c[i].a); free(b->c[i].idx); }
    free(b->c); free(b);
}

/* ---------- flags (bam_str2flag) ---------- */
int parse_flag(const char *s)
{
    char *end;
    long v = strtol(s, &end, 0);
    if (end != s && *end == 0) return v < 0 ? -1 : (int)v;
    static const struct { const char *n; int f; } names[] = {
        {"PAIRED", F_PAIRED}, {"PROPER_PAIR", F_PROPER}, {"UNMAP", F_UNMAP}, {"MUNMAP", F_MUNMAP},
        {"REVERSE", F_REVERSE}, {"MREVERSE", F_MREVERSE}, {"READ1", F_READ1}, {"READ2", F_READ2},
        {"SECONDARY", F_SECONDARY}, {"QCFAIL", F_QCFAIL}, {"DUP", F_DUP}, {"SUPPLEMENTARY", F_SUPP}
    };
    int flag = 0;
    const char *p = s;
    while (*p) {
        const char *e = p; size_t i, n;
        while (*e && *e != ',') e++;
        n = (size_t)(e - p);
        for (i = 0; i < sizeof names / sizeof *names; i++)
            if (strlen(names[i].n) == n && strncasecmp(p, names[i].n, n) == 0) { flag |= names[i].f; break; }
        if (i == sizeof names / sizeof *names) return -1;
        p = *e ? e + 1 : e;
    }
    return flag;
}
