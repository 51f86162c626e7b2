/* fxo.c -- CPU ORACLE (test infrastructure only; see fxo.h).
 *
 * Restates, on a whole-file byte buffer, what the reference computes with its streaming
 * line reader.  Every function cites the reference lines it follows
 * (paths relative to the reference checkout).
 */
#include "fxo.h"
#include <string.h>
#include <stdlib.h>

/* ---- line splitting -------------------------------------------------------------------
 * The reference reads lines with ks_getuntil(ks, '\n', ...) (src/kseq.c:59-109): split on
 * '\n' only, '\r' stays in the line, a final unterminated line is still returned, and an
 * empty tail after the last '\n' yields no line.  `fxo_next_line` restates that on a
 * buffer: returns the line length (without '\n') or -1 at end of input. */
static int64_t fxo_next_line(const uint8_t *buf, int64_t n, int64_t cur, int64_t *next) {
    const uint8_t *nl;
    if (cur >= n) return -1;
    nl = (const uint8_t *)memchr(buf + cur, '\n', (size_t)(n - cur));
    if (nl) { *next = (int64_t)(nl - buf) + 1; return (int64_t)(nl - buf) - cur; }
    *next = n;
    return n - cur;
}

/* the uniform-lines bit of a record from the scan's counters: `bad` lines differ from the first
 * (line_len), the last one (last_len) among them or not; uniform iff no line but the last
 * differs and the last is no longer than the first */
static uint8_t fxo_uniform(int64_t bad, int64_t line_len, int64_t last_len) {
    const int64_t bad_before_last = bad - (last_len != line_len ? 1 : 0);
    return (uint8_t)(bad_before_last == 0 && last_len <= line_len);
}

/* ---- FASTA index scan -------------------------------------------------------------------
 * pyfastx_create_index, src/index.c:230-361.
 *  - position advances by len+1 per line, also for an unterminated last line (230-231),
 *    so the last record's blen is one larger than the bytes present (index.c:348).
 *  - a header is a line whose first byte is '>' (234).
 *  - elen from the header's last byte (267-269); dlen = len - elen (271).
 *  - chrom = bytes after '>' up to the first ' ' or '\t', bounded by dlen (289-301), or
 *    all dlen bytes with full_name (282-285).
 *  - sequence lines: llen = first line's len+1 (330-332); a line whose len+1 differs from
 *    llen counts as bad (325-327); slen += len - elen + 1 (335-338).
 *  - norm = bad <= 1 (237, 342).  The last record is always flushed (341-357).
 * Returns the number of rows (also when it exceeds cap; only cap rows are stored).
 * *no_header is set when the input never had a header line: the reference then still
 * writes one row (start = 0, NULL name); we return that row with nlen = -1.
 *
 * pad[0] is not reference behaviour: it is the "uniform lines" bit the GPU scan keeps for its own
 * kernels (they may index such a record with the slice formula).  With L_1 .. L_k the record's
 * sequence-line lengths counted as len + 1 (the unterminated last line of the file included), the
 * record is uniform iff L_1 = ... = L_{k-1} and L_k <= L_1 (always for k <= 1).  pad[1..5] stay 0. */
int64_t fxo_fasta_scan(const uint8_t *buf, int64_t n, int full_name,
                       fxo_fasta_row *rows, int64_t cap,
                       int64_t *total_slen, int *no_header) {
    int64_t cur = 0, next = 0, len;
    int64_t position = 0, start = 0, seq_len = 0, line_len = 0, bad = 0, total = 0;
    int64_t last_len = 0;   /* len + 1 of the record's latest sequence line (0: none yet) */
    int64_t nrows = 0;
    int32_t dlen = 0, nlen = -1;
    int elen = 1;

    while ((len = fxo_next_line(buf, n, cur, &next)) >= 0) {
        const uint8_t *line = buf + cur;
        position += len + 1;
        if (len > 0 && line[0] == '>') {
            if (start > 0) {
                if (nrows < cap) {
                    fxo_fasta_row *r = &rows[nrows];
                    memset(r, 0, sizeof(*r));
                    r->boff = start;
                    r->blen = position - start - len - 1;
                    r->slen = seq_len;
                    r->llen = line_len;
                    r->elen = (uint8_t)elen;
                    r->norm = (uint8_t)(bad > 1 ? 0 : 1);
                    r->dlen = dlen;
                    r->nlen = nlen;
                    r->pad[0] = fxo_uniform(bad, line_len, last_len);
                }
                ++nrows;
                total += seq_len;
            }
            start = position;
            seq_len = 0; line_len = 0; bad = 0; last_len = 0;
            elen = (line[len - 1] == '\r') ? 2 : 1;
            dlen = (int32_t)(len - elen);
            if (full_name) {
                nlen = dlen;
            } else {
                int32_t k = 0;
                while (k < dlen && line[1 + k] != ' ' && line[1 + k] != '\t') ++k;
                nlen = k;
            }
        } else {
            int64_t temp = len + 1;
            if (line_len > 0 && line_len != temp) ++bad;
            if (line_len == 0) line_len = temp;
            last_len = temp;
            seq_len += len - elen + 1;
        }
        cur = next;
    }
    /* final flush (index.c:341-361) */
    if (nrows < cap) {
        fxo_fasta_row *r = &rows[nrows];
        memset(r, 0, sizeof(*r));
        r->boff = start;
        r->blen = position - start;
        r->slen = seq_len;
        r->llen = line_len;
        r->elen = (uint8_t)elen;
        r->norm = (uint8_t)(bad > 1 ? 0 : 1);
        r->dlen = dlen;
        r->nlen = nlen;
        r->pad[0] = fxo_uniform(bad, line_len, last_len);
    }
    if (no_header) *no_header = (start == 0);
    ++nrows;
    total += seq_len;
    if (total_slen) *total_slen = total;
    return nrows;
}

/* ---- FASTQ index scan -------------------------------------------------------------------
 * pyfastx_fastq_create_index, src/fastq.c:89-171.  Records are four lines by the global
 * line counter (92-95).
 *  line 1: dlen = len (103); name = bytes after '@', minus a trailing '\r' (104-109), cut
 *          at the first ' ' found by strchr, i.e. searching stops at a NUL byte (112-117).
 *  line 2: soff = line start (122); rlen = len minus a trailing '\r' (124-128);
 *          size += rlen (129) -- also for a record that is never completed.
 *  line 4: qoff = line start (133); the row is written (136-145).
 * counts = line_num / 4 (159). */
int64_t fxo_fastq_scan(const uint8_t *buf, int64_t n,
                       fxo_fastq_row *rows, int64_t cap,
                       int64_t *total_size, int64_t *n_lines) {
    int64_t cur = 0, next = 0, len, line_num = 0, nrows = 0, size = 0;
    int64_t soff = 0, rlen = 0;
    int32_t dlen = 0, nlen = 0;

    while ((len = fxo_next_line(buf, n, cur, &next)) >= 0) {
        const uint8_t *line = buf + cur;
        ++line_num;
        switch (line_num % 4) {
        case 1: {
            int64_t l = len - 1, k;
            dlen = (int32_t)len;
            if (l > 0 && line[l] == '\r') --l;   /* name.s[name.l-1], name.s = line+1 */
            if (l < 0) l = 0;
            for (k = 0; k < l; ++k) {
                if (line[1 + k] == 0) { k = l; break; }
                if (line[1 + k] == ' ') break;
            }
            nlen = (int32_t)k;
            break;
        }
        case 2:
            soff = cur;
            rlen = (len > 0 && line[len - 1] == '\r') ? len - 1 : len;
            size += rlen;
            break;
        case 0:
            if (nrows < cap) {
                fxo_fastq_row *r = &rows[nrows];
                r->soff = soff; r->qoff = cur; r->rlen = rlen; r->dlen = dlen; r->nlen = nlen;
            }
            ++nrows;
            break;
        default: break;
        }
        cur = next;
    }
    if (total_size) *total_size = size;
    if (n_lines) *n_lines = line_num;
    return nrows;
}

/* ---- slice -> byte range ------------------------------------------------------------------
 * pyfastx_sequence_subscript, src/sequence.c:498-510 (same math in fasta.c:293-304):
 * 0-based half-open [s,e) on a norm=1 record. */
void fxo_slice_range(const fxo_fasta_row *row, int64_t s, int64_t e,
                     int64_t *offset, int64_t *byte_len) {
    int64_t bpl = row->llen - row->elen;
    int64_t bs = s / bpl, be = e / bpl;
    *offset = row->boff + s + (int64_t)row->elen * bs;
    *byte_len = (e - s) + (be - bs) * (int64_t)row->elen;
}

/* remove_space / remove_space_uppercase, src/util.c:166-194: drop exactly the bytes 10, 13
 * and 32 (jump_table, util.c:157-164; tab 9 is kept); the uppercase variant maps a-z to
 * A-Z (Py_TOUPPER).  Bytes >= 128 index past the reference's 128-entry table (UB there);
 * the oracle keeps them unchanged. */
int64_t fxo_strip(uint8_t *p, int64_t len, int upper) {
    int64_t i, j = 0;
    for (i = 0; i < len; ++i) {
        uint8_t c = p[i];
        if (c == 10 || c == 13 || c == 32) continue;
        if (upper && c >= 'a' && c <= 'z') c = (uint8_t)(c - 32);
        p[j++] = c;
    }
    return j;
}

/* comp_map, src/util.c:228-237, rebuilt from the IUPAC pairs it encodes:
 * A<->T, C<->G, U->A, M<->K, R<->Y, V<->B, H<->D; W S N and everything else map to
 * themselves; case is preserved.  Bytes >= 128: identity (UB in the reference). */
uint8_t fxo_complement_byte(uint8_t b) {
    static const char from[] = "ATCGUMKRYVBHD";
    static const char to[]   = "TAGCAKMYRBVDH";
    uint8_t up = b, low = 0;
    const char *q;
    if (b >= 'a' && b <= 'z') { up = (uint8_t)(b - 32); low = 32; }
    if (up < 'A' || up > 'Z') return b;
    q = (const char *)memchr(from, up, sizeof(from) - 1);
    if (!q) return b;
    return (uint8_t)(to[q - from] + low);
}

/* reverse_seq / complement_seq / reverse_complement_seq, src/util.c:239-269. */
void fxo_transform(uint8_t *p, int64_t len, int flags) {
    int64_t i;
    if (flags & FXO_COMPLEMENT)
        for (i = 0; i < len; ++i) p[i] = fxo_complement_byte(p[i]);
    if (flags & FXO_REVERSE)
        for (i = 0; i < len / 2; ++i) { uint8_t t = p[i]; p[i] = p[len - 1 - i]; p[len - 1 - i] = t; }
}

/* Sequence slice -> bytes.  pyfastx_sequence_get_subseq (src/sequence.c:99-125) +
 * pyfastx_index_fill_cache (src/index.c:694-707) + the getters (sequence.c:337-398):
 *  - norm=1 slices read the covering byte range (fxo_slice_range), strip it and return the
 *    first e-s bytes;
 *  - norm=0 records (and whole records) strip the WHOLE record and index into it
 *    (sequence.c:100-102,108-110).
 * If fewer than e-s bytes survive stripping the reference copies stale buffer contents; the
 * oracle defines those bytes as 0.  Returns e-s. */
int64_t fxo_subseq(const uint8_t *buf, int64_t n, const fxo_fasta_row *row,
                   int64_t s, int64_t e, int flags, uint8_t *out) {
    int64_t want = e - s, off, bytes, got, skip = 0;
    uint8_t *tmp;
    if (want <= 0) return 0;
    if (row->norm && row->llen > row->elen && !(s == 0 && e == row->slen) && !(flags & FXO_WHOLE)) {
        fxo_slice_range(row, s, e, &off, &bytes);
    } else {
        off = row->boff; bytes = row->blen; skip = s;
    }
    if (off > n) off = n;
    if (off + bytes > n) bytes = n - off;
    if (bytes < 0) bytes = 0;
    tmp = (uint8_t *)malloc((size_t)bytes + 1);
    memcpy(tmp, buf + off, (size_t)bytes);
    got = fxo_strip(tmp, bytes, flags & FXO_UPPER);
    memset(out, 0, (size_t)want);
    if (got > skip) {
        int64_t c = got - skip < want ? got - skip : want;
        memcpy(out, tmp + skip, (size_t)c);
    }
    free(tmp);
    fxo_transform(out, want, flags);
    return want;
}

/* A/C/G/T counters as counted by gc_content (src/sequence.c:607-631): both cases. */
static void fxo_acgt(const uint8_t *p, int64_t len, int64_t acgt[4]) {
    int64_t i;
    acgt[0] = acgt[1] = acgt[2] = acgt[3] = 0;
    for (i = 0; i < len; ++i) {
        switch (p[i]) {
        case 'A': case 'a': ++acgt[0]; break;
        case 'C': case 'c': ++acgt[1]; break;
        case 'G': case 'g': ++acgt[2]; break;
        case 'T': case 't': ++acgt[3]; break;
        default: break;
        }
    }
}

/* Batched form of fxo_subseq (what K3 is checked against): packs results at out_off[q];
 * optional acgt[q*4..] counts of the returned bytes. */
int64_t fxo_subseq_batch(const uint8_t *buf, int64_t n, const fxo_fasta_row *rows,
                         const int64_t *row_id, const int64_t *s, const int64_t *e,
                         const int32_t *flags, int64_t nq,
                         const int64_t *out_off, uint8_t *out, int64_t *acgt) {
    int64_t q, total = 0;
    for (q = 0; q < nq; ++q) {
        int64_t len = fxo_subseq(buf, n, &rows[row_id[q]], s[q], e[q], flags[q], out + out_off[q]);
        if (acgt) fxo_acgt(out + out_off[q], len, acgt + 4 * q);
        total += len;
    }
    return total;
}

/* Fasta.fetch, src/fasta.c:384-515: the whole record is loaded and stripped (454-458),
 * 1-based inclusive intervals are concatenated (478-508) and the concatenation is
 * reverse-complemented for strand '-' (510-512).  Returns the output length. */
int64_t fxo_fetch(const uint8_t *buf, int64_t n, const fxo_fasta_row *row,
                  const int64_t *starts, const int64_t *ends, int nintervals,
                  int strand_minus, int upper, uint8_t *out) {
    int64_t bytes = row->blen, off = row->boff, got, j = 0;
    int i;
    uint8_t *tmp;
    if (off > n) off = n;
    if (off + bytes > n) bytes = n - off;
    tmp = (uint8_t *)malloc((size_t)bytes + 1);
    memcpy(tmp, buf + off, (size_t)bytes);
    got = fxo_strip(tmp, bytes, upper);
    for (i = 0; i < nintervals; ++i) {
        int64_t a = starts[i] - 1, len = ends[i] - starts[i] + 1, k;
        for (k = 0; k < len; ++k) out[j++] = (a + k >= 0 && a + k < got) ? tmp[a + k] : 0;
    }
    free(tmp);
    if (strand_minus) fxo_transform(out, j, FXO_REVERSE | FXO_COMPLEMENT);
    return j;
}

/* pyfastx_read_random_reader + seq/qual getters, src/read.c:37-45,152-167,237-249:
 * rlen raw bytes at soff and at qoff, no stripping. */
void fxo_read_fetch(const uint8_t *buf, int64_t n, const fxo_fastq_row *row,
                    uint8_t *seq_out, uint8_t *qual_out) {
    int64_t k;
    for (k = 0; k < row->rlen; ++k) {
        if (seq_out)  seq_out[k]  = (row->soff + k < n) ? buf[row->soff + k] : 0;
        if (qual_out) qual_out[k] = (row->qoff + k < n) ? buf[row->qoff + k] : 0;
    }
}

/* composition, src/sequence.c:727-747 (per-byte histogram). */
void fxo_composition(const uint8_t *p, int64_t len, int64_t counts[256]) {
    int64_t i;
    memset(counts, 0, 256 * sizeof(int64_t));
    for (i = 0; i < len; ++i) ++counts[p[i]];
}

/* (float)(g+c)/(a+c+g+t)*100, src/sequence.c:636 -- float32 divide and multiply. */
float fxo_gc_content(int64_t a, int64_t c, int64_t g, int64_t t) {
    return (float)(g + c) / (a + c + g + t) * 100;
}

/* (float)(g-c)/(g+c), src/sequence.c:692. */
float fxo_gc_skew(int64_t c, int64_t g) {
    return (float)(g - c) / (g + c);
}
