/* fxo -- CPU ORACLE for the pyfastx hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C restatement of the reference algorithms on the hot path (lmdu/pyfastx
 * v2.3.1, files cited per function in fxo.c).  It is NOT the product and is never
 * linked, imported or executed by anything under pyfastx_b200/.  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it,
 * and only as the checker.
 *
 * Pinning: tests/test_oracle_pinned.py checks every function here against
 *   the committed fixtures in tests/golden/, generated from the compiled, unmodified
 *   reference (oracle/_ref, built by oracle/build_ref.sh) by tests/golden/make_golden*.py.
 */
#ifndef FXO_H
#define FXO_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* One `seq` table row (reference DDL: src/index.c:178-188) + where the name lives. */
typedef struct fxo_fasta_row {
    int64_t boff;   /* byte offset of the first sequence byte (index.c:258)            */
    int64_t blen;   /* bytes up to the next header / end position (index.c:243,348)     */
    int64_t slen;   /* sequence length (index.c:335-338)                                */
    int64_t llen;   /* first line length incl. newline (index.c:330-332)                */
    int32_t dlen;   /* header length without '>' and line ending (index.c:271)          */
    int32_t nlen;   /* chrom name length (index.c:282-301)                              */
    uint8_t elen;   /* 1 = \n, 2 = \r\n, decided on the header line (index.c:267-269)   */
    uint8_t norm;   /* <=1 line differing from the first one (index.c:237,342)          */
    uint8_t pad[6]; /* pad[0]: uniform lines, not in the reference (fxo_fasta_scan)     */
} fxo_fasta_row;    /* 48 bytes; name bytes start at boff - elen - dlen                 */

/* One `read` table row (reference DDL: src/fastq.c:29-37). */
typedef struct fxo_fastq_row {
    int64_t soff;   /* offset of the sequence line (fastq.c:122)                        */
    int64_t qoff;   /* offset of the quality line (fastq.c:133)                         */
    int64_t rlen;   /* read length without '\r' (fastq.c:124-128)                       */
    int32_t dlen;   /* length of the name line incl. '@' and '\r' (fastq.c:103)         */
    int32_t nlen;   /* read name length (fastq.c:104-117)                               */
} fxo_fastq_row;    /* 32 bytes; name bytes start at soff - dlen                         */

enum {
    FXO_UPPER      = 1,  /* Fasta(uppercase=True): remove_space_uppercase (util.c:181)  */
    FXO_REVERSE    = 2,  /* Sequence.reverse (sequence.c:353)                           */
    FXO_COMPLEMENT = 4,  /* Sequence.complement (sequence.c:369); both = antisense      */
    FXO_WHOLE      = 16  /* Fasta.fetch: index into the whole stripped record (fasta.c:454-508) */
};

/* index-build scans ------------------------------------------------------------------ */
int64_t fxo_fasta_scan(const uint8_t *buf, int64_t n, int full_name,
                       fxo_fasta_row *rows, int64_t cap,
                       int64_t *total_slen, int *no_header);
int64_t fxo_fastq_scan(const uint8_t *buf, int64_t n,
                       fxo_fastq_row *rows, int64_t cap,
                       int64_t *total_size, int64_t *n_lines);

/* extraction ------------------------------------------------------------------------- */
void    fxo_slice_range(const fxo_fasta_row *row, int64_t s, int64_t e,
                        int64_t *offset, int64_t *byte_len);
int64_t fxo_strip(uint8_t *p, int64_t len, int upper);
void    fxo_transform(uint8_t *p, int64_t len, int flags);
int64_t fxo_subseq(const uint8_t *buf, int64_t n, const fxo_fasta_row *row,
                   int64_t s, int64_t e, int flags, uint8_t *out);
int64_t fxo_subseq_batch(const uint8_t *buf, int64_t n, const fxo_fasta_row *rows,
                         const int64_t *row_id, const int64_t *s, const int64_t *e,
                         const int32_t *flags, int64_t nq,
                         const int64_t *out_off, uint8_t *out, int64_t *acgt);
int64_t fxo_fetch(const uint8_t *buf, int64_t n, const fxo_fasta_row *row,
                  const int64_t *starts, const int64_t *ends, int nintervals,
                  int strand_minus, int upper, uint8_t *out);
void    fxo_read_fetch(const uint8_t *buf, int64_t n, const fxo_fastq_row *row,
                       uint8_t *seq_out, uint8_t *qual_out);

/* composition / GC (float32 arithmetic as in the reference) -------------------------- */
void    fxo_composition(const uint8_t *p, int64_t len, int64_t counts[256]);
float   fxo_gc_content(int64_t a, int64_t c, int64_t g, int64_t t);
float   fxo_gc_skew(int64_t c, int64_t g);
uint8_t fxo_complement_byte(uint8_t b);

#ifdef __cplusplus
}
#endif
#endif
