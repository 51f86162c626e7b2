/* fxg.h -- C-ABI of the H100-native pyfastx hot path (libfxg.so).
 *
 * This is the drop-in boundary: plain C types, caller-owned buffers, int status codes,
 * no Python.h / torch types, callable with the GIL released.  The reference (lmdu/pyfastx
 * v2.3.1) has no FFI of its own -- its hot path is C functions inside a CPython
 * extension -- so each entry point cites the reference function(s) it replaces
 * (paths relative to the reference tree).  INTEGRATION.md shows the binding a maintainer
 * would add on the reference side.
 *
 * Conventions
 *   - every function returns FXG_OK (0) or a negative FXG_E* code; fxg_last_error()
 *     gives a thread-local message for the last failure;
 *   - "dev" pointers are CUDA device pointers on the context's device, "host" pointers
 *     are ordinary (pageable or pinned) host memory;
 *   - all work is enqueued on the context's stream (fxg_ctx_set_stream lets the caller
 *     pass its own cudaStream_t, e.g. torch's current stream); *_host entry points
 *     synchronise before returning, *_dev entry points do not unless stated;
 *   - there is NO CPU fallback anywhere: without a CUDA device every compute entry point
 *     fails with FXG_ENODEV.
 */
#ifndef FXG_H
#define FXG_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define FXG_ABI_VERSION 2

enum {
    FXG_OK       = 0,
    FXG_ENODEV   = -1,  /* no usable CUDA device                           */
    FXG_ECUDA    = -2,  /* CUDA runtime error (see fxg_last_error)         */
    FXG_EINVAL   = -3,  /* bad argument                                    */
    FXG_ENOMEM   = -4,  /* host or device allocation failed                */
    FXG_ECAP     = -5,  /* caller buffer too small (required size returned)*/
    FXG_EIO      = -6,  /* file I/O error                                  */
    FXG_EFORMAT  = -7   /* malformed compressed stream                     */
};

/* ---- row layouts (device and host, little endian) ------------------------------------- */

/* One `seq` table row of the .fxi (DDL: src/index.c:178-188).  48 bytes.
 * chrom name bytes live in the file at [boff - elen - dlen, +nlen). */
typedef struct fxg_fasta_row {
    int64_t boff;     /* offset of first sequence byte            index.c:258      */
    int64_t blen;     /* bytes to next header / end position      index.c:243,348  */
    int64_t slen;     /* sequence length                          index.c:335-338  */
    int64_t llen;     /* first line length incl. line ending      index.c:330-332  */
    int32_t dlen;     /* header length w/o '>' and line ending    index.c:271      */
    int32_t nlen;     /* chrom name length                        index.c:282-301  */
    uint8_t elen;     /* 1 = "\n", 2 = "\r\n" (from the header)   index.c:267-269  */
    uint8_t norm;     /* <= 1 line differing from the first       index.c:237,342  */
    uint8_t pad[6];   /* pad[0] bit 0 (device rows only, not part of the .fxi): every line of the
                       * record except possibly the last has the same length                       */
} fxg_fasta_row;

/* One `read` table row (DDL: src/fastq.c:29-37).  32 bytes.
 * read name bytes live in the file at [soff - dlen, +nlen). */
typedef struct fxg_fastq_row {
    int64_t soff;     /* offset of the sequence line              fastq.c:122      */
    int64_t qoff;     /* offset of the quality line               fastq.c:133      */
    int64_t rlen;     /* read length without '\r'                 fastq.c:124-128  */
    int32_t dlen;     /* name line length incl. '@' and '\r'      fastq.c:103      */
    int32_t nlen;     /* read name length                         fastq.c:104-117  */
} fxg_fastq_row;

/* Totals the scans report next to the rows (the `stat` rows, index.c:367-371,
 * fastq.c:159-171) plus what a multi-GPU shard merge needs (SURVEY.md section 8e). */
typedef struct fxg_scan_stats {
    int64_t n_rows;        /* FASTA: header lines seen; FASTQ: n_lines / 4                 */
    int64_t n_lines;       /* lines incl. an unterminated last line                         */
    int64_t total_len;     /* FASTA: sum(slen) -> stat.seqlen; FASTQ: sum(rlen) -> stat.size */
    int64_t end_position;  /* n, or n+1 when the last line has no '\n' (index.c:231)       */
    int64_t lead_lines;    /* FASTA shard merge: lines before the first header of this buffer */
    int64_t lead_bytes;    /* bytes before the first header (== buffer size if none)       */
    int64_t lead_llen;     /* first line length of that lead part, 0 if none               */
    int64_t reserved;
} fxg_scan_stats;

/* What one shard tells the others in the multi-GPU index build (SURVEY.md section 8e): the fixed struct of the
 * one small all-gather.  128 bytes.  Filled on the device by fxg_scan_begin.
 *   n_rows / n_lines     FASTA header lines / lines (incl. an unterminated last line) of this shard
 *   edge_*               the first (up to 3) lines of the shard: global offset of the line start and line length
 *                        without '\r' -- what the PREVIOUS shard needs to complete a FASTQ read whose four lines
 *                        straddle the boundary (soff/rlen from line 2, qoff from line 4: fastq.c:122-133) */
typedef struct fxg_shard_info {
    int64_t n_rows;
    int64_t n_lines;
    int64_t bytes;         /* shard size                                            */
    int64_t base_offset;   /* file offset of the shard's first byte                 */
    int64_t end_position;  /* bytes, +1 when the last line has no '\n'              */
    int64_t edge_n;        /* valid entries in edge_off / edge_len (<= 3)           */
    int64_t edge_off[3];
    int64_t edge_len[3];
    int64_t reserved[4];
} fxg_shard_info;

/* scan flags */
enum {
    FXG_SCAN_FULL_NAME = 1   /* Fasta(full_name=True): name = whole header (index.c:282-285) */
};

/* per-query extraction flags */
enum {
    FXG_X_UPPER      = 1,   /* Fasta(uppercase=True): remove_space_uppercase  util.c:181-194 */
    FXG_X_REVERSE    = 2,   /* Sequence.reverse                               util.c:251-260 */
    FXG_X_COMPLEMENT = 4,   /* Sequence.complement (both = antisense)         util.c:239-269 */
    FXG_X_RAW        = 8,   /* no whitespace stripping (FASTQ reads)          read.c:37-45   */
    FXG_X_WHOLE      = 16   /* Fasta.fetch semantics: index into the WHOLE stripped record (fasta.c:454-508)
                             * instead of the slice -> byte-range formula; rows whose lines are uniform
                             * (pad[0] bit 0, set by the scan) still take the formula, which is then exact */
};

typedef struct fxg_ctx  fxg_ctx;    /* one per (process, GPU).  NOT thread-safe: a context owns grow-only scratch
                                     * buffers and one stream; every entry point taking a ctx locks the context's
                                     * own mutex, so concurrent callers are serialised (never corrupted), and
                                     * device pointers returned from context scratch (scan rows) stay valid only
                                     * until the next scan on the same context.                                   */
typedef struct fxg_file fxg_file;   /* a FASTA/FASTQ byte stream resident in HBM */
typedef struct fxg_comm fxg_comm;   /* the ranks that share one index build: peer-memory mailboxes (+ the NCCL communicator used to set them up / as fallback) */

/* ---- library / context ----------------------------------------------------------------- */
int         fxg_abi_version(void);
const char *fxg_last_error(void);
int         fxg_device_count(void);
int         fxg_ctx_create(int device, fxg_ctx **out);
void        fxg_ctx_destroy(fxg_ctx *ctx);
int         fxg_ctx_set_stream(fxg_ctx *ctx, void *cuda_stream);
int         fxg_ctx_sync(fxg_ctx *ctx);
int         fxg_ctx_sm_count(fxg_ctx *ctx);

/* measurement hooks (bench.py): with profiling on, the dominant kernels are bracketed by
 * CUDA events on the context's stream; slot 0 = scan (mark) kernel, 1 = FASTA finalize,
 * 2 = extract/reads kernel, 3 = offset prefix-sum kernels, 4 = region-count prefix kernels,
 * 5 = scan lines kernel.  fxg_profile_last_ms waits for
 * the slot's end event.  fxg_ctx_launch_count = kernels launched by this context so far. */
enum { FXG_PROF_SCAN = 0, FXG_PROF_FINALIZE = 1, FXG_PROF_GATHER = 2, FXG_PROF_PLAN = 3, FXG_PROF_PREFIX = 4,
       FXG_PROF_LINES = 5, FXG_PROF_SLOTS = 6 };
int         fxg_profile_enable(fxg_ctx *ctx, int on);
int         fxg_profile_last_ms(fxg_ctx *ctx, int slot, float *ms);
int64_t     fxg_ctx_launch_count(fxg_ctx *ctx);

/* pinned host memory for staging (cudaHostAlloc / cudaFreeHost) */
int         fxg_host_alloc(int64_t nbytes, void **out);
void        fxg_host_free(void *p);

/* ---- file staging: raw bytes -> HBM ------------------------------------------------------
 * Replaces the reference's read side: gzread into a 1 MiB kstream buffer (src/kseq.c:70)
 * for the scan, fseeko+fread per request for random access (src/index.c:683-692,
 * src/read.c:37-45).  The whole file becomes one padded device buffer.
 * fxg_file_alloc (its padding), fxg_file_upload, fxg_file_from_host and fxg_file_slice return with their copies
 * complete, like fxg_file_from_path: the single-query calls (fxg_extract_one_host, fxg_read_one_host) may be served
 * from a stream of the library's own that does not wait for the context's stream. */
int      fxg_file_alloc(fxg_ctx *ctx, int64_t nbytes, fxg_file **out);
int      fxg_file_upload(fxg_ctx *ctx, fxg_file *f, int64_t dst_off, const void *host, int64_t nbytes);
int      fxg_file_from_host(fxg_ctx *ctx, const void *host, int64_t nbytes, fxg_file **out);
int      fxg_file_from_path(fxg_ctx *ctx, const char *path, fxg_file **out);
int      fxg_file_wrap(fxg_ctx *ctx, void *dev_ptr, int64_t nbytes, int64_t capacity, fxg_file **out);
int      fxg_file_download(fxg_ctx *ctx, const fxg_file *f, int64_t src_off, void *host, int64_t nbytes);
void    *fxg_file_devptr(const fxg_file *f);
int64_t  fxg_file_size(const fxg_file *f);
void     fxg_file_free(fxg_file *f);
/* fxg_file_free keeps ONE spare device buffer per device for the next fxg_file_alloc that fits (cudaMalloc / cudaFree of
 * a 10 GB buffer cost more than scanning it); fxg_pool_trim returns the spares to the driver.  FXG_FILE_POOL=0 disables the pool. */
void     fxg_pool_trim(void);

/* ---- K1: FASTA index scan -----------------------------------------------------------------
 * Replaces the scan loop of pyfastx_create_index (src/index.c:226-361) over
 * ks_getuntil2 (src/kseq.c:59-109).  One pass over the resident bytes; rows land in a
 * device array owned by the context (valid until the next scan on this context or
 * fxg_ctx_destroy) and can be copied out with fxg_rows_download.
 *   base_offset : file offset of byte 0 of `f` (added to every boff; 0 for a whole file)
 *   d_rows_out  : receives the device pointer to n_rows fxg_fasta_row
 * Synchronises (the row count is needed on the host). */
int fxg_fasta_scan(fxg_ctx *ctx, const fxg_file *f, int64_t base_offset, int flags,
                   fxg_fasta_row **d_rows_out, fxg_scan_stats *stats);

/* ---- K2: FASTQ index scan -----------------------------------------------------------------
 * Replaces the scan loop of pyfastx_fastq_create_index (src/fastq.c:84-171): strict 4-line records by
 * line number (fastq.c:93); n_rows = complete reads (fastq.c:132-146,159). */
int fxg_fastq_scan(fxg_ctx *ctx, const fxg_file *f, int64_t base_offset,
                   fxg_fastq_row **d_rows_out, fxg_scan_stats *stats);

/* ---- multi-GPU index build: split-phase scan + ONE small all-gather (SURVEY.md section 8e) ----
 * Every rank holds a contiguous byte range of the file that starts at a line start (FASTQ) or at a header
 * line (FASTA); see fxg_split_point_* below.  The scan is split where the only cross-shard dependency sits:
 *   fxg_scan_begin     mark + prefix over the shard (all of the file traffic); leaves the shard's
 *                      fxg_shard_info on the device.  No host synchronisation.
 *   fxg_shard_exchange every rank's fxg_shard_info to every rank, on the context's stream: ONE kernel that stores the
 *                      128-byte block into all ranks' HBM mailboxes over NVLink/NVSwitch (peer memory mapped with CUDA
 *                      IPC at fxg_comm_create) and waits for the peers' flags -- or an in-stream ncclAllGather where
 *                      peer access is unavailable (fxg_comm_uses_p2p).  comm == NULL: single rank, a device copy.
 *   fxg_scan_finish    global line phase (fastq.c:93: line_num % 4 counts from the start of the FILE) and ID
 *                      base from the gathered counts, rows kernel, and for FASTQ the boundary-row merge: a
 *                      read is owned by the shard holding its name line and completed from the next shards'
 *                      edge lines.  ONE host synchronisation at the end.  d_rows_out = this shard's rows
 *                      (FASTQ: owned complete reads only), stats = this shard's totals, all_host (may be NULL)
 *                      receives the nranks gathered structs.
 * fxg_fasta_scan / fxg_fastq_scan are begin + finish with one rank.  mode: 0 = FASTA, 1 = FASTQ. */
int fxg_scan_begin(fxg_ctx *ctx, const fxg_file *f, int mode, int64_t base_offset, int flags,
                   fxg_shard_info *d_info_out /* device, 128 B */);
int fxg_shard_exchange(fxg_ctx *ctx, fxg_comm *comm, const void *d_send, void *d_recv, int64_t bytes_per_rank);
int fxg_scan_finish(fxg_ctx *ctx, const fxg_shard_info *d_all /* device, nranks entries */, int nranks, int rank,
                    void **d_rows_out, fxg_scan_stats *stats, fxg_shard_info *all_host);
/* the three steps in one call (what a rank of the multi-GPU build runs) */
int fxg_scan_sharded(fxg_ctx *ctx, fxg_comm *comm, const fxg_file *f, int mode, int64_t base_offset, int flags,
                     void **d_rows_out, fxg_scan_stats *stats, fxg_shard_info *all_host);

/* communicator: rank 0 creates the id (ncclGetUniqueId), the host layer broadcasts its FXG_COMM_ID_BYTES
 * bytes by any means (torch.distributed, MPI, a file), every rank calls fxg_comm_create (ncclCommInitRank).
 * NCCL is loaded at run time (libnccl.so.2, the copy already in the process if there is one). */
#define FXG_COMM_ID_BYTES 128
int  fxg_comm_unique_id(void *id_out);
int  fxg_comm_create(fxg_ctx *ctx, const void *id, int nranks, int rank, fxg_comm **out);
int  fxg_comm_nranks(const fxg_comm *comm);
int  fxg_comm_rank(const fxg_comm *comm);
/* 1 if fxg_shard_exchange runs over the peer-memory mailboxes (P2P stores into every rank's HBM over NVLink / NVSwitch,
 * mapped with CUDA IPC at fxg_comm_create: one kernel, no collective library on the path), 0 if it falls back to
 * ncclAllGather (IPC or peer access unavailable, or FXG_COMM=nccl). */
int  fxg_comm_uses_p2p(const fxg_comm *comm);
/* after a stream synchronisation: FXG_ECUDA if a mailbox wait timed out (a peer never arrived), else FXG_OK */
int  fxg_comm_check(fxg_comm *comm);
void fxg_comm_destroy(fxg_comm *comm);

/* split points found ON THE DATA: first offset >= from at which a line starts (want_header = 0) or a FASTA
 * header line starts (want_header = 1: '>' at offset 0 or right after '\n', index.c:234); the buffer / file
 * size if there is none.  _dev searches a resident buffer (synchronises), _path reads the file with pread. */
int fxg_split_point_dev(fxg_ctx *ctx, const fxg_file *f, int64_t from, int want_header, int64_t *pos);
int fxg_split_point_path(const char *path, int64_t from, int want_header, int64_t *pos, int64_t *file_size);
/* stage the byte range [begin, end) of a file / of a resident buffer as a shard of its own */
int fxg_file_from_path_range(fxg_ctx *ctx, const char *path, int64_t begin, int64_t end, fxg_file **out);
int fxg_file_slice(fxg_ctx *ctx, const fxg_file *src, int64_t begin, int64_t end, fxg_file **out);

/* copy rows device -> host (row_bytes = 48 or 32) */
int fxg_rows_download(fxg_ctx *ctx, const void *d_rows, int64_t n_rows, int row_bytes, void *host_rows);
int fxg_rows_upload(fxg_ctx *ctx, const void *host_rows, int64_t n_rows, int row_bytes, void **d_rows_out);
void fxg_dev_free(void *d_ptr);

/* One-call, host-buffer form (end-to-end path: H2D staging + scan + D2H rows).
 * rows_cap < n_rows -> FXG_ECAP with stats->n_rows set. */
int fxg_fasta_build_index_host(fxg_ctx *ctx, const void *host_buf, int64_t nbytes, int flags,
                               fxg_fasta_row *rows, int64_t rows_cap, fxg_scan_stats *stats);
int fxg_fastq_build_index_host(fxg_ctx *ctx, const void *host_buf, int64_t nbytes,
                               fxg_fastq_row *rows, int64_t rows_cap, fxg_scan_stats *stats);

/* ---- K3/K4: batched subsequence extraction (+ fused A/C/G/T counts) ----------------------
 * Replaces, per query: the slice -> byte-range math of pyfastx_sequence_subscript
 * (src/sequence.c:498-510), pyfastx_index_random_read + pyfastx_index_fill_cache
 * (src/index.c:683-707), remove_space[_uppercase] (src/util.c:166-194), the strand
 * transforms (src/util.c:239-269 via src/sequence.c:337-398) and, when d_acgt != NULL,
 * the base counting loop of gc_content/gc_skew (src/sequence.c:607-631).
 * Query q = (row_id[q], s[q], e[q], flags[q]) with 0-based half-open [s, e) already
 * clamped to [0, slen] (PySlice_AdjustIndices, sequence.c:446).  Output q is written at
 * d_out + d_out_off[q], length e-s; d_out_off has nq+1 entries (exclusive prefix sum,
 * computed by fxg_extract_plan_dev).  norm=0 records are served by stripping the whole
 * record and indexing into it (sequence.c:100-102). */
int fxg_extract_plan_dev(fxg_ctx *ctx, const int64_t *d_s, const int64_t *d_e, int64_t nq,
                         int64_t *d_out_off, int64_t *total_bytes /* host, may be NULL */);
int fxg_extract_dev(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                    const int64_t *d_row_id, const int64_t *d_s, const int64_t *d_e,
                    const int32_t *d_flags, int64_t nq,
                    const int64_t *d_out_off, uint8_t *d_out, int64_t *d_acgt /* nq*4 or NULL */);
/* host-buffer form: H2D queries, plan, extract, D2H output.  out_off_host has nq+1 entries. */
int fxg_extract_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                     const int64_t *row_id, const int64_t *s, const int64_t *e, const int32_t *flags,
                     int64_t nq, int64_t *out_off_host, uint8_t *out_host, int64_t out_cap,
                     int64_t *acgt_host /* nq*4 or NULL */);

/* ONE query through one kernel launch and one stream synchronisation -- what a per-object getter of the reference
 * costs here (Sequence.seq / .reverse / .complement / .antisense, src/sequence.c:337-398): no plan kernels, no H2D
 * copies (the query travels as kernel arguments), output written straight to mapped pinned memory.  Same bytes as
 * fxg_extract_host with nq = 1. */
int fxg_extract_one_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                         int64_t row_id, int64_t s, int64_t e, int32_t flags, uint8_t *out_host, int64_t out_cap);

/* K4 (full form): per-query byte histogram of the extracted bytes -- the counting loop of
 * pyfastx_sequence_composition (src/sequence.c:727-747) and, summed over records, of the
 * full-index composition scan (src/fasta.c:901-927).  hist_host receives nq x 256 int64. */
int fxg_composition_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                         const int64_t *row_id, const int64_t *s, const int64_t *e, const int32_t *flags,
                         int64_t nq, int64_t *hist_host);

/* ---- K8: exact pattern search on the resident file ------------------------------------------
 * Replaces Sequence.search (src/sequence.c:519-560), which extracts the sequence and scans it with str_n_str
 * (src/util.c:769-783), and extends it to every occurrence in a batch of queries.  The haystack of query
 * q = (row_id[q], s[q], e[q], flags) is exactly the bytes fxg_extract_dev returns for it (FXG_X_UPPER applies); a hit
 * is a start i with hay[i, i+m) == pattern byte for byte (case-sensitive), wholly inside [s, e); overlapping hits all
 * count.  strands: FXG_SEARCH_PLUS matches the pattern, FXG_SEARCH_MINUS its reverse complement (the extraction
 * complement table, case preserved) in the forward haystack; a hit reports its forward start, relative to s[q].
 *   mode FXG_SEARCH_ALL    every hit, in (query, start, minus) order
 *   mode FXG_SEARCH_FIRST  the first hit of each (query, strand) only, in the same order
 * row_id == NULL: one query per row (nq == n_rows), s = 0, e = slen; s and e are then ignored.
 * 1 <= m <= FXG_SEARCH_MAX_PATTERN; flags other than FXG_X_UPPER are FXG_EINVAL.  The result is deterministic.
 * *out is malloc'ed (free with fxg_free_host).  Synchronises after sizing the work, after counting the hits (to size
 * the output; FXG_SEARCH_ALL only) and at the end. */
#define FXG_SEARCH_PIECE        4096   /* stripped bases per work item of a record with uniform lines */
#define FXG_SEARCH_MAX_PATTERN  1024
enum { FXG_SEARCH_PLUS = 1, FXG_SEARCH_MINUS = 2 };          /* strands mask */
enum { FXG_SEARCH_ALL = 0, FXG_SEARCH_FIRST = 1 };            /* mode */
/* 24 B; mismatches: the substitutions of a hit of the search with mismatches below, 0 for the exact search */
typedef struct fxg_search_hit { int64_t query, start; int32_t minus, mismatches; } fxg_search_hit;
int fxg_search_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                    const int64_t *row_id, const int64_t *s, const int64_t *e, int32_t flags, int64_t nq,
                    const uint8_t *pattern, int32_t m, int strands, int mode,
                    fxg_search_hit **out, int64_t *n_out);
/* K8 on FASTQ reads: every occurrence of the pattern in every read of d_rows (the complete reads of a scan or of a
 * loaded .fxi).  The haystack of read i is exactly Read.seq (src/read.c:152-167): the rlen raw bytes at soff, nothing
 * stripped or upper-cased ('\r' is already outside rlen), so a space inside a sequence line is part of the read and a
 * match never runs into the line end, the '+' line, the quality line or the next read.  A hit is a start k with
 * hay[k, k+m) == pattern byte for byte (case-sensitive); overlapping hits all count; strands as for fxg_search_host.
 * query = the read's 0-based row index, start = the forward 0-based start.  Every hit, in (query, start, minus) order;
 * the result is deterministic.  A row whose [soff, soff + rlen) is not inside the buffer has no hits.  Reads longer
 * than FXG_SEARCH_PIECE bases are searched in pieces of FXG_SEARCH_PIECE start positions, shorter ones 32 at a time.
 * 1 <= m <= FXG_SEARCH_MAX_PATTERN; n_rows == 0 gives no hits.  *out is malloc'ed (free with fxg_free_host).
 * Synchronises after sizing the work, after counting the hits and at the end. */
int fxg_search_reads_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                          const uint8_t *pattern, int32_t m, int strands, fxg_search_hit **out, int64_t *n_out);

/* Search with mismatches: every start within max_mismatches substitutions of the pattern.  The haystacks are exactly
 * those of the exact entry points above: for fxg_search_approx_host the bytes extraction returns for the query (10 / 13 /
 * 32 stripped, FXG_X_UPPER applied if set), for fxg_search_reads_approx_host the raw rlen bytes at soff (Read.seq).
 * A hit is a start i with i + m <= len and at most max_mismatches positions j where hay[i + j] != pattern[j]
 * (Hamming distance, substitutions only; byte for byte and case-sensitive, so 'N' against 'A' is a mismatch).  The
 * minus strand compares against the pattern's reverse complement under the extraction table.  A window never extends
 * past its haystack's end: no partial window at a record's or read's end is reported, even if counting the missing
 * bytes as mismatches would keep it within the limit.  Every qualifying start is reported, overlapping ones included,
 * in (query, start, minus) order, deterministically; hit.mismatches is its count (0 .. max_mismatches) against the
 * strand it matched.  The exact entry points write 0 there.  max_mismatches = 0 gives exactly the exact search's hits.
 * 1 <= m <= FXG_SEARCH_MAX_PATTERN and 0 <= max_mismatches < m, else FXG_EINVAL.  There is no first-hit mode.
 * Arguments, row_id == NULL, output and synchronisation are as for fxg_search_host / fxg_search_reads_host. */
int fxg_search_approx_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                           const int64_t *row_id, const int64_t *s, const int64_t *e, int32_t flags, int64_t nq,
                           const uint8_t *pattern, int32_t m, int32_t max_mismatches, int strands,
                           fxg_search_hit **out, int64_t *n_out);
int fxg_search_reads_approx_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                                 const uint8_t *pattern, int32_t m, int32_t max_mismatches, int strands,
                                 fxg_search_hit **out, int64_t *n_out);

/* ---- K5: batched FASTQ read fetch ----------------------------------------------------------
 * Replaces pyfastx_read_random_reader + the seq/qual getters (src/read.c:37-45,152-167,
 * 237-249): for read ids[q] copies rlen raw bytes at soff (seq) and at qoff (qual).
 * Both outputs share out_off (prefix sum of rlen, nq+1 entries, filled by the call). */
int fxg_reads_dev(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                  const int64_t *d_ids, int64_t nq, int32_t flags,
                  int64_t *d_out_off, uint8_t *d_seq_out, uint8_t *d_qual_out, int64_t out_cap,
                  int64_t *total_bytes);
int fxg_reads_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                   const int64_t *ids, int64_t nq, int32_t flags,
                   int64_t *out_off_host, uint8_t *seq_host, uint8_t *qual_host, int64_t out_cap);

/* one read, one kernel launch, one synchronisation: the Read.seq / .qual getters (which: 0 = sequence, 1 = quality) */
int fxg_read_one_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows, int64_t read_id,
                      int which, int32_t flags, int64_t rlen, uint8_t *out_host, int64_t out_cap);

/* ---- K6: BGZF (block-gzip) inputs: member table on the host, member-parallel inflate on the GPU ----
 * Replaces zlib's gzread during the scan (src/kseq.c:70), the second full inflate pass that builds
 * the zran checkpoints (zran_build_index, src/index.c:381-387) and zran_seek + zran_read per random
 * access (src/index.c:685-686, src/read.c:39-40): the whole file is inflated once into HBM (one
 * thread per <= 64 KiB member) and every later access works on the uncompressed bytes.
 * fxg_bgzf_members_host walks the member headers only ('BC' extra field, ISIZE trailer); cmp_off
 * and ucmp_off receive n_members + 1 entries (pass NULL / cap 0 to just count).  FXG_EFORMAT if the
 * stream is plain gzip rather than BGZF (the caller then inflates on the host while staging).
 * d_status receives 0 per good member. */
int fxg_bgzf_members_host(const void *host_buf, int64_t nbytes, int64_t *cmp_off, int64_t *ucmp_off,
                          int64_t cap, int64_t *n_members, int64_t *total_uncompressed);
int fxg_inflate_members_dev(fxg_ctx *ctx, const fxg_file *compressed, const int64_t *d_cmp_off,
                            const int64_t *d_ucmp_off, int64_t n_members, uint8_t *d_out, int64_t out_cap,
                            int32_t *d_status);
int fxg_file_from_bgzf_host(fxg_ctx *ctx, const void *host_buf, int64_t nbytes, fxg_file **out,
                            int64_t *n_members_out);

/* ---- `.fxi` bulk writer (SURVEY.md section 8f-1; host side, no GPU needed) ------------------------------
 * Replaces the per-row INSERT loops and the CREATE UNIQUE INDEX of the reference index build
 * (src/index.c:223-251,363-372; src/fastq.c:81-156): rows (from the scan) and names (one packed buffer,
 * name i = names[name_off[i], name_off[i+1])) are written straight into a SQLite-format file with the
 * reference's schema (src/index.c:178-207, src/fastq.c:29-60) -- table b-trees and the UNIQUE name index
 * are built bottom-up, in parallel, without going through an SQL engine.  Duplicate names: no UNIQUE index
 * is created (the reference ignores that error too, src/index.c:366).  An existing file is replaced.
 *   gz     gzindex rows for a gzip input, in the row-per-field layout of pyfastx_gzip_index_export
 *          (src/util.c:442-540); NULL for plain files
 *   comp   full-index composition rows (src/fasta.c:851-961), NULL / 0 if not computed
 *   meta   FASTQ base / meta rows (src/fastq.c:663-795), NULL if not computed */
typedef struct fxg_gzindex {
    int64_t  compressed_size, uncompressed_size;
    uint32_t spacing, window_size;       /* import requires window_size >= 32768, spacing >= window_size */
    int64_t  npoints;
    const int64_t *cmp_offset;           /* per point: offset of the deflate data in the compressed file  */
    const int64_t *uncmp_offset;         /* per point: offset in the uncompressed stream                  */
    const uint8_t *bits;                 /* per point: bit offset (0..7) of the block start; NULL = all 0 */
    const uint8_t *has_data;             /* per point: 1 = a window follows in `windows`; NULL = none     */
    const uint8_t *windows;              /* window_size bytes per point with has_data, in point order     */
} fxg_gzindex;
typedef struct fxg_comp_row { int64_t seqid, abc, num; } fxg_comp_row;      /* seqid 0 = whole file        */
typedef struct fxg_fastq_meta { int64_t a, c, g, t, n, maxlen, minlen, minqs, maxqs, phred; } fxg_fastq_meta;
int fxg_fxi_write_fasta(const char *path, const fxg_fasta_row *rows, int64_t n_rows, const uint8_t *names,
                        const int64_t *name_off, int64_t total_slen, const fxg_gzindex *gz,
                        const fxg_comp_row *comp, int64_t n_comp);
int fxg_fxi_write_fastq(const char *path, const fxg_fastq_row *rows, int64_t n_rows, const uint8_t *names,
                        const int64_t *name_off, int64_t n_lines, int64_t total_size, const fxg_gzindex *gz,
                        const fxg_fastq_meta *meta);

/* ---- generic (non-BGZF) gzip: one sequential zlib pass on the host that inflates the stream AND collects the zran
 * checkpoints the `.fxi` must carry (replaces gzread during the scan, src/kseq.c:70, and the second inflate pass of
 * zran_build_index, src/index.c:381-387).  One access point per >= `spacing` bytes of output at a deflate block
 * boundary, with the 32 KiB of output in front of it (the published zran.c method); a reader resumes at any point
 * with inflatePrime + inflateSetDictionary.  The inflated bytes are then staged into HBM like a plain file. */
typedef struct fxg_gzip_result fxg_gzip_result;
int            fxg_gzip_inflate_host(const void *comp, int64_t nbytes, uint32_t spacing /* 0 = 1 MiB */, fxg_gzip_result **out);
const uint8_t *fxg_gzip_data(const fxg_gzip_result *r, int64_t *size);
int            fxg_gzip_index(const fxg_gzip_result *r, fxg_gzindex *gz);   /* pointers into r, valid until freed */
void           fxg_gzip_free(fxg_gzip_result *r);
/* Generic gzip with KNOWN checkpoints (the gzindex rows of an existing `.fxi`, or fxg_gzip_index): the compressed bytes go
 * to the device and every checkpoint's segment -- from its (compressed offset, bit offset) with its 32 KiB window to the
 * next checkpoint -- is inflated by its own GPU thread; replaces zran_seek + zran_read of the whole stream
 * (src/index.c:685-686) and the sequential host pass on every later open.  Verified before it is returned: segment
 * statuses, total length and the CRC-32 of the result (per-segment CRCs combined) against the gzip trailer;
 * FXG_EFORMAT otherwise (concatenated members, stale checkpoints): the caller then takes fxg_gzip_inflate_host. */
int            fxg_file_from_gzip_points_host(fxg_ctx *ctx, const void *host_buf, int64_t nbytes, const fxg_gzindex *gz,
                                              fxg_file **out);

/* ---- full-index statistics on the resident file (SURVEY.md section 8f-3) ---------------------------------
 * fxg_fasta_composition  per-record 128-bin byte composition, the counting loop of pyfastx_fasta_calc_composition
 *     (src/fasta.c:851-961): every byte of a record's lines except '\n' (a '\r' lands in bin 13; bytes >= 128,
 *     which index the reference's 128-entry array out of bounds, are dropped).  *out = malloc'ed array of
 *     (seqid, letter, count) rows, count > 0, in (seqid, letter) order, seqid = row index + 1 (free it with
 *     fxg_free_host); total[128] = whole-file counts (the reference's 128 rows with seqid 0).
 * fxg_fastq_stats  A/C/G/T/N totals, min / max read length, min / max quality, phred guess of
 *     pyfastx_fastq_calc_composition (src/fastq.c:663-795).  trailing_seq != 0: d_rows[n_rows] exists and carries
 *     the sequence line of a trailing partial record, whose bases the reference counts as well. */
int  fxg_fasta_composition(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                           int64_t base_offset, fxg_comp_row **out, int64_t *n_out, int64_t *total /* 128 */);
int  fxg_fastq_stats(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                     int64_t base_offset, int trailing_seq, fxg_fastq_meta *out);
void fxg_free_host(void *p);

/* ---- batched name -> row resolution (SURVEY.md section 8f-2; host side) --------------------------------
 * Replaces one sqlite probe per query (pyfastx_index_get_seq_by_name, src/index.c:527-566;
 * pyfastx_fastq_get_read_by_name, src/fastq.c:487-519) by a hash table over the packed names
 * (name i = names[name_off[i], name_off[i+1]); the table BORROWS both arrays: keep them alive).
 * Lookup of a batch runs on several threads; ids_out[i] = 0-based row, -1 if the name does not exist.
 * Duplicate names resolve to the first row. */
typedef struct fxg_nametab fxg_nametab;
int     fxg_nametab_build(const uint8_t *names, const int64_t *name_off, int64_t n, fxg_nametab **out);
int64_t fxg_nametab_find(const fxg_nametab *t, const uint8_t *name, int64_t len);
int     fxg_nametab_lookup(const fxg_nametab *t, const uint8_t *q, const int64_t *q_off, int64_t nq, int64_t *ids_out);
void    fxg_nametab_free(fxg_nametab *t);

/* BGZF writer (bench / test tooling only: the image has no bgzip): 0xff00-byte blocks, raw deflate at `level`, all host
 * threads; *out is malloc'ed (fxg_free_host). */
int fxg_bgzf_compress_host(const void *data, int64_t nbytes, int level, uint8_t **out, int64_t *out_len);

/* ---- synthetic inputs generated directly in HBM (bench / test tooling) -------------------
 * Byte-identical to pyfastx_b200/synth.py.  rec_off has n_records+1 entries (device). */
int fxg_synth_fasta_dev(fxg_ctx *ctx, uint64_t seed, const int64_t *d_lengths, const int64_t *d_rec_off,
                        int64_t n_records, int64_t first_record, int width, uint8_t *d_out);
int fxg_synth_fastq_dev(fxg_ctx *ctx, uint64_t seed, int64_t n_reads, int64_t first_read, int read_len,
                        const int64_t *d_rec_off, uint8_t *d_out);

#ifdef __cplusplus
}
#endif
#endif /* FXG_H */
