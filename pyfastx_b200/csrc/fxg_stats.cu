// fxg_stats.cu -- full-index statistics on the resident file (SURVEY.md section 8f-3), sm_90a.
//
//   FASTA  per-record 128-bin byte composition -> `comp` rows (reference pyfastx_fasta_calc_composition,
//          src/fasta.c:851-961: every byte of the record's lines except '\n' is counted, so a '\r' of a CRLF file
//          lands in bin 13; rows (seqid, letter, count) for count > 0, then 128 rows with seqid 0 = whole file).
//   FASTQ  A/C/G/T/N totals, min/max read length, min/max quality, phred guess -> `base` / `meta` rows
//          (pyfastx_fastq_calc_composition, src/fastq.c:663-795).
// Both re-read the file bytes once (HBM bound in principle; the 128-bin histogram is bound by shared-memory
// read-modify-write: conflict-free per-lane private counters, no atomics in the inner loop).
#include "fxg_common.cuh"
#include <stdlib.h>
#include <string.h>
#include <vector>

namespace fxg {

constexpr int CT_SUB = 8192;            // bytes per warp of the composition kernel
constexpr int CT_WARPS = 2;             // warps per CTA (16 KiB of private counters each)

// first record r in [0, n_rows) with boff + blen > x   (records' byte ranges are disjoint and ascending)
__device__ __forceinline__ int64_t first_record_after(const fxg_fasta_row *rows, int64_t n_rows, int64_t x) {
    int64_t lo = 0, hi = n_rows;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (rows[mid].boff + rows[mid].blen > x) hi = mid; else lo = mid + 1;
    }
    return lo;
}

__global__ void __launch_bounds__(CT_WARPS * 32) comp_hist_kernel(const uint8_t *__restrict__ file, int64_t n, int64_t capacity,
                                                                  const fxg_fasta_row *__restrict__ rows, int64_t n_rows,
                                                                  int64_t base_offset, int64_t row_lo, int64_t row_hi,
                                                                  unsigned long long *__restrict__ hist) {
    __shared__ uint32_t s_cnt[CT_WARPS][128][32];             // [bin][lane]: bank == lane, no conflicts, no atomics
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t (*cnt)[32] = s_cnt[warp];
    for (int b = 0; b < 128; ++b) cnt[b][lane] = 0;
    __syncwarp();
    const int64_t start = ((int64_t)blockIdx.x * CT_WARPS + warp) * CT_SUB;
    if (start >= n) return;
    const int64_t end = start + CT_SUB < n ? start + CT_SUB : n;
    for (int64_t r = first_record_after(rows, n_rows, start + base_offset); r < n_rows; ++r) {
        const int64_t rb = rows[r].boff - base_offset, re = rb + rows[r].blen;
        if (rb >= end) break;
        if (r < row_lo || r >= row_hi) continue;
        const int64_t a = rb > start ? rb : start, b = re < end ? re : end;
        if (b <= a) continue;
        for (int64_t o = (a & ~(int64_t)15) + lane * 16; o < b; o += 512) {
            const uint4 v = *reinterpret_cast<const uint4 *>(file + o);       // o + 16 <= capacity (padded buffer)
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
            const bool whole = o >= a && o + 16 <= b;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const uint32_t c = (w[i >> 2] >> (8 * (i & 3))) & 0xffu;
                if ((whole || (o + i >= a && o + i < b)) && c < 128u) cnt[c][lane] += 1;
            }
        }
        __syncwarp();
        // flush: lane l sums bins l, l+32, l+64, l+96 over the 32 private columns
        unsigned long long *h = hist + (size_t)(r - row_lo) * 128;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int bin = lane + 32 * k;
            uint32_t s = 0;
#pragma unroll 8
            for (int j = 0; j < 32; ++j) { const int col = (j + lane) & 31; s += cnt[bin][col]; cnt[bin][col] = 0; }
            if (s && bin != '\n') atomicAdd(h + bin, (unsigned long long)s);
        }
        __syncwarp();
    }
}

// per record: number of non-zero bins (one warp per record)
__global__ void comp_count_kernel(const unsigned long long *__restrict__ hist, int64_t nrec, int64_t *__restrict__ zeros,
                                  int64_t *__restrict__ cnt) {
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= nrec) return;
    int c = 0;
    for (int k = 0; k < 4; ++k) c += hist[(size_t)r * 128 + lane + 32 * k] != 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) { cnt[r] = c; zeros[r] = 0; }
}

// (seqid, letter, count) triplets in (record, letter) order + whole-file totals
__global__ void comp_emit_kernel(const unsigned long long *__restrict__ hist, int64_t nrec, const int64_t *__restrict__ off,
                                 int64_t first_seqid, fxg_comp_row *__restrict__ out, unsigned long long *__restrict__ total) {
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= nrec) return;
    int64_t o = off[r];
    for (int k = 0; k < 4; ++k) {
        const int bin = lane + 32 * k;
        const unsigned long long v = hist[(size_t)r * 128 + bin];
        const uint32_t m = __ballot_sync(0xffffffffu, v != 0);
        if (v) {
            fxg_comp_row t;
            t.seqid = first_seqid + r; t.abc = bin; t.num = (int64_t)v;
            out[o + __popc(m & ((1u << lane) - 1u))] = t;
            atomicAdd(total + bin, v);
        }
        o += __popc(m);
    }
}

// ---- FASTQ: one warp per read ---------------------------------------------------------------------------
struct FqStats {
    unsigned long long a, c, g, t, n;
    long long maxlen, minlen;
    int minqs, maxqs;
};

// The reference's walk over a quality line of L bytes (src/fastq.c:732-745) shortens the line by one at each '\r' it
// meets and skips it, so byte i is visited iff i + ('\r' before i) < L: a '\r' before the last byte ends the walk
// early.  Exact form for the lines fq_line cannot settle in one pass (L known): -> the walk's length; the visited
// bytes' range goes to mn / mx.
__device__ __forceinline__ int64_t fq_qual_exact(const uint8_t *__restrict__ file, int64_t n, int64_t s, int64_t L, int lane,
                                              int &mn, int &mx) {
    int64_t carry = 0;                                                  // '\r' of the line before this step
    int vis_cr = 0;
    for (int64_t o0 = s & ~(int64_t)15; o0 < s + L; o0 += 512) {
        const int64_t o = o0 + lane * 16;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (o < n) v = *reinterpret_cast<const uint4 *>(file + o);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        int c = 0;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const uint32_t ch = (w[i >> 2] >> (8 * (i & 3))) & 0xffu;
            c += (o + i >= s && o + i < s + L && ch == 13u);
        }
        int incl = c;                                                   // inclusive prefix over the lanes
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        int64_t before = carry + incl - c;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int64_t p = o + i - s;
            if (p >= 0 && p < L) {
                const uint32_t ch = (w[i >> 2] >> (8 * (i & 3))) & 0xffu;
                if (p + before < L) {
                    if (ch == 13u) ++vis_cr;
                    else {
                        const int sc = (int)(signed char)ch;
                        mn = sc < mn ? sc : mn;
                        mx = sc > mx ? sc : mx;
                    }
                }
                before += ch == 13u;
            }
        }
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    return L - __reduce_add_sync(0xffffffffu, vis_cr);
}

// bytes of the line starting at `s` (to the next '\n' or the end of the file), 16 per lane and step.  A sequence
// line counts every byte but '\r'; a quality line gives the reference's length and quality range (fq_qual_exact):
// settled in this pass when its only '\r' is the last byte or it has none, else by a second, exact pass.
template <bool QUAL>
__device__ __forceinline__ void fq_line(const uint8_t *__restrict__ file, int64_t n, int64_t s, int lane,
                                        uint32_t &cA, uint32_t &cC, uint32_t &cG, uint32_t &cT, uint32_t &cOther,
                                        int &mn, int &mx, int64_t &len_out) {
    int64_t len = 0;
    int cr = 0;                                                           // QUAL: this lane's '\r' of the line
    int lmn = 1 << 20, lmx = -(1 << 20);                                  // QUAL: range of the line's other bytes
    bool done = false;
    for (int64_t o0 = s & ~(int64_t)15; !done; o0 += 512) {
        const int64_t o = o0 + lane * 16;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (o < n) v = *reinterpret_cast<const uint4 *>(file + o);           // padded buffer: bytes >= n read as 0
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        const int first = o < s ? (s - o < 16 ? (int)(s - o) : 16) : 0;       // bytes before the line start (first chunk only)
        // position of the first '\n' (or the end of the file) in this lane's 16 bytes
        int stop = 16;
#pragma unroll
        for (int i = 15; i >= 0; --i) {
            const uint32_t ch = (w[i >> 2] >> (8 * (i & 3))) & 0xffu;
            if ((o + i >= n || ch == '\n') && i >= first) stop = i;          // first terminator at or after the line start
        }
        const uint32_t has = __ballot_sync(0xffffffffu, stop < 16);
        // lanes after the one holding the terminator contribute nothing
        const int term_lane = has ? __ffs(has) - 1 : 32;
        const int lim = lane < term_lane ? 16 : (lane == term_lane ? stop : 0);
        int got = 0;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            if (i >= first && i < lim) {
                const uint32_t ch = (w[i >> 2] >> (8 * (i & 3))) & 0xffu;
                ++got;
                if (!QUAL) {
                    if (ch == 'A') ++cA; else if (ch == 'C') ++cC; else if (ch == 'G') ++cG; else if (ch == 'T') ++cT;
                    else if (ch != 13u) ++cOther;
                } else if (ch != 13u) {
                    const int sc = (int)(signed char)ch;                       // the reference compares plain (signed) chars
                    lmn = sc < lmn ? sc : lmn;
                    lmx = sc > lmx ? sc : lmx;
                } else { --got; ++cr; }                                        // '\r' does not count towards the length
            }
        }
        len += __reduce_add_sync(0xffffffffu, got);
        done = has != 0 || o0 + 512 >= n;
    }
    if (QUAL) {
        const int crs = __reduce_add_sync(0xffffffffu, cr);
        const int64_t L = len + crs;                                         // bytes before the terminator
        // no '\r', or one as the last byte (a CRLF line): every byte but the '\r' is visited
        if (crs == 0 || (crs == 1 && file[s + L - 1] == 13u)) {
            mn = lmn < mn ? lmn : mn;
            mx = lmx > mx ? lmx : mx;
        } else {
            len = fq_qual_exact(file, n, s, L, lane, mn, mx);
        }
    }
    len_out = len;
}

__global__ void __launch_bounds__(256) fastq_stats_kernel(const uint8_t *__restrict__ file, int64_t n,
                                                          const fxg_fastq_row *__restrict__ rows, int64_t n_rows,
                                                          int64_t base_offset, int trailing_seq, FqStats *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    uint32_t cA = 0, cC = 0, cG = 0, cT = 0, cO = 0;
    unsigned long long A = 0, Cc = 0, G = 0, T = 0, N = 0;
    int mn = 104, mx = 33;
    long long maxlen = 0, minlen = 10000000000ll;
    const int64_t total = n_rows + (trailing_seq ? 1 : 0);
    for (int64_t r = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5); r < total; r += nwarps) {
        const fxg_fastq_row row = rows[r];
        int64_t len;
        int d0 = 0, d1 = 0;
        fq_line<false>(file, n, row.soff - base_offset, lane, cA, cC, cG, cT, cO, d0, d1, len);
        if (r < n_rows) {
            fq_line<true>(file, n, row.qoff - base_offset, lane, cA, cC, cG, cT, cO, mn, mx, len);
            maxlen = len > maxlen ? len : maxlen;
            minlen = len < minlen ? len : minlen;
        }
        A += cA; Cc += cC; G += cG; T += cT; N += cO;
        cA = cC = cG = cT = cO = 0;
    }
    for (int d = 16; d > 0; d >>= 1) {
        A += (unsigned long long)shfl_down_i64((int64_t)A, d); Cc += (unsigned long long)shfl_down_i64((int64_t)Cc, d);
        G += (unsigned long long)shfl_down_i64((int64_t)G, d); T += (unsigned long long)shfl_down_i64((int64_t)T, d);
        N += (unsigned long long)shfl_down_i64((int64_t)N, d);
        mn = min(mn, __shfl_down_sync(0xffffffffu, mn, d)); mx = max(mx, __shfl_down_sync(0xffffffffu, mx, d));
    }
    if (lane == 0) {
        if (A) atomicAdd(&out->a, A);
        if (Cc) atomicAdd(&out->c, Cc);
        if (G) atomicAdd(&out->g, G);
        if (T) atomicAdd(&out->t, T);
        if (N) atomicAdd(&out->n, N);
        atomicMax(&out->maxlen, maxlen);
        atomicMin(&out->minlen, minlen);
        atomicMin(&out->minqs, mn);
        atomicMax(&out->maxqs, mx);
    }
}

}  // namespace fxg

using namespace fxg;

extern "C" void fxg_free_host(void *p) { free(p); }

// Full-index composition of every record of the resident file: *out receives a malloc'ed array of n_out
// (seqid, letter, count) rows in (seqid, letter) order, seqid 1-based (free with fxg_free_host); total[128] the
// whole-file counts (the 128 seqid = 0 rows of the reference).
extern "C" int fxg_fasta_composition(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                                     int64_t base_offset, fxg_comp_row **out, int64_t *n_out, int64_t *total) {
    FXG_CHECK_ARG(ctx && f && out && n_out && total && n_rows >= 0 && (n_rows == 0 || d_rows), "bad arguments");
    FXG_LOCK(ctx);
    FXG_CUDA(cudaSetDevice(ctx->device));
    *out = nullptr; *n_out = 0;
    memset(total, 0, 128 * sizeof(int64_t));
    if (n_rows == 0) return FXG_OK;
    const int64_t BATCH = (int64_t)1 << 21;                   // records per pass: 2M x 1 KiB of counters
    std::vector<fxg_comp_row> acc;
    int rc;
    if ((rc = ctx->counters.reserve(4096))) return rc;
    unsigned long long *d_total = (unsigned long long *)((uint8_t *)ctx->counters.ptr + 2048);
    FXG_CUDA(cudaMemsetAsync(d_total, 0, 128 * 8, ctx->stream));
    for (int64_t lo = 0; lo < n_rows; lo += BATCH) {
        const int64_t hi = lo + BATCH < n_rows ? lo + BATCH : n_rows, nb = hi - lo;
        // misc: hist[nb][128] u64 | cnt[nb] | zeros[nb] | off[nb+1]
        const size_t hist_b = (size_t)nb * 1024;
        if ((rc = ctx->misc.reserve(hist_b + (size_t)nb * 8 * 3 + 64))) return rc;
        unsigned long long *d_hist = (unsigned long long *)ctx->misc.ptr;
        int64_t *d_cnt = (int64_t *)((uint8_t *)ctx->misc.ptr + hist_b), *d_zero = d_cnt + nb, *d_off = d_zero + nb;
        FXG_CUDA(cudaMemsetAsync(d_hist, 0, hist_b, ctx->stream));
        const int64_t nsub = (f->size + CT_SUB - 1) / CT_SUB;
        ctx->launches += 3;
        comp_hist_kernel<<<(unsigned)((nsub + CT_WARPS - 1) / CT_WARPS), CT_WARPS * 32, 0, ctx->stream>>>(
            f->d, f->size, f->capacity, d_rows, n_rows, base_offset, lo, hi, d_hist);
        comp_count_kernel<<<(unsigned)((nb * 32 + 255) / 256), 256, 0, ctx->stream>>>(d_hist, nb, d_zero, d_cnt);
        FXG_CUDA(cudaGetLastError());
        int64_t n_trip = 0;
        if ((rc = fxg_extract_plan_dev(ctx, d_zero, d_cnt, nb, d_off, &n_trip))) return rc;
        if (n_trip) {
            if ((rc = ctx->row_tmp.reserve((size_t)n_trip * sizeof(fxg_comp_row)))) return rc;
            comp_emit_kernel<<<(unsigned)((nb * 32 + 255) / 256), 256, 0, ctx->stream>>>(d_hist, nb, d_off, lo + 1,
                                                                                        (fxg_comp_row *)ctx->row_tmp.ptr, d_total);
            FXG_CUDA(cudaGetLastError());
            const size_t old = acc.size();
            acc.resize(old + (size_t)n_trip);
            FXG_CUDA(cudaMemcpyAsync(acc.data() + old, ctx->row_tmp.ptr, (size_t)n_trip * sizeof(fxg_comp_row), cudaMemcpyDeviceToHost, ctx->stream));
            FXG_CUDA(cudaStreamSynchronize(ctx->stream));
        }
    }
    FXG_CUDA(cudaMemcpyAsync(total, d_total, 128 * 8, cudaMemcpyDeviceToHost, ctx->stream));
    FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    fxg_comp_row *o = (fxg_comp_row *)malloc(acc.size() * sizeof(fxg_comp_row) + 1);
    if (!o) { fxg_set_error("out of memory (composition rows)"); return FXG_ENOMEM; }
    memcpy(o, acc.data(), acc.size() * sizeof(fxg_comp_row));
    *out = o; *n_out = (int64_t)acc.size();
    return FXG_OK;
}

// A/C/G/T/N totals, min / max read length and quality, phred guess (src/fastq.c:663-795).  n_rows complete reads;
// trailing_seq != 0: row n_rows exists in d_rows and carries the sequence line of a trailing partial record
// (the reference counts its bases too: it walks lines, not reads).
extern "C" int fxg_fastq_stats(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                               int64_t base_offset, int trailing_seq, fxg_fastq_meta *out) {
    FXG_CHECK_ARG(ctx && f && out && n_rows >= 0 && (n_rows == 0 || d_rows), "bad arguments");
    FXG_LOCK(ctx);
    FXG_CUDA(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ctx->counters.reserve(4096))) return rc;
    FqStats init;
    memset(&init, 0, sizeof(init));
    init.maxlen = 0; init.minlen = 10000000000ll; init.minqs = 104; init.maxqs = 33;      // src/fastq.c:667-677
    FqStats *d = (FqStats *)((uint8_t *)ctx->counters.ptr + 3200);
    FXG_CUDA(cudaMemcpyAsync(d, &init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    if (n_rows + (trailing_seq ? 1 : 0) > 0) {
        ctx->launches += 1;
        fastq_stats_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(f->d, f->size, d_rows, n_rows, base_offset, trailing_seq, d);
        FXG_CUDA(cudaGetLastError());
    }
    FqStats h;
    FXG_CUDA(cudaMemcpyAsync(&h, d, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    out->a = (int64_t)h.a; out->c = (int64_t)h.c; out->g = (int64_t)h.g; out->t = (int64_t)h.t; out->n = (int64_t)h.n;
    out->maxlen = h.maxlen; out->minlen = h.minlen; out->minqs = h.minqs; out->maxqs = h.maxqs;
    out->phred = 0;
    if (h.maxqs > 74) out->phred = 64;                          // src/fastq.c:758-764
    if (h.minqs < 59) out->phred = 33;
    return FXG_OK;
}
