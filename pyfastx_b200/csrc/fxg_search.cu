// fxg_search.cu -- K8 exact pattern search on the resident file (sm_90a).
//
// Replaces Sequence.search (src/sequence.c:519-560: extract the sequence, then str_n_str, src/util.c:769-783) and
// extends it to every occurrence in a batch of queries.  The haystack of a query is exactly what extraction returns
// for it: the bytes are found the way serve_query_warp's strip path finds them (fxg_extract.cu), in ONE fused pass
// over the resident file bytes -- a warp streams the covering source range, drops 10 / 13 / 32, upper-cases if asked,
// and stages the kept bytes in its own shared-memory window, where every start position is tested against the
// pattern and its reverse complement.  There is no stripped copy in HBM.
//
// Work items: a query on a record with uniform lines (norm = 1 and the scan's uniform bit) is cut into pieces of
// FXG_SEARCH_PIECE start positions, each staged with the m - 1 bases that follow it (clipped to e) through the slice
// formula (sequence.c:498-510), as extract_one_kernel serves the pieces of such a query.  Any other query is one item: one warp
// streams the record from its first byte with a skip, like gather_one, matching window by window.
//
// Ordered output without atomics or a sort:
//   1. items   per query, the number of items; exclusive prefix -> item offsets (host learns the item total)
//   2. count   per item, the hits of each strand
//   3. ALL:    exclusive prefix of the per-item hits (host learns the output size), then emit: only the items with
//              hits run again, each writing its hits at its offset in (start, minus) order
//      FIRST:  one warp per (query, strand) finds the first item with a hit and runs that item until its first hit
#include "fxg_common.cuh"
#include <stdlib.h>
#include <string.h>
#include <vector>

namespace fxg {

constexpr int SW = 8;                                       // warps per CTA
constexpr int SPIECE = FXG_SEARCH_PIECE;
constexpr int SMAXPAT = FXG_SEARCH_MAX_PATTERN;
// per-warp haystack window: one piece, the m - 1 bases after it, one 512-byte gather round beyond that, and slack for
// the word loads of the last positions
constexpr int SHB = (SPIECE + SMAXPAT - 1 + 512 + 32 + 15) & ~15;
constexpr int SPB = SMAXPAT + 16;                           // pattern buffers (zero padded for word compares)
static_assert(SPIECE % 128 == 0 && SPIECE >= SMAXPAT + 512, "a window shift must not overlap itself");

enum { S_COUNT = 0, S_ALL = 1, S_FIRST = 2 };

struct SearchArgs {
    const uint8_t *file;
    int64_t fsize;
    const fxg_fasta_row *rows;
    int64_t n_rows;
    const int64_t *q_row, *q_s, *q_e;       // q_row == nullptr: query q = (row q, 0, slen)
    int64_t nq;
    int flags, m, strands;
    const uint8_t *pattern;
    const int64_t *item_off;                // nq + 1
    int64_t *tot, *pc;                      // per item: hits on both strands, hits on the plus strand
    const int64_t *hit_off;                 // per item: first output slot (S_ALL)
    fxg_search_hit *out;
};

__device__ __forceinline__ void load_query(const SearchArgs &A, int64_t q, int64_t &s, int64_t &e, fxg_fasta_row &r,
                                           bool &row_ok) {
    const int64_t rid = A.q_row ? A.q_row[q] : q;
    row_ok = rid >= 0 && rid < A.n_rows;
    memset(&r, 0, sizeof(r));
    if (row_ok) r = A.rows[rid];
    s = A.q_row ? A.q_s[q] : 0;
    e = A.q_row ? A.q_e[q] : r.slen;
}
// a query that extract_one_kernel cuts into pieces
__device__ __forceinline__ bool split_row(const fxg_fasta_row &r, bool row_ok) { return row_ok && r.norm && (r.pad[0] & 1); }

// haystack bytes i .. i+3 as one little-endian word (the window is 16-byte aligned)
__device__ __forceinline__ uint32_t word_at(const uint8_t *h, int i) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(h) + (i >> 2);
    return __funnelshift_r(w[0], w[1], 8 * (i & 3));
}
// hay[i + 4, i + m) == P[4, m): the first four bytes were compared by the caller
__device__ __forceinline__ bool rest_equal(const uint8_t *h, int i, const uint8_t *P, int m) {
    const uint32_t *pw = reinterpret_cast<const uint32_t *>(P);
    for (int j = 4; j < m; j += 4) {
        uint32_t d = word_at(h, i + j) ^ pw[j >> 2];
        if (m - j < 4) d &= (1u << (8 * (m - j))) - 1u;
        if (d) return false;
    }
    return true;
}
// bytes of x that are not zero
__device__ __forceinline__ int nonzero_bytes(uint32_t x) { return __popc((((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x) & 0x80808080u); }

// The per-start test, on a start's first (up to) four bytes w against the pattern's p, both masked to m bytes: first(w,
// p); for a start that passed and m > 4, on the whole window: rest(h, i, P, m).  mismatches(h, i, P, m) is what a hit
// reports.  ExactTest is K8's byte-for-byte test.
struct ExactTest {
    __device__ __forceinline__ bool first(uint32_t w, uint32_t p) const { return w == p; }
    __device__ __forceinline__ bool rest(const uint8_t *h, int i, const uint8_t *P, int m) const { return rest_equal(h, i, P, m); }
    __device__ __forceinline__ int mismatches(const uint8_t *, int, const uint8_t *, int) const { return 0; }
};
// At most k substituted bytes (Hamming distance): XOR word by word, count the bytes that differ, stop at the first word
// that takes the count past k.  On uniform random bases 3 of 4 bytes differ, so a start costs about (k + 1) / 3 words.
struct ApproxTest {
    int k;
    __device__ __forceinline__ int mismatches(const uint8_t *h, int i, const uint8_t *P, int m) const {
        const uint32_t *pw = reinterpret_cast<const uint32_t *>(P);
        int n = 0;
        for (int j = 0; j < m && n <= k; j += 4) {
            uint32_t d = word_at(h, i + j) ^ pw[j >> 2];
            if (m - j < 4) d &= (1u << (8 * (m - j))) - 1u;
            n += nonzero_bytes(d);
        }
        return n;
    }
    __device__ __forceinline__ bool first(uint32_t w, uint32_t p) const { return nonzero_bytes(w ^ p) <= k; }
    __device__ __forceinline__ bool rest(const uint8_t *h, int i, const uint8_t *P, int m) const { return mismatches(h, i, P, m) <= k; }
};

// Runs work item p of query q on the strands in `strands` (bit 0 plus, bit 1 minus).  S_COUNT adds the lane's hits to
// cp / cm; S_ALL writes every hit from A.out[out_pos] on; S_FIRST writes the first hit to A.out[out_pos] and returns.
// T: the per-start test (ExactTest, ApproxTest).
template <int MODE, class T>
__device__ void run_item(const SearchArgs &A, const T &test, int64_t q, int64_t p, int strands, uint8_t *__restrict__ hb,
                         const uint8_t *__restrict__ pat, const uint8_t *__restrict__ rc, int lane, int64_t out_pos,
                         int64_t &cp, int64_t &cm) {
    int64_t s, e;
    fxg_fasta_row r;
    bool row_ok;
    load_query(A, q, s, e, r, row_ok);
    const int m = A.m;
    const int64_t len = e - s;
    int64_t a = 0, b = len, c = len;                            // starts [a, b), haystack bytes [a, c) of the query
    if (split_row(r, row_ok)) {
        a = p * SPIECE;
        b = a + SPIECE < len ? a + SPIECE : len;
        c = b + m - 1 < len ? b + m - 1 : len;
    }
    const int64_t ss = s + a, ee = s + c, out_len = c - a;
    const int64_t ntest = (b - a) < (out_len - m + 1) ? (b - a) : (out_len - m + 1);
    // the source range of [ss, ee), as serve_query_warp's strip path takes it; rows pointing outside the buffer
    // give zero bytes, as they do there
    int64_t src = 0, src_len = 0, skip = 0;
    if (row_ok && r.boff >= 0 && r.blen >= 0 && r.boff <= A.fsize && ss >= 0) {
        const int64_t bpl = r.llen - (int64_t)r.elen;
        if (r.norm && bpl > 0 && !(ss == 0 && ee == r.slen)) {
            const int64_t bs = ss / bpl, be = ee / bpl;                          // sequence.c:500-503
            src = r.boff + ss + (int64_t)r.elen * bs;                            // sequence.c:508
            src_len = (ee - ss) + (be - bs) * (int64_t)r.elen;                   // sequence.c:509
        } else {
            src = r.boff; src_len = r.blen; skip = ss;                           // sequence.c:100-102,108-110
        }
    }
    int64_t src_end = src + src_len;
    if (src_end > A.fsize) src_end = A.fsize;
    const int64_t want_end = skip + out_len;
    const bool upper = (A.flags & FXG_X_UPPER) != 0;
    const bool want_p = (strands & 1) != 0, want_m = (strands & 2) != 0;
    const uint32_t pmask = m >= 4 ? 0xffffffffu : (1u << (8 * m)) - 1u;
    const uint32_t pp = *reinterpret_cast<const uint32_t *>(pat) & pmask, pm = *reinterpret_cast<const uint32_t *>(rc) & pmask;
    const uint32_t *hw = reinterpret_cast<const uint32_t *>(hb);
    int64_t done = 0;                                           // kept bytes seen
    int64_t wb = 0;                                             // haystack index (from a) of hb[0]
    int have = 0;                                               // haystack bytes in hb
    int64_t cursor = out_pos;                                   // S_ALL: next output slot
    for (int64_t cbase = src & ~(int64_t)15;; cbase += 512) {
        const bool more = cbase < src_end && done < want_end;
        if (more) {
            const int64_t my = cbase + lane * 16;
            uint4 v = make_uint4(0, 0, 0, 0);
            int lo = 0, hi = 0;
            if (my < src_end && my + 16 > src) {
                v = *reinterpret_cast<const uint4 *>(A.file + my);
                lo = (int)(src > my ? src - my : 0);
                hi = (int)(src_end - my < 16 ? src_end - my : 16);
            }
            const uint32_t wd[4] = {v.x, v.y, v.z, v.w};
            uint32_t keep = 0;                                  // bit j: byte j is kept
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                const uint32_t k = ~(byte_eq_mask(wd[w], 0x0a0a0a0au) | byte_eq_mask(wd[w], 0x0d0d0d0du) |
                                     byte_eq_mask(wd[w], 0x20202020u)) & 0x80808080u;
                keep |= (((k >> 7) & 1u) | ((k >> 14) & 2u) | ((k >> 21) & 4u) | ((k >> 28) & 8u)) << (4 * w);
            }
            keep &= ((1u << hi) - 1u) & ~((1u << lo) - 1u);
            const int cnt = __popc(keep);
            int incl = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += o;
            }
            const int total = __shfl_sync(0xffffffffu, incl, 31);
            int64_t rank = done + (incl - cnt);
            const int64_t r0 = skip + wb;                       // kept rank of hb[0]
            if (keep == 0xffffu && rank >= r0 && rank + 16 <= want_end) {
                // the common case inside a line: all 16 bytes are kept and wanted, no per-byte search of the mask
                uint8_t *d = hb + (rank - r0);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    uint32_t by = (wd[j >> 2] >> (8 * (j & 3))) & 0xffu;
                    if (upper && by - 'a' < 26u) by -= 32;
                    d[j] = (uint8_t)by;
                }
                keep = 0;
            }
            while (keep) {
                const int j = __ffs(keep) - 1;
                keep &= keep - 1;
                if (rank >= r0 && rank < want_end) {
                    const uint32_t wj = j < 8 ? (j < 4 ? v.x : v.y) : (j < 12 ? v.z : v.w);   // no local-memory array
                    uint32_t by = (wj >> (8 * (j & 3))) & 0xffu;
                    if (upper && by >= 'a' && by <= 'z') by -= 32;
                    hb[rank - r0] = (uint8_t)by;
                }
                ++rank;
            }
            done += total;
            __syncwarp();
            int64_t got = done - skip;
            got = got < 0 ? 0 : (got > out_len ? out_len : got);
            have = (int)(got - wb);
        }
        while (wb < ntest) {
            const int64_t wend = wb + SPIECE < ntest ? wb + SPIECE : ntest;
            const int need = (int)((wend + m - 1 < out_len ? wend + m - 1 : out_len) - wb);
            if (have < need) {
                if (more) break;
                // fewer kept bytes than the query asks for (malformed record): extraction defines them as 0
                for (int i = have + lane; i < need; i += 32) hb[i] = 0;
                __syncwarp();
                have = need;
            }
            const int nt = (int)(wend - wb);
            const int64_t start0 = a + wb;
            for (int r0 = 0; r0 < nt; r0 += 128) {
                const int i0 = r0 + 4 * lane;
                const uint32_t W0 = hw[i0 >> 2], W1 = hw[(i0 >> 2) + 1];
                uint32_t hp = 0, hm = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int i = i0 + k;
                    if (i < nt) {
                        const uint32_t w = (k ? __funnelshift_r(W0, W1, 8 * k) : W0) & pmask;
                        if (want_p && test.first(w, pp) && (m <= 4 || test.rest(hb, i, pat, m))) hp |= 1u << k;
                        if (want_m && test.first(w, pm) && (m <= 4 || test.rest(hb, i, rc, m))) hm |= 1u << k;
                    }
                }
                if (MODE == S_COUNT) {
                    cp += __popc(hp);
                    cm += __popc(hm);
                } else if (MODE == S_ALL) {
                    const int n = __popc(hp) + __popc(hm);
                    if (__any_sync(0xffffffffu, n != 0)) {
                        int inc = n;
#pragma unroll
                        for (int d = 1; d < 32; d <<= 1) {
                            const int o = __shfl_up_sync(0xffffffffu, inc, d);
                            if (lane >= d) inc += o;
                        }
                        int64_t o = cursor + (inc - n);
#pragma unroll
                        for (int k = 0; k < 4; ++k) {                         // (start, minus) order
                            if ((hp >> k) & 1u) { fxg_search_hit *h = A.out + o++; h->query = q; h->start = start0 + i0 + k; h->minus = 0; h->mismatches = test.mismatches(hb, i0 + k, pat, m); }
                            if ((hm >> k) & 1u) { fxg_search_hit *h = A.out + o++; h->query = q; h->start = start0 + i0 + k; h->minus = 1; h->mismatches = test.mismatches(hb, i0 + k, rc, m); }
                        }
                        cursor += __shfl_sync(0xffffffffu, inc, 31);
                    }
                } else {
                    const uint32_t h = hp | hm;                                 // one strand is asked for
                    const uint32_t bal = __ballot_sync(0xffffffffu, h != 0);
                    if (bal) {
                        if (lane == __ffs(bal) - 1) {
                            fxg_search_hit *o = A.out + out_pos;
                            o->query = q; o->start = start0 + i0 + __ffs(h) - 1; o->minus = want_m ? 1 : 0; o->mismatches = 0;
                        }
                        return;
                    }
                }
            }
            wb = wend;
            if (wb >= ntest) break;
            // the next window starts PIECE bytes on: keep its first m - 1 bytes and whatever the last round brought
            const int keepn = have - SPIECE;
            __syncwarp();                                       // every lane is done reading the window
            for (int i = lane; i < keepn; i += 32) hb[i] = hb[SPIECE + i];
            __syncwarp();
            have = keepn;
        }
        if (!more || wb >= ntest) break;
    }
}

__global__ void search_items_kernel(SearchArgs A, int64_t *__restrict__ n_items) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= A.nq) return;
    int64_t s, e;
    fxg_fasta_row r;
    bool row_ok;
    load_query(A, q, s, e, r, row_ok);
    const int64_t len = e - s;
    int64_t n = 0;
    if (len >= A.m) n = split_row(r, row_ok) ? (len - A.m + SPIECE) / SPIECE : 1;
    n_items[q] = n;
}

// The count / emit / first-hit pass over the work items, with the per-start test T.
template <int MODE, class T>
__device__ __forceinline__ void search_items(const SearchArgs &A, const T &test) {
    __shared__ __align__(16) uint8_t s_pat[2][SPB];             // the pattern and its reverse complement
    __shared__ __align__(16) uint8_t s_hay[SW][SHB];
    const int m = A.m;
    for (int i = threadIdx.x; i < SPB; i += blockDim.x) {
        s_pat[0][i] = i < m ? A.pattern[i] : 0;
        s_pat[1][i] = i < m ? complement_byte(A.pattern[m - 1 - i]) : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t gw = (int64_t)blockIdx.x * SW + warp, nw = (int64_t)gridDim.x * SW;
    int64_t cp = 0, cm = 0;
    if (MODE != S_FIRST) {
        const int64_t n_items = A.item_off[A.nq];
        for (int64_t it = gw; it < n_items; it += nw) {
            if (MODE == S_ALL && A.tot[it] == 0) continue;
            int64_t lo = 0, hi = A.nq;                              // item_off[lo] <= it < item_off[hi]
            while (hi - lo > 1) {
                const int64_t mid = (lo + hi) >> 1;
                if (A.item_off[mid] <= it) lo = mid; else hi = mid;
            }
            cp = cm = 0;
            run_item<MODE>(A, test, lo, it - A.item_off[lo], A.strands, s_hay[warp], s_pat[0], s_pat[1], lane,
                           MODE == S_ALL ? A.hit_off[it] : 0, cp, cm);
            if (MODE == S_COUNT) {
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) { cp += shfl_down_i64(cp, d); cm += shfl_down_i64(cm, d); }
                if (lane == 0) { A.tot[it] = cp + cm; A.pc[it] = cp; }
            }
            __syncwarp();
        }
    } else {
        for (int64_t w = gw; w < 2 * A.nq; w += nw) {
            const int64_t q = w >> 1;
            const int st = (int)(w & 1);
            int64_t first = -1;
            if ((A.strands >> st) & 1) {
                const int64_t i0 = A.item_off[q], i1 = A.item_off[q + 1];
                for (int64_t b0 = i0; b0 < i1; b0 += 32) {
                    const int64_t it = b0 + lane;
                    int64_t c = 0;
                    if (it < i1) c = st ? A.tot[it] - A.pc[it] : A.pc[it];
                    const uint32_t bal = __ballot_sync(0xffffffffu, c > 0);
                    if (bal) { first = b0 + __ffs(bal) - 1; break; }
                }
            }
            if (lane == 0) A.out[w].query = -1;
            __syncwarp();
            if (first >= 0)
                run_item<S_FIRST>(A, test, q, first - A.item_off[q], 1 << st, s_hay[warp], s_pat[0], s_pat[1], lane, w, cp, cm);
            __syncwarp();
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(SW * 32, 4) search_kernel(SearchArgs A) { search_items<MODE>(A, ExactTest{}); }
// every start within max_mm substitutions; no first-hit mode
template <int MODE>
__global__ void __launch_bounds__(SW * 32, 4) search_approx_kernel(SearchArgs A, int max_mm) {
    search_items<MODE>(A, ApproxTest{max_mm});
}

// ---- K8 on FASTQ reads ----------------------------------------------------------------------------------------------
// The haystack of read i is its raw rlen bytes at soff (Read.seq, src/read.c:152-167).  Work items, in read order: a
// tile is 32 consecutive read ids; each run of short reads (rlen <= SPIECE) between the tile's long reads is one item,
// and each long read adds one item per SPIECE start positions (a piece: those starts and the m - 1 bytes after them, one
// contiguous byte range, since a read is one line).  An item is up to 32 segments, one per lane: the lane's read, or the
// lane's piece.  A round stages as many whole segments as the warp's window holds, each in its own slot of aligned
// 16-byte chunks (every cp.async of the round is issued before any is consumed), then every lane tests the 16 starts of
// one chunk.  A start is tested only below its segment's npos, so no match runs past the end of its read.
constexpr int RW = 4;                                       // warps per CTA
constexpr int RWIN = 8192;                                  // staging window per warp
constexpr int RCH = RWIN / 16;                              // ... in 16-byte chunks
static_assert(RCH >= (15 + SPIECE + SMAXPAT - 1 + 15) / 16, "a piece must fit the window in one round");

struct ReadSearchArgs {
    const uint8_t *file;
    int64_t fsize;
    const fxg_fastq_row *rows;
    int64_t n_rows, n_tiles;
    int m, strands;
    const uint8_t *pattern;
    const int64_t *tile_off;                // n_tiles + 1: first item of each tile
    int64_t *tot;                           // per item: hits on both strands
    const int64_t *hit_off;                 // per item: first output slot (S_ALL)
    fxg_search_hit *out;
};

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Lane's read of tile t: its haystack [soff, soff + len) (len = 0 for a row outside the buffer), whether it is long,
// and how many items it starts.  brk: lanes that end a run of short reads (long reads and lanes past the last row).
__device__ __forceinline__ int64_t tile_items(const ReadSearchArgs &A, int64_t t, int lane, int64_t &soff, int64_t &len,
                                              uint32_t &brk) {
    const int64_t r = t * 32 + lane;
    const bool valid = r < A.n_rows;
    soff = 0;
    len = 0;
    if (valid) {
        const fxg_fastq_row row = A.rows[r];
        if (row.soff >= 0 && row.rlen >= 0 && row.soff <= A.fsize && row.rlen <= A.fsize - row.soff) {
            soff = row.soff;
            len = row.rlen;
        }
    }
    const bool lng = len > SPIECE;
    brk = __ballot_sync(0xffffffffu, lng || !valid);
    if (lng) return (len - A.m + SPIECE) / SPIECE;
    return valid && (lane == 0 || ((brk >> (lane - 1)) & 1u)) ? 1 : 0;
}

__global__ void search_reads_plan_kernel(ReadSearchArgs A, int64_t *__restrict__ n_items) {
    const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= A.n_tiles) return;                                 // warp-uniform
    int64_t soff, len;
    uint32_t brk;
    int64_t n = tile_items(A, t, threadIdx.x & 31, soff, len, brk);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) n += shfl_down_i64(n, d);
    if ((threadIdx.x & 31) == 0) n_items[t] = n;
}

// Every warp runs a contiguous range of items.  S_COUNT writes each item's hits to A.tot; S_ALL re-runs the items with
// hits and writes them from A.hit_off[item] on, in (read, start, minus) order.  T: the per-start test.
template <int MODE, class T>
__device__ __forceinline__ void search_reads_items(const ReadSearchArgs &A, const T &test) {
    __shared__ __align__(16) uint8_t s_pat[2][SPB];
    __shared__ __align__(16) uint8_t s_win[RW][RWIN + 16];      // + one word read past the last chunk
    __shared__ uint8_t s_map[RW][RCH];                           // chunk -> lane whose segment it holds
    const int m = A.m;
    for (int i = threadIdx.x; i < SPB; i += blockDim.x) {
        s_pat[0][i] = i < m ? A.pattern[i] : 0;
        s_pat[1][i] = i < m ? complement_byte(A.pattern[m - 1 - i]) : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *win = s_win[warp], *map = s_map[warp];
    const uint32_t *hw = reinterpret_cast<const uint32_t *>(win);
    const bool want_p = (A.strands & 1) != 0, want_m = (A.strands & 2) != 0;
    const uint32_t pmask = m >= 4 ? 0xffffffffu : (1u << (8 * m)) - 1u;
    const uint32_t pp = *reinterpret_cast<const uint32_t *>(s_pat[0]) & pmask;
    const uint32_t pm = *reinterpret_cast<const uint32_t *>(s_pat[1]) & pmask;

    const int64_t n_items = A.tile_off[A.n_tiles];
    const int64_t nw = (int64_t)gridDim.x * RW, per = (n_items + nw - 1) / nw;
    int64_t it = ((int64_t)blockIdx.x * RW + warp) * per;
    const int64_t it_end = it + per < n_items ? it + per : n_items;
    if (it >= it_end) return;
    int64_t t = 0, hi = A.n_tiles;                              // tile_off[t] <= it < tile_off[hi]
    while (hi - t > 1) {
        const int64_t mid = (t + hi) >> 1;
        if (A.tile_off[mid] <= it) t = mid; else hi = mid;
    }
    int64_t loaded = -1, soff = 0, len = 0, items = 0, excl = 0;
    uint32_t brk = 0;
    for (; it < it_end; ++it) {
        if (MODE == S_ALL && A.tot[it] == 0) continue;
        while (A.tile_off[t + 1] <= it) ++t;
        if (t != loaded) {                                      // lane j holds read 32 t + j: one coalesced 1 KiB load
            loaded = t;
            items = tile_items(A, t, lane, soff, len, brk);
            int64_t inc = items;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int64_t o = shfl_up_i64(inc, d);
                if (lane >= d) inc += o;
            }
            excl = inc - items;
        }
        // the item: lanes [js, je) -- one long read's piece, or a run of short reads
        const int64_t li = it - A.tile_off[t];
        const int js = __ffs(__ballot_sync(0xffffffffu, excl + items > li)) - 1;
        const bool slong = __shfl_sync(0xffffffffu, (int)(len > SPIECE), js) != 0;
        const uint32_t above = brk & ~((2u << js) - 1u);
        const int je = slong ? js + 1 : (above ? __ffs(above) - 1 : 32);
        int64_t a = 0, npos = 0;                                // segment: starts [a, a + npos) of the read
        if (lane >= js && lane < je) {
            if (slong) {
                a = (li - excl) * SPIECE;
                npos = len - m + 1 - a < SPIECE ? len - m + 1 - a : SPIECE;
            } else {
                npos = len - m + 1 > 0 ? len - m + 1 : 0;
            }
        }
        const int64_t so = soff + a;
        const int lead = (int)(so & 15), np = (int)npos;
        const int nch = npos > 0 ? (lead + (int)(npos + m - 1) + 15) >> 4 : 0;
        const int64_t gch = so >> 4;                            // first source chunk of the segment
        int64_t cnt = 0, cursor = MODE == S_ALL ? A.hit_off[it] : 0;
        for (int first = 0;;) {
            // this round: the segments of lanes first .. last whose chunks fit the window
            const int c = lane >= first ? nch : 0;
            int incl = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += o;
            }
            const bool take = lane >= first && incl <= RCH;
            const uint32_t rest = __ballot_sync(0xffffffffu, lane >= first && !take);
            const int C = __shfl_sync(0xffffffffu, incl, rest ? __ffs(rest) - 2 : 31);
            const int P = incl - c;                             // slot of the lane's segment, in chunks
            __syncwarp();                                       // every lane is done with the last round's window
            if (take)
                for (int k = 0; k < c; ++k) map[P + k] = (uint8_t)lane;
            __syncwarp();
            for (int b = 0; b < C; b += 32) {
                const int i = b + lane;
                const int j = i < C ? map[i] : 0;
                const int64_t g = shfl_i64(gch, j);
                const int pj = __shfl_sync(0xffffffffu, P, j);
                if (i < C) cp_async16(win + 16 * i, A.file + ((g + (i - pj)) << 4));
            }
            cp_async_wait_all();
            __syncwarp();
            for (int b = 0; b < C; b += 32) {
                const int ci = b + lane;
                const int j = ci < C ? map[ci] : 0;
                const int pj = __shfl_sync(0xffffffffu, P, j), lj = __shfl_sync(0xffffffffu, lead, j);
                const int nj = __shfl_sync(0xffffffffu, np, j);
                const int k0 = 16 * (ci - pj) - lj;             // segment start of the chunk's byte 0
                const int lo = k0 < 0 ? -k0 : 0, hi2 = nj - k0 < 16 ? nj - k0 : 16;
                const uint32_t valid = ci < C && hi2 > lo ? (0xffffu >> (16 - hi2)) & ~((1u << lo) - 1u) : 0u;
                uint32_t hp = 0, hm = 0;
                if (valid) {
                    const uint4 v = *reinterpret_cast<const uint4 *>(win + 16 * ci);
                    const uint32_t W[5] = {v.x, v.y, v.z, v.w, hw[4 * ci + 4]};
#pragma unroll
                    for (int q = 0; q < 16; ++q) {
                        const uint32_t w = ((q & 3) ? __funnelshift_r(W[q >> 2], W[(q >> 2) + 1], 8 * (q & 3)) : W[q >> 2]) & pmask;
                        hp |= (uint32_t)(want_p && test.first(w, pp)) << q;
                        hm |= (uint32_t)(want_m && test.first(w, pm)) << q;
                    }
                    hp &= valid;
                    hm &= valid;
                    if (m > 4) {
                        for (uint32_t x = hp; x; x &= x - 1u)
                            if (!test.rest(win, 16 * ci + __ffs(x) - 1, s_pat[0], m)) hp &= ~(x & (0u - x));
                        for (uint32_t x = hm; x; x &= x - 1u)
                            if (!test.rest(win, 16 * ci + __ffs(x) - 1, s_pat[1], m)) hm &= ~(x & (0u - x));
                    }
                }
                if (MODE == S_COUNT) {
                    cnt += __popc(hp) + __popc(hm);
                } else {
                    const int64_t aj = shfl_i64(a, j);
                    const int n = __popc(hp) + __popc(hm);
                    if (__any_sync(0xffffffffu, n != 0)) {
                        int inc = n;
#pragma unroll
                        for (int d = 1; d < 32; d <<= 1) {
                            const int o = __shfl_up_sync(0xffffffffu, inc, d);
                            if (lane >= d) inc += o;
                        }
                        int64_t o = cursor + (inc - n);
                        const int64_t rid = t * 32 + j, s0 = aj + k0;
                        for (uint32_t x = hp | hm; x; x &= x - 1u) {                // (start, minus) order
                            const int q = __ffs(x) - 1;
                            if ((hp >> q) & 1u) { fxg_search_hit *h = A.out + o++; h->query = rid; h->start = s0 + q; h->minus = 0; h->mismatches = test.mismatches(win, 16 * ci + q, s_pat[0], m); }
                            if ((hm >> q) & 1u) { fxg_search_hit *h = A.out + o++; h->query = rid; h->start = s0 + q; h->minus = 1; h->mismatches = test.mismatches(win, 16 * ci + q, s_pat[1], m); }
                        }
                        cursor += __shfl_sync(0xffffffffu, inc, 31);
                    }
                }
            }
            if (!rest) break;
            first = __ffs(rest) - 1;
        }
        if (MODE == S_COUNT) {
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) cnt += shfl_down_i64(cnt, d);
            if (lane == 0) A.tot[it] = cnt;
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(RW * 32) search_reads_kernel(ReadSearchArgs A) { search_reads_items<MODE>(A, ExactTest{}); }
// every start within max_mm substitutions
template <int MODE>
__global__ void __launch_bounds__(RW * 32) search_reads_approx_kernel(ReadSearchArgs A, int max_mm) {
    search_reads_items<MODE>(A, ApproxTest{max_mm});
}

}  // namespace fxg

using namespace fxg;

static int search_grid(fxg_ctx *ctx, int64_t warps) {
    int64_t blocks = (warps + SW - 1) / SW;
    const int64_t maxb = (int64_t)ctx->sm_count * 4;
    if (blocks > maxb) blocks = maxb;
    return blocks < 1 ? 1 : (int)blocks;
}

// Every hit of a count pass: the exclusive prefix of the per-item hits d_tot sizes the output (synchronises), emit(out)
// launches the pass that writes it on the device, one D2H copy brings it back.  d_zero and d_hoff: n_items and
// n_items + 1 scratch entries.
template <class Emit>
static int collect_hits(fxg_ctx *ctx, int64_t n_items, const int64_t *d_tot, int64_t *d_zero, int64_t *d_hoff, Emit emit,
                        fxg_search_hit **h, int64_t *n_hits) {
    FXG_CUDA(cudaMemsetAsync(d_zero, 0, (size_t)n_items * 8, ctx->stream));
    int rc = fxg_extract_plan_dev(ctx, d_zero, d_tot, n_items, d_hoff, n_hits);
    if (rc || *n_hits == 0) return rc;
    if ((rc = ctx->row_tmp.reserve((size_t)*n_hits * sizeof(fxg_search_hit) + 64))) return rc;
    fxg_search_hit *d_out = (fxg_search_hit *)ctx->row_tmp.ptr;
    ctx->launches += 1;
    emit(d_out);
    FXG_CUDA(cudaGetLastError());
    fxg_search_hit *p = (fxg_search_hit *)malloc((size_t)*n_hits * sizeof(fxg_search_hit));
    if (!p) { fxg_set_error("out of memory (%lld search hits)", (long long)*n_hits); return FXG_ENOMEM; }
    cudaError_t ce = cudaMemcpyAsync(p, d_out, (size_t)*n_hits * sizeof(fxg_search_hit), cudaMemcpyDeviceToHost, ctx->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(ctx->stream);
    if (ce != cudaSuccess) { free(p); FXG_CUDA(ce); }
    *h = p;
    return FXG_OK;
}

// fxg_search_host (K8's exact test) and fxg_search_approx_host (approx: at most max_mm mismatches, mode FXG_SEARCH_ALL)
static int search_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows, const int64_t *row_id,
                       const int64_t *s, const int64_t *e, int32_t flags, int64_t nq, const uint8_t *pattern, int32_t m,
                       bool approx, int32_t max_mm, int strands, int mode, fxg_search_hit **out, int64_t *n_out) {
    if (!ctx && fxg_device_count() == 0) {
        fxg_set_error("no CUDA device available; libfxg has no CPU fallback");
        return FXG_ENODEV;
    }
    FXG_CHECK_ARG(ctx && f && out && n_out && pattern && nq >= 0 && n_rows >= 0, "bad arguments");
    FXG_CHECK_ARG(m >= 1 && m <= FXG_SEARCH_MAX_PATTERN, "pattern length must be 1 .. FXG_SEARCH_MAX_PATTERN");
    FXG_CHECK_ARG(!approx || (max_mm >= 0 && max_mm < m), "max_mismatches must be 0 .. m - 1");
    FXG_CHECK_ARG(strands >= 1 && strands <= 3, "strands must be FXG_SEARCH_PLUS, FXG_SEARCH_MINUS or both");
    FXG_CHECK_ARG(mode == FXG_SEARCH_ALL || mode == FXG_SEARCH_FIRST, "mode must be FXG_SEARCH_ALL or FXG_SEARCH_FIRST");
    FXG_CHECK_ARG((flags & ~FXG_X_UPPER) == 0, "flags other than FXG_X_UPPER are not searchable");
    FXG_CHECK_ARG(row_id ? (nq == 0 || (s && e)) : nq == n_rows, "row_id, s, e: all or none (then nq == n_rows)");
    FXG_CHECK_ARG(nq == 0 || d_rows, "d_rows == NULL");
    *out = nullptr;
    *n_out = 0;
    FXG_LOCK(ctx);
    FXG_CUDA(cudaSetDevice(ctx->device));
    fxg_search_hit *h = nullptr;
    int64_t n_hits = 0;
    if (nq > 0) {
        // misc: [row | s | e] | n_items | zeros | item_off (nq + 1) | pattern
        const size_t qb = (size_t)nq * 8, nqa = row_id ? 3 : 0;
        int rc = ctx->misc.reserve(qb * (nqa + 2) + qb + 8 + SPB + 64);
        if (rc) return rc;
        int64_t *base = (int64_t *)ctx->misc.ptr;
        int64_t *d_row = row_id ? base : nullptr, *d_s = row_id ? base + nq : nullptr, *d_e = row_id ? base + 2 * nq : nullptr;
        int64_t *d_nit = base + nqa * nq, *d_zero = d_nit + nq, *d_ioff = d_zero + nq;
        uint8_t *d_pat = (uint8_t *)(d_ioff + nq + 1);
        if (row_id) {
            FXG_CUDA(cudaMemcpyAsync(d_row, row_id, qb, cudaMemcpyHostToDevice, ctx->stream));
            FXG_CUDA(cudaMemcpyAsync(d_s, s, qb, cudaMemcpyHostToDevice, ctx->stream));
            FXG_CUDA(cudaMemcpyAsync(d_e, e, qb, cudaMemcpyHostToDevice, ctx->stream));
        }
        FXG_CUDA(cudaMemcpyAsync(d_pat, pattern, (size_t)m, cudaMemcpyHostToDevice, ctx->stream));
        FXG_CUDA(cudaMemsetAsync(d_zero, 0, qb, ctx->stream));
        SearchArgs A;
        memset(&A, 0, sizeof(A));
        A.file = f->d; A.fsize = f->size; A.rows = d_rows; A.n_rows = n_rows;
        A.q_row = d_row; A.q_s = d_s; A.q_e = d_e; A.nq = nq;
        A.flags = flags; A.m = m; A.strands = strands; A.pattern = d_pat; A.item_off = d_ioff;
        ctx->launches += 1;
        search_items_kernel<<<(unsigned)((nq + 255) / 256), 256, 0, ctx->stream>>>(A, d_nit);
        FXG_CUDA(cudaGetLastError());
        int64_t n_items = 0;
        if ((rc = fxg_extract_plan_dev(ctx, d_zero, d_nit, nq, d_ioff, &n_items))) return rc;     // synchronises
        if (n_items > 0) {
            // search scratch: tot | pc | zeros | hit_off (n_items + 1)
            if ((rc = ctx->search.reserve((size_t)n_items * 32 + 8 + 64))) return rc;
            A.tot = (int64_t *)ctx->search.ptr;
            A.pc = A.tot + n_items;
            int64_t *d_zero2 = A.pc + n_items, *d_hoff = d_zero2 + n_items;
            A.hit_off = d_hoff;
            {
                FxgProfScope prof(ctx, FXG_PROF_GATHER);
                if (!approx) search_kernel<S_COUNT><<<search_grid(ctx, n_items), SW * 32, 0, ctx->stream>>>(A);
                else search_approx_kernel<S_COUNT><<<search_grid(ctx, n_items), SW * 32, 0, ctx->stream>>>(A, max_mm);
            }
            FXG_CUDA(cudaGetLastError());
            if (mode == FXG_SEARCH_ALL) {
                rc = collect_hits(ctx, n_items, A.tot, d_zero2, d_hoff, [&](fxg_search_hit *o) {
                    A.out = o;
                    if (!approx) search_kernel<S_ALL><<<search_grid(ctx, n_items), SW * 32, 0, ctx->stream>>>(A);
                    else search_approx_kernel<S_ALL><<<search_grid(ctx, n_items), SW * 32, 0, ctx->stream>>>(A, max_mm);
                }, &h, &n_hits);
                if (rc) return rc;
            } else {
                if ((rc = ctx->row_tmp.reserve((size_t)nq * 2 * sizeof(fxg_search_hit) + 64))) return rc;
                A.out = (fxg_search_hit *)ctx->row_tmp.ptr;
                ctx->launches += 1;
                search_kernel<S_FIRST><<<search_grid(ctx, 2 * nq), SW * 32, 0, ctx->stream>>>(A);
                FXG_CUDA(cudaGetLastError());
                std::vector<fxg_search_hit> slot((size_t)nq * 2);
                FXG_CUDA(cudaMemcpyAsync(slot.data(), A.out, slot.size() * sizeof(fxg_search_hit), cudaMemcpyDeviceToHost, ctx->stream));
                FXG_CUDA(cudaStreamSynchronize(ctx->stream));
                h = (fxg_search_hit *)malloc(slot.size() * sizeof(fxg_search_hit));
                if (!h) { fxg_set_error("out of memory (%lld search hits)", (long long)nq * 2); return FXG_ENOMEM; }
                for (int64_t q = 0; q < nq; ++q) {                   // slot 2q: plus strand, 2q + 1: minus strand
                    const fxg_search_hit &p = slot[2 * q], &mi = slot[2 * q + 1];
                    const bool hp = p.query >= 0, hm = mi.query >= 0;
                    if (hp && hm && mi.start < p.start) { h[n_hits++] = mi; h[n_hits++] = p; }
                    else { if (hp) h[n_hits++] = p; if (hm) h[n_hits++] = mi; }
                }
            }
        }
    }
    if (!h) {
        h = (fxg_search_hit *)malloc(sizeof(fxg_search_hit));
        if (!h) { fxg_set_error("out of memory"); return FXG_ENOMEM; }
    }
    *out = h;
    *n_out = n_hits;
    return FXG_OK;
}

extern "C" int fxg_search_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                               const int64_t *row_id, const int64_t *s, const int64_t *e, int32_t flags, int64_t nq,
                               const uint8_t *pattern, int32_t m, int strands, int mode, fxg_search_hit **out,
                               int64_t *n_out) {
    return search_host(ctx, f, d_rows, n_rows, row_id, s, e, flags, nq, pattern, m, false, 0, strands, mode, out, n_out);
}

extern "C" int fxg_search_approx_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                                      const int64_t *row_id, const int64_t *s, const int64_t *e, int32_t flags, int64_t nq,
                                      const uint8_t *pattern, int32_t m, int32_t max_mismatches, int strands,
                                      fxg_search_hit **out, int64_t *n_out) {
    return search_host(ctx, f, d_rows, n_rows, row_id, s, e, flags, nq, pattern, m, true, max_mismatches,
                       strands, FXG_SEARCH_ALL, out, n_out);
}

// reads kernels: the most CTAs of 4 warps an SM holds (the window is static shared memory, so ask for the largest
// carveout); per_sm[0] for the exact kernels, per_sm[1] for the approximate ones
static int search_reads_grid(fxg_ctx *ctx, int64_t n_items, bool approx) {
    static int per_sm[2] = {0, 0};
    if (!per_sm[0]) {
        const void *k[2][2] = {{(const void *)search_reads_kernel<S_COUNT>, (const void *)search_reads_kernel<S_ALL>},
                               {(const void *)search_reads_approx_kernel<S_COUNT>, (const void *)search_reads_approx_kernel<S_ALL>}};
        for (int a = 0; a < 2; ++a)
            for (int i = 0; i < 2; ++i) {
                cudaFuncSetAttribute(k[a][i], cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
                int nb = 0;
                if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k[a][i], RW * 32, 0) != cudaSuccess || nb < 1) nb = 1;
                if (i == S_COUNT) per_sm[a] = nb;                   // the grid is sized by the count kernel
            }
    }
    int64_t blocks = (n_items + RW - 1) / RW;
    const int64_t maxb = (int64_t)ctx->sm_count * per_sm[approx ? 1 : 0];
    if (blocks > maxb) blocks = maxb;
    return blocks < 1 ? 1 : (int)blocks;
}

// fxg_search_reads_host (K8's exact test) and fxg_search_reads_approx_host (approx: at most max_mm mismatches)
static int search_reads_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                             const uint8_t *pattern, int32_t m, bool approx, int32_t max_mm, int strands, fxg_search_hit **out,
                             int64_t *n_out) {
    if (!ctx && fxg_device_count() == 0) {
        fxg_set_error("no CUDA device available; libfxg has no CPU fallback");
        return FXG_ENODEV;
    }
    FXG_CHECK_ARG(ctx && f && out && n_out && pattern && n_rows >= 0, "bad arguments");
    FXG_CHECK_ARG(m >= 1 && m <= FXG_SEARCH_MAX_PATTERN, "pattern length must be 1 .. FXG_SEARCH_MAX_PATTERN");
    FXG_CHECK_ARG(!approx || (max_mm >= 0 && max_mm < m), "max_mismatches must be 0 .. m - 1");
    FXG_CHECK_ARG(strands >= 1 && strands <= 3, "strands must be FXG_SEARCH_PLUS, FXG_SEARCH_MINUS or both");
    FXG_CHECK_ARG(n_rows == 0 || d_rows, "d_rows == NULL");
    *out = nullptr;
    *n_out = 0;
    FXG_LOCK(ctx);
    FXG_CUDA(cudaSetDevice(ctx->device));
    fxg_search_hit *h = nullptr;
    int64_t n_hits = 0;
    if (n_rows > 0) {
        // misc: n_items per tile | zeros | tile_off (n_tiles + 1) | pattern
        const int64_t n_tiles = (n_rows + 31) / 32;
        const size_t tb = (size_t)n_tiles * 8;
        int rc = ctx->misc.reserve(tb * 3 + 8 + SPB + 64);
        if (rc) return rc;
        int64_t *d_nit = (int64_t *)ctx->misc.ptr, *d_zero = d_nit + n_tiles, *d_toff = d_zero + n_tiles;
        uint8_t *d_pat = (uint8_t *)(d_toff + n_tiles + 1);
        FXG_CUDA(cudaMemcpyAsync(d_pat, pattern, (size_t)m, cudaMemcpyHostToDevice, ctx->stream));
        FXG_CUDA(cudaMemsetAsync(d_zero, 0, tb, ctx->stream));
        ReadSearchArgs A;
        memset(&A, 0, sizeof(A));
        A.file = f->d; A.fsize = f->size; A.rows = d_rows; A.n_rows = n_rows; A.n_tiles = n_tiles;
        A.m = m; A.strands = strands; A.pattern = d_pat; A.tile_off = d_toff;
        ctx->launches += 1;
        search_reads_plan_kernel<<<(unsigned)((n_tiles + 7) / 8), 256, 0, ctx->stream>>>(A, d_nit);
        FXG_CUDA(cudaGetLastError());
        int64_t n_items = 0;
        if ((rc = fxg_extract_plan_dev(ctx, d_zero, d_nit, n_tiles, d_toff, &n_items))) return rc;     // synchronises
        // search scratch: tot | zeros | hit_off (n_items + 1)
        if ((rc = ctx->search.reserve((size_t)n_items * 24 + 8 + 64))) return rc;
        A.tot = (int64_t *)ctx->search.ptr;
        int64_t *d_zero2 = A.tot + n_items, *d_hoff = d_zero2 + n_items;
        A.hit_off = d_hoff;
        const int grid = search_reads_grid(ctx, n_items, approx);
        {
            FxgProfScope prof(ctx, FXG_PROF_GATHER);
            if (!approx) search_reads_kernel<S_COUNT><<<grid, RW * 32, 0, ctx->stream>>>(A);
            else search_reads_approx_kernel<S_COUNT><<<grid, RW * 32, 0, ctx->stream>>>(A, max_mm);
        }
        FXG_CUDA(cudaGetLastError());
        rc = collect_hits(ctx, n_items, A.tot, d_zero2, d_hoff, [&](fxg_search_hit *o) {
            A.out = o;
            if (!approx) search_reads_kernel<S_ALL><<<grid, RW * 32, 0, ctx->stream>>>(A);
            else search_reads_approx_kernel<S_ALL><<<grid, RW * 32, 0, ctx->stream>>>(A, max_mm);
        }, &h, &n_hits);
        if (rc) return rc;
    }
    if (!h) {
        h = (fxg_search_hit *)malloc(sizeof(fxg_search_hit));
        if (!h) { fxg_set_error("out of memory"); return FXG_ENOMEM; }
    }
    *out = h;
    *n_out = n_hits;
    return FXG_OK;
}

extern "C" int fxg_search_reads_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                                     const uint8_t *pattern, int32_t m, int strands, fxg_search_hit **out, int64_t *n_out) {
    return search_reads_host(ctx, f, d_rows, n_rows, pattern, m, false, 0, strands, out, n_out);
}

extern "C" int fxg_search_reads_approx_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                                            const uint8_t *pattern, int32_t m, int32_t max_mismatches, int strands,
                                            fxg_search_hit **out, int64_t *n_out) {
    return search_reads_host(ctx, f, d_rows, n_rows, pattern, m, true, max_mismatches, strands, out, n_out);
}
