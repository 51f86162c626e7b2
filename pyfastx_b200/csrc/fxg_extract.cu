// fxg_extract.cu -- K3/K4 batched subsequence extraction and K5 batched read fetch (sm_90a).
//
// Replaces, per query, the reference chain
//   pyfastx_sequence_subscript  (src/sequence.c:498-510)  slice -> (offset, byte_len)
//   pyfastx_index_random_read   (src/index.c:683-692)     fseeko + fread of the byte range
//   remove_space[_uppercase]    (src/util.c:166-194)      drop 10/13/32, optional toupper
//   reverse/complement getters  (src/util.c:239-269)      strand transforms via comp_map
//   gc_content counting loop    (src/sequence.c:607-631)  A/C/G/T counters (fused, optional)
// and for FASTQ  pyfastx_read_random_reader (src/read.c:37-45): raw copies of rlen bytes.
//
// A batch of queries goes to extract_bulk_kernel: a warp owns up to 32 queries, and for records with
// uniform lines the covering source bytes of every 1 KiB output piece arrive in shared memory by one
// TMA bulk copy, from which every lane assembles aligned 16-byte output words (slice formula).
// Every other query -- norm = 0 records, odd lines, short or raw queries, a failed layout check --
// is served by one whole warp (serve_query_warp): the uniform-line pull path (pull_one) where it
// applies, else the general strip path (gather_one), which streams the covering byte range in
// 512-byte rounds and ranks the kept bytes with a warp prefix sum ("strip" semantics, exact also
// for records with an odd line).  A single query (extract_one_kernel, extract_service_kernel) and
// FASTQ reads (reads_kernel, read_one_kernel) use the same per-warp code.
#include "fxg_common.cuh"
#include <stdlib.h>
#include <string.h>
#include <chrono>

namespace fxg {

constexpr int XTHREADS = 256;
constexpr int XWARPS = XTHREADS / 32;
constexpr int XSTAGE = 512 + 32;   // staging bytes per warp (512 payload + alignment slack)

struct GatherJob {
    int64_t src;       // first source byte (buffer relative)
    int64_t src_len;   // bytes to scan
    int64_t skip;      // kept bytes to skip before emitting (norm=0 records)
    int64_t out_len;   // bytes to emit
    uint8_t *dst;      // output position
    int     flags;
};

__device__ __forceinline__ uint32_t keep_mask16(const uint4 &v) {
    // combined-mask layout (see chunk_eq_mask): 1 = byte is one of 10, 13, 32
    return chunk_eq_mask(v, 0x0a0a0a0au) | chunk_eq_mask(v, 0x0d0d0d0du) | chunk_eq_mask(v, 0x20202020u);
}
// combined-mask bit for chunk byte `off` (0..15)
__device__ __forceinline__ uint32_t bit_of_off(int off) { return 1u << (8 * (off & 3) + 7 - (off >> 2)); }

// counts of bytes equal (case-insensitively) to the letter in c4 (lower case x4), within `valid` (0x80 per byte)
__device__ __forceinline__ int count_letter(uint32_t w, uint32_t c4, uint32_t valid) {
    return __popc(byte_eq_mask(w | 0x20202020u, c4) & valid);
}
// the same for one byte
__device__ __forceinline__ void count_byte(uint32_t b, int &cA, int &cC, int &cG, int &cT) {
    b |= 0x20u;
    cA += b == 'a'; cC += b == 'c'; cG += b == 'g'; cT += b == 't';
}

template <bool WANT_ACGT>
__device__ void gather_one(const uint8_t *__restrict__ file, int64_t fsize, const GatherJob &job,
                           const uint8_t *__restrict__ s_lut, uint8_t *__restrict__ stage,
                           int lane, int64_t *acgt_out) {
    const bool raw = (job.flags & FXG_X_RAW) != 0;
    const bool upper = (job.flags & FXG_X_UPPER) != 0;
    const bool comp = (job.flags & FXG_X_COMPLEMENT) != 0;
    const bool rev = (job.flags & FXG_X_REVERSE) != 0;
    int64_t src_end = job.src + job.src_len;
    if (src_end > fsize) src_end = fsize;                       // fread past EOF returns short
    const int64_t want_end = job.skip + job.out_len;            // kept-rank window [skip, want_end)
    int64_t done = 0;                                           // kept bytes seen so far
    int cntA = 0, cntC = 0, cntG = 0, cntT = 0;

    for (int64_t cbase = job.src & ~(int64_t)15; cbase < src_end && done < want_end; cbase += 512) {
        const int64_t my = cbase + lane * 16;
        uint4 v = make_uint4(0, 0, 0, 0);
        uint32_t valid = 0;                                      // combined-mask bits of in-range bytes
        if (my < src_end && my + 16 > job.src) {
            v = *reinterpret_cast<const uint4 *>(file + my);
            const int lo = (int)(job.src > my ? job.src - my : 0);
            const int hi = (int)(src_end - my < 16 ? src_end - my : 16);
            // combined-mask bits of bytes lo..hi-1, byte by byte: no byte at or past hi may count, or a range holding
            // fewer kept bytes than requested would take the kept byte after its end instead of the zero fill below
            // (test_edge_layouts_gpu.py::test_slice_short_of_kept_bytes)
            uint32_t m = 0;
#pragma unroll
            for (int off = 0; off < 16; ++off)
                if (off >= lo && off < hi) m |= bit_of_off(off);
            valid = m;
        }
        uint32_t keep = raw ? valid : (valid & ~keep_mask16(v));
        const int cnt = __popc(keep);
        // warp exclusive prefix of cnt
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += o;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        int64_t rank = done + (incl - cnt);                      // rank of this lane's first kept byte
        // this round emits kept ranks [r0, r1)
        const int64_t r0 = done > job.skip ? done : job.skip;
        int64_t r1 = done + total;
        if (r1 > want_end) r1 = want_end;
        const int nout = (int)(r1 > r0 ? r1 - r0 : 0);
        if (nout > 0) {
            // output byte index of rank r is (r - skip), or out_len-1-(r-skip) when reversed.
            // the round's outputs form one contiguous range [o0, o0+nout)
            const int64_t o0 = rev ? (job.out_len - (r1 - job.skip)) : (r0 - job.skip);
            uint8_t *g0 = job.dst + o0;
            const int a = (int)((uintptr_t)g0 & 15);
            if (cnt) {
                const uint32_t words[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int off = 0; off < 16; ++off) {
                    if (keep & bit_of_off(off)) {
                        if (rank >= r0 && rank < r1) {
                            uint32_t b = (words[off >> 2] >> (8 * (off & 3))) & 0xffu;
                            if (upper && b >= 'a' && b <= 'z') b -= 32;
                            if (comp) b = s_lut[b];
                            const int pos = rev ? (int)(r1 - 1 - rank) : (int)(rank - r0);
                            stage[a + pos] = (uint8_t)b;
                        }
                        ++rank;
                    }
                }
            }
            __syncwarp();
            // flush: aligned 16-byte words; ragged ends byte-wise
            const int nwords = (a + nout + 15) >> 4;
            for (int w = lane; w < nwords; w += 32) {
                const int lo = (w == 0) ? a : 0;
                const int hi = ((w + 1) * 16 <= a + nout) ? 16 : (a + nout - w * 16);
                uint8_t *gw = g0 - a + w * 16;
                // the counts are taken from exactly the bytes stored: the whole word, or the ragged bytes one by one
                if (lo == 0 && hi == 16) {
                    const uint4 sv = *reinterpret_cast<const uint4 *>(stage + w * 16);
                    *reinterpret_cast<uint4 *>(gw) = sv;
                    if (WANT_ACGT) {
                        const uint32_t sw[4] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            cntA += count_letter(sw[q], 0x61616161u, 0x80808080u);
                            cntC += count_letter(sw[q], 0x63636363u, 0x80808080u);
                            cntG += count_letter(sw[q], 0x67676767u, 0x80808080u);
                            cntT += count_letter(sw[q], 0x74747474u, 0x80808080u);
                        }
                    }
                } else {
                    for (int i = lo; i < hi; ++i) {
                        const uint8_t b = stage[w * 16 + i];
                        gw[i] = b;
                        if (WANT_ACGT) count_byte(b, cntA, cntC, cntG, cntT);
                    }
                }
            }
            __syncwarp();
        }
        done += total;
    }
    // fewer kept bytes than requested (malformed record): the reference returns stale buffer
    // bytes there; we define them as 0 (documented in DESIGN.md)
    {
        const int64_t emitted = (done > job.skip ? (done < want_end ? done : want_end) - job.skip : 0);
        if (emitted < job.out_len) {
            const int64_t missing = job.out_len - emitted;
            uint8_t *z = rev ? job.dst : job.dst + emitted;
            for (int64_t i = lane; i < missing; i += 32) z[i] = 0;
        }
    }
    if (WANT_ACGT) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            cntA += __shfl_down_sync(0xffffffffu, cntA, d);
            cntC += __shfl_down_sync(0xffffffffu, cntC, d);
            cntG += __shfl_down_sync(0xffffffffu, cntG, d);
            cntT += __shfl_down_sync(0xffffffffu, cntT, d);
        }
        if (lane == 0 && acgt_out) { acgt_out[0] = cntA; acgt_out[1] = cntC; acgt_out[2] = cntG; acgt_out[3] = cntT; }
    }
}

// ---- fast path ("pull"): records with uniform lines ---------------------------------------------
// Output-driven: every lane assembles one aligned 16-byte OUTPUT word per round.  The kept rank of
// its first byte gives the source position through the slice formula (sequence.c:498-510):
//   src(k) = boff + k + elen * (k / bpl)
// Six aligned 32-bit loads cover the <= 18 source bytes; two funnel-shift extractions (before /
// after the line break) are merged with a byte mask.  The layout assumption is VERIFIED on the
// fly (no strippable byte among the kept ones, '\r' where elen = 2 says so); any violation makes
// the warp redo the query with the general strip path, so results stay exact.
// tables: 0 = complement, 1 = upper, 2 = upper then complement
template <bool WANT_ACGT>
__device__ bool pull_one(const uint8_t *__restrict__ file, int64_t boff, int64_t s, int64_t out_len, uint32_t bpl,
                         int elen, int flags, uint8_t *__restrict__ dst, const uint8_t (*__restrict__ s_lut)[256],
                         int lane, int64_t *acgt_out) {
    const bool raw = (flags & FXG_X_RAW) != 0;
    const bool rev = (flags & FXG_X_REVERSE) != 0;
    const bool upper = (flags & FXG_X_UPPER) != 0, comp = (flags & FXG_X_COMPLEMENT) != 0;
    const uint8_t *tbl = comp ? (upper ? s_lut[2] : s_lut[0]) : s_lut[1];
    const bool xform = upper || comp;
    const int a = (int)((uintptr_t)dst & 15);
    const int64_t nwords = (a + out_len + 15) >> 4;
    int64_t q_s = 0;
    uint32_t rem_s = 0;
    if (!raw) {
        if ((uint64_t)s < (1ull << 32)) { const uint32_t qq = (uint32_t)s / bpl; q_s = qq; rem_s = (uint32_t)s - qq * bpl; }
        else { q_s = s / (int64_t)bpl; rem_s = (uint32_t)(s - q_s * (int64_t)bpl); }
    }
    bool bad = false;
    int cntA = 0, cntC = 0, cntG = 0, cntT = 0;
    for (int64_t w0 = 0; w0 < nwords; w0 += 32) {
        const int64_t w = w0 + lane;
        if (w < nwords) {
            const int64_t jw = 16 * w - a;                              // output index of slot 0
            const int lo = jw < 0 ? (int)(-jw) : 0;
            const int hi = (jw + 16 > out_len) ? (int)(out_len - jw) : 16;
            const int nb = hi - lo;                                     // valid slots [lo, hi)
            const uint32_t d = (uint32_t)(rev ? (out_len - (jw + hi)) : (jw + lo));   // first kept rank - s
            uint32_t dq = 0, c = 0xffffffffu;
            if (!raw) {
                const uint32_t t = rem_s + d;
                dq = t / bpl;
                c = bpl - (t - dq * bpl);                               // bytes left on this line
            }
            const int64_t p = boff + s + (int64_t)d + (int64_t)elen * (q_s + (int64_t)dq);
            const uint32_t *wp = reinterpret_cast<const uint32_t *>(file + (p & ~(int64_t)3));
            uint32_t W[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) W[i] = wp[i];
            const int o1 = (int)(p & 3);
            uint32_t V[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) V[i] = __funnelshift_r(W[i], W[i + 1], o1 * 8);
            if (c < (uint32_t)nb) {                                     // a line break inside this word
                const int o2 = o1 + elen, ws2 = o2 >> 2, bs2 = (o2 & 3) * 8;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const uint32_t lo_w = ws2 ? W[i + 1] : W[i], hi_w = ws2 ? W[(i + 2 < 6) ? i + 2 : 5] : W[i + 1];
                    const uint32_t e2 = __funnelshift_r(lo_w, hi_w, bs2);
                    const int rel = (int)c - 4 * i;                     // bytes of this word taken before the break
                    const uint32_t m = rel <= 0 ? 0xffffffffu : (rel >= 4 ? 0u : (0xffffffffu << (8 * rel)));
                    V[i] = (V[i] & ~m) | (e2 & m);
                }
                if (elen == 2 && file[p + c] != '\r') bad = true;      // the skipped byte must be strippable
            } else if (c == (uint32_t)nb && elen == 2 && file[p + c] != '\r') {
                bad = true;                                             // a break right after the word: checked here too
            }
            // valid-byte masks (0x80 per byte) of the first nb bytes
            uint32_t vb[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int rel = nb - 4 * i;
                vb[i] = rel >= 4 ? 0x80808080u : (rel <= 0 ? 0u : (0x80808080u & ((1u << (8 * rel)) - 1u)));
            }
            if (!raw) {
                // conservative layout check: every kept byte must be >= 0x40 (letters); anything below
                // (which includes the strippable 10 / 13 / 32, but also digits, '*', '-') sends the query
                // to the general strip path, so the result is exact either way
                uint32_t all = 0x40404040u;
#pragma unroll
                for (int i = 0; i < 4; ++i) all &= ((V[i] | (V[i] >> 1)) | ~(vb[i] >> 1));
                if ((all & 0x40404040u) != 0x40404040u) bad = true;
            }
            if (xform) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const uint32_t x = V[i];
                    V[i] = (uint32_t)tbl[x & 0xff] | ((uint32_t)tbl[(x >> 8) & 0xff] << 8) |
                           ((uint32_t)tbl[(x >> 16) & 0xff] << 16) | ((uint32_t)tbl[x >> 24] << 24);
                }
            }
            uint8_t *gw = dst + jw;                                     // 16-byte aligned
            // the counts are taken from exactly the bytes stored: the whole word, or the ragged bytes one by one
            if (nb == 16) {
                if (WANT_ACGT) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        cntA += count_letter(V[i], 0x61616161u, 0x80808080u);
                        cntC += count_letter(V[i], 0x63636363u, 0x80808080u);
                        cntG += count_letter(V[i], 0x67676767u, 0x80808080u);
                        cntT += count_letter(V[i], 0x74747474u, 0x80808080u);
                    }
                }
                uint4 o;
                if (rev) {
                    o.x = __byte_perm(V[3], 0, 0x0123); o.y = __byte_perm(V[2], 0, 0x0123);
                    o.z = __byte_perm(V[1], 0, 0x0123); o.w = __byte_perm(V[0], 0, 0x0123);
                } else { o.x = V[0]; o.y = V[1]; o.z = V[2]; o.w = V[3]; }
                *reinterpret_cast<uint4 *>(gw) = o;
            } else {                                                    // ragged first / last word
                uint32_t tmp[4] = {V[0], V[1], V[2], V[3]};
                for (int i = 0; i < nb; ++i) {
                    const int k = rev ? nb - 1 - i : i;
                    const uint8_t b = (uint8_t)(tmp[k >> 2] >> (8 * (k & 3)));
                    gw[lo + i] = b;
                    if (WANT_ACGT) count_byte(b, cntA, cntC, cntG, cntT);
                }
            }
        }
    }
    bad = __any_sync(0xffffffffu, bad);
    if (bad) return false;
    if (WANT_ACGT) {
#pragma unroll
        for (int dd = 16; dd > 0; dd >>= 1) {
            cntA += __shfl_down_sync(0xffffffffu, cntA, dd);
            cntC += __shfl_down_sync(0xffffffffu, cntC, dd);
            cntG += __shfl_down_sync(0xffffffffu, cntG, dd);
            cntT += __shfl_down_sync(0xffffffffu, cntT, dd);
        }
        if (lane == 0 && acgt_out) { acgt_out[0] = cntA; acgt_out[1] = cntC; acgt_out[2] = cntG; acgt_out[3] = cntT; }
    }
    return true;
}

__device__ __forceinline__ void init_luts(uint8_t (*s_lut)[256]) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        const int up = (i >= 'a' && i <= 'z') ? i - 32 : i;
        s_lut[0][i] = complement_byte(i);
        s_lut[1][i] = (uint8_t)up;
        s_lut[2][i] = complement_byte(up);
    }
}

// ---- whole-warp service of one query: the uniform-line pull path, else the general strip path ----
template <bool WANT_ACGT>
__device__ void serve_query_warp(const uint8_t *__restrict__ file, int64_t fsize, int64_t capacity,
                                 const fxg_fasta_row &r, bool row_ok, int64_t s, int64_t e, int flags, uint8_t *dst,
                                 const uint8_t (*__restrict__ s_lut)[256], uint8_t *__restrict__ stage, int lane,
                                 int64_t *acgt_q) {
    GatherJob job;
    job.flags = flags;
    job.dst = dst;
    job.skip = 0;
    job.src = 0; job.src_len = 0;
    job.out_len = e > s ? e - s : 0;
    bool done = false;
    // rows come from a scan or from a loaded .fxi: offsets that point outside the buffer never reach a load
    row_ok = row_ok && r.boff >= 0 && r.blen >= 0 && r.boff <= fsize && s >= 0;
    if (row_ok && job.out_len > 0) {
        const int64_t bpl = r.llen - (int64_t)r.elen;
        const bool whole = (s == 0 && e == r.slen);
        const bool uniform = (r.pad[0] & 1) != 0;
        // fast path: uniform lines, sane sizes, source window inside the buffer
        if (r.norm && uniform && bpl >= 16 && bpl < (1ll << 30) && job.out_len < (1ll << 30) && e <= r.slen &&
            r.boff + r.blen + 32 <= capacity && !(flags & FXG_X_RAW)) {
            done = pull_one<WANT_ACGT>(file, r.boff, s, job.out_len, (uint32_t)bpl, (int)r.elen, flags, job.dst, s_lut,
                                       lane, acgt_q);
        }
        if (!done) {
            const bool formula_ok = !(flags & FXG_X_WHOLE) || uniform;
            if (r.norm && bpl > 0 && !whole && formula_ok) {
                const int64_t bs = s / bpl, be = e / bpl;                       // sequence.c:500-503
                job.src = r.boff + s + (int64_t)r.elen * bs;                    // sequence.c:508
                job.src_len = (e - s) + (be - bs) * (int64_t)r.elen;            // sequence.c:509
            } else {
                job.src = r.boff; job.src_len = r.blen; job.skip = s;           // sequence.c:100-102,108-110
            }
        }
    }
    if (!done) {
        if (job.out_len > 0) gather_one<WANT_ACGT>(file, fsize, job, s_lut[0], stage, lane, acgt_q);
        else if (WANT_ACGT && lane == 0) { acgt_q[0] = acgt_q[1] = acgt_q[2] = acgt_q[3] = 0; }
    }
}

// ---- uniform-line output words ----------------------------------------------------------------------------
// Helpers of the bulk kernel below: the 16-byte transform of kept bytes, and the assembly of any 16 output bytes of a
// query on uniform lines straight from the file (the ragged first / last word of a query).

// Complement of four bytes at once for the letters that make up almost all nucleotide data: A C G T N in either
// case.  (b >> 1) & 7 is a perfect hash of these five letters (A 0, C 1, T 2, G 3, N 7), so ONE byte-permute
// looks up all four complements in an 8-entry register table; a second permute with the table of the letters
// themselves verifies that every byte really was one of the five -- any other byte (IUPAC codes, '*', '-', ...)
// makes `ok` false and the caller uses the 256-entry shared-memory LUT for that word.  Case is preserved.
__device__ __forceinline__ uint32_t comp4_acgtn(uint32_t w, bool &ok) {
    const uint32_t h = (w >> 1) & 0x07070707u;
    const uint32_t t = h | (h >> 4);
    const uint32_t sel = __byte_perm(t, 0u, 0x4420u);                    // nibbles h0 h1 h2 h3
    const uint32_t up = __byte_perm(0x47544341u, 0x4E000000u, sel);      // the letter each hash stands for (upper case)
    const uint32_t cm = __byte_perm(0x43414754u, 0x4E000000u, sel);      // its complement
    ok = (w & 0xDFDFDFDFu) == up;
    return cm | (w & 0x20202020u);
}

// upper-case / complement of 16 kept bytes (all in 0x40..0x7f, checked by the caller)
__device__ __forceinline__ void xform16(uint32_t V[4], bool upper, bool comp, const uint8_t (*__restrict__ s_lut)[256]) {
    if (comp) {
        bool f0, f1, f2, f3;
        uint32_t c0 = comp4_acgtn(V[0], f0), c1 = comp4_acgtn(V[1], f1), c2 = comp4_acgtn(V[2], f2), c3 = comp4_acgtn(V[3], f3);
        if (f0 && f1 && f2 && f3) {
            if (upper) { c0 &= 0xDFDFDFDFu; c1 &= 0xDFDFDFDFu; c2 &= 0xDFDFDFDFu; c3 &= 0xDFDFDFDFu; }
            V[0] = c0; V[1] = c1; V[2] = c2; V[3] = c3;
        } else {
            const uint8_t *tbl = upper ? s_lut[2] : s_lut[0];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t x = V[i];
                V[i] = (uint32_t)tbl[x & 0xff] | ((uint32_t)tbl[(x >> 8) & 0xff] << 8) |
                       ((uint32_t)tbl[(x >> 16) & 0xff] << 16) | ((uint32_t)tbl[x >> 24] << 24);
            }
        }
    } else if (upper) {
        // bytes are in 0x40..0x7f here: 'a'..'z' = 0x61..0x7a lose bit 5
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t x = V[i];
            const uint32_t ge = (x + 0x1f1f1f1fu) & 0x80808080u;            // byte >= 0x61
            const uint32_t le = ~(x + 0x05050505u) & 0x80808080u;           // byte <= 0x7a
            V[i] = x & ~((ge & le) >> 2);
        }
    }
}

// The 16 output bytes [j0, j0+16) of a query (0 <= j0 <= out_len-16) as four little-endian words, in two
// steps so that the loads of several words can be in flight together.
// fq = file + boff + s + elen*(s/bpl): source address of kept rank 0;  rem_s = s % bpl;  inv = 2^32 / bpl.
struct WordReq { const uint32_t *wp; int o1; uint32_t c; };

__device__ __forceinline__ WordReq ow_locate(const uint8_t *__restrict__ fq, uint32_t rem_s, uint32_t bpl, uint32_t inv,
                                             int elen, uint32_t out_len, bool rev, uint32_t j0) {
    const uint32_t r = rev ? out_len - 16u - j0 : j0;               // first kept rank of the word (source order)
    const uint32_t t = rem_s + r;
    uint32_t dq = __umulhi(t, inv);                                  // t / bpl: one below at most
    uint32_t rr = t - dq * bpl;
    if (rr >= bpl) { ++dq; rr -= bpl; }
    WordReq q;
    q.c = bpl - rr;                                                  // bytes left on this line
    const uint8_t *p = fq + (r + (uint32_t)elen * dq);              // slice formula, sequence.c:498-510
    q.wp = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)3);
    q.o1 = (int)(reinterpret_cast<uintptr_t>(p) & 3);
    return q;
}
__device__ __forceinline__ void ow_load(const WordReq &q, uint32_t W[6]) {
#pragma unroll
    for (int i = 0; i < 6; ++i) W[i] = __ldg(q.wp + i);
}
// Returns false if the bytes contradict the uniform-line layout (the query is then redone by the general path).
__device__ __forceinline__ bool ow_finish(const uint32_t W[6], const WordReq &q, int elen, bool rev, bool upper, bool comp,
                                          const uint8_t (*__restrict__ s_lut)[256], uint32_t o[4]) {
    const int o1 = q.o1;
    const uint32_t c = q.c;
    uint32_t V[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) V[i] = __funnelshift_r(W[i], W[i + 1], o1 * 8);
    bool ok = true;
    if (c < 16u) {                                                   // one line break inside the word
        if (elen == 2) {                                             // the first skipped byte must be '\r'
            const uint32_t vw = c < 8u ? (c < 4u ? V[0] : V[1]) : (c < 12u ? V[2] : V[3]);
            ok = ((vw >> (8 * (c & 3u))) & 0xffu) == 0x0du;
        }
        const int o2 = o1 + elen, ws2 = o2 >> 2, bs2 = (o2 & 3) * 8;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t lo_w = ws2 ? W[i + 1] : W[i], hi_w = ws2 ? W[(i + 2 < 6) ? i + 2 : 5] : W[i + 1];
            const uint32_t e2 = __funnelshift_r(lo_w, hi_w, bs2);
            const int rel = (int)c - 4 * i;                          // bytes of this word taken before the break
            const uint32_t m = rel <= 0 ? 0xffffffffu : (rel >= 4 ? 0u : (0xffffffffu << (8 * rel)));
            V[i] = (V[i] & ~m) | (e2 & m);
        }
    }
    // conservative layout check: every kept byte must be a letter-range byte (>= 0x40, < 0x80); anything else --
    // which includes the strippable 10 / 13 / 32 -- sends the query to the general strip path
    const uint32_t all = V[0] & V[1] & V[2] & V[3], hi = V[0] | V[1] | V[2] | V[3];
    ok = ok && (all & 0x40404040u) == 0x40404040u && (hi & 0x80808080u) == 0u;
    xform16(V, upper, comp, s_lut);
    if (rev) {
        o[0] = __byte_perm(V[3], 0, 0x0123); o[1] = __byte_perm(V[2], 0, 0x0123);
        o[2] = __byte_perm(V[1], 0, 0x0123); o[3] = __byte_perm(V[0], 0, 0x0123);
    } else { o[0] = V[0]; o[1] = V[1]; o[2] = V[2]; o[3] = V[3]; }
    return ok;
}

// ---- bulk-copy pull path: the covering source range of every 1 KiB output piece travels global -> shared memory
//      as ONE 1-D TMA bulk copy (cp.async.bulk, completion counted on an mbarrier), several pieces in flight per warp ----
// Assembling output words from global loads makes the L1 data pipe the limiter (six 4-byte loads per 16 output bytes,
// each touching a different cache line per query), not DRAM (DESIGN.md section 4).  Here the file bytes
// never pass through the load/store unit as global loads: the TMA engine writes them to shared memory, every lane
// assembles its aligned 16-byte output words from three 8-byte shared-memory loads, and a warp's stores are 512
// contiguous bytes.
//   * a warp owns a batch of `bq` queries (one per lane: descriptor + index row in registers, the constants the
//     consumers need in shared memory);
//   * a query is cut into items of BK_WORDS aligned output words; the items of the batch are enumerated in order by
//     two warp-uniform cursors (issue / consume) and run through a ring of BK_NS slots per warp: the lane that owns the
//     query computes the covering, 16-byte aligned source range (slice formula, sequence.c:498-510) and issues the
//     bulk copy; all lanes consume;
//   * the layout assumption is verified on every word (every kept byte in 0x40..0x7f, '\r' where a CRLF break is
//     expected); failures and queries that do not qualify (norm = 0, odd lines, < 16 bytes, RAW ...) are redone by
//     serve_query_warp (the per-warp pull path, else the general strip path), one query per warp at a time.
#ifndef FXG_BK_NS
#define FXG_BK_NS 4
#endif
constexpr int BK_NS = FXG_BK_NS;               // slots (items in flight) per warp
constexpr int BK_WORDS = 64;                   // aligned 16-byte output words per item
constexpr int BK_OUT = BK_WORDS * 16;          // output bytes per item
constexpr int BK_SLOT = 1280;                  // >= BK_OUT + 16 (ragged-word reach) + 2 * ((BK_OUT + 16) / 16 + 2) + 30 + 32
constexpr size_t BK_OFF_BAR = (size_t)XWARPS * BK_NS * BK_SLOT;
constexpr size_t BK_OFF_G0 = BK_OFF_BAR + (size_t)XWARPS * BK_NS * 8;
constexpr size_t BK_OFF_QC = (BK_OFF_G0 + (size_t)XWARPS * BK_NS * 4 + 15) & ~(size_t)15;
constexpr size_t BK_OFF_LUT = BK_OFF_QC + (size_t)XWARPS * 32 * 32;
constexpr size_t BK_OFF_STAGE = BK_OFF_LUT + 3 * 256;
constexpr size_t BK_SMEM = BK_OFF_STAGE + (size_t)XWARPS * XSTAGE;

__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}

template <bool WANT_ACGT>
__global__ void __launch_bounds__(XTHREADS, 3) extract_bulk_kernel(
    const uint8_t *__restrict__ file, int64_t fsize, int64_t capacity, const fxg_fasta_row *__restrict__ rows,
    int64_t n_rows, const int64_t *__restrict__ q_row, const int64_t *__restrict__ q_s,
    const int64_t *__restrict__ q_e, const int32_t *__restrict__ q_flags, int64_t nq,
    const int64_t *__restrict__ out_off, uint8_t *__restrict__ out, int64_t *__restrict__ acgt, int bq) {
    extern __shared__ __align__(128) uint8_t bk_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *slots = bk_smem + (size_t)warp * BK_NS * BK_SLOT;
    uint64_t *bars = reinterpret_cast<uint64_t *>(bk_smem + BK_OFF_BAR) + warp * BK_NS;
    int *g0s = reinterpret_cast<int *>(bk_smem + BK_OFF_G0) + warp * BK_NS;
    uint4 *qc = reinterpret_cast<uint4 *>(bk_smem + BK_OFF_QC) + warp * 64;          // two uint4 per lane
    uint8_t (*s_lut)[256] = reinterpret_cast<uint8_t (*)[256]>(bk_smem + BK_OFF_LUT);
    uint8_t *stage = bk_smem + BK_OFF_STAGE + (size_t)warp * XSTAGE;
    init_luts(s_lut);
    if (lane < BK_NS) mbar_init(&bars[lane], 1);
    mbar_fence_init();
    __syncthreads();
    uint32_t it_issue = 0, it_cons = 0;                     // items issued / consumed by this warp since the launch
    const int64_t step = (int64_t)gridDim.x * XWARPS * bq;
    for (int64_t qb = ((int64_t)blockIdx.x * XWARPS + warp) * bq; qb < nq; qb += step) {
        const int64_t q = qb + lane;
        const bool valid = lane < bq && q < nq;
        int64_t rid = -1, s = 0, e = 0, off = 0;
        int flags = 0;
        if (valid) { rid = q_row[q]; s = q_s[q]; e = q_e[q]; off = out_off[q]; flags = q_flags ? q_flags[q] : 0; }
        const bool row_ok = rid >= 0 && rid < n_rows;
        union RowU { fxg_fasta_row r; uint4 v[3]; } ru;
        ru.v[0] = ru.v[1] = ru.v[2] = make_uint4(0, 0, 0, 0);
        if (row_ok) {
            const uint4 *p4 = reinterpret_cast<const uint4 *>(rows + rid);
            ru.v[0] = p4[0]; ru.v[1] = p4[1]; ru.v[2] = p4[2];
        }
        const fxg_fasta_row &r = ru.r;
        const int64_t out_len64 = e > s ? e - s : 0;
        const int64_t bpl64 = r.llen - (int64_t)r.elen;
        const bool fast = row_ok && out_len64 >= 16 && out_len64 < (1ll << 30) && r.norm && (r.pad[0] & 1) != 0 &&
                          bpl64 >= 16 && bpl64 < (1ll << 30) && s >= 0 && s < (1ll << 32) && e <= r.slen &&
                          r.boff >= 0 && r.boff + r.blen + 32 <= capacity && !(flags & FXG_X_RAW);
        // per-lane constants of the lane's own query
        uint32_t bpl = 16, out_len = 0, rem_s = 0, inv = 0, pk = 0;
        const uint8_t *fq = file;
        uint8_t *dst0 = out;
        int np = 0;
        if (fast) {
            bpl = (uint32_t)bpl64; out_len = (uint32_t)out_len64;
            const uint32_t q_s32 = (uint32_t)s / bpl;
            rem_s = (uint32_t)s - q_s32 * bpl;
            inv = (uint32_t)(0x100000000ull / bpl);
            fq = file + r.boff + s + (int64_t)r.elen * (int64_t)q_s32;
            uint8_t *dst = out + off;
            const uint32_t a = (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15);
            dst0 = dst - a;
            pk = a | ((uint32_t)r.elen << 4) | ((flags & FXG_X_REVERSE) ? 0x100u : 0u) | ((flags & FXG_X_UPPER) ? 0x200u : 0u) |
                 ((flags & FXG_X_COMPLEMENT) ? 0x400u : 0u);
            // items cover the FULL aligned output words only; a ragged first / last word is written by the batch epilogue
            const uint32_t tot = a + out_len;
            const uint32_t nfull = ((tot + 15u) >> 4) - (a ? 1u : 0u) - ((tot & 15u) ? 1u : 0u);
            np = (int)((nfull + BK_WORDS - 1) / BK_WORDS);
        }
        // source range of one item of the lane's own query: (offset of the 16-byte aligned start relative to fq, bytes)
        auto item_range = [&](int p, int &g0, uint32_t &bytes) {
            const int a = (int)(pk & 15u), elen = (int)((pk >> 4) & 15u);
            const int tot = a + (int)out_len;
            const int olo = (p * BK_WORDS + (a ? 1 : 0)) * 16 - a;                // output bytes of the item's full words
            int ohi = olo + BK_OUT;
            const int oend = (tot & ~15) - a;
            if (ohi > oend) ohi = oend;
            const bool rev = (pk & 0x100u) != 0;
            const uint32_t ra = rev ? out_len - (uint32_t)ohi : (uint32_t)olo;
            const uint32_t rb1 = (rev ? out_len - (uint32_t)olo : (uint32_t)ohi) - 1u;          // last kept rank of the item
            uint32_t t1 = rem_s + ra, d1 = __umulhi(t1, inv);
            if (t1 - d1 * bpl >= bpl) ++d1;
            uint32_t t2 = rem_s + rb1, d2 = __umulhi(t2, inv);
            if (t2 - d2 * bpl >= bpl) ++d2;
            // rel2 also covers the byte after the last kept one: the '\r' of a break that follows the item's last word
            const int rel1 = (int)(ra + (uint32_t)elen * d1), rel2 = (int)(rb1 + (uint32_t)elen * d2) + (elen == 2 ? 2 : 1);
            const int fqa = (int)(reinterpret_cast<uintptr_t>(fq) & 15);
            g0 = rel1 - ((fqa + rel1) & 15);
            const int g1 = rel2 + ((16 - ((fqa + rel2) & 15)) & 15);
            bytes = (uint32_t)(g1 - g0);
            if (bytes > (uint32_t)(BK_SLOT - 32)) bytes = (uint32_t)(BK_SLOT - 32);             // cannot happen (BK_SLOT bound)
        };
        int g0_first = 0;
        uint32_t bytes_first = 16;
        if (np > 0) item_range(0, g0_first, bytes_first);        // all lanes at once: most queries are a single item
        __syncwarp();                                        // the previous batch's consumers are done with qc
        qc[2 * lane] = make_uint4(bpl, inv, rem_s, out_len);
        qc[2 * lane + 1] = make_uint4(pk, (uint32_t)np, (uint32_t)reinterpret_cast<uintptr_t>(dst0),
                                      (uint32_t)(reinterpret_cast<uintptr_t>(dst0) >> 32));
        const uint32_t nz = __ballot_sync(0xffffffffu, np > 0);        // lanes whose query runs through the ring
        __syncwarp();
        uint32_t badmask = 0;
        // cursors over the batch's items (warp-uniform): lane (= query) and item index within the query
        int ji = nz ? __ffs(nz) - 1 : 32, pi = 0;              // next item to issue
        int jc = ji, pc = 0;                                    // next item to consume

        auto issue = [&]() {                                    // issues item (ji, pi) and advances the cursor
            const int slot = (int)(it_issue % BK_NS);
            if (lane == ji) {
                int g0 = g0_first;
                uint32_t bytes = bytes_first;
                if (pi > 0) item_range(pi, g0, bytes);
                g0s[slot] = g0;
                mbar_expect_tx(&bars[slot], bytes);
                tma_load_1d(slots + (size_t)slot * BK_SLOT, fq + g0, bytes, &bars[slot]);
            }
            ++it_issue;
            const int np_i = __shfl_sync(0xffffffffu, np, ji & 31);
            if (pi + 1 < np_i) ++pi;
            else {
                const uint32_t rest = ji < 31 ? nz & (0xffffffffu << (ji + 1)) : 0u;
                ji = rest ? __ffs(rest) - 1 : 32;
                pi = 0;
            }
        };

        for (int k = 0; k < BK_NS && ji < 32; ++k) issue();
        __syncwarp();
        int cntA = 0, cntC = 0, cntG = 0, cntT = 0;
        while (jc < 32) {
            const int slot = (int)(it_cons % BK_NS);
            const uint32_t parity = (it_cons / BK_NS) & 1u;
            ++it_cons;
            {
                uint32_t spins = 0;
                while (!mbar_try_wait(&bars[slot], parity))
                    if (++spins > (1u << 22)) __trap();      // a lost completion must not hang the device
            }
            const int base_rel = g0s[slot];
            const uint4 qa = qc[2 * jc], qd = qc[2 * jc + 1];
            const uint32_t j_bpl = qa.x, j_inv = qa.y, j_rem = qa.z, j_len = qa.w, j_pk = qd.x;
            const int j_np = (int)qd.y;
            uint8_t *j_dst0 = reinterpret_cast<uint8_t *>((uintptr_t)qd.z | ((uintptr_t)qd.w << 32));
            const uint32_t a = j_pk & 15u;
            const int elen = (int)((j_pk >> 4) & 15u);
            const bool rev = (j_pk & 0x100u) != 0, upper = (j_pk & 0x200u) != 0, comp = (j_pk & 0x400u) != 0;
            const uint32_t w_beg = a ? 1u : 0u, w_end = (a + j_len) >> 4;          // the query's full words [w_beg, w_end)
            const int lenm16 = (int)j_len - 16;
            const uint8_t *sl = slots + (size_t)slot * BK_SLOT;
            bool bad = false;
#pragma unroll
            for (int k = 0; k < BK_WORDS / 32; ++k) {
                const uint32_t w = w_beg + (uint32_t)pc * BK_WORDS + (uint32_t)lane + 32u * k;
                if (w < w_end) {
                    const int j0 = (int)(16u * w) - (int)a;                             // first output byte of the word
                    const uint32_t rk = (uint32_t)(rev ? lenm16 - j0 : j0);          // first kept rank (source order)
                    const uint32_t tt = j_rem + rk;
                    uint32_t dq = __umulhi(tt, j_inv);
                    uint32_t rr = tt - dq * j_bpl;
                    if (rr >= j_bpl) { ++dq; rr -= j_bpl; }
                    const uint32_t c = j_bpl - rr;                                    // bytes left on this source line
                    const int soff = (int)(rk + (uint32_t)elen * dq) - base_rel;    // position in the slot
                    // five 4-byte shared-memory loads from the 4-byte aligned position (the select network that 8- or 16-byte
                    // loads need costs ALU-pipe instructions, and the ALU pipe is what limits this kernel)
                    const uint32_t *cp = reinterpret_cast<const uint32_t *>(sl + (soff & ~3));
                    const int sh = (soff & 3) * 8;
                    const uint32_t y0 = cp[0], y1 = cp[1], y2 = cp[2], y3 = cp[3], y4 = cp[4];
                    uint32_t V[4] = {__funnelshift_r(y0, y1, sh), __funnelshift_r(y1, y2, sh), __funnelshift_r(y2, y3, sh),
                                     __funnelshift_r(y3, y4, sh)};
                    bool ok = true;
                    if (c < 16u) {                                                    // one line break inside the word
                        uint32_t y5 = 0u;
                        if (elen == 2) {
                            if (sh == 24) y5 = cp[5];
                            const uint32_t vw = c < 8u ? (c < 4u ? V[0] : V[1]) : (c < 12u ? V[2] : V[3]);
                            ok = ((vw >> (8 * (c & 3u))) & 0xffu) == 0x0du;           // the first skipped byte must be '\r'
                        }
                        const uint32_t v4 = __funnelshift_r(y4, y5, sh);
                        const int es = 8 * elen;
                        const uint32_t E[4] = {__funnelshift_r(V[0], V[1], es), __funnelshift_r(V[1], V[2], es),
                                               __funnelshift_r(V[2], V[3], es), __funnelshift_r(V[3], v4, es)};
                        const int c8 = 8 * (int)c;
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            // bytes of word i at or after the break come from E: mask = ~0 << 8 * clamp(c - 4 i, 0, 4)
                            const uint32_t m = __funnelshift_lc(0u, 0xffffffffu, max(c8 - 32 * i, 0));
                            V[i] = (V[i] & ~m) | (E[i] & m);
                        }
                    } else if (c == 16u && elen == 2) {
                        // a break right after the word, between two words: its '\r' is byte 16, in the slot (item_range)
                        ok = ((y4 >> sh) & 0xffu) == 0x0du;
                    }
                    // conservative layout check: every kept byte must lie in 0x40..0x7f (letters)
                    const uint32_t all = V[0] & V[1] & V[2] & V[3], hi = V[0] | V[1] | V[2] | V[3];
                    if (((~all & 0x40404040u) | (hi & 0x80808080u)) != 0u || !ok) bad = true;
                    xform16(V, upper, comp, s_lut);
                    uint32_t o[4];
                    if (rev) {
                        o[0] = __byte_perm(V[3], 0, 0x0123); o[1] = __byte_perm(V[2], 0, 0x0123);
                        o[2] = __byte_perm(V[1], 0, 0x0123); o[3] = __byte_perm(V[0], 0, 0x0123);
                    } else { o[0] = V[0]; o[1] = V[1]; o[2] = V[2]; o[3] = V[3]; }
                    *reinterpret_cast<uint4 *>(j_dst0 + 16u * w) = make_uint4(o[0], o[1], o[2], o[3]);
                    if (WANT_ACGT) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            cntA += count_letter(o[i], 0x61616161u, 0x80808080u);
                            cntC += count_letter(o[i], 0x63636363u, 0x80808080u);
                            cntG += count_letter(o[i], 0x67676767u, 0x80808080u);
                            cntT += count_letter(o[i], 0x74747474u, 0x80808080u);
                        }
                    }
                }
            }
            if (bad) badmask |= 1u << jc;                       // per lane; OR-reduced after the batch
            const bool last_item = pc + 1 >= j_np;
            if (WANT_ACGT && last_item) {                      // last item of the query: its counts
#pragma unroll
                for (int dd = 16; dd > 0; dd >>= 1) {
                    cntA += __shfl_down_sync(0xffffffffu, cntA, dd);
                    cntC += __shfl_down_sync(0xffffffffu, cntC, dd);
                    cntG += __shfl_down_sync(0xffffffffu, cntG, dd);
                    cntT += __shfl_down_sync(0xffffffffu, cntT, dd);
                }
                if (lane == 0) {
                    int64_t *aq = acgt + 4 * (qb + jc);
                    aq[0] = cntA; aq[1] = cntC; aq[2] = cntG; aq[3] = cntT;
                }
                cntA = cntC = cntG = cntT = 0;
            }
            if (!last_item) ++pc;
            else {
                const uint32_t rest = jc < 31 ? nz & (0xffffffffu << (jc + 1)) : 0u;
                jc = rest ? __ffs(rest) - 1 : 32;
                pc = 0;
            }
            __syncwarp();                                      // every lane is done with the slot
            if (ji < 32) issue();
        }
        // batch epilogue: every lane writes the ragged first / last word of its OWN query (at most 15 bytes each) from
        // the nearest complete 16 output bytes, read with plain loads (the sectors are in L2: the items just fetched them)
        {
            bool mybad = false;
            int rA = 0, rC = 0, rG = 0, rT = 0;
            if (fast) {
                const uint32_t a = pk & 15u;
                const int elen = (int)((pk >> 4) & 15u);
                const bool rev = (pk & 0x100u) != 0, upper = (pk & 0x200u) != 0, comp = (pk & 0x400u) != 0;
                const uint32_t total = a + out_len, hi_last = total & 15u, nwords = (total + 15u) >> 4;
#pragma unroll 1
                for (int side = 0; side < 2; ++side) {
                    const bool first = side == 0;
                    if (first ? a == 0u : hi_last == 0u) continue;
                    uint32_t o[4], WE[6];
                    const WordReq re = ow_locate(fq, rem_s, bpl, inv, elen, out_len, rev, first ? 0u : out_len - 16u);
                    ow_load(re, WE);
                    if (!ow_finish(WE, re, elen, rev, upper, comp, s_lut, o)) mybad = true;
                    uint64_t lo = (uint64_t)o[0] | ((uint64_t)o[1] << 32), hi2 = (uint64_t)o[2] | ((uint64_t)o[3] << 32);
                    uint32_t b_lo, b_hi;                                     // slots [b_lo, b_hi) of the word are ours
                    uint8_t *gw;
                    if (first) {
                        const uint32_t s8 = 8u * a;                          // outputs 0.. move up to slot a
                        if (s8 < 64u) { hi2 = (hi2 << s8) | (lo >> (64u - s8)); lo <<= s8; } else { hi2 = lo << (s8 - 64u); lo = 0; }
                        b_lo = a; b_hi = 16u; gw = dst0;
                    } else {
                        const uint32_t s8 = 8u * (16u - hi_last);            // the last hi_last outputs move down to slot 0
                        if (s8 < 64u) { lo = (lo >> s8) | (hi2 << (64u - s8)); hi2 >>= s8; } else { lo = hi2 >> (s8 - 64u); hi2 = 0; }
                        b_lo = 0u; b_hi = hi_last; gw = dst0 + 16u * (nwords - 1u);
                    }
                    const uint32_t x[4] = {(uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi2, (uint32_t)(hi2 >> 32)};
#pragma unroll
                    for (uint32_t i = 0; i < 4; ++i) {
                        const uint32_t b0 = 4u * i;
                        uint32_t vm = 0;
                        if (b_lo <= b0 && b0 + 4u <= b_hi) { *reinterpret_cast<uint32_t *>(gw + b0) = x[i]; vm = 0x80808080u; }
                        else {
#pragma unroll
                            for (uint32_t b = 0; b < 4; ++b)
                                if (b0 + b >= b_lo && b0 + b < b_hi) { gw[b0 + b] = (uint8_t)(x[i] >> (8u * b)); vm |= 0x80u << (8u * b); }
                        }
                        if (WANT_ACGT) {
                            rA += count_letter(x[i], 0x61616161u, vm);
                            rC += count_letter(x[i], 0x63636363u, vm);
                            rG += count_letter(x[i], 0x67676767u, vm);
                            rT += count_letter(x[i], 0x74747474u, vm);
                        }
                    }
                }
                if (WANT_ACGT) {                                     // the items' lane 0 wrote the full words' counts (np > 0)
                    int64_t *aq = acgt + 4 * q;
                    if (np > 0) { aq[0] += rA; aq[1] += rC; aq[2] += rG; aq[3] += rT; }
                    else { aq[0] = rA; aq[1] = rC; aq[2] = rG; aq[3] = rT; }
                }
            }
            badmask = __reduce_or_sync(0xffffffffu, badmask) | __ballot_sync(0xffffffffu, mybad);
        }
        // queries the bulk path could not serve (or that failed its layout check): whole warp, one at a time
        uint32_t fb = __ballot_sync(0xffffffffu, valid && (!fast || ((badmask >> lane) & 1u)) && (out_len64 > 0 || WANT_ACGT));
        while (fb) {
            const int src = __ffs(fb) - 1;
            fb &= fb - 1;
            const int64_t b_rid = shfl_i64(rid, src), b_s = shfl_i64(s, src), b_e = shfl_i64(e, src), b_off = shfl_i64(off, src);
            const int b_flags = __shfl_sync(0xffffffffu, flags, src);
            const bool b_ok = b_rid >= 0 && b_rid < n_rows;
            RowU bu;
            bu.v[0] = bu.v[1] = bu.v[2] = make_uint4(0, 0, 0, 0);
            if (b_ok) {
                const uint4 *p4 = reinterpret_cast<const uint4 *>(rows + b_rid);
                bu.v[0] = p4[0]; bu.v[1] = p4[1]; bu.v[2] = p4[2];
            }
            serve_query_warp<WANT_ACGT>(file, fsize, capacity, bu.r, b_ok, b_s, b_e, b_flags, out + b_off, s_lut, stage, lane,
                                        WANT_ACGT ? acgt + 4 * (qb + src) : nullptr);
            __syncwarp();
        }
    }
}

// ---- one query, ONE launch, ONE synchronisation: what a per-object getter (Sequence.seq, .antisense, ...) costs ----
// The query's output range is cut into `chunk`-byte pieces, one per warp; a piece of a query is itself a query, exact
// for records with uniform lines (the slice formula) -- any other record is served whole by warp 0.  The output goes
// straight to mapped pinned host memory (or to device scratch for long sequences).
__global__ void __launch_bounds__(XTHREADS) extract_one_kernel(
    const uint8_t *__restrict__ file, int64_t fsize, int64_t capacity, const fxg_fasta_row *__restrict__ rows,
    int64_t n_rows, int64_t rid, int64_t s, int64_t e, int flags, int64_t chunk, uint8_t *__restrict__ out) {
    __shared__ uint8_t s_lut[3][256];
    __shared__ __align__(16) uint8_t s_stage[XWARPS][XSTAGE];
    init_luts(s_lut);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool row_ok = rid >= 0 && rid < n_rows;
    fxg_fasta_row r;
    memset(&r, 0, sizeof(r));
    if (row_ok) r = rows[rid];
    const int64_t gw = (int64_t)blockIdx.x * XWARPS + warp;
    const bool splittable = row_ok && r.norm && (r.pad[0] & 1) != 0 && !(flags & FXG_X_RAW);
    int64_t ss = s, ee = e;
    if (splittable) { ss = s + gw * chunk; ee = ss + chunk < e ? ss + chunk : e; }
    else if (gw != 0) return;
    if (ss >= ee) return;
    const int64_t ooff = (flags & FXG_X_REVERSE) ? e - ee : ss - s;      // reversed strands fill the output back to front
    serve_query_warp<false>(file, fsize, capacity, r, row_ok, ss, ee, flags, out + ooff, s_lut, s_stage[warp], lane, nullptr);
}

// K5: FASTQ reads: raw copies of rlen bytes at soff (sequence) and qoff (quality)
// ---- single-query SERVICE: a resident one-CTA kernel that is handed queries through mapped host memory ----
// `fa[name][s:e].seq` is one query per Python call; as a kernel launch plus a stream synchronisation it costs several
// times the query's work in driver round trips.
// While a caller keeps asking, this kernel stays resident instead: warp 0 polls a 128-byte request block in mapped pinned
// host memory (ONE coalesced 128-byte read per poll), the CTA serves the query exactly like extract_one_kernel, the bytes go
// straight to mapped host memory, a system-wide fence and a sequence number tell the spinning host thread that they are
// there.  No launch, no stream synchronisation, no driver call on the path.  The kernel leaves by itself after
// FXG_SVC_IDLE_CYCLES without a request (and whenever the host sets `stop`), so it never holds the device for longer
// than that: device-wide synchronisations (cudaFree ...) elsewhere in the process wait at most one idle period.
// Request block (two 64-byte halves; a PCIe read may complete them separately): the host writes the second half with
// `tail` last, then the first half with `head` last; the request is valid when head == tail == the expected number.
struct __align__(128) OneRequest {
    unsigned long long head;          // half A
    const uint8_t *file; long long fsize, capacity; const fxg_fasta_row *rows; long long n_rows, rid, s;
    long long e;                      // half B
    int flags, stop;
    long long pad[5];
    unsigned long long tail;
};
static_assert(sizeof(OneRequest) == 128, "OneRequest layout");
#ifndef FXG_SVC_IDLE_CYCLES
#define FXG_SVC_IDLE_CYCLES 4000000ll      // ~2 ms at 1.9 GHz
#endif

__global__ void __launch_bounds__(XTHREADS) extract_service_kernel(const OneRequest *req, volatile unsigned long long *resp,
                                                                    unsigned long long next_seq, uint8_t *__restrict__ out) {
    __shared__ uint8_t s_lut[3][256];
    __shared__ __align__(16) uint8_t s_stage[XWARPS][XSTAGE];
    __shared__ __align__(16) uint32_t s_req[32];
    __shared__ int s_go;
    init_luts(s_lut);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (;;) {
        if (warp == 0) {
            const long long t0 = clock64();
            int go = 0;
            for (;;) {
                uint32_t w;
                asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(w) : "l"(reinterpret_cast<const uint32_t *>(req) + lane) : "memory");
                const unsigned long long head = (unsigned long long)__shfl_sync(0xffffffffu, w, 0) | ((unsigned long long)__shfl_sync(0xffffffffu, w, 1) << 32);
                const unsigned long long tail = (unsigned long long)__shfl_sync(0xffffffffu, w, 30) | ((unsigned long long)__shfl_sync(0xffffffffu, w, 31) << 32);
                const int stop = (int)__shfl_sync(0xffffffffu, w, 19);
                if (head == next_seq && tail == next_seq) { s_req[lane] = w; go = 1; break; }
                if (stop || clock64() - t0 > FXG_SVC_IDLE_CYCLES) break;
            }
            if (lane == 0) s_go = go;
        }
        __syncthreads();
        if (!s_go) return;
        const OneRequest *q = reinterpret_cast<const OneRequest *>(s_req);
        const uint8_t *file = q->file;
        const int64_t fsize = q->fsize, capacity = q->capacity, n_rows = q->n_rows, rid = q->rid, s = q->s, e = q->e;
        const fxg_fasta_row *rows = q->rows;
        const int flags = q->flags;
        if (q->pad[0] == 1) {
            // a FASTQ read: rows are fxg_fastq_row, rid = read id, s = 0 (sequence) / 1 (quality) -- read_one_kernel's job
            if (warp == 0 && rid >= 0 && rid < n_rows) {
                const fxg_fastq_row rr = reinterpret_cast<const fxg_fastq_row *>(rows)[rid];
                if (rr.rlen > 0) {
                    const int which = (int)s;
                    GatherJob job;
                    job.skip = 0; job.src_len = rr.rlen; job.out_len = rr.rlen;
                    job.src = which ? rr.qoff : rr.soff;
                    job.dst = out;
                    job.flags = (which ? (flags & FXG_X_REVERSE) : flags) | FXG_X_RAW;      // qualities are never complemented
                    const bool fastr = rr.rlen < (1ll << 30) && job.src >= 0 && job.src + rr.rlen + 32 <= capacity;
                    if (!fastr || !pull_one<false>(file, job.src, 0, rr.rlen, 1u << 30, 1, job.flags, job.dst, s_lut, lane, nullptr))
                        gather_one<false>(file, fsize, job, s_lut[0], s_stage[0], lane, nullptr);
                }
            }
            __threadfence_system();
            __syncthreads();
            if (threadIdx.x == 0) { *resp = next_seq; __threadfence_system(); }
            ++next_seq;
            continue;
        }
        const bool row_ok = rid >= 0 && rid < n_rows;
        fxg_fasta_row r;
        memset(&r, 0, sizeof(r));
        if (row_ok) r = rows[rid];
        const int64_t len = e - s;
        int64_t warps = (len + 2047) / 2048;
        if (warps > XWARPS) warps = XWARPS;
        const int64_t chunk = ((len + warps - 1) / warps + 15) & ~(int64_t)15;
        const bool splittable = row_ok && r.norm && (r.pad[0] & 1) != 0 && !(flags & FXG_X_RAW);
        int64_t ss = s, ee = e;
        bool mine = true;
        if (splittable) { ss = s + warp * chunk; ee = ss + chunk < e ? ss + chunk : e; }
        else if (warp != 0) mine = false;
        if (mine && ss < ee) {
            const int64_t ooff = (flags & FXG_X_REVERSE) ? e - ee : ss - s;
            serve_query_warp<false>(file, fsize, capacity, r, row_ok, ss, ee, flags, out + ooff, s_lut, s_stage[warp], lane, nullptr);
        }
        __threadfence_system();                     // the output bytes are in host memory before the number is
        __syncthreads();
        if (threadIdx.x == 0) { *resp = next_seq; __threadfence_system(); }
        ++next_seq;
    }
}

__global__ void __launch_bounds__(XTHREADS) reads_kernel(
    const uint8_t *__restrict__ file, int64_t fsize, int64_t capacity, const fxg_fastq_row *__restrict__ rows,
    int64_t n_rows, const int64_t *__restrict__ ids, int64_t nq, int flags, const int64_t *__restrict__ out_off,
    uint8_t *__restrict__ seq_out, uint8_t *__restrict__ qual_out) {
    __shared__ uint8_t s_lut[3][256];
    __shared__ __align__(16) uint8_t s_stage[XWARPS][XSTAGE];
    init_luts(s_lut);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t nwarps = (int64_t)gridDim.x * XWARPS;
    for (int64_t q = (int64_t)blockIdx.x * XWARPS + warp; q < nq; q += nwarps) {
        const int64_t id = ids[q];
        if (id < 0 || id >= n_rows) continue;
        const fxg_fastq_row r = rows[id];
        if (r.rlen <= 0 || r.soff < 0 || r.qoff < 0 || r.soff > fsize || r.qoff > fsize) continue;   // untrusted rows (loaded .fxi)
        const bool fast = r.rlen < (1ll << 30) && r.soff + r.rlen + 32 <= capacity && r.qoff + r.rlen + 32 <= capacity &&
                          r.soff >= 0 && r.qoff >= 0;
        GatherJob job;
        job.skip = 0; job.src_len = r.rlen; job.out_len = r.rlen;
        if (seq_out) {
            job.src = r.soff; job.dst = seq_out + out_off[q]; job.flags = flags | FXG_X_RAW;
            if (!fast || !pull_one<false>(file, r.soff, 0, r.rlen, 1u << 30, 1, job.flags, job.dst, s_lut, lane, nullptr))
                gather_one<false>(file, fsize, job, s_lut[0], s_stage[warp], lane, nullptr);
        }
        if (qual_out) {
            job.src = r.qoff; job.dst = qual_out + out_off[q];
            job.flags = (flags & FXG_X_REVERSE) | FXG_X_RAW;      // qualities are never complemented
            if (!fast || !pull_one<false>(file, r.qoff, 0, r.rlen, 1u << 30, 1, job.flags, job.dst, s_lut, lane, nullptr))
                gather_one<false>(file, fsize, job, s_lut[0], s_stage[warp], lane, nullptr);
        }
    }
}

// one FASTQ read, one launch: sequence (which = 0) or quality (which = 1) bytes of read `id` (src/read.c:37-45,152-249)
__global__ void __launch_bounds__(32) read_one_kernel(const uint8_t *__restrict__ file, int64_t fsize, int64_t capacity,
                                                      const fxg_fastq_row *__restrict__ rows, int64_t n_rows, int64_t id,
                                                      int which, int flags, uint8_t *__restrict__ out) {
    __shared__ uint8_t s_lut[3][256];
    __shared__ __align__(16) uint8_t s_stage[1][XSTAGE];
    init_luts(s_lut);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    if (id < 0 || id >= n_rows) return;
    const fxg_fastq_row r = rows[id];
    if (r.rlen <= 0) return;
    GatherJob job;
    job.skip = 0; job.src_len = r.rlen; job.out_len = r.rlen;
    job.src = which ? r.qoff : r.soff;
    job.dst = out;
    job.flags = (which ? (flags & FXG_X_REVERSE) : flags) | FXG_X_RAW;      // qualities are never complemented
    const bool fast = r.rlen < (1ll << 30) && job.src >= 0 && job.src + r.rlen + 32 <= capacity;
    if (!fast || !pull_one<false>(file, job.src, 0, r.rlen, 1u << 30, 1, job.flags, job.dst, s_lut, lane, nullptr))
        gather_one<false>(file, fsize, job, s_lut[0], s_stage[0], lane, nullptr);
}

// ---- exclusive prefix sum of lengths (3 small kernels; < 2 % of the gather traffic) -----------
constexpr int PS_ITEMS = 2048;   // per block
__global__ void ps_block_sums(const int64_t *s, const int64_t *e, const fxg_fastq_row *rows, const int64_t *ids,
                              int64_t n_rows, int64_t nq, int64_t *block_sums) {
    __shared__ int64_t red[8];
    const int64_t b0 = (int64_t)blockIdx.x * PS_ITEMS;
    int64_t acc = 0;
    for (int i = threadIdx.x; i < PS_ITEMS; i += blockDim.x) {
        const int64_t q = b0 + i;
        if (q < nq) {
            int64_t len;
            if (rows) { const int64_t id = ids[q]; len = (id >= 0 && id < n_rows) ? rows[id].rlen : 0; }
            else { len = e[q] - s[q]; }
            acc += len > 0 ? len : 0;
        }
    }
    for (int d = 16; d > 0; d >>= 1) acc += shfl_down_i64(acc, d);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t t = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
        block_sums[blockIdx.x] = t;
    }
}
__global__ void ps_scan_sums(int64_t *block_sums, int64_t nblocks, int64_t *total) {
    // single block, sequential over chunks of blockDim
    __shared__ int64_t carry;
    __shared__ int64_t wsum[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t b = 0; b < nblocks; b += blockDim.x) {
        const int64_t i = b + threadIdx.x;
        const int64_t v = i < nblocks ? block_sums[i] : 0;
        int64_t incl = v;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t o = shfl_i64(incl, lane >= d ? lane - d : lane);
            if (lane >= d) incl += o;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        int64_t wb = 0;
        for (int w = 0; w < warp; ++w) wb += wsum[w];
        const int64_t base = carry;
        if (i < nblocks) block_sums[i] = base + wb + incl - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = base + wb + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0 && total) *total = carry;
}
__global__ void ps_write_offsets(const int64_t *s, const int64_t *e, const fxg_fastq_row *rows, const int64_t *ids,
                                 int64_t n_rows, int64_t nq, const int64_t *block_sums, int64_t *out_off) {
    // each thread owns PS_ITEMS / blockDim consecutive items
    __shared__ int64_t wsum[32];
    const int per = PS_ITEMS / blockDim.x;
    const int64_t q0 = (int64_t)blockIdx.x * PS_ITEMS + (int64_t)threadIdx.x * per;
    int64_t loc[16];
    int64_t acc = 0;
    for (int i = 0; i < per; ++i) {
        const int64_t q = q0 + i;
        int64_t len = 0;
        if (q < nq) {
            if (rows) { const int64_t id = ids[q]; len = (id >= 0 && id < n_rows) ? rows[id].rlen : 0; }
            else { len = e[q] - s[q]; }
            if (len < 0) len = 0;
        }
        loc[i] = acc;
        acc += len;
    }
    int64_t incl = acc;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t o = shfl_i64(incl, lane >= d ? lane - d : lane);
        if (lane >= d) incl += o;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    int64_t wb = 0;
    for (int w = 0; w < warp; ++w) wb += wsum[w];
    const int64_t base = block_sums[blockIdx.x] + wb + incl - acc;
    for (int i = 0; i < per; ++i) {
        const int64_t q = q0 + i;
        if (q < nq) out_off[q] = base + loc[i];
    }
    if (q0 + per >= nq && q0 < nq + per) {
        // the thread that covers index nq-1 also writes out_off[nq]
        if (q0 <= nq - 1 && nq - 1 < q0 + per) out_off[nq] = base + acc;
    }
}

// per-query 256-bin histogram of the packed output (one CTA per query, 64-bit shared bins)
__global__ void hist_kernel(const uint8_t *__restrict__ out, const int64_t *__restrict__ out_off, int64_t *__restrict__ hist) {
    __shared__ unsigned long long bins[256];
    const int64_t q = blockIdx.x;
    bins[threadIdx.x] = 0;
    __syncthreads();
    const int64_t b = out_off[q], e = out_off[q + 1];
    for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) atomicAdd(&bins[out[i]], 1ull);
    __syncthreads();
    hist[q * 256 + threadIdx.x] = (int64_t)bins[threadIdx.x];
}

}  // namespace fxg

using namespace fxg;

static int prefix_lengths(fxg_ctx *ctx, const int64_t *d_s, const int64_t *d_e, const fxg_fastq_row *rows,
                          const int64_t *ids, int64_t n_rows, int64_t nq, int64_t *d_out_off, int64_t *total_host) {
    FXG_CUDA(cudaSetDevice(ctx->device));
    if (nq == 0) {
        FXG_CUDA(cudaMemsetAsync(d_out_off, 0, sizeof(int64_t), ctx->stream));
        if (total_host) *total_host = 0;
        return FXG_OK;
    }
    const int64_t nblocks = (nq + PS_ITEMS - 1) / PS_ITEMS;
    int rc = ctx->plan.reserve((size_t)(nblocks + 2) * sizeof(int64_t));
    if (rc) return rc;
    int64_t *bs = (int64_t *)ctx->plan.ptr;
    {
    FxgProfScope prof(ctx, FXG_PROF_PLAN, 3);
    ps_block_sums<<<(unsigned)nblocks, 256, 0, ctx->stream>>>(d_s, d_e, rows, ids, n_rows, nq, bs);
    ps_scan_sums<<<1, 1024, 0, ctx->stream>>>(bs, nblocks, bs + nblocks);
    ps_write_offsets<<<(unsigned)nblocks, 256, 0, ctx->stream>>>(d_s, d_e, rows, ids, n_rows, nq, bs, d_out_off);
    }
    FXG_CUDA(cudaGetLastError());
    if (total_host) {
        FXG_CUDA(cudaMemcpyAsync(total_host, bs + nblocks, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
        FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    return FXG_OK;
}

extern "C" int fxg_extract_plan_dev(fxg_ctx *ctx, const int64_t *d_s, const int64_t *d_e, int64_t nq,
                                    int64_t *d_out_off, int64_t *total_bytes) {
    FXG_CHECK_ARG(ctx && d_out_off && nq >= 0 && (nq == 0 || (d_s && d_e)), "bad arguments");
    FXG_LOCK(ctx);
    return prefix_lengths(ctx, d_s, d_e, nullptr, nullptr, 0, nq, d_out_off, total_bytes);
}

static int gather_grid(fxg_ctx *ctx, int64_t nq) {
    int64_t blocks = (nq + XWARPS - 1) / XWARPS;
    const int64_t maxb = (int64_t)ctx->sm_count * 8;
    if (blocks > maxb) blocks = maxb;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

extern "C" int fxg_extract_dev(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                               const int64_t *d_row_id, const int64_t *d_s, const int64_t *d_e,
                               const int32_t *d_flags, int64_t nq, const int64_t *d_out_off, uint8_t *d_out,
                               int64_t *d_acgt) {
    FXG_CHECK_ARG(ctx && f && nq >= 0, "bad arguments");
    FXG_LOCK(ctx);
    if (nq == 0) return FXG_OK;
    FXG_CHECK_ARG(d_rows && d_row_id && d_s && d_e && d_out_off && d_out, "null device pointer");
    FXG_CUDA(cudaSetDevice(ctx->device));
    FxgProfScope prof(ctx, FXG_PROF_GATHER);
    static int ctas_per_sm[2] = {0, 0};                     // [with counts]
    const int v = d_acgt ? 1 : 0;
    if (!ctas_per_sm[v]) {
        int nb = 0;
        if (v) {
            FXG_CUDA(cudaFuncSetAttribute(extract_bulk_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BK_SMEM));
            FXG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, extract_bulk_kernel<true>, XTHREADS, BK_SMEM));
        } else {
            FXG_CUDA(cudaFuncSetAttribute(extract_bulk_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BK_SMEM));
            FXG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, extract_bulk_kernel<false>, XTHREADS, BK_SMEM));
        }
        ctas_per_sm[v] = nb > 0 ? nb : 1;
    }
    const int64_t resident_warps = (int64_t)ctx->sm_count * ctas_per_sm[v] * XWARPS;
    // queries per warp batch: a lane per query when there is enough work to fill the machine that way
    int bq = nq >= resident_warps * 32 ? 32 : (nq >= resident_warps * 16 ? 16 : 8);
    if (const char *b = getenv("FXG_BK_BQ")) { const int v = atoi(b); if (v >= 1 && v <= 32) bq = v; }   // tests: force a batch width
    int64_t blocks = (nq + (int64_t)XWARPS * bq - 1) / ((int64_t)XWARPS * bq);
    const int64_t maxb = (int64_t)ctx->sm_count * ctas_per_sm[v];
    if (blocks > maxb) blocks = maxb;
    if (v)
        extract_bulk_kernel<true><<<(unsigned)blocks, XTHREADS, BK_SMEM, ctx->stream>>>(
            f->d, f->size, f->capacity, d_rows, n_rows, d_row_id, d_s, d_e, d_flags, nq, d_out_off, d_out, d_acgt, bq);
    else
        extract_bulk_kernel<false><<<(unsigned)blocks, XTHREADS, BK_SMEM, ctx->stream>>>(
            f->d, f->size, f->capacity, d_rows, n_rows, d_row_id, d_s, d_e, d_flags, nq, d_out_off, d_out, nullptr, bq);
    FXG_CUDA(cudaGetLastError());
    return FXG_OK;
}

extern "C" int fxg_extract_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                                const int64_t *row_id, const int64_t *s, const int64_t *e, const int32_t *flags,
                                int64_t nq, int64_t *out_off_host, uint8_t *out_host, int64_t out_cap,
                                int64_t *acgt_host) {
    FXG_CHECK_ARG(ctx && f && nq >= 0, "bad arguments");
    FXG_LOCK(ctx);
    if (nq == 0) { if (out_off_host) out_off_host[0] = 0; return FXG_OK; }
    FXG_CHECK_ARG(row_id && s && e && out_off_host && out_host, "null host pointer");
    FXG_CUDA(cudaSetDevice(ctx->device));
    const size_t qb = (size_t)nq * sizeof(int64_t);
    // device layout in ctx->misc: row_id | s | e | out_off(nq+1) | flags | acgt
    const size_t need = qb * 3 + (size_t)(nq + 1) * 8 + (size_t)nq * 4 + 16 + (acgt_host ? (size_t)nq * 32 : 0);
    int rc = ctx->misc.reserve(need + 64);
    if (rc) return rc;
    uint8_t *base = (uint8_t *)ctx->misc.ptr;
    int64_t *d_row = (int64_t *)base, *d_s = d_row + nq, *d_e = d_s + nq, *d_off = d_e + nq;
    int32_t *d_fl = (int32_t *)(d_off + nq + 1);
    int64_t *d_acgt = acgt_host ? (int64_t *)(((uintptr_t)(d_fl + nq) + 15) & ~(uintptr_t)15) : nullptr;
    FXG_CUDA(cudaMemcpyAsync(d_row, row_id, qb, cudaMemcpyHostToDevice, ctx->stream));
    FXG_CUDA(cudaMemcpyAsync(d_s, s, qb, cudaMemcpyHostToDevice, ctx->stream));
    FXG_CUDA(cudaMemcpyAsync(d_e, e, qb, cudaMemcpyHostToDevice, ctx->stream));
    if (flags) FXG_CUDA(cudaMemcpyAsync(d_fl, flags, (size_t)nq * 4, cudaMemcpyHostToDevice, ctx->stream));
    int64_t total = 0;
    rc = prefix_lengths(ctx, d_s, d_e, nullptr, nullptr, 0, nq, d_off, &total);
    if (rc) return rc;
    if (total > out_cap) { fxg_set_error("output needs %lld bytes, capacity %lld", (long long)total, (long long)out_cap); return FXG_ECAP; }
    if ((rc = ctx->row_tmp.reserve((size_t)total + 64))) return rc;
    uint8_t *d_out = (uint8_t *)ctx->row_tmp.ptr;
    rc = fxg_extract_dev(ctx, f, d_rows, n_rows, d_row, d_s, d_e, flags ? d_fl : nullptr, nq, d_off, d_out, d_acgt);
    if (rc) return rc;
    FXG_CUDA(cudaMemcpyAsync(out_off_host, d_off, (size_t)(nq + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (total) FXG_CUDA(cudaMemcpyAsync(out_host, d_out, (size_t)total, cudaMemcpyDeviceToHost, ctx->stream));
    if (acgt_host) FXG_CUDA(cudaMemcpyAsync(acgt_host, d_acgt, (size_t)nq * 32, cudaMemcpyDeviceToHost, ctx->stream));
    FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    return FXG_OK;
}

extern "C" int fxg_reads_dev(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                             const int64_t *d_ids, int64_t nq, int32_t flags, int64_t *d_out_off,
                             uint8_t *d_seq_out, uint8_t *d_qual_out, int64_t out_cap, int64_t *total_bytes) {
    FXG_CHECK_ARG(ctx && f && nq >= 0 && d_out_off, "bad arguments");
    FXG_LOCK(ctx);
    FXG_CUDA(cudaSetDevice(ctx->device));
    int64_t total = 0;
    int rc = prefix_lengths(ctx, nullptr, nullptr, d_rows, d_ids, n_rows, nq, d_out_off, &total);
    if (rc) return rc;
    if (total_bytes) *total_bytes = total;
    if (total > out_cap) { fxg_set_error("output needs %lld bytes, capacity %lld", (long long)total, (long long)out_cap); return FXG_ECAP; }
    if (nq == 0 || (!d_seq_out && !d_qual_out)) return FXG_OK;
    FxgProfScope prof(ctx, FXG_PROF_GATHER);
    reads_kernel<<<gather_grid(ctx, nq), XTHREADS, 0, ctx->stream>>>(f->d, f->size, f->capacity, d_rows, n_rows, d_ids, nq, flags,
                                                                    d_out_off, d_seq_out, d_qual_out);
    FXG_CUDA(cudaGetLastError());
    return FXG_OK;
}

extern "C" int fxg_reads_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows,
                              const int64_t *ids, int64_t nq, int32_t flags, int64_t *out_off_host,
                              uint8_t *seq_host, uint8_t *qual_host, int64_t out_cap) {
    FXG_CHECK_ARG(ctx && f && nq >= 0 && out_off_host, "bad arguments");
    FXG_LOCK(ctx);
    if (nq == 0) { out_off_host[0] = 0; return FXG_OK; }
    FXG_CUDA(cudaSetDevice(ctx->device));
    int rc = ctx->misc.reserve((size_t)nq * 8 + (size_t)(nq + 1) * 8 + 64);
    if (rc) return rc;
    int64_t *d_ids = (int64_t *)ctx->misc.ptr, *d_off = d_ids + nq;
    FXG_CUDA(cudaMemcpyAsync(d_ids, ids, (size_t)nq * 8, cudaMemcpyHostToDevice, ctx->stream));
    int64_t total = 0;
    rc = prefix_lengths(ctx, nullptr, nullptr, d_rows, d_ids, n_rows, nq, d_off, &total);
    if (rc) return rc;
    if (total > out_cap) { fxg_set_error("output needs %lld bytes, capacity %lld", (long long)total, (long long)out_cap); return FXG_ECAP; }
    if ((rc = ctx->row_tmp.reserve((size_t)total * 2 + 128))) return rc;
    uint8_t *d_seq = (uint8_t *)ctx->row_tmp.ptr;
    uint8_t *d_qual = d_seq + fxg_round_up(total + 16, 16);
    ctx->launches += 1;
    reads_kernel<<<gather_grid(ctx, nq), XTHREADS, 0, ctx->stream>>>(f->d, f->size, f->capacity, d_rows, n_rows, d_ids, nq, flags, d_off,
                                                                    seq_host ? d_seq : nullptr, qual_host ? d_qual : nullptr);
    FXG_CUDA(cudaGetLastError());
    FXG_CUDA(cudaMemcpyAsync(out_off_host, d_off, (size_t)(nq + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (seq_host && total) FXG_CUDA(cudaMemcpyAsync(seq_host, d_seq, (size_t)total, cudaMemcpyDeviceToHost, ctx->stream));
    if (qual_host && total) FXG_CUDA(cudaMemcpyAsync(qual_host, d_qual, (size_t)total, cudaMemcpyDeviceToHost, ctx->stream));
    FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    return FXG_OK;
}

extern "C" int fxg_composition_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                                    const int64_t *row_id, const int64_t *s, const int64_t *e, const int32_t *flags,
                                    int64_t nq, int64_t *hist_host) {
    FXG_CHECK_ARG(ctx && f && nq >= 0 && (nq == 0 || (row_id && s && e && hist_host)), "bad arguments");
    FXG_LOCK(ctx);
    if (nq == 0) return FXG_OK;
    FXG_CUDA(cudaSetDevice(ctx->device));
    const size_t qb = (size_t)nq * sizeof(int64_t);
    int rc = ctx->misc.reserve(qb * 3 + (size_t)(nq + 1) * 8 + (size_t)nq * 4 + 64 + (size_t)nq * 2048);
    if (rc) return rc;
    int64_t *d_row = (int64_t *)ctx->misc.ptr, *d_s = d_row + nq, *d_e = d_s + nq, *d_off = d_e + nq;
    int32_t *d_fl = (int32_t *)(d_off + nq + 1);
    int64_t *d_hist = (int64_t *)(((uintptr_t)(d_fl + nq) + 15) & ~(uintptr_t)15);
    FXG_CUDA(cudaMemcpyAsync(d_row, row_id, qb, cudaMemcpyHostToDevice, ctx->stream));
    FXG_CUDA(cudaMemcpyAsync(d_s, s, qb, cudaMemcpyHostToDevice, ctx->stream));
    FXG_CUDA(cudaMemcpyAsync(d_e, e, qb, cudaMemcpyHostToDevice, ctx->stream));
    if (flags) FXG_CUDA(cudaMemcpyAsync(d_fl, flags, (size_t)nq * 4, cudaMemcpyHostToDevice, ctx->stream));
    FXG_CUDA(cudaMemsetAsync(d_hist, 0, (size_t)nq * 2048, ctx->stream));
    int64_t total = 0;
    rc = prefix_lengths(ctx, d_s, d_e, nullptr, nullptr, 0, nq, d_off, &total);
    if (rc) return rc;
    if ((rc = ctx->row_tmp.reserve((size_t)total + 64))) return rc;
    uint8_t *d_out = (uint8_t *)ctx->row_tmp.ptr;
    rc = fxg_extract_dev(ctx, f, d_rows, n_rows, d_row, d_s, d_e, flags ? d_fl : nullptr, nq, d_off, d_out, nullptr);
    if (rc) return rc;
    ctx->launches += 1;
    hist_kernel<<<(unsigned)nq, 256, 0, ctx->stream>>>(d_out, d_off, d_hist);
    FXG_CUDA(cudaGetLastError());
    FXG_CUDA(cudaMemcpyAsync(hist_host, d_hist, (size_t)nq * 2048, cudaMemcpyDeviceToHost, ctx->stream));
    FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    return FXG_OK;
}

// ---- host side of the single-query service ----
static const int FXG_EAGAIN_INTERNAL = -1000;
static bool svc_enabled() {
    static int on = -1;
    if (on < 0) { const char *e = getenv("FXG_ONE_SERVICE"); on = (e && e[0] == '0') ? 0 : 1; }
    return on != 0;
}
// Called by fxg_ctx_destroy.  Freeing a buffer that a query named needs no stop: cudaFree, and the file pool's
// cudaDeviceSynchronize before it hands a buffer on, wait for the resident kernel, which leaves after its idle period.
void fxg_svc_stop(fxg_ctx *ctx) {
    if (!ctx->svc_req) return;
    OneRequest *rq = (OneRequest *)ctx->svc_req;
    ((volatile OneRequest *)rq)->stop = 1;
    __sync_synchronize();
    if (ctx->svc_stream) cudaStreamSynchronize(ctx->svc_stream);
    ((volatile OneRequest *)rq)->stop = 0;
    ctx->svc_running = false;
}
static int svc_launch(fxg_ctx *ctx) {
    void *d_req = nullptr, *d_resp = nullptr, *d_out = nullptr;
    FXG_CUDA(cudaHostGetDevicePointer(&d_req, ctx->svc_req, 0));
    FXG_CUDA(cudaHostGetDevicePointer(&d_resp, ctx->svc_resp, 0));
    FXG_CUDA(cudaHostGetDevicePointer(&d_out, ctx->h_one, 0));
    ctx->launches += 1;
    extract_service_kernel<<<1, XTHREADS, 0, ctx->svc_stream>>>((const OneRequest *)d_req, (volatile unsigned long long *)d_resp,
                                                                ctx->svc_next, (uint8_t *)d_out);
    FXG_CUDA(cudaGetLastError());
    ctx->svc_running = true;
    return FXG_OK;
}
static int svc_query(fxg_ctx *ctx, const fxg_file *f, const void *d_rows_any, int64_t n_rows, int64_t row_id, int64_t s,
                     int64_t e, int32_t flags, int kind = 0) {
    const fxg_fasta_row *d_rows = (const fxg_fasta_row *)d_rows_any;
    if (!ctx->svc_req) {
        if (cudaHostAlloc(&ctx->svc_req, 256, cudaHostAllocMapped) != cudaSuccess) { cudaGetLastError(); ctx->svc_req = nullptr; return FXG_EAGAIN_INTERNAL; }
        memset(ctx->svc_req, 0, 256);
        ctx->svc_resp = (uint8_t *)ctx->svc_req + 128;
        if (cudaStreamCreateWithFlags(&ctx->svc_stream, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); return FXG_EAGAIN_INTERNAL; }
        ctx->svc_next = 1;
    }
    // results of earlier work on the context's stream (staging, scan, row uploads) must be complete: every host entry point
    // that produces them synchronises before it returns (the file staging calls too, include/fxg.h), so there is nothing
    // to wait for here
    volatile OneRequest *rq = (volatile OneRequest *)ctx->svc_req;
    const unsigned long long n = ctx->svc_next;
    // second half first, `tail` last; then the first half, `head` last (x86 keeps the store order)
    rq->e = e; rq->flags = flags; rq->stop = 0; rq->pad[0] = kind;
    __sync_synchronize();
    rq->tail = n;
    __sync_synchronize();
    rq->file = f->d; rq->fsize = f->size; rq->capacity = f->capacity; rq->rows = d_rows; rq->n_rows = n_rows; rq->rid = row_id; rq->s = s;
    __sync_synchronize();
    rq->head = n;
    __sync_synchronize();
    if (!ctx->svc_running) { int rc = svc_launch(ctx); if (rc) return rc; }
    volatile unsigned long long *resp = (volatile unsigned long long *)ctx->svc_resp;
    // spin on the response word; look at the stream (a driver call) only every 100 us: that is where a kernel that
    // left after its idle period, or a failed one, is noticed
    uint32_t spins = 0;
    auto t_last = std::chrono::steady_clock::now();
    while (*resp != n) {
        if ((++spins & 255u) == 0) {
            const auto now = std::chrono::steady_clock::now();
            if (std::chrono::duration<double>(now - t_last).count() < 100e-6) continue;
            t_last = now;
            const cudaError_t q = cudaStreamQuery(ctx->svc_stream);
            if (q == cudaSuccess) {                      // the kernel left (idle period over) before it saw the request
                if (*resp == n) break;
                int rc = svc_launch(ctx);
                if (rc) return rc;
            } else if (q != cudaErrorNotReady) {
                cudaGetLastError();
                fxg_set_error("single-query service failed: %s", cudaGetErrorString(q));
                ctx->svc_running = false;
                return FXG_ECUDA;
            }
            if (spins > (1u << 28)) { fxg_set_error("single-query service timed out"); return FXG_ECUDA; }
        }
    }
    __sync_synchronize();
    ctx->svc_next = n + 1;
    return FXG_OK;
}

// One query through one kernel launch and one stream synchronisation (no plan kernels, no H2D copies: the query
// travels as kernel arguments).  Same result as fxg_extract_host with nq = 1.
extern "C" int fxg_extract_one_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fasta_row *d_rows, int64_t n_rows,
                                    int64_t row_id, int64_t s, int64_t e, int32_t flags, uint8_t *out_host, int64_t out_cap) {
    FXG_CHECK_ARG(ctx && f && d_rows && (out_host || e <= s), "bad arguments");
    FXG_LOCK(ctx);
    const int64_t len = e > s ? e - s : 0;
    if (len == 0) return FXG_OK;
    if (len > out_cap) { fxg_set_error("output needs %lld bytes, capacity %lld", (long long)len, (long long)out_cap); return FXG_ECAP; }
    FXG_CUDA(cudaSetDevice(ctx->device));
    const int64_t ONE_PINNED = 1 << 20;
    if (!ctx->h_one) FXG_CUDA(cudaHostAlloc(&ctx->h_one, (size_t)ONE_PINNED + 64, cudaHostAllocMapped));
    uint8_t *d_out;
    const bool direct = len <= ONE_PINNED;
    if (direct && svc_enabled() && len <= 65536) {
        int rc = svc_query(ctx, f, d_rows, n_rows, row_id, s, e, flags);
        if (rc == FXG_OK) { memcpy(out_host, ctx->h_one, (size_t)len); return FXG_OK; }
        if (rc != FXG_EAGAIN_INTERNAL) return rc;       // else: the service is unavailable, take the launch path
    }
    if (direct) {
        void *dp = nullptr;
        FXG_CUDA(cudaHostGetDevicePointer(&dp, ctx->h_one, 0));
        d_out = (uint8_t *)dp;
    } else {
        int rc = ctx->row_tmp.reserve((size_t)len + 64);
        if (rc) return rc;
        d_out = (uint8_t *)ctx->row_tmp.ptr;
    }
    // pieces of >= 2 KiB, multiples of 16 bytes, at most 8 warps x 4 CTAs per SM worth of them
    int64_t warps = (len + 2047) / 2048;
    const int64_t maxw = (int64_t)ctx->sm_count * 4 * XWARPS;
    if (warps > maxw) warps = maxw;
    int64_t chunk = ((len + warps - 1) / warps + 15) & ~(int64_t)15;
    warps = (len + chunk - 1) / chunk;
    const unsigned grid = (unsigned)((warps + XWARPS - 1) / XWARPS);
    {
        FxgProfScope prof(ctx, FXG_PROF_GATHER);
        extract_one_kernel<<<grid, XTHREADS, 0, ctx->stream>>>(f->d, f->size, f->capacity, d_rows, n_rows, row_id, s, e, flags, chunk, d_out);
    }
    FXG_CUDA(cudaGetLastError());
    if (!direct) FXG_CUDA(cudaMemcpyAsync(out_host, d_out, (size_t)len, cudaMemcpyDeviceToHost, ctx->stream));
    FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (direct) memcpy(out_host, ctx->h_one, (size_t)len);
    return FXG_OK;
}

// One read through one kernel launch and one stream synchronisation (the Read.seq / .qual getters).
extern "C" int fxg_read_one_host(fxg_ctx *ctx, const fxg_file *f, const fxg_fastq_row *d_rows, int64_t n_rows, int64_t read_id,
                                 int which, int32_t flags, int64_t rlen, uint8_t *out_host, int64_t out_cap) {
    FXG_CHECK_ARG(ctx && f && d_rows && (out_host || rlen <= 0), "bad arguments");
    FXG_LOCK(ctx);
    if (rlen <= 0) return FXG_OK;
    if (rlen > out_cap) { fxg_set_error("output needs %lld bytes, capacity %lld", (long long)rlen, (long long)out_cap); return FXG_ECAP; }
    FXG_CUDA(cudaSetDevice(ctx->device));
    const int64_t ONE_PINNED = 1 << 20;
    if (!ctx->h_one) FXG_CUDA(cudaHostAlloc(&ctx->h_one, (size_t)ONE_PINNED + 64, cudaHostAllocMapped));
    const bool direct = rlen <= ONE_PINNED;
    uint8_t *d_out;
    if (direct && svc_enabled() && rlen <= 65536) {
        int rc = svc_query(ctx, f, d_rows, n_rows, read_id, which ? 1 : 0, rlen, flags, 1);
        if (rc == FXG_OK) { memcpy(out_host, ctx->h_one, (size_t)rlen); return FXG_OK; }
        if (rc != FXG_EAGAIN_INTERNAL) return rc;
    }
    if (direct) {
        void *dp = nullptr;
        FXG_CUDA(cudaHostGetDevicePointer(&dp, ctx->h_one, 0));
        d_out = (uint8_t *)dp;
    } else {
        int rc = ctx->row_tmp.reserve((size_t)rlen + 64);
        if (rc) return rc;
        d_out = (uint8_t *)ctx->row_tmp.ptr;
    }
    ctx->launches += 1;
    read_one_kernel<<<1, 32, 0, ctx->stream>>>(f->d, f->size, f->capacity, d_rows, n_rows, read_id, which, flags, d_out);
    FXG_CUDA(cudaGetLastError());
    if (!direct) FXG_CUDA(cudaMemcpyAsync(out_host, d_out, (size_t)rlen, cudaMemcpyDeviceToHost, ctx->stream));
    FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (direct) memcpy(out_host, ctx->h_one, (size_t)rlen);
    return FXG_OK;
}
