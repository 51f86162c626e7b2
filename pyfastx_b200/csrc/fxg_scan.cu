// fxg_scan.cu -- K1 (FASTA) and K2 (FASTQ) index-build scans for sm_90a.
//
// Replaces the per-line loops of pyfastx_create_index (reference src/index.c:226-361) and
// pyfastx_fastq_create_index (src/fastq.c:84-171), both driven by ks_getuntil2
// (src/kseq.c:59-109).  The file bytes resident in HBM are read ONCE; everything after that
// works on compact per-region records (newline lists, FASTA line facts).
//
// Design (see DESIGN.md section 3):
//   mark    one warp per 2 KiB region, no communication between warps at all: 4 coalesced
//           16-byte loads per lane, exact SWAR newline masks (3 ALU ops per 32-bit word),
//           ballot-ranked compaction into the region's segment of the newline list
//           {position in region | '\r' before | '>' after}, plus the region's counts
//           {#newlines, #header starts}.  This kernel carries all of the file traffic and is
//           a pure stream: nothing in it waits on another CTA.
//   prefix  exclusive prefix of the region counts (small kernels over 4 bytes per region; FASTA keeps
//           block sums only).
//   rows    reads only the newline list (and the file bytes of header / read-name lines).  Every
//           quantity the reference carries from line to line is re-expressed as a local rule on
//           (this line, previous line, global line index, global header ordinal):
//             - a header line writes boff / dlen / elen / name length / its line index;
//             - a sequence line that follows a header writes llen;
//             - a sequence line whose length differs from the previous sequence line raises an
//               "event" (count, min/max line index, sum of length deltas) on its record.
//           FASTA: mark itself settles every line k >= 2 of a region that changes a record into a line
//           fact (name cut included), and writes the newline list only for general regions (more than
//           32 newlines or 3 facts).  fasta_rows_kernel scans the region counts per CTA (no per-region
//           prefix array), resolves lines 0 and 1 of each region from the region before it and applies
//           the facts; fasta_general_kernel runs the general regions from their newline list; a tiny
//           finalize kernel then derives blen, slen, norm per record from neighbouring headers and the
//           event summary (proof of equivalence with index.c:325-342 in DESIGN.md).
//           FASTQ (fastq_records_kernel): no per-record state at all, line k of the file writes
//           field k%4 of row k/4; one lane builds the whole row of a read from five consecutive
//           newline positions, and reads the name line once to find the name cut.
//           Regions the fast paths cannot settle go through full_region, lane per line.
//
// An earlier single-pass variant (TMA tile ring + decoupled look-back inside one kernel) stayed far below
// DRAM speed: every tile's shared-memory slot stayed occupied for the thousands of cycles its look-back spent
// waiting on L2 round trips.  Splitting the dependency out of the streaming kernel removes that wait.
#include "fxg_common.cuh"
#include <stdlib.h>
#include <string.h>
#include <limits.h>

namespace fxg {

#ifndef FXG_MARK_MINB
#define FXG_MARK_MINB 6
#endif
constexpr int REGION   = 2048;            // bytes per warp
constexpr int SEGCAP   = 128;             // newline-list entries kept per region (lines >= 16 B on average)
constexpr int MARK_WARPS = 8;             // warps per CTA of the mark / rows kernels
// FASTA mark: each warp prefetches into L2 the region this many regions ahead, a little more than one wave of the grid
// (132 SMs x 6 CTAs x 8 warps = 6336 regions on an H100), so the warps of the next wave find their bytes in L2
constexpr int64_t MARK_AHEAD = 8192;
constexpr int PS_THREADS = 256, PS_PER_THREAD = 16, PS_BLOCK = PS_THREADS * PS_PER_THREAD;   // regions per prefix block
constexpr int64_t NOPOS = INT64_MIN / 4;
constexpr uint32_t E_POS = 0x07ffu, E_CR = 1u << 14, E_HDR = 1u << 15;
// FASTA region record.  Every region keeps its first two entries (fw); bits 11..13 of the first entry are free and
// carry the number of line facts (FW_NF) or FW_GEN: the region is settled by full_region from its newline list.
// A line fact describes one line k >= 2 of the region that changes a record (a header, the first sequence line
// after a header, a change of line length):
//   x = newline position | k << 11 | header starts before entry k << 16 | kind << 21
//   y = LF_HDR: dlen | nlen << 11 | (elen - 1) << 22 | LF_CUT_UNKNOWN;  LF_LLEN: len + 1;  LF_EVENT: change of len
constexpr uint32_t FW_NF_SHIFT = 11, FW_NF = 3u << FW_NF_SHIFT, FW_GEN = 1u << 13;
constexpr int LF_MAX = 3, LF_STRIDE = 4;  // facts per region; uint2 slots per region (32 bytes)
constexpr uint32_t LF_HDR = 0, LF_LLEN = 1, LF_EVENT = 2, LF_CUT_UNKNOWN = 1u << 23;
constexpr uint32_t NAME_SCAN = 64;        // header bytes mark searches for the name cut

struct __align__(16) FastaTmp {   // per header slot (slot 0 = lines before the first header)
    int64_t  boff;       // header thread
    int64_t  lineidx;    // header thread: buffer-local line index of the header line
    int64_t  llen;       // first sequence line (len + 1)
    uint64_t S;          // sum of (L - prevL) over events (wrapping)
    uint64_t evmax;      // max line index of an event
    uint64_t evminc;     // max of ~lineidx  (== ~min)
    uint32_t D;          // number of events
    int32_t  dlen;
    int32_t  nlen;
    uint32_t elen;
};
static_assert(sizeof(FastaTmp) == 64, "FastaTmp layout");

struct ScanTotals {     // device, 128 bytes; every phase-B kernel reads its sizes from here (no host round trip)
    uint64_t nl;        // newlines (incl. the virtual one at n)
    uint64_t hdr;       // header starts
    int64_t  n_eff;     // n + 1 if the last line has no '\n'
    uint64_t sum_len;   // FASTA: sum(slen) (finalize); FASTQ: sum(rlen)
    int64_t  lead_lines, lead_bytes, lead_llen;
    int64_t  first_line;   // FASTQ: global index of this shard's first line (shard_prefix_kernel)
    int64_t  nrows;        // row slots phase B writes: FASTA header count; FASTQ incl. partially owned rows
    int64_t  row0;         // FASTQ: index of the first row whose name line lies in this shard (0 or 1)
    int64_t  n_owned;      // FASTQ: complete reads whose name line lies in this shard
    int64_t  total_lines;  // lines of all shards
    int64_t  pad[4];
};
static_assert(sizeof(ScanTotals) == 128, "ScanTotals layout");
static_assert(sizeof(fxg_shard_info) == 128, "fxg_shard_info layout");

struct ScanParams;
struct ScanParams {
    const uint8_t *file;
    int64_t   n;            // bytes
    int64_t   capacity;     // readable bytes at file (multiple of 16)
    int64_t   nreg;         // regions that can hold a newline: ceil((n + 1) / REGION)
    int64_t   base_offset;  // added to every file offset written to rows
    int64_t   first_line;   // FASTQ: global index of the first line of this buffer (kernels load it from totals)
    int       flags;
    uint2    *rc;           // per region: {newlines | header starts << 16, last entry | the one before << 16}
                            // (padded to PS_BLOCK with zeros)
    uint32_t *fw;           // FASTA, per region: first entry | second << 16, FW_* flags in the first (padded to PS_BLOCK)
    uint2    *lf;           // FASTA, per region: up to LF_MAX line facts (written only where FW_NF is not 0);
                            // a general region's slot holds its exclusive {newlines, header starts} instead
    uint32_t *gblk;         // FASTA, per prefix block: 1 if it has a general region (fasta_rows_kernel)
    uint16_t *seg;          // per region: SEGCAP entries, file order (FASTA: general regions only)
    ulonglong2 *ex;         // FASTQ, per region: exclusive {newlines, header starts}
    ulonglong2 *bs;         // per prefix block
    ScanTotals *totals;
    FastaTmp *tmp;          // FASTA
    int64_t   tmp_cap;      // slots
    fxg_fastq_row *qrows;   // FASTQ
    int64_t   qrows_cap;
    const ScanParams *self; // the same struct in GLOBAL memory: the rare noinline paths take this pointer -- passing the
                            // kernel parameter by reference made every thread copy all 200 bytes to its local memory
                            // (r02 ncu: 1 GB of DRAM writes per 5 GB FASTQ came from that copy alone)
};

// the REGION bytes at p (16-byte aligned) into L2, one bulk request without registers held
__device__ __forceinline__ void prefetch_l2(const uint8_t *p) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(p), "n"(REGION) : "memory");
}
__device__ __forceinline__ uint4 ld_stream16(const uint8_t *p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// =============================================================================================
// mark: newline list + counts of one 2 KiB region per warp
// =============================================================================================
// Pass 1, V = 2 (r02): every lane tests 64 CONTIGUOUS bytes.  The loads stay coalesced (lane l takes 16 bytes of each
// of the four 512-byte quarters); the region is transposed on its way through shared memory, where pass 2 needs it
// anyway: 16-byte unit u is stored at u ^ ((u >> 3) & 7), which makes both the quarter-major stores and the lane-major
// loads (units 4l .. 4l+3) bank-conflict free.  With contiguous bytes per lane the file order of the newlines is the
// lane order, so ONE pair of ballots ranks the whole region (r01: one or two ballots and a rank per quarter), and
// the per-byte flags are packed into a position-ordered 64-bit mask by integer multiply-adds -- work for the FMA pipe
// where the r01 code kept the ALU pipe busy.  V = 1 tests every 16-byte chunk where it was loaded.
// One region per warp: a warp that also had the next region's loads in flight was slower (2, 4, 8 regions at 4 or 5
// CTAs per SM for the extra registers) than one region per warp at 6 CTAs per SM.  The kernel is not bound by
// instruction issue: skipping the shared-memory copy and pass 2 for headerless regions did not make it faster
// (DESIGN.md section 3, the read floor of mark's shape).
__device__ __forceinline__ uint32_t swz_unit(uint32_t u) { return u ^ ((u >> 3) & 7u); }
// byte p (0 .. REGION-1) of a region held in swizzled (V = 2) or linear (V = 1) shared memory
template <int V>
__device__ __forceinline__ uint32_t region_byte(const uint8_t *sb, uint32_t p) {
    return V == 2 ? sb[(swz_unit(p >> 4) << 4) | (p & 15u)] : sb[p];
}

template <int MODE, int V>   // MODE: 0 = FASTA, 1 = FASTQ; V: pass-1 variant
__global__ void __launch_bounds__(MARK_WARPS * 32, FXG_MARK_MINB) mark_kernel(const ScanParams P) {
    __shared__ uint4    s_data[MARK_WARPS * (REGION / 16)];   // the regions' bytes (neighbour-byte lookups)
    __shared__ uint16_t s_ent[MARK_WARPS][SEGCAP];         // newline positions, then complete entries
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r = (int64_t)blockIdx.x * MARK_WARPS + warp;
    if (r >= P.nreg) return;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const int64_t n = P.n;
    const uint8_t *file = P.file;
    const uint32_t k0a = reg_const(0x0a0a0a0au), k7f = reg_const(0x7f7f7f7fu), k80 = reg_const(0x80808080u);
    const int64_t base = r * REGION;

    // the 2 KiB of the region: four coalesced 16-byte streaming loads per lane, all in flight together
    uint4 v[4];
    if (base + REGION <= n) {
        const uint8_t *src = file + base + lane * 16;
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = ld_stream16(src + j * 512);
        // more of the file in flight than the registers of 48 warps per SM hold, at no register cost
        if (MODE == 0 && lane == 0 && base + (MARK_AHEAD + 1) * REGION <= n) prefetch_l2(file + base + MARK_AHEAD * REGION);
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t o = base + j * 512 + lane * 16;
            if (o + 16 <= n) { v[j] = ld_stream16(file + o); continue; }
            // the chunk that contains EOF (or lies past it): bytes >= n read as 0, and a file that does
            // not end in '\n' gets a virtual newline at n (kseq returns the last line all the same)
            const bool virt = n > 0 && file[n - 1] != '\n';
            uint32_t w[4] = {0, 0, 0, 0};
            for (int i = 0; i < 16; ++i) {
                const int64_t x = o + i;
                const uint32_t b = x < n ? file[x] : ((virt && x == n) ? 0x0au : 0u);
                w[i >> 2] |= b << ((i & 3) * 8);
            }
            v[j] = make_uint4(w[0], w[1], w[2], w[3]);
        }
    }
    uint32_t nlc = 0;
    uint16_t *ent = s_ent[warp];

    if constexpr (V == 2) {
        // ---- pass 1 (V2): transpose through shared memory, 64 contiguous bytes per lane, one ranking for the region ----
        uint4 *sd = s_data + warp * (REGION / 16);
#pragma unroll
        for (int j = 0; j < 4; ++j) sd[swz_unit((uint32_t)(j * 32 + lane))] = v[j];
        __syncwarp();
        uint32_t lo = 0, hi = 0;                      // bit p of hi:lo <-> byte 64 * lane + p is a newline
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint4 x = sd[swz_unit((uint32_t)(4 * lane + i))];
            const uint32_t w4[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const uint32_t f = byte_eq_mask_r(w4[c], k0a, k7f, k80);            // 0x80 per newline byte
                const uint32_t nib = (f * 0x00204081u) >> 28;                       // the four flags as a nibble, byte order
                const int k = 4 * i + c;
                if (k < 8) lo = nib * (1u << (4 * k)) + lo;                         // multiply-adds: FMA pipe
                else hi = nib * (1u << (4 * (k - 8))) + hi;
            }
        }
        {
            const uint32_t c = (uint32_t)(__popc(lo) + __popc(hi));
            const uint32_t b1 = __ballot_sync(0xffffffffu, c >= 1u), b2 = __ballot_sync(0xffffffffu, c >= 2u);
            const uint32_t b3 = __ballot_sync(0xffffffffu, c >= 3u);
            const uint32_t pbase = (uint32_t)lane * 64u;
            if (!b3) {
                // lines of 32 bytes or more: at most two newlines in a lane's 64 bytes
                const uint32_t idx = (uint32_t)(__popc(b1 & lt_mask) + __popc(b2 & lt_mask));
                nlc = (uint32_t)(__popc(b1) + __popc(b2));
                if (c) {
                    const uint32_t p1 = lo ? (uint32_t)(__ffs(lo) - 1) : 32u + (uint32_t)(__ffs(hi) - 1);
                    if (idx < (uint32_t)SEGCAP) ent[idx] = (uint16_t)(pbase + p1);
                    if (c >= 2u) {
                        if (lo) lo &= lo - 1u; else hi &= hi - 1u;
                        const uint32_t p2 = lo ? (uint32_t)(__ffs(lo) - 1) : 32u + (uint32_t)(__ffs(hi) - 1);
                        if (idx + 1u < (uint32_t)SEGCAP) ent[idx + 1u] = (uint16_t)(pbase + p2);
                    }
                }
            } else {
                // short lines: exclusive scan of the per-lane counts, every lane walks its own newlines in order
                uint32_t incl = c;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t o2 = __shfl_up_sync(0xffffffffu, incl, d);
                    if (lane >= d) incl += o2;
                }
                nlc = __shfl_sync(0xffffffffu, incl, 31);
                uint32_t idx = incl - c;
                while (lo) { if (idx < (uint32_t)SEGCAP) ent[idx] = (uint16_t)(pbase + (uint32_t)(__ffs(lo) - 1)); lo &= lo - 1u; ++idx; }
                while (hi) { if (idx < (uint32_t)SEGCAP) ent[idx] = (uint16_t)(pbase + 32u + (uint32_t)(__ffs(hi) - 1)); hi &= hi - 1u; ++idx; }
            }
        }
        __syncwarp();
    } else {
        // ---- pass 1: positions, ranked in file order (chunk-major, lane-minor) ------------------
        uint32_t m[4];
        int cmax = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            s_data[warp * (REGION / 16) + j * 32 + lane] = v[j];
            m[j] = chunk_eq_mask_r(v[j], k0a, k7f, k80);
            cmax = max(cmax, __popc(m[j]));
        }
        const bool any2 = __any_sync(0xffffffffu, cmax >= 2);          // e.g. the "+" line of a FASTQ record
        const bool multi = any2 && __any_sync(0xffffffffu, cmax >= 3);
        if (!any2) {
            // the usual FASTA case: no lane holds two newlines in its 16 bytes -> one ballot per chunk
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t bn = __ballot_sync(0xffffffffu, m[j] != 0);
                if (m[j]) {
                    const uint32_t idx = nlc + __popc(bn & lt_mask);
                    if (idx < (uint32_t)SEGCAP) ent[idx] = (uint16_t)(j * 512 + lane * 16 + chunk_bit_to_off(__ffs(m[j]) - 1));
                }
                nlc += __popc(bn);
            }
        } else if (!multi) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = __popc(m[j]);
                const uint32_t bn1 = __ballot_sync(0xffffffffu, c >= 1);
                const uint32_t bn2 = __ballot_sync(0xffffffffu, c >= 2);
                if (c) {
                    const uint32_t idx = nlc + __popc(bn1 & lt_mask) + __popc(bn2 & lt_mask);
                    const int xo = j * 512 + lane * 16;
                    int oa = chunk_bit_to_off(__ffs(m[j]) - 1);
                    if (c == 2) {
                        const uint32_t m2 = m[j] & (m[j] - 1);
                        const int ob = chunk_bit_to_off(__ffs(m2) - 1);
                        const int hi = max(oa, ob);
                        oa = min(oa, ob);
                        if (idx + 1 < (uint32_t)SEGCAP) ent[idx + 1] = (uint16_t)(xo + hi);
                    }
                    if (idx < (uint32_t)SEGCAP) ent[idx] = (uint16_t)(xo + oa);
                }
                nlc += __popc(bn1) + __popc(bn2);
            }
        }
        if (multi) {
            // short lines: three or more newlines inside one lane's 16 bytes -> shuffle scan per chunk, then each lane
            // walks its own newlines in byte order (word, then byte within the word)
            nlc = 0;
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                uint32_t mj = 0;
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) if (jj == j) mj = m[jj];
                const uint32_t c = (uint32_t)__popc(mj);
                uint32_t incl = c;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t o2 = __shfl_up_sync(0xffffffffu, incl, d);
                    if (lane >= d) incl += o2;
                }
                uint32_t idx = nlc + incl - c;
#pragma unroll 1
                for (int w = 0; w < 4; ++w) {
                    uint32_t mw = mj & (0x80808080u >> w);
                    while (mw) {
                        if (idx < (uint32_t)SEGCAP) ent[idx] = (uint16_t)(j * 512 + lane * 16 + chunk_bit_to_off(__ffs(mw) - 1));
                        mw &= mw - 1;
                        ++idx;
                    }
                }
                nlc += __shfl_sync(0xffffffffu, incl, 31);
            }
        }
        __syncwarp();
    }

    // ---- pass 2: one lane per newline: neighbour byte -> flag; counts; write-out --------------
    const uint8_t *sb = reinterpret_cast<const uint8_t *>(s_data + warp * (REGION / 16));
    uint32_t hc = 0;
    if (nlc <= (uint32_t)SEGCAP) {
        uint16_t *dst = P.seg + r * SEGCAP;
        const uint32_t nround = (nlc + 15u) & ~15u;         // whole 32-byte sectors, zero padded
        bool general = MODE == 1 || nlc > 32u;              // FASTA writes the newline list of general regions only
        uint32_t nfacts = 0;
        for (uint32_t k0 = 0; k0 < nround; k0 += 32) {
            const uint32_t k = k0 + lane;
            uint32_t e = 0;
            if (k < nlc) {
                const uint32_t pos = ent[k];
                e = pos;
                if (MODE == 0) {
                    const uint32_t next = pos < (uint32_t)(REGION - 1) ? region_byte<V>(sb, pos + 1u)
                                                                      : (base + REGION < n ? (uint32_t)file[base + REGION] : 0u);
                    if (next == '>') e |= E_HDR;
                } else {
                    const uint32_t prev = pos > 0 ? region_byte<V>(sb, pos - 1u) : (base > 0 ? (uint32_t)file[base - 1] : 0u);
                    if (prev == '\r') e |= E_CR;
                }
            }
            if (MODE == 0) {
                const uint32_t hb = __ballot_sync(0xffffffffu, (e & E_HDR) != 0);
                hc += __popc(hb);
                if (k0 == 0) {
                    // lines that change a record: header lines, the line after a header, and lines whose length
                    // differs from the previous line's.  k >= 2: the line and both newlines before it lie in the
                    // region, so it is settled here, one lane per line, into a line fact.
                    const uint32_t e1 = __shfl_up_sync(0xffffffffu, e, 1), e2 = __shfl_up_sync(0xffffffffu, e, 2);
                    const uint32_t p = e & E_POS, p1 = e1 & E_POS, L = p - p1, dL = L - (p1 - (e2 & E_POS));
                    const bool it = lane >= 2 && k < nlc && (((e1 | e2) & E_HDR) != 0 || dL != 0u);
                    const uint32_t imask = __ballot_sync(0xffffffffu, it);
                    nfacts = (uint32_t)__popc(imask);
                    general |= nfacts > (uint32_t)LF_MAX;
                    if (!general) {
                        uint32_t kind = LF_EVENT, y = dL;
                        if (e1 & E_HDR) {
                            const uint32_t elen = region_byte<V>(sb, p - 1u) == '\r' ? 2u : 1u, dlen = L - 1u - elen;
                            kind = LF_HDR;
                            y = dlen | (dlen << 11) | ((elen - 1u) << 22);
                        } else if (e2 & E_HDR) {
                            kind = LF_LLEN;
                            y = L;
                        }
                        // the name cut: first ' ' or '\t' of the header, all lanes testing its bytes at once
                        uint32_t hm = __ballot_sync(0xffffffffu, it && kind == LF_HDR && !(P.flags & FXG_SCAN_FULL_NAME));
                        while (hm) {
                            const int f = __ffs(hm) - 1;
                            hm &= hm - 1u;
                            const uint32_t s1 = __shfl_sync(0xffffffffu, p1 + 2u, f), dlen = __shfl_sync(0xffffffffu, y & E_POS, f);
                            const uint32_t lim = min(dlen, NAME_SCAN);
                            uint32_t cut = dlen > NAME_SCAN ? ~0u : dlen;
                            for (uint32_t o = 0; o < lim; o += 32) {
                                const uint32_t b = o + lane < lim ? region_byte<V>(sb, s1 + o + lane) : 0u;
                                const uint32_t m = __ballot_sync(0xffffffffu, b == ' ' || b == '\t');
                                if (m) { cut = o + (uint32_t)(__ffs(m) - 1); break; }
                            }
                            if (lane == f) y = cut == ~0u ? (y | LF_CUT_UNKNOWN) : ((y & ~(E_POS << 11)) | (cut << 11));
                        }
                        if (it)
                            P.lf[r * LF_STRIDE + __popc(imask & lt_mask)] =
                                make_uint2(p | ((uint32_t)k << 11) | ((uint32_t)__popc(hb & lt_mask) << 16) | (kind << 21), y);
                    }
                }
            }
            if (general && k < nround) dst[k] = (uint16_t)e;
            if (k < nlc) ent[k] = (uint16_t)e;                   // complete entries (for the region records)
        }
        __syncwarp();
        if (lane == 0) {
            const uint32_t last = nlc >= 1 ? ent[nlc - 1] : 0u, prev = nlc >= 2 ? ent[nlc - 2] : 0u;
            P.rc[r] = make_uint2(nlc | (hc << 16), last | (prev << 16));
            if (MODE == 0) {
                const uint32_t f0 = nlc >= 1 ? ent[0] : 0u, f1 = nlc >= 2 ? ent[1] : 0u;
                P.fw[r] = f0 | (f1 << 16) | (general ? FW_GEN : nfacts << FW_NF_SHIFT);
            }
        }
    } else {
        // dense region: only the counts; the rows kernels re-read the bytes
        if (MODE == 0) {
            uint32_t myh = 0;
            for (int x = lane; x < REGION; x += 32)
                if (region_byte<V>(sb, (uint32_t)x) == '\n') {
                    const uint32_t next = x < REGION - 1 ? region_byte<V>(sb, (uint32_t)x + 1u) : (base + REGION < n ? (uint32_t)file[base + REGION] : 0u);
                    myh += next == '>';
                }
            hc = __reduce_add_sync(0xffffffffu, myh);
        }
        if (lane == 0) {
            P.rc[r] = make_uint2(nlc | (hc << 16), 0u);
            if (MODE == 0) P.fw[r] = FW_GEN;
        }
    }
}

// =============================================================================================
// prefix over the region counts
// =============================================================================================
// per block of PS_BLOCK regions: {sum newlines, sum header starts}
__global__ void __launch_bounds__(PS_THREADS) prefix_reduce_kernel(const uint2 *rc, ulonglong2 *bs) {
    __shared__ uint32_t sm[16];
    const uint4 *p = reinterpret_cast<const uint4 *>(rc + (size_t)blockIdx.x * PS_BLOCK + (size_t)threadIdx.x * PS_PER_THREAD);
    uint32_t a = 0, b = 0;
#pragma unroll
    for (int i = 0; i < PS_PER_THREAD / 2; ++i) {
        const uint4 q = p[i];
        a += (q.x & 0xffffu) + (q.z & 0xffffu);
        b += (q.x >> 16) + (q.z >> 16);
    }
    a = __reduce_add_sync(0xffffffffu, a);
    b = __reduce_add_sync(0xffffffffu, b);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { sm[warp] = a; sm[8 + warp] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t ta = 0, tb = 0;
        for (int w = 0; w < PS_THREADS / 32; ++w) { ta += sm[w]; tb += sm[8 + w]; }
        bs[blockIdx.x] = make_ulonglong2(ta, tb);
    }
}

// exclusive scan of the block sums (one CTA), seeds, totals
__global__ void __launch_bounds__(1024) prefix_blocks_kernel(ulonglong2 *bs, int64_t nb, const uint8_t *file, int64_t n,
                                                             int mode, ScanTotals *tot) {
    __shared__ uint64_t s_a[32], s_b[32];
    __shared__ uint64_t s_ca, s_cb;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { s_ca = 0; s_cb = (mode == 0 && n > 0 && file[0] == '>') ? 1u : 0u; }   // header at byte 0
    __syncthreads();
    for (int64_t b0 = 0; b0 < nb; b0 += 1024) {
        const int64_t i = b0 + threadIdx.x;
        const ulonglong2 v = i < nb ? bs[i] : make_ulonglong2(0, 0);
        uint64_t a = v.x, b = v.y;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t oa = (uint64_t)shfl_up_i64((int64_t)a, d), ob = (uint64_t)shfl_up_i64((int64_t)b, d);
            if (lane >= d) { a += oa; b += ob; }
        }
        if (lane == 31) { s_a[warp] = a; s_b[warp] = b; }
        __syncthreads();
        uint64_t wa = 0, wb = 0;
        for (int w = 0; w < warp; ++w) { wa += s_a[w]; wb += s_b[w]; }
        const uint64_t ca = s_ca, cb = s_cb;
        if (i < nb) bs[i] = make_ulonglong2(ca + wa + a - v.x, cb + wb + b - v.y);
        __syncthreads();
        if (threadIdx.x == 1023) { s_ca = ca + wa + a; s_cb = cb + wb + b; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const bool virt = n > 0 && file[n - 1] != '\n';
        tot->nl = s_ca; tot->hdr = s_cb; tot->n_eff = n + (virt ? 1 : 0);
    }
}

// per region: exclusive {newlines, header starts}
__global__ void __launch_bounds__(PS_THREADS) prefix_expand_kernel(const uint2 *rc, const ulonglong2 *bs, ulonglong2 *ex,
                                                                 int64_t nreg) {
    __shared__ uint32_t s_a[PS_THREADS / 32], s_b[PS_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t r0 = (size_t)blockIdx.x * PS_BLOCK + (size_t)threadIdx.x * PS_PER_THREAD;
    const uint4 *p = reinterpret_cast<const uint4 *>(rc + r0);
    uint32_t c[PS_PER_THREAD];
    uint32_t a = 0, b = 0;
#pragma unroll
    for (int i = 0; i < PS_PER_THREAD / 2; ++i) {
        const uint4 q = p[i];
        c[2 * i] = q.x; c[2 * i + 1] = q.z;
        a += (q.x & 0xffffu) + (q.z & 0xffffu);
        b += (q.x >> 16) + (q.z >> 16);
    }
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t oa = __shfl_up_sync(0xffffffffu, ia, d), ob = __shfl_up_sync(0xffffffffu, ib, d);
        if (lane >= d) { ia += oa; ib += ob; }
    }
    if (lane == 31) { s_a[warp] = ia; s_b[warp] = ib; }
    __syncthreads();
    uint32_t wa = 0, wb = 0;
    for (int w = 0; w < warp; ++w) { wa += s_a[w]; wb += s_b[w]; }
    const ulonglong2 bb = bs[blockIdx.x];
    uint64_t ea = bb.x + wa + ia - a, eb = bb.y + wb + ib - b;
#pragma unroll
    for (int i = 0; i < PS_PER_THREAD; ++i) {
        if ((int64_t)(r0 + i) < nreg) ex[r0 + i] = make_ulonglong2(ea, eb);
        ea += c[i] & 0xffffu; eb += c[i] >> 16;
    }
}

// =============================================================================================
// lines: one thread per line, from the newline list
// =============================================================================================
// First k in [0, limit) with h[k] == a or h[k] == b, else limit.  Word-wise: four aligned 32-bit
// loads in flight per step instead of one dependent byte load per character.  Reads whole aligned
// words up to 18 bytes past h + limit (the caller checks the buffer capacity).
__device__ __forceinline__ int64_t find_first_of2(const uint8_t *h, int64_t limit, uint32_t a4, uint32_t b4, int *which) {
    const int mis = (int)((uintptr_t)h & 3);
    const uint32_t *wp = reinterpret_cast<const uint32_t *>(h - mis);
    *which = 0;
    for (int64_t k = -mis; k < limit; k += 16, wp += 4) {
        const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2], w3 = wp[3];
        uint32_t ma[4] = {byte_eq_mask(w0, a4), byte_eq_mask(w1, a4), byte_eq_mask(w2, a4), byte_eq_mask(w3, a4)};
        uint32_t mb[4] = {byte_eq_mask(w0, b4), byte_eq_mask(w1, b4), byte_eq_mask(w2, b4), byte_eq_mask(w3, b4)};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint32_t m = ma[i] | mb[i];
            const int64_t kk = k + 4 * i;
            if (kk < 0) m &= 0xffffffffu << (8 * (int)(-kk));        // bytes before h (only the first word)
            if (m) {
                const int byte = (__ffs(m) - 1) >> 3;
                const int64_t pos = kk + byte;
                if (pos >= limit) return limit;
                *which = ((mb[i] >> (8 * byte)) & 0x80u) ? 2 : 1;
                return pos;
            }
        }
    }
    return limit;
}

struct Prev2 {            // the two newlines before some point: [1] nearest, [0] the one before
    int64_t  pos1, pos0;  // NOPOS if there is none; -1 = the virtual newline before byte 0
    uint32_t h1, h0;      // the line starting after that newline begins with '>'
};

template <int MODE>
__device__ __forceinline__ uint32_t is_hdr_at(const ScanParams &P, int64_t x) {     // does a header line start at byte x?
    return (MODE == 0 && x < P.n && P.file[x] == '>') ? 1u : 0u;
}
__device__ __forceinline__ bool nl_at(const ScanParams &P, int64_t x) {             // incl. the virtual newline at n
    return x < P.n ? P.file[x] == '\n' : (x == P.n && P.n > 0 && P.file[P.n - 1] != '\n');
}

// ---- FASTA record slot updates, shared by the line walk (do_line) and the line facts ----
// name length: bytes of the header line starting at s (its '>') before the first ' ' or '\t'
__device__ __forceinline__ int64_t fasta_name_len(const ScanParams &P, int64_t s, int64_t dlen) {
    int64_t nlen = 0;
    if (s + 1 + dlen + 20 <= P.capacity) {
        int which;
        nlen = find_first_of2(P.file + s + 1, dlen, 0x20202020u, 0x09090909u, &which);
    } else {
        while (nlen < dlen) {
            const uint8_t ch = P.file[s + 1 + nlen];
            if (ch == ' ' || ch == '\t') break;
            ++nlen;
        }
    }
    return nlen;
}
// header line ending in the newline at p
__device__ __forceinline__ void fasta_header(const ScanParams &P, int64_t slot, int64_t p, int64_t lineidx, int64_t dlen,
                                             int64_t nlen, int elen) {
    if (slot < P.tmp_cap) {
        FastaTmp *t = &P.tmp[slot];
        t->boff = P.base_offset + p + 1;
        t->lineidx = lineidx;
        t->dlen = (int32_t)dlen;
        t->nlen = (int32_t)nlen;
        t->elen = (uint32_t)elen;
    }
}
// sequence line whose length differs from the previous sequence line's by dL (slot < tmp_cap)
__device__ __forceinline__ void fasta_event(const ScanParams &P, int64_t slot, int64_t lineidx, int64_t dL) {
    FastaTmp *t = &P.tmp[slot];
    atomicAdd(&t->D, 1u);
    atomicMax((unsigned long long *)&t->evmax, (unsigned long long)lineidx);
    atomicMax((unsigned long long *)&t->evminc, ~(unsigned long long)lineidx);
    atomicAdd((unsigned long long *)&t->S, (unsigned long long)dL);
}

// ---- one line: newline at p, previous newlines pm1, pm2; h1 / h2: the line starting after pm1 / pm2 is a
//      header; hcount: header starts up to and including the one after pm1 (= record ordinal + 1);
//      cr: the byte before p is '\r' (FASTQ entries carry it; FASTA looks it up for header lines only) ----
template <int MODE>
__device__ __forceinline__ void do_line(const ScanParams &P, int64_t first_line, int64_t p, int64_t pm1, int64_t pm2, bool h1, bool h2,
                                        int64_t hcount, int64_t lineidx, bool cr, unsigned long long &my_size) {
    const uint8_t *file = P.file;
    const int64_t s = pm1 + 1;
    const int64_t L = p - pm1;                            // len + 1
    if (MODE == 0) {
        const int64_t slot = hcount;                      // rec + 1
        if (h1) {
            const int elen = (p >= 1 && (p - 1 < P.n ? file[p - 1] : 0) == '\r') ? 2 : 1;
            const int64_t dlen = L - 1 - elen;
            const int64_t nlen = (P.flags & FXG_SCAN_FULL_NAME) ? dlen : fasta_name_len(P, s, dlen);
            fasta_header(P, slot, p, lineidx, dlen, nlen, elen);
        } else if (slot < P.tmp_cap) {
            const bool prev_exists = pm1 >= 0;
            if (!prev_exists || h2) {
                P.tmp[slot].llen = L;
            } else {
                const int64_t prevL = pm1 - pm2;
                if (L != prevL) fasta_event(P, slot, lineidx, L - prevL);
            }
        }
    } else {
        const int64_t gline = first_line + lineidx;
        const int ph = (int)(gline & 3);
        const int64_t row = (gline >> 2) - (first_line >> 2);
        const int64_t len = L - 1;
        if (ph == 1) {
            const int64_t rlen = (len > 0 && cr) ? len - 1 : len;
            my_size += (unsigned long long)rlen;
            if (row < P.qrows_cap) { P.qrows[row].soff = P.base_offset + s; P.qrows[row].rlen = rlen; }
        } else if (row < P.qrows_cap) {
            if (ph == 0) {
                int64_t l = len - 1;
                if (l > 0 && cr) --l;
                if (l < 0) l = 0;
                int64_t k = 0;
                if (s + 1 + l + 20 <= P.capacity) {
                    int which;
                    k = find_first_of2(file + s + 1, l, 0x20202020u, 0x00000000u, &which);
                    if (which == 2) k = l;          // a NUL before any space: strchr() finds nothing (fastq.c:112)
                } else {
                    for (; k < l; ++k) {
                        const uint8_t ch = file[s + 1 + k];
                        if (ch == 0) { k = l; break; }
                        if (ch == ' ') break;
                    }
                }
                *reinterpret_cast<int2 *>(&P.qrows[row].dlen) = make_int2((int)len, (int)k);
            } else if (ph == 3) {
                P.qrows[row].qoff = P.base_offset + s;
            }
        }
    }
}

// ---- the two newlines before region r (warp-uniform): walk back over the region records, 32 at a time.
//      General path: long lines (more than ~60 KiB without a newline) and neighbours of dense regions. ----
template <int MODE>
__device__ __noinline__ Prev2 carry_walk(const ScanParams *Pg, int64_t r) {
    const ScanParams &P = *Pg;
    Prev2 cy;
    const int lane = threadIdx.x & 31;
    cy.pos1 = cy.pos0 = NOPOS; cy.h1 = cy.h0 = 0;
    int need = 2;
    auto push = [&](int64_t pos, uint32_t h) {
        if (need == 2) { cy.pos1 = pos; cy.h1 = h; } else { cy.pos0 = pos; cy.h0 = h; }
        --need;
    };
    int64_t q = r - 1;
    while (need > 0 && q >= 0) {
        const int64_t qq = q - lane;
        const uint32_t c = qq >= 0 ? (P.rc[qq].x & 0xffffu) : 0u;
        const uint32_t nz = __ballot_sync(0xffffffffu, c != 0);
        if (!nz) { q -= 32; continue; }
        const int f = __ffs(nz) - 1;
        q -= f;
        const int cq = (int)__shfl_sync(0xffffffffu, c, f);
        if (cq <= SEGCAP) {
            const uint32_t y = P.rc[q].y;                      // the region's last entry | the one before << 16
            push(q * REGION + (int64_t)(y & E_POS), MODE == 0 ? ((y >> 15) & 1u) : 0u);
            if (need > 0 && cq >= 2) push(q * REGION + (int64_t)((y >> 16) & E_POS), MODE == 0 ? (y >> 31) : 0u);
        } else {
            for (int64_t x = q * REGION + REGION - 1; x >= q * REGION && need > 0; --x)
                if (nl_at(P, x)) push(x, is_hdr_at<MODE>(P, x + 1));
        }
        q -= 1;
    }
    if (need > 0) push(-1, is_hdr_at<MODE>(P, 0));            // the virtual newline before byte 0
    return cy;
}

// ---- dense region (more than SEGCAP newlines in 2 KiB): re-read the bytes; every lane owns 64 of them ----
template <int MODE>
__device__ __noinline__ unsigned long long dense_region(const ScanParams *Pg, int64_t first_line, int64_t r, Prev2 cy,
                                                        ulonglong2 exv) {
    const ScanParams &P = *Pg;
    unsigned long long my_size = 0;
    const int lane = threadIdx.x & 31;
    const uint8_t *file = P.file;
    const int64_t b0 = r * REGION + lane * 64;
    // per lane: count, header count, last two newlines
    uint32_t c = 0, h = 0;
    Prev2 inc; inc.pos1 = inc.pos0 = NOPOS; inc.h1 = inc.h0 = 0;
    for (int i = 0; i < 64; ++i) {
        const int64_t x = b0 + i;
        if (nl_at(P, x)) {
            const uint32_t hh = is_hdr_at<MODE>(P, x + 1);
            ++c; h += hh;
            inc.pos0 = inc.pos1; inc.h0 = inc.h1; inc.pos1 = x; inc.h1 = hh;
        }
    }
    // inclusive scans: counts, and the "last two newlines" pair (the right operand wins slot by slot)
    uint32_t ic = c, ih = h;
    uint32_t icnt = c > 2 ? 2 : c;                        // how many of inc's slots are filled (0..2)
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t oc = __shfl_up_sync(0xffffffffu, ic, d), oh = __shfl_up_sync(0xffffffffu, ih, d);
        const int64_t op1 = shfl_up_i64(inc.pos1, d), op0 = shfl_up_i64(inc.pos0, d);
        const uint32_t oh1 = __shfl_up_sync(0xffffffffu, inc.h1, d), oh0 = __shfl_up_sync(0xffffffffu, inc.h0, d);
        const uint32_t ocnt = __shfl_up_sync(0xffffffffu, icnt, d);
        if (lane >= d) {
            ic += oc; ih += oh;
            if (icnt == 0) { inc.pos1 = op1; inc.h1 = oh1; inc.pos0 = op0; inc.h0 = oh0; icnt = ocnt; }
            else if (icnt == 1 && ocnt >= 1) { inc.pos0 = op1; inc.h0 = oh1; icnt = 2; }
        }
    }
    // exclusive = inclusive of lane-1, completed from the region carry
    Prev2 pv;
    pv.pos1 = shfl_up_i64(inc.pos1, 1); pv.pos0 = shfl_up_i64(inc.pos0, 1);
    pv.h1 = __shfl_up_sync(0xffffffffu, inc.h1, 1); pv.h0 = __shfl_up_sync(0xffffffffu, inc.h0, 1);
    uint32_t pcnt = __shfl_up_sync(0xffffffffu, icnt, 1);
    if (lane == 0) pcnt = 0;
    if (pcnt == 0) pv = cy;
    else if (pcnt == 1) { pv.pos0 = cy.pos1; pv.h0 = cy.h1; }
    int64_t idx = (int64_t)exv.x + (ic - c);
    int64_t hcount = (int64_t)exv.y + (ih - h);
    for (int i = 0; i < 64 && c; ++i) {
        const int64_t x = b0 + i;
        if (!nl_at(P, x)) continue;
        const bool cr = x > 0 && file[x - 1] == '\r';
        do_line<MODE>(P, first_line, x, pv.pos1, pv.pos0, pv.h1 != 0, pv.h0 != 0, hcount, idx, cr, my_size);
        const uint32_t hh = is_hdr_at<MODE>(P, x + 1);
        hcount += hh; ++idx;
        pv.pos0 = pv.pos1; pv.h0 = pv.h1; pv.pos1 = x; pv.h1 = hh;
    }
    return my_size;
}

// ---- the lines of one region with at most SEGCAP newlines, warp-cooperative: batches of 32 entries.
//      E0 / E1: the first two batches (entry k0 + lane), loaded by the caller. ----
template <int MODE>
__device__ __forceinline__ void region_batches(const ScanParams &P, int64_t first_line, int64_t r, int nl, Prev2 cy, ulonglong2 X,
                                               uint32_t E0, uint32_t E1, unsigned long long &my_size) {
    const int lane = threadIdx.x & 31;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const int64_t base = r * REGION;
    const uint16_t *sg = P.seg + r * SEGCAP;
    int64_t hrun = (int64_t)X.y;                      // header starts through the newline before the batch
    for (int k0 = 0; k0 < nl; k0 += 32) {
        const int k = k0 + lane;
        const bool valid = k < nl;
        uint32_t e = k0 == 0 ? E0 : (k0 == 32 ? E1 : (valid ? (uint32_t)sg[k] : 0u));
        if (!valid) e = 0;
        const uint32_t hb = __ballot_sync(0xffffffffu, (e & E_HDR) != 0);
        const uint32_t e1 = __shfl_up_sync(0xffffffffu, e, 1), e2 = __shfl_up_sync(0xffffffffu, e, 2);
        if (valid) {
            int64_t pm1, pm2;
            bool h1, h2;
            if (lane >= 1) { pm1 = base + (e1 & E_POS); h1 = (e1 & E_HDR) != 0; } else { pm1 = cy.pos1; h1 = cy.h1 != 0; }
            if (lane >= 2) { pm2 = base + (e2 & E_POS); h2 = (e2 & E_HDR) != 0; }
            else if (lane == 1) { pm2 = cy.pos1; h2 = cy.h1 != 0; }
            else { pm2 = cy.pos0; h2 = cy.h0 != 0; }
            do_line<MODE>(P, first_line, base + (e & E_POS), pm1, pm2, h1, h2, hrun + __popc(hb & lt_mask), (int64_t)X.x + k,
                          (e & E_CR) != 0, my_size);
        }
        // carry for the next batch (only reached when this one was full)
        const uint32_t l31 = __shfl_sync(0xffffffffu, e, 31), l30 = __shfl_sync(0xffffffffu, e, 30);
        cy.pos1 = base + (l31 & E_POS); cy.h1 = (l31 >> 15) & 1u;
        cy.pos0 = base + (l30 & E_POS); cy.h0 = (l30 >> 15) & 1u;
        hrun += __popc(hb);
    }
}

// ---- general path for one region: everything looked up from scratch ----
// X: exclusive {newlines, header starts} of the region
template <int MODE>
__device__ __noinline__ unsigned long long full_region(const ScanParams *Pg, int64_t first_line, int64_t r, ulonglong2 X) {
    const ScanParams &P = *Pg;
    unsigned long long my_size = 0;
    const int lane = threadIdx.x & 31;
    const int nl = (int)(P.rc[r].x & 0xffffu);
    if (nl == 0) return 0;
    Prev2 cy = carry_walk<MODE>(Pg, r);
    if (MODE != 0) cy.h1 = cy.h0 = 0;
    if (nl <= SEGCAP) region_batches<MODE>(P, first_line, r, nl, cy, X, P.seg[r * SEGCAP + lane], P.seg[r * SEGCAP + 32 + lane], my_size);
    else my_size += dense_region<MODE>(Pg, first_line, r, cy, X);
    return my_size;
}

// FASTQ fast path: one LANE per read.  A warp takes RG consecutive regions, flattens their newline lists
// (plus two look-ahead regions) into shared memory, and every lane assembles the whole 32-byte row of one
// read from five consecutive newline positions -- straight-line code, one row store, the name cut searched
// by all lanes at once.  Ownership: a warp covers every line inside its span (the up-to-three leading lines
// of a read that began earlier are written field by field) and completes the reads that START in its span
// as far as its window reaches; lines past the window are (also) covered by the warp that owns their
// region, which writes identical values.  Spans containing a dense region use the general path.
constexpr int RG = 8;                          // regions per warp
constexpr int RWIN = RG + 2;                   // + look-ahead
static_assert(RWIN * REGION <= 32768, "window positions must fit 15 bits");

__global__ void __launch_bounds__(MARK_WARPS * 32) fastq_records_kernel(const ScanParams Pin) {
    __shared__ uint16_t s_flat[MARK_WARPS][RWIN * SEGCAP];      // position in window | '\r' before << 15
    const ScanParams &P = Pin;
    const int64_t first_line = Pin.totals->first_line;          // global line phase, known only after the exchange
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r0 = ((int64_t)blockIdx.x * MARK_WARPS + warp) * RG;
    if (r0 >= P.nreg) return;
    unsigned long long my_size = 0;
    const uint8_t *file = P.file;

    // lane l <-> region r0 - 1 + l  (l = 0: the region before the span; 1..RG: the span; then the look-ahead)
    const int64_t rl = r0 - 1 + lane;
    uint2 rec = make_uint2(0u, 0u);
    uint64_t exl = 0;
    if (lane <= RWIN && rl >= 0 && rl < P.nreg) { rec = P.rc[rl]; exl = P.ex[rl].x; }
    const uint32_t nll = rec.x & 0xffffu;
    const uint32_t densem = __ballot_sync(0xffffffffu, nll > (uint32_t)SEGCAP);
    if (densem & (((1u << RG) - 1u) << 1)) {                       // a dense region inside the span
        for (int i = 0; i < RG; ++i)
            if (r0 + i < P.nreg) my_size += full_region<1>(P.self, first_line, r0 + i, P.ex[r0 + i]);
    } else {
        const uint64_t ex0 = (uint64_t)shfl_i64((int64_t)exl, 1);    // lines before the span
        // ---- flatten the window ----
        uint16_t *flat = s_flat[warp];
        // Two entries per lane and load: 64 per region cover every region of a typical short-read file in one load.
        int W = 0, Ls = 0;                                           // entries in the window / in the span
        bool closed = false;                                         // a dense look-ahead region ends the window
#pragma unroll
        for (int i = 0; i < RWIN; ++i) {
            const int nl = (int)__shfl_sync(0xffffffffu, nll, i + 1);
            if (nl > SEGCAP) closed = true;
            if (!closed) {
                const int k = 2 * lane;
                const uint32_t E2 = k < nl ? reinterpret_cast<const uint32_t *>(P.seg + (r0 + i) * SEGCAP)[lane] : 0u;
                const uint32_t e0 = E2 & 0xffffu, e1 = E2 >> 16;
                if (k < nl) flat[W + k] = (uint16_t)((i * REGION + (int)(e0 & E_POS)) | ((e0 & E_CR) ? 0x8000u : 0u));
                if (k + 1 < nl) flat[W + k + 1] = (uint16_t)((i * REGION + (int)(e1 & E_POS)) | ((e1 & E_CR) ? 0x8000u : 0u));
                if (nl > 64) {                                       // lines shorter than 32 bytes on average
                    const uint16_t *sg = P.seg + (r0 + i) * SEGCAP;
                    for (int kk = 64 + lane; kk < nl; kk += 32) {
                        const uint32_t e = sg[kk];
                        flat[W + kk] = (uint16_t)((i * REGION + (int)(e & E_POS)) | ((e & E_CR) ? 0x8000u : 0u));
                    }
                }
                W += nl;
            }
            if (i == RG - 1) Ls = W;
        }
        __syncwarp();
        // ---- the newline before the span ----
        int64_t carry;
        {
            const uint32_t pn = __shfl_sync(0xffffffffu, nll, 0), py = __shfl_sync(0xffffffffu, rec.y, 0);
            if (r0 == 0) carry = -1;
            else if (pn >= 1 && pn <= (uint32_t)SEGCAP) carry = (r0 - 1) * REGION + (int64_t)(py & E_POS);
            else carry = carry_walk<1>(P.self, r0).pos1;
        }
        const int64_t span_base = r0 * REGION;
        auto POS = [&](int f) -> int64_t { return f < 0 ? carry : span_base + (int64_t)(flat[f] & 0x7fffu); };
        auto CR = [&](int f) -> bool { return (flat[f] & 0x8000u) != 0; };
        const int64_t g0 = first_line + (int64_t)ex0;                // global line index of flat[0]
        const int64_t row0 = first_line >> 2;
        int lead = (int)((4 - (g0 & 3)) & 3);
        if (lead > Ls) lead = Ls;
        // ---- (a) leading lines of a read that started before the span: field by field ----
        if (lane < lead) {
            const int f = lane;
            const int64_t g = g0 + f;
            const int ph = (int)(g & 3);
            const int64_t row = (g >> 2) - row0;
            const int64_t pm1 = POS(f - 1), p = POS(f);
            if (ph == 1) {
                const int64_t len = p - pm1 - 1;
                const int64_t rlen = (len > 0 && CR(f)) ? len - 1 : len;
                my_size += (unsigned long long)rlen;
                if (row < P.qrows_cap) { P.qrows[row].soff = P.base_offset + pm1 + 1; P.qrows[row].rlen = rlen; }
            } else if (ph == 3) {
                if (row < P.qrows_cap) P.qrows[row].qoff = P.base_offset + pm1 + 1;
            }
        }
        // ---- (b) reads that start inside the span: one lane each ----
        for (int fb = lead; fb < Ls; fb += 128) {
            const int f = fb + 4 * lane;
            int64_t row = 0, soff = 0, rlen = 0, qoff = 0, len = 0, k = 0;
            bool have1 = false, have3 = false;
            const bool mine = f < Ls;
            if (mine) {
                row = ((g0 + f) >> 2) - row0;
                have1 = f + 1 < W; have3 = f + 3 < W;
                const int64_t pm1 = POS(f - 1), p0 = POS(f);
                len = p0 - pm1 - 1;                                  // name line incl. '@' and '\r'
                int64_t l = len - 1;
                if (l > 0 && CR(f)) --l;
                if (l < 0) l = 0;
                const int64_t s = pm1 + 1;
                if (s + 1 + l + 20 <= P.capacity) {
                    int which;
                    k = find_first_of2(file + s + 1, l, 0x20202020u, 0x00000000u, &which);
                    if (which == 2) k = l;          // a NUL before any space: strchr() finds nothing (fastq.c:112)
                } else {
                    for (; k < l; ++k) {
                        const uint8_t ch = file[s + 1 + k];
                        if (ch == 0) { k = l; break; }
                        if (ch == ' ') break;
                    }
                }
                if (have1) {
                    const int64_t p1 = POS(f + 1);
                    const int64_t len1 = p1 - p0 - 1;
                    soff = P.base_offset + p0 + 1;
                    rlen = (len1 > 0 && CR(f + 1)) ? len1 - 1 : len1;
                    if (f + 1 < Ls) my_size += (unsigned long long)rlen;
                }
                if (have3) qoff = P.base_offset + POS(f + 2) + 1;
            }
            // ---- row stores.  A lane holds one 32-byte row = one DRAM sector; written as two 16-byte halves by ONE
            //      lane, every store instruction leaves half-filled sectors.  Neighbouring lanes swap halves instead, so
            //      that each instruction writes whole sectors: lanes (2j, 2j+1) write row 2j, then row 2j+1. ----
            const bool full = mine && have3 && row < P.qrows_cap;
            const int other_full = __shfl_xor_sync(0xffffffffu, full ? 1 : 0, 1);   // every lane must reach the shuffle
            const bool pair_full = full && other_full != 0;
            longlong2 a, b;
            a.x = soff; a.y = qoff;
            b.x = rlen; b.y = (long long)(((unsigned long long)(uint32_t)(int)k << 32) | (uint32_t)(int)len);
            const bool odd = (lane & 1) != 0;
            const longlong2 send = odd ? a : b;
            longlong2 recv;
            recv.x = shfl_i64(send.x, lane ^ 1);
            recv.y = shfl_i64(send.y, lane ^ 1);
            if (pair_full) {
                fxg_fastq_row *q0 = &P.qrows[odd ? row - 1 : row];                 // row of the even lane
                reinterpret_cast<longlong2 *>(q0)[odd ? 1 : 0] = odd ? recv : a;   // row 2j:   even lane's a, even lane's b
                reinterpret_cast<longlong2 *>(q0 + 1)[odd ? 1 : 0] = odd ? b : recv;   // row 2j+1: odd lane's a, odd lane's b
            } else if (mine && row < P.qrows_cap) {
                fxg_fastq_row *q = &P.qrows[row];
                if (have3) {
                    reinterpret_cast<longlong2 *>(q)[0] = a;
                    reinterpret_cast<longlong2 *>(q)[1] = b;
                } else {
                    *reinterpret_cast<int2 *>(&q->dlen) = make_int2((int)len, (int)k);
                    if (have1) { q->soff = soff; q->rlen = rlen; }
                }
            }
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) my_size += (unsigned long long)shfl_down_i64((int64_t)my_size, d);
    if (lane == 0 && my_size) atomicAdd((unsigned long long *)&P.totals->sum_len, my_size);
}

// FASTA rows: one CTA per prefix block, ROWS_PER_THREAD consecutive regions per thread.  The regions' exclusive
// counts are scanned here from rc (there is no per-region prefix array for FASTA).  Only lines that change a
// record do any work: lines 0 and 1 of a region go through do_line (the newlines before them are the previous
// region's last two entries, or are found by carry_walk), lines k >= 2 are the line facts mark wrote.  A general
// region (more than 32 newlines, more than LF_MAX facts, dense) has no line facts; its exclusive counts go into its
// fact slot instead, for fasta_general_kernel.
constexpr int ROWS_THREADS = 1024, ROWS_PER_THREAD = PS_BLOCK / ROWS_THREADS;
static_assert(ROWS_PER_THREAD == 4, "one uint4 of first-entry words per thread");

__global__ void __launch_bounds__(ROWS_THREADS) fasta_rows_kernel(const ScanParams P) {
    __shared__ uint32_t s_a[ROWS_THREADS / 32], s_b[ROWS_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r0 = (int64_t)blockIdx.x * PS_BLOCK + (int64_t)threadIdx.x * ROWS_PER_THREAD;
    const uint4 qa = reinterpret_cast<const uint4 *>(P.rc + r0)[0], qb = reinterpret_cast<const uint4 *>(P.rc + r0)[1];
    const uint4 fv = *reinterpret_cast<const uint4 *>(P.fw + r0);
    const uint2 rcv[ROWS_PER_THREAD] = {make_uint2(qa.x, qa.y), make_uint2(qa.z, qa.w), make_uint2(qb.x, qb.y), make_uint2(qb.z, qb.w)};
    const uint32_t fwv[ROWS_PER_THREAD] = {fv.x, fv.y, fv.z, fv.w};
    uint2 pv = r0 >= 1 ? P.rc[r0 - 1] : make_uint2(0u, 0u);
    // exclusive {newlines, header starts} of the thread's first region
    uint32_t a = 0, b = 0;
#pragma unroll
    for (int i = 0; i < ROWS_PER_THREAD; ++i) { a += rcv[i].x & 0xffffu; b += rcv[i].x >> 16; }
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t oa = __shfl_up_sync(0xffffffffu, ia, d), ob = __shfl_up_sync(0xffffffffu, ib, d);
        if (lane >= d) { ia += oa; ib += ob; }
    }
    const ulonglong2 bb = P.bs[blockIdx.x];
    if (lane == 31) { s_a[warp] = ia; s_b[warp] = ib; }
    __syncthreads();
    uint32_t wa = 0, wb = 0;
    for (int w = 0; w < warp; ++w) { wa += s_a[w]; wb += s_b[w]; }
    ulonglong2 X = make_ulonglong2(bb.x + wa + ia - a, bb.y + wb + ib - b);
    unsigned long long dummy = 0;
    bool any_general = false;
#pragma unroll
    for (int i = 0; i < ROWS_PER_THREAD; ++i) {
        const int64_t r = r0 + i, base = r * REGION;
        const uint32_t nl = rcv[i].x & 0xffffu, fw = fwv[i], pnl = pv.x & 0xffffu;
        const bool general = nl != 0 && (fw & FW_GEN) != 0;
        const bool walk = nl != 0 && !general && (r == 0 || pnl < 2u || pnl > (uint32_t)SEGCAP);
        Prev2 cy;                                     // the two newlines before the region
        cy.pos1 = base - REGION + (int64_t)(pv.y & E_POS); cy.h1 = (pv.y >> 15) & 1u;
        cy.pos0 = base - REGION + (int64_t)((pv.y >> 16) & E_POS); cy.h0 = pv.y >> 31;
        uint32_t wm = __ballot_sync(0xffffffffu, walk);
        while (wm) {
            const int f = __ffs(wm) - 1;
            wm &= wm - 1u;
            const Prev2 c = carry_walk<0>(P.self, shfl_i64(r, f));
            if (lane == f) cy = c;
        }
        if (general) *reinterpret_cast<ulonglong2 *>(P.lf + r * LF_STRIDE) = X;
        any_general |= general;
        if (nl != 0 && !general) {
            const uint32_t f0 = fw & 0xffffu, f1 = fw >> 16;
            const int64_t p0 = base + (int64_t)(f0 & E_POS);
            do_line<0>(P, 0, p0, cy.pos1, cy.pos0, cy.h1 != 0, cy.h0 != 0, (int64_t)X.y, (int64_t)X.x, false, dummy);
            if (nl >= 2u)
                do_line<0>(P, 0, base + (int64_t)(f1 & E_POS), p0, cy.pos1, (f0 & E_HDR) != 0, cy.h1 != 0,
                           (int64_t)X.y + ((f0 & E_HDR) ? 1 : 0), (int64_t)X.x + 1, false, dummy);
            const uint32_t nf = (fw & FW_NF) >> FW_NF_SHIFT;
            for (uint32_t j = 0; j < nf; ++j) {
                const uint2 lf = P.lf[r * LF_STRIDE + j];
                const int64_t slot = (int64_t)X.y + ((lf.x >> 16) & 31u), lineidx = (int64_t)X.x + ((lf.x >> 11) & 31u);
                if (slot >= P.tmp_cap) continue;
                const uint32_t kind = lf.x >> 21;
                if (kind == LF_HDR) {
                    const int64_t p = base + (int64_t)(lf.x & E_POS), dlen = lf.y & E_POS;
                    const int elen = 1 + (int)((lf.y >> 22) & 1u);
                    const int64_t nlen = (lf.y & LF_CUT_UNKNOWN) ? fasta_name_len(P, p - dlen - elen, dlen) : (int64_t)((lf.y >> 11) & E_POS);
                    fasta_header(P, slot, p, lineidx, dlen, nlen, elen);
                } else if (kind == LF_LLEN) {
                    P.tmp[slot].llen = lf.y;
                } else {
                    fasta_event(P, slot, lineidx, (int32_t)lf.y);
                }
            }
        }
        X.x += nl; X.y += rcv[i].x >> 16;
        pv = rcv[i];
    }
    const int block_general = __syncthreads_or(any_general ? 1 : 0);
    if (threadIdx.x == 0) P.gblk[blockIdx.x] = block_general ? 1u : 0u;
}

// FASTA general regions: one LANE per region screens the first-entries word (and loads the exclusive counts
// fasta_rows_kernel left in the fact slot), then the warp runs its general regions one after the other.
__global__ void __launch_bounds__(MARK_WARPS * 32) fasta_general_kernel(const ScanParams P) {
    __shared__ ulonglong2 s_x[MARK_WARPS][32];     // the lanes' counts, so that no register holds them across the calls
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t R0 = ((int64_t)blockIdx.x * MARK_WARPS + warp) * 32;
    if (R0 >= P.nreg) return;
    const int64_t r = R0 + lane;
    if (!P.gblk[R0 / PS_BLOCK]) return;          // no general region in this prefix block (the usual case)
    const bool general = r < P.nreg && (P.fw[r] & FW_GEN) != 0;   // mark flags only regions with newlines
    if (general) s_x[warp][lane] = *reinterpret_cast<const ulonglong2 *>(P.lf + r * LF_STRIDE);
    uint32_t gm = __ballot_sync(0xffffffffu, general);
    while (gm) {
        const int f = __ffs(gm) - 1;
        gm &= gm - 1u;
        full_region<0>(P.self, 0, R0 + f, s_x[warp][f]);
    }
}

// ---- FASTA finalize: per-record fields from neighbouring headers + event summary ------------
// blen  = next header start - boff (or end position)                       index.c:243,348
// slen  = blen - n_lines * elen  (sum over lines of len - elen + 1)        index.c:335-338
// norm  = [#lines differing from the first <= 1], from the events (DESIGN.md proof)  index.c:325-342
// The row count comes from the device totals (grid-stride), so the host never waits for it.
__global__ void __launch_bounds__(256) fasta_finalize_kernel(const FastaTmp *tmp, int64_t tmp_cap, int64_t rows_cap,
                                                             int64_t base_offset, ScanTotals *tot, fxg_fasta_row *rows) {
    int64_t nrows = (int64_t)tot->hdr;
    if (nrows > rows_cap || nrows + 1 > tmp_cap) nrows = 0;        // capacity miss: the host regrows and reruns phase B
    unsigned long long slen_acc = 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += stride) {
        const FastaTmp t = tmp[r + 1];
        int64_t next_h, next_line;
        if (r + 1 < nrows) {
            const FastaTmp nx = tmp[r + 2];
            next_h = nx.boff - (1 + nx.dlen + (int64_t)nx.elen);
            next_line = nx.lineidx;
        } else {
            next_h = base_offset + tot->n_eff;
            next_line = (int64_t)tot->nl;
        }
        const int64_t blen = next_h - t.boff;
        const int64_t nlines = next_line - t.lineidx - 1;
        const int64_t slen = blen - nlines * (int64_t)t.elen;
        int norm;
        if (t.D == 0) norm = 1;
        else if (t.D == 1) norm = ((int64_t)t.evmax == t.lineidx + nlines) ? 1 : 0;
        else if (t.D == 2) norm = ((t.evmax - (~t.evminc) == 1) && t.S == 0) ? 1 : 0;
        else norm = 0;
        fxg_fasta_row o;
        o.boff = t.boff; o.blen = blen; o.slen = slen; o.llen = t.llen;
        o.dlen = t.dlen; o.nlen = t.nlen; o.elen = (uint8_t)t.elen; o.norm = (uint8_t)norm;
        for (int i = 0; i < 6; ++i) o.pad[i] = 0;
        // uniform lines: no length change at all, or a single SHORTER line at the very end
        o.pad[0] = (t.D == 0 || (t.D == 1 && (int64_t)t.evmax == t.lineidx + nlines && (int64_t)t.S < 0)) ? 1 : 0;
        rows[r] = o;
        slen_acc += (unsigned long long)slen;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) slen_acc += (unsigned long long)shfl_down_i64((int64_t)slen_acc, d);
    if ((threadIdx.x & 31) == 0 && slen_acc) atomicAdd((unsigned long long *)&tot->sum_len, slen_acc);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        // lead part = lines before the first header of this buffer (multi-GPU shard merge)
        const FastaTmp l = tmp[0];
        tot->lead_llen = l.llen;
        if (nrows > 0) {
            const FastaTmp f = tmp[1];
            tot->lead_lines = f.lineidx;
            tot->lead_bytes = f.boff - base_offset - (1 + f.dlen + (int64_t)f.elen);
        }
    }
}

// ---- phase A tail: what this shard tells the others (fxg_shard_info), one warp ----------------
// The first up-to-three lines are read off the newline list (or the bytes of a dense region).
__global__ void __launch_bounds__(32) edge_kernel(const ScanParams P, int mode, fxg_shard_info *info) {
    const int lane = threadIdx.x;
    int found = 0;
    int64_t pos[3] = {0, 0, 0};
    for (int64_t r0 = 0; r0 < P.nreg && found < 3; r0 += 32) {
        const int64_t r = r0 + lane;
        const uint32_t c = r < P.nreg ? (P.rc[r].x & 0xffffu) : 0u;
        uint32_t nz = __ballot_sync(0xffffffffu, c != 0);
        while (nz && found < 3) {
            const int fl = __ffs(nz) - 1;
            nz &= nz - 1;
            const int64_t q = r0 + fl;
            // the region's bytes, 16 per lane and 512 per step (FASTA keeps no newline list for most regions)
            for (int64_t x0 = q * REGION; x0 < q * REGION + REGION && found < 3; x0 += 512) {
                const int64_t x = x0 + lane * 16;
                uint32_t m = 0;                                // bit i: byte x + i is a newline
                if (x + 16 <= P.n) {
                    const uint4 v = *reinterpret_cast<const uint4 *>(P.file + x);
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int i = 0; i < 16; ++i) m |= (((w[i >> 2] >> (8 * (i & 3))) & 0xffu) == '\n' ? 1u : 0u) << i;
                } else {
                    for (int i = 0; i < 16; ++i) m |= (nl_at(P, x + i) ? 1u : 0u) << i;
                }
                uint32_t any = __ballot_sync(0xffffffffu, m != 0);
                while (any && found < 3) {
                    const int fl2 = __ffs(any) - 1;
                    any &= any - 1u;
                    uint32_t mm = __shfl_sync(0xffffffffu, m, fl2);
                    while (mm && found < 3) { pos[found++] = x0 + fl2 * 16 + (__ffs(mm) - 1); mm &= mm - 1u; }
                }
            }
        }
    }
    if (lane == 0) {
        const ScanTotals t = *P.totals;
        fxg_shard_info o;
        o.n_rows = mode == 0 ? (int64_t)t.hdr : 0;
        o.n_lines = (int64_t)t.nl;
        o.bytes = P.n;
        o.base_offset = P.base_offset;
        o.end_position = t.n_eff;
        o.edge_n = found;
        int64_t start = 0;
        for (int j = 0; j < 3; ++j) {
            o.edge_off[j] = 0; o.edge_len[j] = 0;
            if (j < found) {
                const int64_t p = pos[j];
                const bool cr = p > start && p - 1 < P.n && P.file[p - 1] == '\r';
                o.edge_off[j] = P.base_offset + start;
                o.edge_len[j] = p - start - (cr ? 1 : 0);
                start = p + 1;
            }
        }
        for (int j = 0; j < 4; ++j) o.reserved[j] = 0;
        *info = o;
    }
}

// ---- phase B head: global line phase / row-slot count from the gathered shard infos -------------
__global__ void shard_prefix_kernel(const fxg_shard_info *all, int nranks, int rank, int mode, ScanTotals *tot) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int64_t F = 0, T = 0;
    for (int p = 0; p < nranks; ++p) {
        const int64_t nlp = all[p].n_lines;
        if (p < rank) F += nlp;
        T += nlp;
    }
    if (mode == 0) F = 0;                       // FASTA line indices stay buffer-local
    tot->first_line = F;
    tot->total_lines = T;
    const int64_t nl = (int64_t)tot->nl;
    tot->nrows = mode == 0 ? (int64_t)tot->hdr : (F + nl + 3) / 4 - F / 4;
    tot->sum_len = 0;                           // (re)accumulated by phase B
}

// zero what phase B accumulates into: FASTA record slots; FASTQ the two possibly partial boundary rows
__global__ void __launch_bounds__(256) clear_kernel(const ScanParams P, int mode, int64_t tmp_slots) {
    const int64_t nrows = P.totals->nrows;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (mode == 0) {
        int64_t slots = nrows + 2;
        if (slots > tmp_slots) slots = tmp_slots;
        uint4 *p = reinterpret_cast<uint4 *>(P.tmp);
        for (int64_t i = t0; i < slots * 4; i += stride) p[i] = make_uint4(0u, 0u, 0u, 0u);
    } else if (t0 < 4) {
        const int64_t row = t0 < 2 ? 0 : nrows - 1;
        if (row >= 0 && row < P.qrows_cap) reinterpret_cast<uint4 *>(P.qrows + row)[t0 & 1] = make_uint4(0u, 0u, 0u, 0u);
    }
}

// ---- FASTQ boundary-row merge (one thread): a read belongs to the shard that holds its name line; the lines
//      of the shard's last read that lie in later shards come from those shards' edge lines (fastq.c:122-133) ----
__global__ void fastq_stitch_kernel(const ScanParams P, const fxg_shard_info *all, int nranks, int rank) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    ScanTotals *tot = P.totals;
    const int64_t F = tot->first_line, n = (int64_t)tot->nl, T = tot->total_lines;
    const int64_t first_read = (F + 3) / 4;                    // first read whose name line is >= F
    int64_t last_read = n > 0 ? (F + n - 1) / 4 : first_read - 1;   // last read whose name line is < F + n
    if (last_read > T / 4 - 1) last_read = T / 4 - 1;          // only complete reads are rows (fastq.c:132-146,159)
    const int64_t owned = last_read >= first_read ? last_read - first_read + 1 : 0;
    tot->row0 = first_read - F / 4;
    tot->n_owned = owned;
    if (owned == 0) return;
    const int64_t row = last_read - F / 4;
    if (row >= P.qrows_cap) return;
    for (int ph = 1; ph <= 3; ph += 2) {
        const int64_t g = 4 * last_read + ph;
        if (g < F + n) continue;                               // the line is ours: already written
        int64_t Fp = F + n;
        for (int p = rank + 1; p < nranks; ++p) {
            const int64_t np = all[p].n_lines;
            if (g < Fp + np) {
                const int64_t j = g - Fp;
                if (j < all[p].edge_n) {
                    if (ph == 1) { P.qrows[row].soff = all[p].edge_off[j]; P.qrows[row].rlen = all[p].edge_len[j]; }
                    else P.qrows[row].qoff = all[p].edge_off[j];
                }
                break;
            }
            Fp += np;
        }
    }
}

// ---- split point on resident data: first line start (or header line start) at or after `from` ----
__global__ void __launch_bounds__(256) split_point_kernel(const uint8_t *file, int64_t n, int64_t from, int want_header,
                                                          long long *out) {
    __shared__ long long s_best;
    if (threadIdx.x == 0) s_best = LLONG_MAX;
    __syncthreads();
    if (from <= 0) {
        if (!want_header || (n > 0 && file[0] == '>')) { if (threadIdx.x == 0) *out = 0; return; }
        from = 1;
    }
    for (int64_t c0 = from - 1; c0 < n; c0 += 256 * 16) {
        const int64_t a = c0 + threadIdx.x * 16;
        long long mine = LLONG_MAX;
        for (int i = 0; i < 16; ++i) {
            const int64_t x = a + i;
            if (x < n && file[x] == '\n' && (!want_header || (x + 1 < n && file[x + 1] == '>'))) { mine = x + 1; break; }
        }
        if (mine != LLONG_MAX) atomicMin(&s_best, mine);
        __syncthreads();
        if (s_best != LLONG_MAX) break;
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = s_best == LLONG_MAX ? n : s_best;
}

}  // namespace fxg

// =============================================================================================
// host side
// =============================================================================================
using namespace fxg;

// Row capacity policy: phase B is launched without knowing the row count on the host.  The buffers are
// grow-only; a first scan of a file sizes them from the byte count (typical records), every kernel bounds
// checks against the capacity, and a miss (known at the single synchronisation) regrows and reruns phase B.
static int64_t guess_rows(int mode, int64_t n) { return (mode == 0 ? n / 1024 : n / 200) + 4096; }

static int scan_params(fxg_ctx *ctx, const fxg_file *f, int mode, int64_t base_offset, int flags, bool reserve,
                       ScanParams *out, int64_t *tmp_slots) {
    const int64_t n = f->size;
    const int64_t nreg = (n + 1 + REGION - 1) / REGION;     // room for a virtual newline at n
    const int64_t nb = (nreg + PS_BLOCK - 1) / PS_BLOCK;
    const int64_t nreg_pad = nb * PS_BLOCK;
    // tile_desc: rc[nreg_pad] | bs[nb] | FASTQ: ex[nreg];  FASTA: fw[nreg_pad] | gblk[nb] | lf[nreg * LF_STRIDE]
    const size_t off_bs = fxg_round_up((int64_t)nreg_pad * 8, 256);
    const size_t off_x = off_bs + fxg_round_up(nb * (int64_t)sizeof(ulonglong2), 256);
    const size_t off_gb = off_x + fxg_round_up(nreg_pad * (int64_t)sizeof(uint32_t), 256);
    const size_t off_lf = off_gb + fxg_round_up(nb * (int64_t)sizeof(uint32_t), 256);
    const size_t tile_bytes = mode == 0 ? off_lf + (size_t)nreg * LF_STRIDE * sizeof(uint2) : off_x + (size_t)nreg * sizeof(ulonglong2);
    int rc;
    if (reserve) {
        if ((rc = ctx->counters.reserve(1024))) return rc;
        if ((rc = ctx->tile_desc.reserve(tile_bytes))) return rc;
        if ((rc = ctx->seg.reserve((size_t)nreg * SEGCAP * sizeof(uint16_t)))) return rc;
        const int64_t want = guess_rows(mode, n);
        if (mode == 0) {
            if (ctx->row_tmp.cap < (size_t)(want + 2) * sizeof(FastaTmp) && (rc = ctx->row_tmp.reserve((size_t)(want + 2) * sizeof(FastaTmp)))) return rc;
            if (ctx->rows.cap < (size_t)(want + 1) * sizeof(fxg_fasta_row) && (rc = ctx->rows.reserve((size_t)(want + 1) * sizeof(fxg_fasta_row)))) return rc;
        } else if (ctx->rows.cap < (size_t)(want + 2) * sizeof(fxg_fastq_row)) {
            if ((rc = ctx->rows.reserve((size_t)(want + 2) * sizeof(fxg_fastq_row)))) return rc;
        }
    }
    ScanParams P;
    memset(&P, 0, sizeof(P));
    P.file = f->d; P.n = n; P.capacity = f->capacity & ~(int64_t)15; P.nreg = nreg;
    P.base_offset = base_offset; P.first_line = 0; P.flags = flags;
    P.rc = (uint2 *)ctx->tile_desc.ptr;
    P.bs = (ulonglong2 *)((uint8_t *)ctx->tile_desc.ptr + off_bs);
    if (mode == 0) {
        P.fw = (uint32_t *)((uint8_t *)ctx->tile_desc.ptr + off_x);
        P.gblk = (uint32_t *)((uint8_t *)ctx->tile_desc.ptr + off_gb);
        P.lf = (uint2 *)((uint8_t *)ctx->tile_desc.ptr + off_lf);
    } else {
        P.ex = (ulonglong2 *)((uint8_t *)ctx->tile_desc.ptr + off_x);
    }
    P.seg = (uint16_t *)ctx->seg.ptr;
    P.totals = (ScanTotals *)((uint8_t *)ctx->counters.ptr + 64);
    *tmp_slots = 0;
    if (mode == 0) {
        *tmp_slots = (int64_t)(ctx->row_tmp.cap / sizeof(FastaTmp));
        P.tmp = (FastaTmp *)ctx->row_tmp.ptr;
        P.tmp_cap = *tmp_slots - 1;                              // slots 0 .. tmp_cap-1 are written
    } else {
        P.qrows = (fxg_fastq_row *)ctx->rows.ptr;
        P.qrows_cap = (int64_t)(ctx->rows.cap / sizeof(fxg_fastq_row));
    }
    *out = P;
    return FXG_OK;
}

static fxg_shard_info *own_info(fxg_ctx *ctx) { return (fxg_shard_info *)((uint8_t *)ctx->counters.ptr + 256); }

// phase A: mark + prefix + edge.  No host synchronisation.
extern "C" int fxg_scan_begin(fxg_ctx *ctx, const fxg_file *f, int mode, int64_t base_offset, int flags,
                              fxg_shard_info *d_info_out) {
    FXG_CHECK_ARG(ctx && f && (mode == 0 || mode == 1), "null ctx/file or bad mode");
    FXG_LOCK(ctx);
    FXG_CUDA(cudaSetDevice(ctx->device));
    ctx->run.active = false;
    ScanParams P;
    int64_t tmp_slots;
    int rc = scan_params(ctx, f, mode, base_offset, flags, true, &P, &tmp_slots);
    if (rc) return rc;
    const int64_t n = f->size, nreg = P.nreg;
    const int64_t nb = (nreg + PS_BLOCK - 1) / PS_BLOCK, nreg_pad = nb * PS_BLOCK;
    FXG_CUDA(cudaMemsetAsync(ctx->counters.ptr, 0, 1024, ctx->stream));
    if (nreg_pad > nreg) FXG_CUDA(cudaMemsetAsync(P.rc + nreg, 0, (size_t)(nreg_pad - nreg) * 8, ctx->stream));
    const unsigned grid = (unsigned)((nreg + MARK_WARPS - 1) / MARK_WARPS);
    {
        FxgProfScope prof(ctx, FXG_PROF_SCAN);
        // pass-1 variant per format: V1 is the faster one for FASTA, V2 for FASTQ (DESIGN.md section 3)
        if (mode == 0) mark_kernel<0, 1><<<grid, MARK_WARPS * 32, 0, ctx->stream>>>(P);
        else mark_kernel<1, 2><<<grid, MARK_WARPS * 32, 0, ctx->stream>>>(P);
    }
    FXG_CUDA(cudaGetLastError());
    {
        FxgProfScope prof(ctx, FXG_PROF_PREFIX, mode == 0 ? 3 : 4);
        prefix_reduce_kernel<<<(unsigned)nb, PS_THREADS, 0, ctx->stream>>>(P.rc, P.bs);
        prefix_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(P.bs, nb, P.file, n, mode, P.totals);
        // FASTA: the rows pass scans the region counts itself (fasta_rows_kernel)
        if (mode == 1) prefix_expand_kernel<<<(unsigned)nb, PS_THREADS, 0, ctx->stream>>>(P.rc, P.bs, P.ex, nreg);
        edge_kernel<<<1, 32, 0, ctx->stream>>>(P, mode, own_info(ctx));
    }
    FXG_CUDA(cudaGetLastError());
    if (d_info_out)
        FXG_CUDA(cudaMemcpyAsync(d_info_out, own_info(ctx), sizeof(fxg_shard_info), cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->run.active = true; ctx->run.mode = mode; ctx->run.flags = flags; ctx->run.file = f; ctx->run.base_offset = base_offset;
    return FXG_OK;
}

static int launch_phase_b(fxg_ctx *ctx, const ScanParams &P0, int mode, int64_t tmp_slots, const fxg_shard_info *d_all,
                          int nranks, int rank) {
    // the parameter block also goes to global memory (P.self) for the rare noinline paths of the rows kernels
    int rc0 = ctx->params.reserve(512);
    if (rc0) return rc0;
    if (!ctx->h_counters) FXG_CUDA(cudaHostAlloc(&ctx->h_counters, 8192, cudaHostAllocDefault));
    ScanParams P = P0;
    P.self = (const ScanParams *)ctx->params.ptr;
    static_assert(sizeof(ScanParams) <= 512, "ScanParams staging");
    memcpy((uint8_t *)ctx->h_counters + 4096, &P, sizeof(P));
    FXG_CUDA(cudaMemcpyAsync(ctx->params.ptr, (uint8_t *)ctx->h_counters + 4096, sizeof(P), cudaMemcpyHostToDevice, ctx->stream));
    const int64_t nreg = P.nreg;
    {
        FxgProfScope prof(ctx, FXG_PROF_LINES, mode == 0 ? 4 : 3);
        shard_prefix_kernel<<<1, 32, 0, ctx->stream>>>(d_all, nranks, rank, mode, P.totals);
        clear_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(P, mode, tmp_slots);
        if (mode == 0) {
            const int64_t nb = (nreg + PS_BLOCK - 1) / PS_BLOCK;
            fasta_rows_kernel<<<(unsigned)nb, ROWS_THREADS, 0, ctx->stream>>>(P);
            fasta_general_kernel<<<(unsigned)((nreg + MARK_WARPS * 32 - 1) / (MARK_WARPS * 32)), MARK_WARPS * 32, 0, ctx->stream>>>(P);
        } else {
            const unsigned lgrid = (unsigned)((nreg + MARK_WARPS * RG - 1) / (MARK_WARPS * RG));
            fastq_records_kernel<<<lgrid, MARK_WARPS * 32, 0, ctx->stream>>>(P);
        }
    }
    FXG_CUDA(cudaGetLastError());
    {
        FxgProfScope prof(ctx, FXG_PROF_FINALIZE);
        if (mode == 0)
            fasta_finalize_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(
                P.tmp, P.tmp_cap, (int64_t)(ctx->rows.cap / sizeof(fxg_fasta_row)), P.base_offset, P.totals,
                (fxg_fasta_row *)ctx->rows.ptr);
        else
            fastq_stitch_kernel<<<1, 32, 0, ctx->stream>>>(P, d_all, nranks, rank);
    }
    FXG_CUDA(cudaGetLastError());
    return FXG_OK;
}

// phase B + collect: ONE host synchronisation (two when a capacity guess was too small)
extern "C" int fxg_scan_finish(fxg_ctx *ctx, const fxg_shard_info *d_all, int nranks, int rank, void **d_rows_out,
                               fxg_scan_stats *stats, fxg_shard_info *all_host) {
    FXG_CHECK_ARG(ctx && stats && nranks >= 1 && rank >= 0 && rank < nranks, "bad arguments");
    FXG_LOCK(ctx);
    FXG_CHECK_ARG(ctx->run.active, "fxg_scan_finish without fxg_scan_begin");
    FXG_CUDA(cudaSetDevice(ctx->device));
    ctx->run.active = false;
    const int mode = ctx->run.mode;
    const fxg_file *f = ctx->run.file;
    if (!d_all) { FXG_CHECK_ARG(nranks == 1, "d_all == NULL with more than one rank"); d_all = own_info(ctx); }
    memset(stats, 0, sizeof(*stats));
    if (d_rows_out) *d_rows_out = nullptr;
    if (!ctx->h_counters) FXG_CUDA(cudaHostAlloc(&ctx->h_counters, 8192, cudaHostAllocDefault));
    FXG_CHECK_ARG((size_t)nranks * sizeof(fxg_shard_info) + 256 <= 4096 || !all_host, "too many ranks for all_host");
    ScanTotals *ht = (ScanTotals *)ctx->h_counters;
    fxg_shard_info *hall = (fxg_shard_info *)((uint8_t *)ctx->h_counters + 256);
    for (int attempt = 0; attempt < 2; ++attempt) {
        ScanParams P;
        int64_t tmp_slots;
        int rc = scan_params(ctx, f, mode, ctx->run.base_offset, ctx->run.flags, false, &P, &tmp_slots);
        if (rc) return rc;
        if ((rc = launch_phase_b(ctx, P, mode, tmp_slots, d_all, nranks, rank))) return rc;
        FXG_CUDA(cudaMemcpyAsync(ht, P.totals, sizeof(ScanTotals), cudaMemcpyDeviceToHost, ctx->stream));
        if (all_host)
            FXG_CUDA(cudaMemcpyAsync(hall, d_all, (size_t)nranks * sizeof(fxg_shard_info), cudaMemcpyDeviceToHost, ctx->stream));
        FXG_CUDA(cudaStreamSynchronize(ctx->stream));
        // capacity check (exact, after the fact)
        bool fits;
        if (mode == 0) fits = ht->nrows + 2 <= tmp_slots && (size_t)(ht->nrows + 1) * sizeof(fxg_fasta_row) <= ctx->rows.cap;
        else fits = ht->nrows <= P.qrows_cap;
        if (fits) break;
        if (attempt == 1) { fxg_set_error("row buffers still too small after regrowing"); return FXG_ENOMEM; }
        if (mode == 0) {
            if ((rc = ctx->row_tmp.reserve((size_t)(ht->nrows + 2) * sizeof(FastaTmp)))) return rc;
            if ((rc = ctx->rows.reserve((size_t)(ht->nrows + 1) * sizeof(fxg_fasta_row)))) return rc;
        } else if ((rc = ctx->rows.reserve((size_t)(ht->nrows + 2) * sizeof(fxg_fastq_row)))) return rc;
    }
    stats->n_lines = (int64_t)ht->nl;
    stats->end_position = ht->n_eff;
    stats->total_len = (int64_t)ht->sum_len;
    if (mode == 0) {
        stats->n_rows = ht->nrows;
        stats->lead_llen = ht->lead_llen;
        if (ht->nrows > 0) { stats->lead_lines = ht->lead_lines; stats->lead_bytes = ht->lead_bytes; }
        else { stats->lead_lines = (int64_t)ht->nl; stats->lead_bytes = f->size; }
        if (d_rows_out) *d_rows_out = ctx->rows.ptr;
    } else {
        stats->n_rows = ht->n_owned;                 // complete reads whose name line lies in this shard
        stats->lead_lines = ht->first_line;          // global index of the shard's first line
        stats->reserved = ht->total_lines;
        if (d_rows_out) *d_rows_out = (fxg_fastq_row *)ctx->rows.ptr + ht->row0;
    }
    if (all_host) memcpy(all_host, hall, (size_t)nranks * sizeof(fxg_shard_info));
    return FXG_OK;
}

extern "C" int fxg_scan_sharded(fxg_ctx *ctx, fxg_comm *comm, const fxg_file *f, int mode, int64_t base_offset, int flags,
                                void **d_rows_out, fxg_scan_stats *stats, fxg_shard_info *all_host) {
    FXG_CHECK_ARG(ctx && f && stats, "null ctx/file/stats");
    FXG_LOCK(ctx);
    const int nranks = comm ? fxg_comm_nranks(comm) : 1, rank = comm ? fxg_comm_rank(comm) : 0;
    int rc = ctx->misc.reserve((size_t)nranks * sizeof(fxg_shard_info) + 256);
    if (rc) return rc;
    fxg_shard_info *d_all = (fxg_shard_info *)ctx->misc.ptr;
    if ((rc = fxg_scan_begin(ctx, f, mode, base_offset, flags, nullptr))) return rc;
    if ((rc = fxg_shard_exchange(ctx, comm, own_info(ctx), d_all, sizeof(fxg_shard_info)))) return rc;
    if ((rc = fxg_scan_finish(ctx, d_all, nranks, rank, d_rows_out, stats, all_host))) return rc;
    return comm ? fxg_comm_check(comm) : FXG_OK;
}

extern "C" int fxg_fasta_scan(fxg_ctx *ctx, const fxg_file *f, int64_t base_offset, int flags,
                              fxg_fasta_row **d_rows_out, fxg_scan_stats *stats) {
    FXG_CHECK_ARG(ctx && f && stats, "null ctx/file/stats");
    FXG_LOCK(ctx);
    int rc = fxg_scan_begin(ctx, f, 0, base_offset, flags, nullptr);
    if (rc) return rc;
    return fxg_scan_finish(ctx, nullptr, 1, 0, (void **)d_rows_out, stats, nullptr);
}

extern "C" int fxg_fastq_scan(fxg_ctx *ctx, const fxg_file *f, int64_t base_offset,
                              fxg_fastq_row **d_rows_out, fxg_scan_stats *stats) {
    FXG_CHECK_ARG(ctx && f && stats, "null ctx/file/stats");
    FXG_LOCK(ctx);
    int rc = fxg_scan_begin(ctx, f, 1, base_offset, 0, nullptr);
    if (rc) return rc;
    return fxg_scan_finish(ctx, nullptr, 1, 0, (void **)d_rows_out, stats, nullptr);
}

extern "C" int fxg_split_point_dev(fxg_ctx *ctx, const fxg_file *f, int64_t from, int want_header, int64_t *pos) {
    FXG_CHECK_ARG(ctx && f && pos && from >= 0, "bad arguments");
    FXG_LOCK(ctx);
    FXG_CUDA(cudaSetDevice(ctx->device));
    if (from >= f->size) { *pos = f->size; return FXG_OK; }
    int rc;
    if ((rc = ctx->counters.reserve(1024))) return rc;
    long long *d = (long long *)((uint8_t *)ctx->counters.ptr + 512);
    ctx->launches += 1;
    split_point_kernel<<<1, 256, 0, ctx->stream>>>(f->d, f->size, from, want_header, d);
    FXG_CUDA(cudaGetLastError());
    long long h = 0;
    FXG_CUDA(cudaMemcpyAsync(&h, d, 8, cudaMemcpyDeviceToHost, ctx->stream));
    FXG_CUDA(cudaStreamSynchronize(ctx->stream));
    *pos = (int64_t)h;
    return FXG_OK;
}
