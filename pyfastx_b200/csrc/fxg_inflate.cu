// fxg_inflate.cu -- K6: DEFLATE decoding on the GPU (sm_90a), for BGZF members and for plain gzip from checkpoints.
//
// Replaces, for block-gzipped inputs, the reference's zlib read side: gzread during the index scan
// (src/kseq.c:70) and zran_seek + zran_read per random access (src/index.c:685-686,
// src/read.c:39-40).  A BGZF file is a series of independent gzip members (<= 64 KiB of output
// each) whose sizes are in the 'BC' extra field, so
//   * the host walks the member headers (no inflation) and gets, per member, the compressed range
//     and -- from the ISIZE trailer -- the uncompressed offset: this is the checkpoint table that
//     zran would have to inflate the whole file for (src/index.c:381-387);
//   * one THREAD per member inflates it straight into its slot of the uncompressed HBM buffer
//     (inflate_thread_kernel, with the fxi::Decoder of fxg_inflate_core.cuh);
//   * crc_members_kernel checks every member's output against its gzip trailer;
//   * the K1/K2 scans and K3/K5 gathers then run on that buffer exactly as for plain files.
// A plain (non-BGZF) gzip stream has no independent entry points until one serial pass has recorded
// checkpoints (csrc/fxg_gzip.cpp); with those, inflate_points_kernel decodes a segment per thread.
#include "fxg_common.cuh"
#include <zlib.h>
#include <vector>
#include "fxg_inflate_core.cuh"
#include <stdlib.h>
#include <string.h>

namespace fxg {

// ---- a thread per member -----------------------------------------------------------------------------
// The Huffman decode of one member is serial: a warp working on one member would issue every instruction
// for ONE useful lane.  Here 32 members share a warp: each lane runs an fxi::Decoder on its own member
// with its own 2.2 KB of decode tables; up to 1,152 members are in flight per SM.
__device__ const uint16_t D_LEN_BASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__device__ const uint8_t D_LEN_EXTRA[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__device__ const uint16_t D_DIST_BASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__device__ const uint8_t D_DIST_EXTRA[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__device__ const uint8_t D_CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

constexpr int MT_THREADS = 64;                                      // members per CTA
#ifndef FXG_MT_WARPS
#define FXG_MT_WARPS 36
#endif
constexpr int MT_WARPS_PER_SM = FXG_MT_WARPS;                                 // resident warps the launch aims for: 36 is the most
                                                                    // the register file holds at 56 registers; on 132 SMs that is 152,064
                                                                    // members per round (C5's 155,577: one round and a short tail)
constexpr int SYM_BATCH = 32;                                      // symbols per lane between member / block checks

__global__ void __launch_bounds__(MT_THREADS, MT_WARPS_PER_SM * 32 / MT_THREADS) inflate_thread_kernel(const uint8_t *__restrict__ in, int64_t in_size,
                                                                   const int64_t *__restrict__ cmp_off,
                                                                   const int64_t *__restrict__ ucmp_off, int64_t n_members,
                                                                   uint8_t *out, int64_t out_cap, int32_t *__restrict__ status,
                                                                   fxi::MemberTables *tables) {
    // decode tables live in global memory (2.2 KB per lane, L1/L2 resident where hot): shared memory would
    // cap the SM at ~96 members in flight, far too few to hide the latency of the serial decode chains
    fxi::MemberTables &T = tables[(size_t)blockIdx.x * MT_THREADS + threadIdx.x];
    const fxi::DeflateConsts K = {D_LEN_BASE, D_LEN_EXTRA, D_DIST_BASE, D_DIST_EXTRA, D_CL_ORDER};
    const int64_t step = (int64_t)gridDim.x * MT_THREADS;
    int64_t m = (int64_t)blockIdx.x * MT_THREADS + threadIdx.x;
    fxi::Decoder d;
    d.state = fxi::Decoder::DONE; d.status = 0;
    bool have = false, finished = false;
    // All lanes advance in lock step -- one symbol per lane and step, reconverging after every step -- so
    // the warp never splits into fragments that the scheduler would run one after the other.
    for (;;) {
        if (d.state == fxi::Decoder::DONE) {                       // next member for this lane
            if (have) { status[m] = d.status; m += step; have = false; }
            if (!finished) {
                if (m < n_members) { d.begin(in, in_size, cmp_off[m], cmp_off[m + 1], out_cap, ucmp_off[m], ucmp_off[m + 1]); have = true; }
                else finished = true;
            }
        }
        if (__all_sync(0xffffffffu, finished)) break;
        if (d.state == fxi::Decoder::NEED_BLOCK) d.begin_block(out, T, K);
        __syncwarp();
#pragma unroll 1
        for (int k = 0; k < SYM_BATCH; ++k) {
            if (d.state == fxi::Decoder::SYMBOLS) d.step_symbol(out, out_cap, T, K);
            __syncwarp();
        }
    }
}

// ---- CRC-32 of every member's output against its gzip trailer (zlib, which the reference reads through, rejects a
//      member whose CRC does not match; a bit flip that still decodes to the right length must not reach the index) ----
// One thread per member, slicing-by-4 with the four 256-entry tables in shared memory; 16-byte loads once the output
// pointer is aligned.  Sets status 9 for a member whose inflate status was 0 and whose CRC differs.
constexpr int CRC_THREADS = 128;

// The four slicing-by-4 tables of CRC-32 (polynomial 0xEDB88320), built by the whole CTA into shared memory.
__device__ __forceinline__ void crc_build_tables(uint32_t (*T)[256]) {
    for (int i = threadIdx.x; i < 256; i += CRC_THREADS) {
        uint32_t c = (uint32_t)i;
        for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
        T[0][i] = c;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += CRC_THREADS) {
        uint32_t c = T[0][i];
        for (int t = 1; t < 4; ++t) { c = T[0][c & 0xffu] ^ (c >> 8); T[t][i] = c; }
    }
    __syncthreads();
}

// CRC-32 of p[0, len): bytewise up to 16-byte alignment, then four words per 16-byte load, then the tail bytewise.
__device__ __forceinline__ uint32_t crc32_range(const uint32_t (*T)[256], const uint8_t *p, int64_t len) {
    uint32_t crc = 0xffffffffu;
    auto word = [&](uint32_t w) {
        crc ^= w;
        crc = T[3][crc & 0xffu] ^ T[2][(crc >> 8) & 0xffu] ^ T[1][(crc >> 16) & 0xffu] ^ T[0][crc >> 24];
    };
    while (len > 0 && (reinterpret_cast<uintptr_t>(p) & 15u)) { crc = T[0][(crc ^ *p) & 0xffu] ^ (crc >> 8); ++p; --len; }
    for (; len >= 16; len -= 16, p += 16) {
        const uint4 v = *reinterpret_cast<const uint4 *>(p);
        word(v.x); word(v.y); word(v.z); word(v.w);
    }
    for (; len > 0; --len, ++p) crc = T[0][(crc ^ *p) & 0xffu] ^ (crc >> 8);
    return ~crc;
}

__global__ void __launch_bounds__(CRC_THREADS) crc_members_kernel(const uint8_t *__restrict__ comp, const int64_t *__restrict__ cmp_off,
                                                                  const int64_t *__restrict__ ucmp_off, int64_t n_members,
                                                                  const uint8_t *__restrict__ out, int32_t *__restrict__ status) {
    __shared__ uint32_t T[4][256];
    crc_build_tables(T);
    const int64_t m = (int64_t)blockIdx.x * CRC_THREADS + threadIdx.x;
    if (m >= n_members || status[m] != 0) return;
    const uint32_t crc = crc32_range(T, out + ucmp_off[m], ucmp_off[m + 1] - ucmp_off[m]);
    const uint8_t *t = comp + cmp_off[m + 1] - 8;                      // CRC32, ISIZE: the last eight bytes of the member
    const uint32_t want = (uint32_t)t[0] | ((uint32_t)t[1] << 8) | ((uint32_t)t[2] << 16) | ((uint32_t)t[3] << 24);
    if (crc != want) status[m] = 9;
}

// ---- generic gzip: one thread per zran checkpoint (SURVEY.md section 8f-4) ----
// A plain .gz file is one serial deflate stream; its checkpoints (compressed offset, bit offset, the 32 KiB of output in
// front of it -- collected by the one sequential pass of csrc/fxg_gzip.cpp, or loaded from the `.fxi`) are independent
// entry points: every thread decodes the segment from its checkpoint to the next one (both deflate block boundaries)
// into the shared output buffer, taking the bytes its first matches reach back to from the checkpoint's window.  The
// same fxi::Decoder as the BGZF kernel, started with begin_at().  `seg_crc` receives the CRC-32 of every segment's
// output; the host combines them (crc32_combine) and compares with the gzip trailer.
__global__ void __launch_bounds__(64) inflate_points_kernel(const uint8_t *__restrict__ in, int64_t in_size, const int64_t *__restrict__ cmp_off,
                                                            const uint8_t *__restrict__ bits, const int64_t *__restrict__ ucmp_off,
                                                            const int32_t *__restrict__ win_index, const uint8_t *__restrict__ windows,
                                                            int wsize, int64_t n_points, uint8_t *out, int64_t out_cap,
                                                            int32_t *__restrict__ status, fxi::MemberTables *tables) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_points) return;
    const fxi::DeflateConsts K = {D_LEN_BASE, D_LEN_EXTRA, D_DIST_BASE, D_DIST_EXTRA, D_CL_ORDER};
    const int32_t wi = win_index[i];
    status[i] = fxi::inflate_segment(in, in_size, cmp_off[i], (int)bits[i], out, out_cap, ucmp_off[i], ucmp_off[i + 1],
                                     wi >= 0 ? windows + (size_t)wi * wsize : nullptr, wi >= 0 ? wsize : 0, tables[i], K);
}

// CRC-32 of out[off[i], off[i + 1]) per segment
__global__ void __launch_bounds__(CRC_THREADS) crc_segments_kernel(const int64_t *__restrict__ off, int64_t n, const uint8_t *__restrict__ out,
                                                                   uint32_t *__restrict__ crc_out) {
    __shared__ uint32_t T[4][256];
    crc_build_tables(T);
    const int64_t m = (int64_t)blockIdx.x * CRC_THREADS + threadIdx.x;
    if (m >= n) return;
    crc_out[m] = crc32_range(T, out + off[m], off[m + 1] - off[m]);
}

}  // namespace fxg

using namespace fxg;

// Host: walk the BGZF member headers.  cmp_off / ucmp_off receive n_members + 1 entries.
// Replaces the SECOND full inflate pass the reference needs to build its random-access
// checkpoints (zran_build_index, src/index.c:381-387): BGZF carries the member sizes in the headers.
extern "C" int fxg_bgzf_members_host(const void *host_buf, int64_t nbytes, int64_t *cmp_off, int64_t *ucmp_off,
                                     int64_t cap, int64_t *n_members, int64_t *total_uncompressed) {
    FXG_CHECK_ARG(host_buf && n_members && total_uncompressed && nbytes >= 0, "bad arguments");
    const uint8_t *b = (const uint8_t *)host_buf;
    int64_t p = 0, n = 0, u = 0;
    while (p < nbytes) {
        if (nbytes - p < 18 || b[p] != 0x1f || b[p + 1] != 0x8b || b[p + 2] != 8 || !(b[p + 3] & 4)) {
            fxg_set_error("not a BGZF member at offset %lld", (long long)p);
            return FXG_EFORMAT;
        }
        const int xlen = b[p + 10] | (b[p + 11] << 8);
        int64_t q = p + 12, xe = p + 12 + xlen;
        int64_t bsize = -1;
        while (q + 4 <= xe && xe <= nbytes) {
            const int slen = b[q + 2] | (b[q + 3] << 8);
            if (b[q] == 'B' && b[q + 1] == 'C' && slen == 2 && q + 6 <= xe) bsize = (b[q + 4] | (b[q + 5] << 8)) + 1;
            q += 4 + slen;
        }
        if (bsize < 0 || p + bsize > nbytes || bsize < xlen + 20) {
            fxg_set_error("gzip member without a valid BGZF 'BC' field at offset %lld", (long long)p);
            return FXG_EFORMAT;
        }
        const uint8_t *t = b + p + bsize - 4;
        const int64_t isize = (int64_t)t[0] | ((int64_t)t[1] << 8) | ((int64_t)t[2] << 16) | ((int64_t)t[3] << 24);
        if (n < cap) {
            if (cmp_off) cmp_off[n] = p;
            if (ucmp_off) ucmp_off[n] = u;
        }
        ++n;
        p += bsize;
        u += isize;
    }
    if (n < cap) {
        if (cmp_off) cmp_off[n] = p;
        if (ucmp_off) ucmp_off[n] = u;
    }
    *n_members = n;
    *total_uncompressed = u;
    return n + 1 <= cap || (!cmp_off && !ucmp_off) ? FXG_OK : FXG_ECAP;
}

extern "C" int fxg_inflate_members_dev(fxg_ctx *ctx, const fxg_file *compressed, const int64_t *d_cmp_off,
                                       const int64_t *d_ucmp_off, int64_t n_members, uint8_t *d_out, int64_t out_cap,
                                       int32_t *d_status) {
    FXG_CHECK_ARG(ctx && compressed && n_members >= 0, "bad arguments");
    FXG_LOCK(ctx);
    if (n_members == 0) return FXG_OK;
    FXG_CHECK_ARG(d_cmp_off && d_ucmp_off && d_out && d_status, "null device pointer");
    FXG_CUDA(cudaSetDevice(ctx->device));
    FxgProfScope prof(ctx, FXG_PROF_GATHER);
    int64_t blocks = (n_members + MT_THREADS - 1) / MT_THREADS;
    const int64_t maxb = (int64_t)ctx->sm_count * (MT_WARPS_PER_SM * 32 / MT_THREADS);
    if (blocks > maxb) blocks = maxb;
    int rc = ctx->misc.reserve((size_t)blocks * MT_THREADS * sizeof(fxi::MemberTables));
    if (rc) return rc;
    inflate_thread_kernel<<<(unsigned)blocks, MT_THREADS, 0, ctx->stream>>>(compressed->d, compressed->size, d_cmp_off, d_ucmp_off,
                                                                            n_members, d_out, out_cap, d_status,
                                                                            (fxi::MemberTables *)ctx->misc.ptr);
    FXG_CUDA(cudaGetLastError());
    const char *ce = getenv("FXG_BGZF_CRC");
    if (!(ce && ce[0] == '0')) {                                 // member CRCs against their trailers (status 9 = mismatch)
        ctx->launches += 1;
        crc_members_kernel<<<(unsigned)((n_members + CRC_THREADS - 1) / CRC_THREADS), CRC_THREADS, 0, ctx->stream>>>(
            compressed->d, d_cmp_off, d_ucmp_off, n_members, d_out, d_status);
        FXG_CUDA(cudaGetLastError());
    }
    return FXG_OK;
}

// Host-buffer convenience: BGZF bytes in host memory -> uncompressed fxg_file resident in HBM.
extern "C" int fxg_file_from_bgzf_host(fxg_ctx *ctx, const void *host_buf, int64_t nbytes, fxg_file **out,
                                       int64_t *n_members_out) {
    FXG_CHECK_ARG(ctx && host_buf && out, "bad arguments");
    FXG_LOCK(ctx);
    *out = nullptr;
    int64_t n = 0, total = 0;
    int rc = fxg_bgzf_members_host(host_buf, nbytes, nullptr, nullptr, 0, &n, &total);
    if (rc) return rc;
    int64_t *tab = (int64_t *)malloc((size_t)(n + 1) * 2 * sizeof(int64_t));
    if (!tab) { fxg_set_error("out of host memory"); return FXG_ENOMEM; }
    rc = fxg_bgzf_members_host(host_buf, nbytes, tab, tab + n + 1, n + 1, &n, &total);
    fxg_file *cf = nullptr, *uf = nullptr;
    void *d_tab = nullptr;
    int32_t *d_status = nullptr;
    int32_t *h_status = nullptr;
    if (!rc) rc = fxg_file_alloc_async(ctx, nbytes, &cf);           // the stream is synchronised below
    if (!rc) rc = fxg_file_upload_async(ctx, cf, 0, host_buf, nbytes);
    if (!rc) rc = fxg_file_alloc_async(ctx, total, &uf);
    if (!rc) rc = fxg_rows_upload(ctx, tab, (n + 1) * 2, (int)sizeof(int64_t), &d_tab);
    if (!rc && cudaMalloc((void **)&d_status, (size_t)(n + 1) * sizeof(int32_t)) != cudaSuccess) { fxg_set_error("cudaMalloc failed"); rc = FXG_ENOMEM; }
    if (!rc) rc = fxg_inflate_members_dev(ctx, cf, (const int64_t *)d_tab, (const int64_t *)d_tab + n + 1, n, uf->d, total, d_status);
    if (!rc && !(h_status = (int32_t *)malloc((size_t)(n + 1) * sizeof(int32_t)))) { fxg_set_error("out of host memory"); rc = FXG_ENOMEM; }
    if (!rc) {
        cudaError_t e = cudaMemcpyAsync(h_status, d_status, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { fxg_set_error("inflate failed: %s", cudaGetErrorString(e)); rc = FXG_ECUDA; }
        for (int64_t i = 0; !rc && i < n; ++i)
            if (h_status[i]) {
                fxg_set_error(h_status[i] == 9 ? "BGZF member %lld: CRC-32 of the inflated bytes differs from the member trailer (status %d)"
                                               : "BGZF member %lld is corrupt (inflate status %d)", (long long)i, h_status[i]);
                rc = FXG_EFORMAT;
            }
    }
    free(tab); free(h_status);
    if (d_tab) cudaFree(d_tab);
    if (d_status) cudaFree(d_status);
    if (cf) fxg_file_free(cf);
    if (rc) { if (uf) fxg_file_free(uf); return rc; }
    *out = uf;
    if (n_members_out) *n_members_out = n;
    return FXG_OK;
}

// Generic gzip with known checkpoints (from the `.fxi` of an earlier open, or from fxg_gzip_inflate_host): the compressed
// bytes go to the device and every checkpoint's segment is inflated by its own thread -- no sequential host pass.
// The CRC-32 of the result (per-segment CRCs combined on the host) must equal the gzip trailer's, as must the length;
// anything else returns FXG_EFORMAT and the caller takes the sequential host path.
extern "C" int fxg_file_from_gzip_points_host(fxg_ctx *ctx, const void *host_buf, int64_t nbytes, const fxg_gzindex *gz, fxg_file **out) {
    FXG_CHECK_ARG(ctx && host_buf && gz && out && nbytes >= 18, "bad arguments");
    FXG_LOCK(ctx);
    *out = nullptr;
    const int64_t n = gz->npoints, total = gz->uncompressed_size;
    FXG_CHECK_ARG(n >= 1 && total >= 0 && gz->cmp_offset && gz->uncmp_offset && gz->compressed_size == nbytes, "bad checkpoint table");
    const uint8_t *hb = (const uint8_t *)host_buf;
    const uint32_t want_crc = (uint32_t)hb[nbytes - 8] | ((uint32_t)hb[nbytes - 7] << 8) | ((uint32_t)hb[nbytes - 6] << 16) | ((uint32_t)hb[nbytes - 5] << 24);
    const uint32_t want_len = (uint32_t)hb[nbytes - 4] | ((uint32_t)hb[nbytes - 3] << 8) | ((uint32_t)hb[nbytes - 2] << 16) | ((uint32_t)hb[nbytes - 1] << 24);
    if (want_len != (uint32_t)total) { fxg_set_error("gzip trailer length differs from the checkpoint table's"); return FXG_EFORMAT; }
    std::vector<int64_t> uo((size_t)n + 1);
    std::vector<int32_t> wi((size_t)n, -1);
    std::vector<uint8_t> bt((size_t)n, 0);
    int64_t nw = 0;
    for (int64_t i = 0; i < n; ++i) {
        uo[(size_t)i] = gz->uncmp_offset[i];
        if (gz->bits) bt[(size_t)i] = gz->bits[i];
        if (gz->has_data && gz->has_data[i]) wi[(size_t)i] = (int32_t)nw++;
        if (i && (gz->uncmp_offset[i] <= gz->uncmp_offset[i - 1] || gz->cmp_offset[i] < gz->cmp_offset[i - 1])) { fxg_set_error("checkpoints out of order"); return FXG_EFORMAT; }
        if (i && !(gz->has_data && gz->has_data[i])) { fxg_set_error("checkpoint %lld has no window", (long long)i); return FXG_EFORMAT; }
    }
    uo[(size_t)n] = total;
    if (uo[0] != 0 || uo[(size_t)n - 1] >= total + (total == 0) || (nw && (gz->window_size != 32768 || !gz->windows))) { fxg_set_error("unusable checkpoint table"); return FXG_EFORMAT; }
    FXG_CUDA(cudaSetDevice(ctx->device));
    fxg_file *cf = nullptr, *uf = nullptr;
    void *d_co = nullptr, *d_uo = nullptr, *d_bt = nullptr, *d_wi = nullptr, *d_win = nullptr;
    int32_t *d_status = nullptr;
    uint32_t *d_crc = nullptr;
    std::vector<int32_t> h_status((size_t)n);
    std::vector<uint32_t> h_crc((size_t)n);
    int rc = fxg_file_alloc_async(ctx, nbytes, &cf);                // the stream is synchronised below
    if (!rc) rc = fxg_file_upload_async(ctx, cf, 0, host_buf, nbytes);
    if (!rc) rc = fxg_file_alloc_async(ctx, total, &uf);
    if (!rc) rc = fxg_rows_upload(ctx, gz->cmp_offset, n, 8, &d_co);
    if (!rc) rc = fxg_rows_upload(ctx, uo.data(), n + 1, 8, &d_uo);
    if (!rc) rc = fxg_rows_upload(ctx, bt.data(), n, 1, &d_bt);
    if (!rc) rc = fxg_rows_upload(ctx, wi.data(), n, 4, &d_wi);
    if (!rc && nw) rc = fxg_rows_upload(ctx, gz->windows, nw, (int)gz->window_size, &d_win);
    if (!rc && (cudaMalloc((void **)&d_status, (size_t)n * 4) != cudaSuccess || cudaMalloc((void **)&d_crc, (size_t)n * 4) != cudaSuccess)) { cudaGetLastError(); fxg_set_error("cudaMalloc failed"); rc = FXG_ENOMEM; }
    if (!rc) rc = ctx->misc.reserve((size_t)n * sizeof(fxi::MemberTables));
    if (!rc) {
        ctx->launches += 2;
        inflate_points_kernel<<<(unsigned)((n + 63) / 64), 64, 0, ctx->stream>>>(cf->d, cf->size, (const int64_t *)d_co, (const uint8_t *)d_bt,
                                                                               (const int64_t *)d_uo, (const int32_t *)d_wi, (const uint8_t *)d_win,
                                                                               (int)gz->window_size, n, uf->d, total, d_status,
                                                                               (fxi::MemberTables *)ctx->misc.ptr);
        crc_segments_kernel<<<(unsigned)((n + CRC_THREADS - 1) / CRC_THREADS), CRC_THREADS, 0, ctx->stream>>>((const int64_t *)d_uo, n, uf->d, d_crc);
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(h_status.data(), d_status, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(h_crc.data(), d_crc, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { fxg_set_error("inflate from checkpoints failed: %s", cudaGetErrorString(e)); rc = FXG_ECUDA; }
    }
    if (!rc) {
        uLong crc = crc32(0L, Z_NULL, 0);
        for (int64_t i = 0; i < n && !rc; ++i) {
            if (h_status[(size_t)i]) { fxg_set_error("segment %lld of the gzip stream is corrupt (inflate status %d)", (long long)i, h_status[(size_t)i]); rc = FXG_EFORMAT; }
            crc = crc32_combine(crc, (uLong)h_crc[(size_t)i], (z_off_t)(uo[(size_t)i + 1] - uo[(size_t)i]));
        }
        if (!rc && (uint32_t)crc != want_crc) { fxg_set_error("CRC-32 of the inflated bytes differs from the gzip trailer (several members, or stale checkpoints)"); rc = FXG_EFORMAT; }
    }
    for (void *p : {d_co, d_uo, d_bt, d_wi, d_win, (void *)d_status, (void *)d_crc}) if (p) cudaFree(p);
    if (cf) fxg_file_free(cf);
    if (rc) { if (uf) fxg_file_free(uf); return rc; }
    *out = uf;
    return FXG_OK;
}
