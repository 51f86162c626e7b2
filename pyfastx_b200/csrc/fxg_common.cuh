// fxg_common.cuh -- shared device helpers and host-side context for libfxg.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <mutex>
#include "../../include/fxg.h"

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
void fxg_set_error(const char *fmt, ...);
// fxg_file_alloc / fxg_file_upload without their closing stream synchronisation (fxg_api.cu), for library calls that
// synchronise the context's stream before they return
int fxg_file_alloc_async(fxg_ctx *c, int64_t nbytes, fxg_file **out);
int fxg_file_upload_async(fxg_ctx *c, fxg_file *f, int64_t dst_off, const void *host, int64_t nbytes);

#define FXG_CUDA(call)                                                                    \
    do {                                                                                  \
        cudaError_t e__ = (call);                                                         \
        if (e__ != cudaSuccess) {                                                         \
            fxg_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),        \
                          __FILE__, __LINE__);                                            \
            return (e__ == cudaErrorNoDevice || e__ == cudaErrorInsufficientDriver)       \
                       ? FXG_ENODEV : (e__ == cudaErrorMemoryAllocation ? FXG_ENOMEM : FXG_ECUDA); \
        }                                                                                 \
    } while (0)

#define FXG_CHECK_ARG(cond, msg)                                                          \
    do {                                                                                  \
        if (!(cond)) { fxg_set_error("invalid argument: %s", msg); return FXG_EINVAL; }   \
    } while (0)

// grow-only device scratch buffer
struct FxgScratch {
    void  *ptr = nullptr;
    size_t cap = 0;
    int reserve(size_t bytes);
    void release();
};

struct fxg_file {
    uint8_t *d = nullptr;   // device bytes; buffer capacity >= size rounded up to FXG_FILE_PAD
    int64_t  size = 0;
    int64_t  capacity = 0;   // logical capacity (zero padded up to here)
    int64_t  alloc_cap = 0;  // bytes really allocated (a pooled buffer may be larger than `capacity`)
    bool     owned = false;
    int      device = 0;
};

// state of a split-phase scan between fxg_scan_begin and fxg_scan_finish
struct FxgScanRun {
    bool     active = false;
    int      mode = 0, flags = 0;
    const fxg_file *file = nullptr;
    int64_t  base_offset = 0;
};

struct fxg_ctx {
    std::recursive_mutex mu;             // every entry point that touches scratch or the stream holds it
    FxgScanRun   run;
    int          device = 0;
    int          sm_count = 0;
    cudaStream_t stream = nullptr;
    bool         own_stream = false;
    // staging (pinned double buffers for pageable host memory)
    void        *pinned[2] = {nullptr, nullptr};
    size_t       pinned_bytes = 0;
    cudaEvent_t  pinned_ev[2] = {nullptr, nullptr};
    void        *ring = nullptr;         // pinned ring of the path stager (32 x 16 MiB), one event per slot
    cudaEvent_t  ring_ev[32] = {};
    // scan scratch
    FxgScratch   tile_desc, seg, row_tmp, rows, counters, params, plan, misc, stage_file;
    FxgScratch   search;                 // pattern search: per-item hit counts and offsets (fxg_search_host)
    void        *h_counters = nullptr;   // pinned, small
    void        *h_one = nullptr;        // pinned + mapped: output of single-query launches (fxg_extract_one_host)
    // single-query service (resident kernel fed through mapped host memory)
    void        *svc_req = nullptr, *svc_resp = nullptr;
    cudaStream_t svc_stream = nullptr;
    unsigned long long svc_next = 1;
    bool         svc_running = false;
    // measurement hooks
    bool         profiling = false;
    cudaEvent_t  prof_ev[FXG_PROF_SLOTS][2] = {};
    bool         prof_valid[FXG_PROF_SLOTS] = {};
    int64_t      launches = 0;
    int64_t      collectives = 0;
};

#define FXG_LOCK(ctx) std::lock_guard<std::recursive_mutex> fxg_lock__((ctx)->mu)

// brackets a kernel launch with events when profiling is on; always counts the launch
struct FxgProfScope {
    fxg_ctx *c; int slot;
    FxgProfScope(fxg_ctx *ctx, int s, int nlaunch = 1) : c(ctx), slot(s) {
        c->launches += nlaunch;
        if (c->profiling) cudaEventRecord(c->prof_ev[slot][0], c->stream);
    }
    ~FxgProfScope() {
        if (c->profiling) { cudaEventRecord(c->prof_ev[slot][1], c->stream); c->prof_valid[slot] = true; }
    }
};

static const int64_t FXG_FILE_PAD = 65536;   // device file buffers are padded with zeros

inline int64_t fxg_round_up(int64_t v, int64_t m) { return (v + m - 1) / m * m; }

// ---------------------------------------------------------------------------------------
// device side: PTX wrappers (mbarrier + 1-D TMA bulk copy), byte tricks
// ---------------------------------------------------------------------------------------
#ifdef __CUDACC__
namespace fxg {

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D TMA bulk copy global -> shared, completion counted on an mbarrier (SASS: UBLKCP).
// dst, src 16-byte aligned; bytes a multiple of 16.
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// 0x80 in every byte of w that equals `c` (c < 0x80).  Exact, 3 ALU ops when the constants
// live in registers (one LOP3 per boolean step):
//   u = (w ^ c4) & 0x7f7f7f7f ; t = u + 0x7f7f7f7f ; r = ~(t | w) & 0x80808080
__device__ __forceinline__ uint32_t byte_eq_mask_r(uint32_t w, uint32_t c4, uint32_t k7f, uint32_t k80) {
    uint32_t u, r;
    asm("lop3.b32 %0, %1, %2, %3, 0x28;" : "=r"(u) : "r"(w), "r"(c4), "r"(k7f));   // (a ^ b) & c
    const uint32_t t = u + k7f;
    asm("lop3.b32 %0, %1, %2, %3, 0x02;" : "=r"(r) : "r"(t), "r"(w), "r"(k80));    // ~(a | b) & c
    return r;
}
__device__ __forceinline__ uint32_t byte_eq_mask(uint32_t w, uint32_t c4) {
    uint32_t u = (w ^ c4) & 0x7f7f7f7fu;
    uint32_t t = u + 0x7f7f7f7fu;
    return ~(t | w) & 0x80808080u;
}
// Combined 16-bit-population word for a 16-byte chunk: bit (8*b + 7 - w) <-> byte 4*w + b.
__device__ __forceinline__ uint32_t chunk_eq_mask(const uint4 &v, uint32_t c4) {
    return byte_eq_mask(v.x, c4) | (byte_eq_mask(v.y, c4) >> 1) | (byte_eq_mask(v.z, c4) >> 2) |
           (byte_eq_mask(v.w, c4) >> 3);
}
// same with the three constants held in registers by the caller (hot loops)
__device__ __forceinline__ uint32_t chunk_eq_mask_r(const uint4 &v, uint32_t c4, uint32_t k7f, uint32_t k80) {
    return byte_eq_mask_r(v.x, c4, k7f, k80) | (byte_eq_mask_r(v.y, c4, k7f, k80) >> 1) |
           (byte_eq_mask_r(v.z, c4, k7f, k80) >> 2) | (byte_eq_mask_r(v.w, c4, k7f, k80) >> 3);
}
// keeps a constant in a register (defeats immediate folding)
__device__ __forceinline__ uint32_t reg_const(uint32_t v) {
    uint32_t r;
    asm volatile("mov.b32 %0, %1;" : "=r"(r) : "r"(v));
    return r;
}
// byte offset (0..15) of combined-mask bit beta
__device__ __forceinline__ int chunk_bit_to_off(int beta) { return ((7 - (beta & 7)) << 2) + (beta >> 3); }

// complement LUT: comp_map (src/util.c:228-237) extended to 256 entries with identity for
// bytes >= 128 (the reference indexes a 128-entry table out of bounds there).  Extraction's strand
// transforms and the reverse-complement pattern of pattern search both use it.
__device__ __forceinline__ uint8_t complement_byte(int b) {
    const int low = (b >= 'a' && b <= 'z') ? 32 : 0;
    const int up = b - low;
    int r = up;
    switch (up) {
    case 'A': r = 'T'; break; case 'T': r = 'A'; break; case 'U': r = 'A'; break;
    case 'C': r = 'G'; break; case 'G': r = 'C'; break;
    case 'M': r = 'K'; break; case 'K': r = 'M'; break;
    case 'R': r = 'Y'; break; case 'Y': r = 'R'; break;
    case 'V': r = 'B'; break; case 'B': r = 'V'; break;
    case 'H': r = 'D'; break; case 'D': r = 'H'; break;
    default: break;
    }
    return (uint8_t)(r + low);
}

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_u32(uint32_t *p, uint32_t v) {
    asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int64_t ld_cg_i64(const int64_t *p) { return __ldcg(reinterpret_cast<const long long *>(p)); }
__device__ __forceinline__ uint64_t ld_cg_u64(const uint64_t *p) {
    return __ldcg(reinterpret_cast<const unsigned long long *>(p));
}

__device__ __forceinline__ int64_t shfl_i64(int64_t v, int src) {
    int lo = __shfl_sync(0xffffffffu, (int)(uint32_t)(uint64_t)v, src);
    int hi = __shfl_sync(0xffffffffu, (int)(uint32_t)((uint64_t)v >> 32), src);
    return (int64_t)(((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo);
}
__device__ __forceinline__ int64_t shfl_up_i64(int64_t v, int d) {
    int lo = __shfl_up_sync(0xffffffffu, (int)(uint32_t)(uint64_t)v, d);
    int hi = __shfl_up_sync(0xffffffffu, (int)(uint32_t)((uint64_t)v >> 32), d);
    return (int64_t)(((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo);
}
__device__ __forceinline__ int64_t shfl_down_i64(int64_t v, int d) {
    int lo = __shfl_down_sync(0xffffffffu, (int)(uint32_t)(uint64_t)v, d);
    int hi = __shfl_down_sync(0xffffffffu, (int)(uint32_t)((uint64_t)v >> 32), d);
    return (int64_t)(((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo);
}

}  // namespace fxg
#endif  // __CUDACC__
