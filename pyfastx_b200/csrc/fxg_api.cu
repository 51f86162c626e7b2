// fxg_api.cu -- context, error reporting, HBM file buffers and pinned-chunk staging.
#include "fxg_common.cuh"
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <thread>
#include <vector>
#include <atomic>
#include <mutex>

static thread_local char g_err[512] = "";

void fxg_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void fxg_pool_drain(int device);

int FxgScratch::reserve(size_t bytes) {
    if (bytes <= cap) return FXG_OK;
    if (ptr) cudaFree(ptr);
    ptr = nullptr; cap = 0;
    size_t want = bytes + bytes / 8 + 4096;
    cudaError_t e = cudaMalloc(&ptr, want);
    if (e != cudaSuccess) {
        cudaGetLastError();
        int dev = 0;
        cudaGetDevice(&dev);
        fxg_pool_drain(dev);
        want = bytes;
        e = cudaMalloc(&ptr, want);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        ptr = nullptr;
        fxg_set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
        return FXG_ENOMEM;
    }
    cap = want;
    return FXG_OK;
}
void FxgScratch::release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr; cap = 0;
}

extern "C" int fxg_abi_version(void) { return FXG_ABI_VERSION; }
extern "C" const char *fxg_last_error(void) { return g_err; }

extern "C" int fxg_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

static const size_t PINNED_CHUNK = (size_t)256 << 20;

extern "C" int fxg_ctx_create(int device, fxg_ctx **out) {
    FXG_CHECK_ARG(out, "out == NULL");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        fxg_set_error("no CUDA device available (%s); libfxg has no CPU fallback",
                      e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
        return FXG_ENODEV;
    }
    FXG_CHECK_ARG(device >= 0 && device < n, "device index out of range");
    FXG_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    FXG_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {               // sm_90a code loads on compute capability 9.0 only
        fxg_set_error("device %d is sm_%d%d; libfxg is built for sm_90a only", device, prop.major, prop.minor);
        return FXG_ENODEV;
    }
    fxg_ctx *c = new fxg_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    FXG_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
    *out = c;
    return FXG_OK;
}

void fxg_svc_stop(fxg_ctx *ctx);

extern "C" void fxg_ctx_destroy(fxg_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    fxg_svc_stop(c);
    if (c->svc_stream) cudaStreamDestroy(c->svc_stream);
    if (c->svc_req) cudaFreeHost(c->svc_req);
    cudaStreamSynchronize(c->stream);
    if (c->h_counters) cudaFreeHost(c->h_counters);
    if (c->h_one) cudaFreeHost(c->h_one);
    if (c->ring) { cudaFreeHost(c->ring); for (int i = 0; i < 32; ++i) if (c->ring_ev[i]) cudaEventDestroy(c->ring_ev[i]); }
    for (int i = 0; i < 2; ++i) {
        if (c->pinned[i]) cudaFreeHost(c->pinned[i]);
        if (c->pinned_ev[i]) cudaEventDestroy(c->pinned_ev[i]);
    }
    for (int i = 0; i < FXG_PROF_SLOTS; ++i)
        for (int j = 0; j < 2; ++j) if (c->prof_ev[i][j]) cudaEventDestroy(c->prof_ev[i][j]);
    c->tile_desc.release(); c->seg.release(); c->row_tmp.release(); c->rows.release();
    c->counters.release(); c->params.release(); c->plan.release(); c->misc.release(); c->stage_file.release();
    c->search.release();
    if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

extern "C" int fxg_ctx_set_stream(fxg_ctx *c, void *cuda_stream) {
    FXG_CHECK_ARG(c, "ctx == NULL");
    FXG_LOCK(c);
    FXG_CUDA(cudaSetDevice(c->device));
    FXG_CUDA(cudaStreamSynchronize(c->stream));
    if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
    c->stream = (cudaStream_t)cuda_stream;
    c->own_stream = false;
    return FXG_OK;
}

extern "C" int fxg_ctx_sync(fxg_ctx *c) {
    FXG_CHECK_ARG(c, "ctx == NULL");
    FXG_LOCK(c);
    FXG_CUDA(cudaSetDevice(c->device));
    FXG_CUDA(cudaStreamSynchronize(c->stream));
    return FXG_OK;
}

extern "C" int fxg_ctx_sm_count(fxg_ctx *c) { return c ? c->sm_count : 0; }

extern "C" int fxg_profile_enable(fxg_ctx *c, int on) {
    FXG_CHECK_ARG(c, "ctx == NULL");
    FXG_LOCK(c);
    FXG_CUDA(cudaSetDevice(c->device));
    if (on && !c->prof_ev[0][0])
        for (int i = 0; i < FXG_PROF_SLOTS; ++i)
            for (int j = 0; j < 2; ++j) FXG_CUDA(cudaEventCreate(&c->prof_ev[i][j]));
    c->profiling = on != 0;
    for (int i = 0; i < FXG_PROF_SLOTS; ++i) c->prof_valid[i] = false;
    return FXG_OK;
}
extern "C" int fxg_profile_last_ms(fxg_ctx *c, int slot, float *ms) {
    FXG_CHECK_ARG(c && ms && slot >= 0 && slot < FXG_PROF_SLOTS, "bad arguments");
    FXG_LOCK(c);
    FXG_CHECK_ARG(c->prof_valid[slot], "no measurement recorded for this slot");
    FXG_CUDA(cudaEventSynchronize(c->prof_ev[slot][1]));
    FXG_CUDA(cudaEventElapsedTime(ms, c->prof_ev[slot][0], c->prof_ev[slot][1]));
    return FXG_OK;
}
extern "C" int64_t fxg_ctx_launch_count(fxg_ctx *c) { return c ? c->launches : 0; }

extern "C" int fxg_host_alloc(int64_t nbytes, void **out) {
    FXG_CHECK_ARG(out && nbytes >= 0, "bad arguments");
    *out = nullptr;
    FXG_CUDA(cudaHostAlloc(out, (size_t)(nbytes > 0 ? nbytes : 1), cudaHostAllocPortable));
    return FXG_OK;
}
extern "C" void fxg_host_free(void *p) {
    if (p) cudaFreeHost(p);
}

// ---- device file buffers ------------------------------------------------------------------
// One spare buffer per device is kept when a file is freed and handed to the next file that fits: cudaMalloc /
// cudaFree of a 10 GB buffer cost more than the scan of that buffer.  FXG_FILE_POOL=0 turns it off;
// any failed device allocation drains it and retries.
struct FxgFilePool {
    std::mutex mu;
    uint8_t *d[16] = {};
    int64_t cap[16] = {};
};
static FxgFilePool g_pool;
static bool pool_enabled() {
    static int on = -1;
    if (on < 0) { const char *e = getenv("FXG_FILE_POOL"); on = (e && e[0] == '0') ? 0 : 1; }
    return on != 0;
}
void fxg_pool_drain(int device) {
    std::lock_guard<std::mutex> g(g_pool.mu);
    for (int i = 0; i < 16; ++i)
        if ((device < 0 || device == i) && g_pool.d[i]) { cudaSetDevice(i); cudaFree(g_pool.d[i]); g_pool.d[i] = nullptr; g_pool.cap[i] = 0; }
}
extern "C" void fxg_pool_trim(void) { fxg_pool_drain(-1); }

// The public staging entry points (fxg_file_alloc / _upload / _from_host / _slice) return with their copies complete:
// the single-query service reads file buffers from a stream of its own, which does not wait for the context's stream.
// fxg_file_alloc_async / fxg_file_upload_async only enqueue; library calls that synchronise before they return anyway
// (the path stager, the one-call index builds, the GPU inflate paths) use them directly.
static int file_done(fxg_ctx *c, fxg_file **out, int rc) {
    if (rc == FXG_OK) {
        const cudaError_t e = cudaStreamSynchronize(c->stream);
        if (e == cudaSuccess) return FXG_OK;
        fxg_set_error("file staging failed: %s", cudaGetErrorString(e));
        rc = FXG_ECUDA;
    }
    if (out && *out) { fxg_file_free(*out); *out = nullptr; }
    return rc;
}

int fxg_file_alloc_async(fxg_ctx *c, int64_t nbytes, fxg_file **out) {
    *out = nullptr;
    FXG_CUDA(cudaSetDevice(c->device));
    fxg_file *f = new fxg_file();
    f->size = nbytes;
    f->capacity = fxg_round_up(nbytes + 1, FXG_FILE_PAD) + FXG_FILE_PAD;
    f->alloc_cap = f->capacity;
    f->owned = true;
    f->device = c->device;
    if (pool_enabled() && c->device < 16) {
        std::lock_guard<std::mutex> g(g_pool.mu);
        const int64_t have = g_pool.cap[c->device];
        if (g_pool.d[c->device] && have >= f->capacity && have <= 2 * f->capacity + ((int64_t)256 << 20)) {
            f->d = g_pool.d[c->device];
            f->alloc_cap = have;
            g_pool.d[c->device] = nullptr; g_pool.cap[c->device] = 0;
        }
    }
    if (f->d) {
        cudaDeviceSynchronize();             // nothing that used the buffer in its previous life is still running
    } else {
        cudaError_t e = cudaMalloc((void **)&f->d, (size_t)f->capacity);
        if (e != cudaSuccess) {
            cudaGetLastError();
            fxg_pool_drain(c->device);
            e = cudaMalloc((void **)&f->d, (size_t)f->capacity);
        }
        if (e != cudaSuccess) {
            cudaGetLastError();
            delete f;
            fxg_set_error("cudaMalloc(%lld) for file buffer failed: %s", (long long)nbytes, cudaGetErrorString(e));
            return FXG_ENOMEM;
        }
    }
    // zero the padding (never contains '\n'); data region is overwritten by uploads
    const int64_t pad_from = nbytes & ~(int64_t)15;
    *out = f;
    FXG_CUDA(cudaMemsetAsync(f->d + pad_from, 0, (size_t)(f->capacity - pad_from), c->stream));
    return FXG_OK;
}

extern "C" int fxg_file_alloc(fxg_ctx *c, int64_t nbytes, fxg_file **out) {
    FXG_CHECK_ARG(c && out && nbytes >= 0, "bad arguments");
    FXG_LOCK(c);
    return file_done(c, out, fxg_file_alloc_async(c, nbytes, out));
}

static bool host_ptr_is_pinned(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

static int ensure_pinned(fxg_ctx *c) {
    if (c->pinned[0]) return FXG_OK;
    for (int i = 0; i < 2; ++i) {
        FXG_CUDA(cudaHostAlloc(&c->pinned[i], PINNED_CHUNK, cudaHostAllocDefault));
        FXG_CUDA(cudaEventCreateWithFlags(&c->pinned_ev[i], cudaEventDisableTiming));
    }
    c->pinned_bytes = PINNED_CHUNK;
    return FXG_OK;
}

// parallel memcpy into a pinned staging buffer (a single core cannot feed PCIe Gen5)
static void parallel_memcpy(void *dst, const void *src, size_t n) {
    const size_t kMin = (size_t)4 << 20;
    unsigned nt = std::thread::hardware_concurrency();
    if (nt > 16) nt = 16;
    if (nt < 1) nt = 1;
    if (n < 2 * kMin || nt == 1) { memcpy(dst, src, n); return; }
    std::vector<std::thread> th;
    const size_t per = (n + nt - 1) / nt;
    for (unsigned i = 0; i < nt; ++i) {
        const size_t o = (size_t)i * per;
        if (o >= n) break;
        const size_t len = (o + per <= n) ? per : n - o;
        th.emplace_back([=] { memcpy((char *)dst + o, (const char *)src + o, len); });
    }
    for (auto &t : th) t.join();
}

int fxg_file_upload_async(fxg_ctx *c, fxg_file *f, int64_t dst_off, const void *host, int64_t nbytes) {
    FXG_CHECK_ARG(dst_off >= 0 && nbytes >= 0 && dst_off + nbytes <= f->size, "upload range outside file");
    FXG_CUDA(cudaSetDevice(c->device));
    if (nbytes == 0) return FXG_OK;
    if (host_ptr_is_pinned(host)) {
        // pinned source: DMA straight from the caller's buffer, in chunks so the copy engine pipelines
        const int64_t chunk = (int64_t)256 << 20;
        for (int64_t o = 0; o < nbytes; o += chunk) {
            const int64_t len = (nbytes - o < chunk) ? nbytes - o : chunk;
            FXG_CUDA(cudaMemcpyAsync(f->d + dst_off + o, (const char *)host + o, (size_t)len,
                                     cudaMemcpyHostToDevice, c->stream));
        }
        return FXG_OK;
    }
    int rc = ensure_pinned(c);
    if (rc) return rc;
    int which = 0;
    for (int64_t o = 0; o < nbytes; o += (int64_t)c->pinned_bytes, which ^= 1) {
        const int64_t len = (nbytes - o < (int64_t)c->pinned_bytes) ? nbytes - o : (int64_t)c->pinned_bytes;
        FXG_CUDA(cudaEventSynchronize(c->pinned_ev[which]));   // previous DMA out of this buffer done
        parallel_memcpy(c->pinned[which], (const char *)host + o, (size_t)len);
        FXG_CUDA(cudaMemcpyAsync(f->d + dst_off + o, c->pinned[which], (size_t)len, cudaMemcpyHostToDevice, c->stream));
        FXG_CUDA(cudaEventRecord(c->pinned_ev[which], c->stream));
    }
    return FXG_OK;
}

extern "C" int fxg_file_upload(fxg_ctx *c, fxg_file *f, int64_t dst_off, const void *host, int64_t nbytes) {
    FXG_CHECK_ARG(c && f && (host || nbytes == 0), "bad arguments");
    FXG_LOCK(c);
    return file_done(c, nullptr, fxg_file_upload_async(c, f, dst_off, host, nbytes));
}

extern "C" int fxg_file_from_host(fxg_ctx *c, const void *host, int64_t nbytes, fxg_file **out) {
    FXG_CHECK_ARG(c && out && nbytes >= 0 && (host || nbytes == 0), "bad arguments");
    FXG_LOCK(c);
    int rc = fxg_file_alloc_async(c, nbytes, out);
    if (rc == FXG_OK) rc = fxg_file_upload_async(c, *out, 0, host, nbytes);
    return file_done(c, out, rc);
}

// NUMA node that holds the page-cache pages of bytes [begin, end) of an open file (sampled at three offsets), -1 if unknown.
// Readers pinned to that node copy a tmpfs file faster than unpinned ones on a multi-socket host (tools/stage_probe.cu).
static int file_numa_node(int fd, int64_t begin, int64_t end) {
    if (end <= begin) return -1;
    const long pg = sysconf(_SC_PAGESIZE);
    int votes[64] = {0};
    int best = -1;
    // inside the staged range: ranks of a sharded build read different parts of the file, which may sit on different nodes
    const int64_t offs[3] = {begin / pg * pg, ((begin + end) / 2) / pg * pg, (end - 1) / pg * pg};
    for (int i = 0; i < 3; ++i) {
        void *m = mmap(nullptr, (size_t)pg, PROT_READ, MAP_SHARED, fd, (off_t)offs[i]);
        if (m == MAP_FAILED) continue;
        volatile char sink = *(volatile char *)m;
        (void)sink;
        int node = -1;
        if (syscall(SYS_get_mempolicy, &node, nullptr, 0ul, m, 3ul /* MPOL_F_NODE | MPOL_F_ADDR */) == 0 && node >= 0 && node < 64) {
            ++votes[node];
            if (best < 0 || votes[node] > votes[best]) best = node;
        }
        munmap(m, (size_t)pg);
    }
    return best;
}
static bool node_cpuset(int node, cpu_set_t *cs) {
    char pth[128], buf[4096];
    snprintf(pth, sizeof pth, "/sys/devices/system/node/node%d/cpulist", node);
    FILE *f = fopen(pth, "r");
    if (!f) return false;
    const bool got = fgets(buf, sizeof buf, f) != nullptr;
    fclose(f);
    if (!got) return false;
    CPU_ZERO(cs);
    int n = 0;
    for (char *p = buf; *p;) {
        char *e;
        long a = strtol(p, &e, 10);
        if (e == p) break;
        long b = a;
        if (*e == '-') { p = e + 1; b = strtol(p, &e, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int)c, cs); ++n; }
        p = (*e == ',') ? e + 1 : e;
        if (*e != ',' && *e != '-') break;
    }
    return n > 0;
}

// bytes [begin, end) of `path` (end < 0: to the end of the file) -> a device buffer of their own.
// A ring of 16 MiB pinned pieces: ~20 persistent reader threads (pinned to the NUMA node that holds the file's
// page-cache pages) pread the next free piece, the calling thread issues one cudaMemcpyAsync per finished piece, in
// order, and retires pieces as their copies complete -- reads and DMA overlap piece by piece, without per-chunk
// thread spawns or barriers (tools/stage_probe.cu compares it with a double buffer of large chunks).
static const int64_t RING_PIECE = (int64_t)16 << 20;
static const int RING_SLOTS = 32;
static int stage_path_range(fxg_ctx *c, const char *path, int64_t begin, int64_t end, fxg_file **out) {
    FXG_CHECK_ARG(c && path && out && begin >= 0, "bad arguments");
    *out = nullptr;
    int fd = open(path, O_RDONLY);
    if (fd < 0) { fxg_set_error("cannot open %s", path); return FXG_EIO; }
    struct stat st;
    if (fstat(fd, &st) != 0) { close(fd); fxg_set_error("cannot stat %s", path); return FXG_EIO; }
    if (end < 0 || end > (int64_t)st.st_size) end = (int64_t)st.st_size;
    if (begin > end) begin = end;
    const int64_t n = end - begin;
    int rc = fxg_file_alloc_async(c, n, out);                           // the stream is synchronised below
    if (rc) { close(fd); if (*out) { fxg_file_free(*out); *out = nullptr; } return rc; }
    if (!c->ring) {
        cudaError_t e = cudaHostAlloc(&c->ring, (size_t)(RING_PIECE * RING_SLOTS), cudaHostAllocDefault);
        if (e != cudaSuccess) { cudaGetLastError(); c->ring = nullptr; close(fd); fxg_file_free(*out); *out = nullptr; fxg_set_error("cudaHostAlloc of the staging ring failed: %s", cudaGetErrorString(e)); return FXG_ENOMEM; }
        for (int i = 0; i < RING_SLOTS; ++i) cudaEventCreateWithFlags(&c->ring_ev[i], cudaEventDisableTiming);
    }
    const int64_t np = (n + RING_PIECE - 1) / RING_PIECE;
    int nt = 20;
    if (const char *e = getenv("FXG_STAGE_THREADS")) { const int v = atoi(e); if (v >= 1 && v <= 256) nt = v; }
    const unsigned hw = std::thread::hardware_concurrency();
    if (hw && (unsigned)nt > hw) nt = (int)hw;
    if ((int64_t)nt > np) nt = (int)(np > 0 ? np : 1);
    cpu_set_t cs;
    bool pin = false;
    const char *pe = getenv("FXG_STAGE_PIN");
    if (!(pe && pe[0] == '0') && n >= ((int64_t)256 << 20)) {
        const int node = file_numa_node(fd, begin, end);
        pin = node >= 0 && node_cpuset(node, &cs);
        if (getenv("FXG_TIMING")) fprintf(stderr, "[fxg timing] staging: file pages on NUMA node %d, %d readers%s\n", node, nt, pin ? " pinned there" : "");
    }
    std::vector<std::atomic<int>> ready((size_t)(np > 0 ? np : 1));
    for (auto &r : ready) r.store(0, std::memory_order_relaxed);
    std::atomic<int64_t> next(0), retired_a(0);
    std::atomic<int> bad(0);
    char *ring = (char *)c->ring;
    std::vector<std::thread> th;
    for (int i = 0; i < nt && np > 0; ++i) th.emplace_back([&, pin] {
        if (pin) sched_setaffinity(0, sizeof(cs), &cs);
        for (;;) {
            const int64_t p = next.fetch_add(1);
            if (p >= np || bad.load(std::memory_order_relaxed)) return;
            while (p - retired_a.load(std::memory_order_acquire) >= RING_SLOTS) {      // the slot's previous piece is still in flight
                if (bad.load(std::memory_order_relaxed)) return;
                std::this_thread::yield();
            }
            const int64_t o = p * RING_PIECE, len = n - o < RING_PIECE ? n - o : RING_PIECE;
            char *dst = ring + (p % RING_SLOTS) * RING_PIECE;
            int64_t done = 0;
            while (done < len) {
                const ssize_t r = pread(fd, dst + done, (size_t)(len - done), (off_t)(begin + o + done));
                if (r <= 0) { bad.store(1); return; }
                done += r;
            }
            ready[(size_t)p].store(1, std::memory_order_release);
        }
    });
    int64_t issued = 0, retired = 0;
    cudaError_t cerr = cudaSuccess;
    while (retired < np && !bad.load(std::memory_order_relaxed) && cerr == cudaSuccess) {
        bool progress = false;
        while (issued < np && ready[(size_t)issued].load(std::memory_order_acquire)) {
            const int64_t o = issued * RING_PIECE, len = n - o < RING_PIECE ? n - o : RING_PIECE;
            cerr = cudaMemcpyAsync((*out)->d + o, ring + (issued % RING_SLOTS) * RING_PIECE, (size_t)len, cudaMemcpyHostToDevice, c->stream);
            if (cerr != cudaSuccess) break;
            cudaEventRecord(c->ring_ev[issued % RING_SLOTS], c->stream);
            ++issued;
            progress = true;
        }
        while (retired < issued && cudaEventQuery(c->ring_ev[retired % RING_SLOTS]) == cudaSuccess) {
            ++retired;
            retired_a.store(retired, std::memory_order_release);
            progress = true;
        }
        if (!progress) std::this_thread::yield();
    }
    if (cerr != cudaSuccess) bad.store(1);
    for (auto &t : th) t.join();
    close(fd);
    cudaStreamSynchronize(c->stream);
    if (bad.load()) {
        cudaGetLastError();
        fxg_file_free(*out); *out = nullptr;
        if (cerr != cudaSuccess) { fxg_set_error("H2D failed: %s", cudaGetErrorString(cerr)); return FXG_ECUDA; }
        fxg_set_error("read error on %s", path);
        return FXG_EIO;
    }
    return FXG_OK;
}

extern "C" int fxg_file_from_path(fxg_ctx *c, const char *path, fxg_file **out) {
    FXG_CHECK_ARG(c, "ctx == NULL");
    FXG_LOCK(c);
    return stage_path_range(c, path, 0, -1, out);
}

extern "C" int fxg_file_from_path_range(fxg_ctx *c, const char *path, int64_t begin, int64_t end, fxg_file **out) {
    FXG_CHECK_ARG(c, "ctx == NULL");
    FXG_LOCK(c);
    return stage_path_range(c, path, begin, end, out);
}

extern "C" int fxg_file_slice(fxg_ctx *c, const fxg_file *src, int64_t begin, int64_t end, fxg_file **out) {
    FXG_CHECK_ARG(c && src && out && begin >= 0 && end >= begin && end <= src->size, "bad arguments");
    FXG_LOCK(c);
    int rc = fxg_file_alloc_async(c, end - begin, out);
    if (rc == FXG_OK && end > begin) {
        const cudaError_t e = cudaMemcpyAsync((*out)->d, src->d + begin, (size_t)(end - begin), cudaMemcpyDeviceToDevice, c->stream);
        if (e != cudaSuccess) { fxg_set_error("device copy failed: %s", cudaGetErrorString(e)); rc = FXG_ECUDA; }
    }
    return file_done(c, out, rc);
}

// Split point on a host file (SURVEY.md section 8e): first offset >= from where a line (or a FASTA header line,
// index.c:234) starts; the file size if there is none.  Reads 1 MiB windows with pread.
extern "C" int fxg_split_point_path(const char *path, int64_t from, int want_header, int64_t *pos, int64_t *file_size) {
    FXG_CHECK_ARG(path && pos && from >= 0, "bad arguments");
    int fd = open(path, O_RDONLY);
    if (fd < 0) { fxg_set_error("cannot open %s", path); return FXG_EIO; }
    struct stat st;
    if (fstat(fd, &st) != 0) { close(fd); fxg_set_error("cannot stat %s", path); return FXG_EIO; }
    const int64_t n = (int64_t)st.st_size;
    if (file_size) *file_size = n;
    *pos = n;
    if (from >= n) { close(fd); return FXG_OK; }
    std::vector<char> buf((size_t)1 << 20);
    if (from == 0) {
        char c0 = 0;
        if (!want_header || (pread(fd, &c0, 1, 0) == 1 && c0 == '>')) { *pos = 0; close(fd); return FXG_OK; }
        from = 1;
    }
    // candidates: x in [from-1, n) with byte[x] == '\n' (and byte[x+1] == '>'), answer x + 1
    for (int64_t o = from - 1; o < n;) {
        const ssize_t got = pread(fd, buf.data(), buf.size(), (off_t)o);
        if (got <= 0) { close(fd); fxg_set_error("read error on %s", path); return FXG_EIO; }
        const char *b = buf.data();
        const char *p = b;
        const char *e = b + got;
        while ((p = (const char *)memchr(p, '\n', (size_t)(e - p))) != nullptr) {
            const int64_t x = o + (p - b);
            if (!want_header) { *pos = x + 1; close(fd); return FXG_OK; }
            if (p + 1 < e) {
                if (p[1] == '>') { *pos = x + 1; close(fd); return FXG_OK; }
            } else if (x + 1 < n) {
                char c1 = 0;
                if (pread(fd, &c1, 1, (off_t)(x + 1)) == 1 && c1 == '>') { *pos = x + 1; close(fd); return FXG_OK; }
            }
            ++p;
        }
        o += got;
    }
    close(fd);
    return FXG_OK;
}

extern "C" int fxg_file_wrap(fxg_ctx *c, void *dev_ptr, int64_t nbytes, int64_t capacity, fxg_file **out) {
    FXG_CHECK_ARG(c && out && dev_ptr && nbytes >= 0 && capacity >= nbytes, "bad arguments");
    FXG_LOCK(c);
    FXG_CHECK_ARG(((uintptr_t)dev_ptr & 15) == 0, "device pointer must be 16-byte aligned");
    FXG_CHECK_ARG(capacity >= fxg_round_up(nbytes, 16), "capacity must cover nbytes rounded up to 16");
    fxg_file *f = new fxg_file();
    f->d = (uint8_t *)dev_ptr; f->size = nbytes; f->capacity = capacity; f->owned = false; f->device = c->device;
    *out = f;
    return FXG_OK;
}

extern "C" int fxg_file_download(fxg_ctx *c, const fxg_file *f, int64_t src_off, void *host, int64_t nbytes) {
    FXG_CHECK_ARG(c && f && host && src_off >= 0 && nbytes >= 0 && src_off + nbytes <= f->size, "bad arguments");
    FXG_LOCK(c);
    FXG_CUDA(cudaSetDevice(c->device));
    FXG_CUDA(cudaMemcpyAsync(host, f->d + src_off, (size_t)nbytes, cudaMemcpyDeviceToHost, c->stream));
    FXG_CUDA(cudaStreamSynchronize(c->stream));
    return FXG_OK;
}

extern "C" void *fxg_file_devptr(const fxg_file *f) { return f ? f->d : nullptr; }
extern "C" int64_t fxg_file_size(const fxg_file *f) { return f ? f->size : 0; }
extern "C" void fxg_file_free(fxg_file *f) {
    if (!f) return;
    if (f->owned && f->d) {
        uint8_t *spare = f->d;
        int64_t cap = f->alloc_cap;
        if (pool_enabled() && f->device < 16 && cap >= ((int64_t)64 << 20)) {
            std::lock_guard<std::mutex> g(g_pool.mu);
            if (cap > g_pool.cap[f->device]) {          // keep the larger one
                std::swap(spare, g_pool.d[f->device]);
                std::swap(cap, g_pool.cap[f->device]);
            }
        }
        if (spare) { cudaSetDevice(f->device); cudaFree(spare); }
    }
    delete f;
}

// ---- rows up/down ------------------------------------------------------------------------------
extern "C" int fxg_rows_download(fxg_ctx *c, const void *d_rows, int64_t n_rows, int row_bytes, void *host_rows) {
    FXG_CHECK_ARG(c && (n_rows == 0 || (d_rows && host_rows)) && n_rows >= 0 && row_bytes > 0, "bad arguments");
    FXG_LOCK(c);
    FXG_CUDA(cudaSetDevice(c->device));
    if (n_rows) {
        FXG_CUDA(cudaMemcpyAsync(host_rows, d_rows, (size_t)n_rows * row_bytes, cudaMemcpyDeviceToHost, c->stream));
        FXG_CUDA(cudaStreamSynchronize(c->stream));
    }
    return FXG_OK;
}

extern "C" int fxg_rows_upload(fxg_ctx *c, const void *host_rows, int64_t n_rows, int row_bytes, void **d_rows_out) {
    FXG_CHECK_ARG(c && d_rows_out && n_rows >= 0 && row_bytes > 0 && (n_rows == 0 || host_rows), "bad arguments");
    FXG_LOCK(c);
    FXG_CUDA(cudaSetDevice(c->device));
    *d_rows_out = nullptr;
    void *d = nullptr;
    FXG_CUDA(cudaMalloc(&d, (size_t)(n_rows > 0 ? n_rows : 1) * row_bytes));
    if (n_rows) {
        cudaError_t e = cudaMemcpyAsync(d, host_rows, (size_t)n_rows * row_bytes, cudaMemcpyHostToDevice, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) { cudaFree(d); fxg_set_error("rows upload failed: %s", cudaGetErrorString(e)); return FXG_ECUDA; }
    }
    *d_rows_out = d;
    return FXG_OK;
}

extern "C" void fxg_dev_free(void *d) {
    if (d) cudaFree(d);
}

// ---- one-call host-buffer index builds (end-to-end path) ------------------------------------------
// The device copy lives in a context-owned, grow-only buffer: repeated builds do not pay
// cudaMalloc / cudaFree of a multi-gigabyte buffer every call.
static int stage_into_ctx(fxg_ctx *c, const void *host_buf, int64_t nbytes, fxg_file *view) {
    FXG_CUDA(cudaSetDevice(c->device));
    const int64_t cap = fxg_round_up(nbytes + 1, FXG_FILE_PAD) + FXG_FILE_PAD;
    int rc = c->stage_file.reserve((size_t)cap);
    if (rc) return rc;
    view->d = (uint8_t *)c->stage_file.ptr;
    view->size = nbytes; view->capacity = cap; view->owned = false; view->device = c->device;
    const int64_t pad_from = nbytes & ~(int64_t)15;
    FXG_CUDA(cudaMemsetAsync(view->d + pad_from, 0, (size_t)(cap - pad_from), c->stream));
    return fxg_file_upload_async(c, view, 0, host_buf, nbytes);        // the build synchronises before it returns
}

extern "C" int fxg_fasta_build_index_host(fxg_ctx *c, const void *host_buf, int64_t nbytes, int flags,
                                          fxg_fasta_row *rows, int64_t rows_cap, fxg_scan_stats *stats) {
    FXG_CHECK_ARG(c && stats && (host_buf || nbytes == 0), "bad arguments");
    FXG_LOCK(c);
    fxg_file f;
    int rc = stage_into_ctx(c, host_buf, nbytes, &f);
    if (rc) return rc;
    fxg_fasta_row *d_rows = nullptr;
    rc = fxg_fasta_scan(c, &f, 0, flags, &d_rows, stats);
    if (rc == FXG_OK) {
        if (stats->n_rows > rows_cap) { fxg_set_error("rows_cap %lld < n_rows %lld", (long long)rows_cap, (long long)stats->n_rows); rc = FXG_ECAP; }
        else rc = fxg_rows_download(c, d_rows, stats->n_rows, (int)sizeof(fxg_fasta_row), rows);
    }
    return rc;
}

extern "C" int fxg_fastq_build_index_host(fxg_ctx *c, const void *host_buf, int64_t nbytes,
                                          fxg_fastq_row *rows, int64_t rows_cap, fxg_scan_stats *stats) {
    FXG_CHECK_ARG(c && stats && (host_buf || nbytes == 0), "bad arguments");
    FXG_LOCK(c);
    fxg_file f;
    int rc = stage_into_ctx(c, host_buf, nbytes, &f);
    if (rc) return rc;
    fxg_fastq_row *d_rows = nullptr;
    rc = fxg_fastq_scan(c, &f, 0, &d_rows, stats);
    if (rc == FXG_OK) {
        if (stats->n_rows > rows_cap) { fxg_set_error("rows_cap %lld < n_rows %lld", (long long)rows_cap, (long long)stats->n_rows); rc = FXG_ECAP; }
        else rc = fxg_rows_download(c, d_rows, stats->n_rows, (int)sizeof(fxg_fastq_row), rows);
    }
    return rc;
}
