// Read floor of the FASTA mark kernel's shape (needs an H100):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/mark_floor tools/mark_floor.cu && /tmp/mark_floor [GB]
// Fills a buffer in HBM with the C2 byte pattern (80-column lines of ACGT, a header line every ~10 KB) and times, at
// mark's launch shape (one warp per 2 KiB region, 8 warps per CTA, four 16-byte streaming loads per lane, no loop):
//   (a) the loads and a trivial reduction (XOR of the words);
//   (b) the loads, the SWAR newline test of mark_kernel and the count.
// Each kernel writes one 4-byte word per region.  Mark writes 12 bytes per region and stages the region in shared
// memory, so (b) is a floor for mark, not a model of it.  The card, its power limit and SM clock are printed first.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int REGION = 2048, WARPS = 8;
constexpr int64_t REC = 16 + 125 * 81;   // ">r%013d\n"-style header of 16 bytes, then 125 lines of 80 bases

__global__ void fill_kernel(uint8_t *f, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t rec = i / REC, o = i % REC;
        uint8_t b;
        if (o < 16) {
            int64_t d = rec;   // digit o - 2 of the record number, 13 digits
            for (int k = (int)o; k < 14; ++k) d /= 10;
            b = o == 0 ? '>' : o == 1 ? 'r' : o == 15 ? '\n' : (uint8_t)('0' + d % 10);
        } else {
            const int64_t l = (o - 16) % 81;
            uint64_t h = (uint64_t)i * 0x9e3779b97f4a7c15ull;
            b = l == 80 ? '\n' : "ACGT"[(h >> 61) & 3];
        }
        f[i] = b;
    }
}

__device__ __forceinline__ uint4 ld_stream16(const uint8_t *p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t nl_mask(uint32_t w) {   // 0x80 per '\n' byte (mark's exact SWAR test)
    const uint32_t u = (w ^ 0x0a0a0a0au) & 0x7f7f7f7fu;
    return ~((u + 0x7f7f7f7fu) | w) & 0x80808080u;
}

template <int KIND>   // 0: loads + XOR, 1: loads + SWAR newline count
__global__ void __launch_bounds__(WARPS * 32) floor_kernel(const uint8_t *file, int64_t nreg, uint32_t *out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r = (int64_t)blockIdx.x * WARPS + warp;
    if (r >= nreg) return;
    const uint8_t *src = file + r * REGION + lane * 16;
    uint4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = ld_stream16(src + j * 512);
    uint32_t acc = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (KIND == 0) acc ^= v[j].x ^ v[j].y ^ v[j].z ^ v[j].w;
        else acc += __popc(nl_mask(v[j].x) | (nl_mask(v[j].y) >> 1) | (nl_mask(v[j].z) >> 2) | (nl_mask(v[j].w) >> 3));
    }
    acc = KIND == 0 ? __reduce_xor_sync(0xffffffffu, acc) : __reduce_add_sync(0xffffffffu, acc);
    if (lane == 0) out[r] = acc;
}

static void card_info() {
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, 0));
    printf("device: %s, %d SMs\n", p.name, p.multiProcessorCount);
    fflush(stdout);
    if (system("nvidia-smi --query-gpu=name,power.limit,clocks.max.sm,clocks.sm --format=csv,noheader") != 0)
        printf("nvidia-smi: not available\n");
    fflush(stdout);
}

int main(int argc, char **argv) {
    const double gb = argc > 1 ? atof(argv[1]) : 10.16;
    const int iters = argc > 2 ? atoi(argv[2]) : 20;
    card_info();
    const int64_t nreg = (int64_t)(gb * 1e9) / REGION, n = nreg * REGION;
    uint8_t *f;
    uint32_t *out;
    CK(cudaMalloc(&f, n));
    CK(cudaMalloc(&out, nreg * sizeof(uint32_t)));
    fill_kernel<<<132 * 16, 256>>>(f, n);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    const unsigned grid = (unsigned)((nreg + WARPS - 1) / WARPS);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    std::vector<float> t[2];
    auto launch = [&](int k) {
        if (k == 0) floor_kernel<0><<<grid, WARPS * 32>>>(f, nreg, out);
        else floor_kernel<1><<<grid, WARPS * 32>>>(f, nreg, out);
    };
    for (int w = 0; w < 3; ++w) { launch(0); launch(1); }
    CK(cudaDeviceSynchronize());
    for (int i = 0; i < iters; ++i)
        for (int k = 0; k < 2; ++k) {   // alternating (a), (b)
            CK(cudaEventRecord(e0));
            launch(k);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            t[k].push_back(ms);
        }
    CK(cudaGetLastError());
    // the newline count of the whole buffer, as a check that (b) computed what it claims
    std::vector<uint32_t> h(nreg);
    CK(cudaMemcpy(h.data(), out, nreg * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    uint64_t nl = 0;
    for (uint32_t c : h) nl += c;
    const int64_t full = n / REC, rest = n % REC;
    const uint64_t want = (uint64_t)full * 126 + (rest >= 16) + (rest > 96 ? (rest - 97) / 81 + 1 : 0);
    printf("newlines counted %llu, expected %llu\n", (unsigned long long)nl, (unsigned long long)want);
    const char *name[2] = {"(a) loads + XOR", "(b) loads + SWAR newline count"};
    for (int k = 0; k < 2; ++k) {
        std::sort(t[k].begin(), t[k].end());
        const double med = t[k][t[k].size() / 2];
        printf("%-32s %.2f GB, %d launches: min %.4f ms, median %.4f ms, max %.4f ms (%.3f TB/s at the median)\n",
               name[k], n / 1e9, iters, t[k].front(), med, t[k].back(), n / (med * 1e-3) / 1e12);
    }
    CK(cudaFree(f));
    CK(cudaFree(out));
    return nl == want ? 0 : 2;
}
