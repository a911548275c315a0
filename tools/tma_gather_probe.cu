// Micro-benchmark: how fast can one warp stage 32 records of 48 bytes into shared memory with bulk TMA when the records are
//   (a) one contiguous 1536-byte block (one cp.async.bulk)            — what the render kernels do today (sorted copy), or
//   (b) 32 scattered 48-byte records (32 cp.async.bulk, one per lane) — a gather straight from the per-Gaussian array, or
//   (c) 32 scattered records through plain 128-bit loads + shared-memory stores (no TMA)?
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_gather_probe tools/tma_gather_probe.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

struct __align__(16) Rec { float4 a, b, c; };

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do { asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory"); } while (!ok);
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

constexpr int kWarps = 4, kStages = 3;
struct __align__(128) Ring { Rec rec[kStages][32]; uint64_t full[kStages]; uint64_t pad[13]; };

template <int MODE>
__global__ void __launch_bounds__(kWarps * 32) probe(const Rec *rec, const unsigned *ids, int n_ids, int iters, float *sink) {
    __shared__ Ring rings[kWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    Ring &rg = rings[warp];
    if (lane == 0) { for (int i = 0; i < kStages; i++) mbar_init(&rg.full[i], 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncwarp();
    const int gw = (blockIdx.x * kWarps + warp);
    unsigned phase = 0;
    float acc = 0.f;
    auto issue = [&](int it) {
        const int st = it % kStages;
        const unsigned base = (unsigned)(((size_t)gw * 977 + (size_t)it * 32) % (size_t)(n_ids - 32));
        if (MODE == 0) {
            if (lane == 0) { mbar_expect_tx(&rg.full[st], 32 * sizeof(Rec)); tma_bulk_g2s(&rg.rec[st][0], rec + ids[base] % (unsigned)(n_ids - 32), 32 * sizeof(Rec), &rg.full[st]); }
        } else if (MODE == 1) {
            if (lane == 0) mbar_expect_tx(&rg.full[st], 32 * sizeof(Rec));
            __syncwarp();
            tma_bulk_g2s(&rg.rec[st][lane], rec + ids[base + lane], sizeof(Rec), &rg.full[st]);
        } else {
            const Rec *src = rec + ids[base + lane];
            const float4 a = __ldg(&src->a), b = __ldg(&src->b), c = __ldg(&src->c);
            rg.rec[st][lane].a = a; rg.rec[st][lane].b = b; rg.rec[st][lane].c = c;
        }
    };
    for (int it = 0; it < kStages - 1 && it < iters; it++) issue(it);
    for (int it = 0; it < iters; it++) {
        if (it + kStages - 1 < iters) issue(it + kStages - 1);
        const int st = it % kStages;
        if (MODE != 2) { mbar_wait(&rg.full[st], (phase >> st) & 1u); phase ^= 1u << st; } else __syncwarp();
        acc += rg.rec[st][lane].a.x + rg.rec[st][(lane + 7) & 31].c.w;       // consume
        __syncwarp();
    }
    if (acc == 12345.678f) sink[0] = acc;
}

int main() {
    const int P = 100000, iters = 2000;
    Rec *rec; unsigned *ids; float *sink;
    cudaMalloc(&rec, sizeof(Rec) * P); cudaMemset(rec, 0, sizeof(Rec) * P);
    unsigned *h = (unsigned *)malloc(4 * P);
    srand(1); for (int i = 0; i < P; i++) h[i] = (unsigned)(rand() % (P - 32));
    cudaMalloc(&ids, 4 * P); cudaMemcpy(ids, h, 4 * P, cudaMemcpyHostToDevice); cudaMalloc(&sink, 4);
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    for (int per_sm = 2; per_sm <= 12; per_sm += 5) {
        for (int mode = 0; mode < 3; mode++) {
            cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
            const int grid = sms * per_sm;
            for (int rep = 0; rep < 2; rep++) {
                cudaEventRecord(e0);
                if (mode == 0) probe<0><<<grid, kWarps * 32>>>(rec, ids, P, iters, sink);
                else if (mode == 1) probe<1><<<grid, kWarps * 32>>>(rec, ids, P, iters, sink);
                else probe<2><<<grid, kWarps * 32>>>(rec, ids, P, iters, sink);
                cudaEventRecord(e1); cudaEventSynchronize(e1);
            }
            float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
            const double chunks = (double)grid * kWarps * iters;
            printf("warps/SM %2d mode %d (%s): %.3f ms, %.1f M chunks/s, %.1f ns per 32-record chunk per SM, %.1f GB/s  err=%s\n", per_sm * kWarps, mode,
                   mode == 0 ? "1 x 1536 B bulk" : mode == 1 ? "32 x 48 B bulk gather" : "32 x 48 B LDG gather", ms, chunks / ms / 1e3,
                   ms * 1e6 / (chunks / sms), chunks * 1536 / ms / 1e6, cudaGetErrorString(cudaGetLastError()));
        }
    }
    return 0;
}
