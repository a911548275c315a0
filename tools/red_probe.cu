// Micro-benchmark: how long does L2 take to absorb the moment reductions of one backward render of the bench view when each
// (record, sub-tile) pair sends its ten floats as
//   (a) 10 x red.global.add.f32                       (b) 5 x red.global.add.v2.f32
//   (c) v4 [0..3] + v4 [4..7] + v2 [8..9]             (d1) v4 [0..3] + v4 [4..7] + f32 [8] + f32 [9]
//   (d2) v4 [0..3] + v2 [4..5] + v2 [6..7] + v2 [8..9]
// into 48-byte rows (kGradRecFloats = 12) of a 256-aligned [rows x 12] float array?  8 lanes per warp instruction, each on a
// different row, as in render_bwd_body's flush.  Row patterns:
//   contended: the 8 warps of a CTA send the same rows in the same order (a tile's 8 sub-tile items run together and park the
//              same records) — the worst case of the kernel's pattern;
//   random:    every (warp, flush, lane) draws its own row.
// Only the reductions run: the result is the time of that stream alone, not its share of the kernel.
// Usage: red_probe [pairs] [rows] [launches]      (tools/red_probe.py builds and runs it)
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int kRowFloats = 12, kWarps = 8, kLanes = 8;

__device__ __forceinline__ void red1(float *a, float v) { asm volatile("red.global.add.f32 [%0], %1;" ::"l"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void red2(float *a, float x, float y) { asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(a), "f"(x), "f"(y) : "memory"); }
__device__ __forceinline__ void red4(float *a, float x, float y, float z, float w) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}

// row_ids: [CTAs][kWarps][flushes][kLanes]; one CTA = one tile's 8 sub-tile warps
template <int MODE>
__global__ void __launch_bounds__(kWarps * 32) probe(const int *__restrict__ row_ids, int flushes, float *__restrict__ rows) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane >= kLanes) return;
    const int *ids = row_ids + ((size_t)blockIdx.x * kWarps + warp) * flushes * kLanes + lane;
    const float v = 1e-3f * (float)(lane + 1);
    for (int f = 0; f < flushes; f++) {
        float *d = rows + (size_t)__ldg(ids + f * kLanes) * kRowFloats;
        if (MODE == 0) {
#pragma unroll
            for (int i = 0; i < 10; i++) red1(d + i, v);
        } else if (MODE == 1) {
#pragma unroll
            for (int i = 0; i < 10; i += 2) red2(d + i, v, v);
        } else if (MODE == 2) {
            red4(d, v, v, v, v); red4(d + 4, v, v, v, v); red2(d + 8, v, v);
        } else if (MODE == 3) {
            red4(d, v, v, v, v); red4(d + 4, v, v, v, v); red1(d + 8, v); red1(d + 9, v);
        } else {
            red4(d, v, v, v, v); red2(d + 4, v, v); red2(d + 6, v, v); red2(d + 8, v, v);
        }
    }
}

static unsigned long long g_rng = 0x9E3779B97F4A7C15ull;
static unsigned rnd(unsigned n) { g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17; return (unsigned)(g_rng % n); }

// 8 distinct rows for one warp instruction
static void draw8(int *out, int nrows) {
    for (int l = 0; l < kLanes; l++) {
        int r;
        bool dup;
        do { r = (int)rnd((unsigned)nrows); dup = false; for (int k = 0; k < l; k++) dup |= out[k] == r; } while (dup);
        out[l] = r;
    }
}

int main(int argc, char **argv) {
    const long long pairs = argc > 1 ? atoll(argv[1]) : 590000;
    const int nrows = argc > 2 ? atoi(argv[2]) : 100000;
    const int launches = argc > 3 ? atoi(argv[3]) : 200;
    const int flushes = 9;                                      // per warp; CTAs = pairs / (8 warps x 9 flushes x 8 lanes)
    const int ctas = (int)((pairs + kWarps * flushes * kLanes - 1) / (kWarps * flushes * kLanes));
    const long long real_pairs = (long long)ctas * kWarps * flushes * kLanes;
    const size_t n_ids = (size_t)ctas * kWarps * flushes * kLanes;

    std::vector<int> contended(n_ids), random(n_ids);
    for (int c = 0; c < ctas; c++)
        for (int f = 0; f < flushes; f++) {
            int r8[kLanes];
            draw8(r8, nrows);
            for (int w = 0; w < kWarps; w++)
                for (int l = 0; l < kLanes; l++) contended[(((size_t)c * kWarps + w) * flushes + f) * kLanes + l] = r8[l];
        }
    for (size_t i = 0; i < n_ids; i += kLanes) draw8(&random[i], nrows);

    int *d_ids[2];
    float *d_rows;
    CK(cudaMalloc(&d_ids[0], n_ids * 4)); CK(cudaMalloc(&d_ids[1], n_ids * 4));
    CK(cudaMemcpy(d_ids[0], contended.data(), n_ids * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_ids[1], random.data(), n_ids * 4, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&d_rows, (size_t)nrows * kRowFloats * 4));
    CK(cudaMemset(d_rows, 0, (size_t)nrows * kRowFloats * 4));
    if (((size_t)d_rows & 255) != 0) { fprintf(stderr, "rows not 256-aligned\n"); return 1; }

    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device %s, %d SMs\n", prop.name, prop.multiProcessorCount);
    printf("pairs %lld (%d CTAs x %d warps x %d flushes x %d lanes), rows %d x %d B, %d launches per timing\n",
           real_pairs, ctas, kWarps, flushes, kLanes, nrows, kRowFloats * 4, launches);

    typedef void (*K)(const int *, int, float *);
    const K kern[5] = {probe<0>, probe<1>, probe<2>, probe<3>, probe<4>};
    const char *name[5] = {"a_10xf32", "b_5xv2", "c_v4v4v2", "d1_v4v4f32f32", "d2_v4v2v2v2"};
    const int ops[5] = {10, 5, 3, 4, 4};
    const char *pat[2] = {"contended", "random"};
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int p = 0; p < 2; p++)
        for (int rep = 0; rep < 2; rep++)                       // two passes: the second shows the spread
            for (int m = 0; m < 5; m++) {
                for (int i = 0; i < 20; i++) kern[m]<<<ctas, kWarps * 32>>>(d_ids[p], flushes, d_rows);
                CK(cudaGetLastError());
                CK(cudaEventRecord(e0));
                for (int i = 0; i < launches; i++) kern[m]<<<ctas, kWarps * 32>>>(d_ids[p], flushes, d_rows);
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
                float ms;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                const double us = 1e3 * ms / launches;
                const double red_ops = (double)real_pairs * ops[m];
                printf("RESULT pattern=%s pass=%d variant=%s ops_per_pair=%d us=%.2f red_ops_per_s=%.3e floats_per_s=%.3e\n",
                       pat[p], rep, name[m], ops[m], us, red_ops / (us * 1e-6), (double)real_pairs * 10 / (us * 1e-6));
            }
    CK(cudaDeviceSynchronize());
    return 0;
}
