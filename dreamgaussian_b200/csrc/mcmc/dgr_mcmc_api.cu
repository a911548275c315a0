// dgr_mcmc_api.cu — the C ABI of include/dgr_mcmc.h over the kernels of dgr_mcmc.cuh (libdgr_mcmc.so).
#include <cuda_runtime.h>

#include <cmath>
#include <string>

#include "../../../include/dgr_mcmc.h"
#include "dgr_mcmc.cuh"

using namespace dgr;

namespace {
thread_local std::string g_err;

int fail(int code, const char *what, const char *detail = nullptr) {
    g_err = what;
    if (detail) { g_err += ": "; g_err += detail; }
    return code;
}
}  // namespace

#define DGR_CUDA(call)                                                                         \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess) return fail((int)e_, #call, cudaGetErrorString(e_));            \
    } while (0)
// launch a kernel (the statement in __VA_ARGS__) and check the launch
#define MCMC_KERNEL(...)                                                                       \
    do {                                                                                       \
        __VA_ARGS__;                                                                           \
        cudaError_t e_ = cudaGetLastError();                                                   \
        if (e_ != cudaSuccess) return fail((int)e_, "kernel launch", cudaGetErrorString(e_));  \
    } while (0)

extern "C" {

const char *dgr_mcmc_last_error(void) { return g_err.c_str(); }

int dgr_mcmc_relocation(int32_t n, const float *opacity, const float *scale, const int32_t *ratio, float *new_opacity, float *new_scale,
                        void *stream) {
    if (n < 0) return fail(-1, "dgr_mcmc_relocation: n < 0");
    if (n == 0) return 0;
    if (!opacity || !scale || !ratio || !new_opacity || !new_scale) return fail(-1, "dgr_mcmc_relocation: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    MCMC_KERNEL(mcmc_relocation_kernel<<<(n + kMcmcThreads - 1) / kMcmcThreads, kMcmcThreads, 0, st>>>(
                                             n, opacity, scale, ratio, new_opacity, new_scale));
    return 0;
}

size_t dgr_mcmc_scratch_bytes(int32_t P, int32_t n_add) { return McmcLayout(P, n_add).total; }

int dgr_mcmc_refine(int32_t P, int32_t n_add, const DgrDensifyTensors *t, const float *u_relocate, const float *u_add, float min_opacity,
                    void *scratch_v, size_t scratch_bytes, int32_t *n_relocated, void *stream) {
    if (P < 0 || n_add < 0) return fail(-1, "dgr_mcmc_refine: negative P or n_add");
    if (!t) return fail(-1, "dgr_mcmc_refine: NULL tensors");
    if (!(min_opacity >= 0.f && min_opacity < 1.f)) return fail(-1, "dgr_mcmc_refine: min_opacity outside [0, 1)");
    McmcTensors T;
    for (int k = 0; k < kMcmcTensors; k++) {
        T.in[k] = t->in[k]; T.m_in[k] = t->exp_avg_in[k]; T.v_in[k] = t->exp_avg_sq_in[k];
        T.out[k] = t->out[k]; T.m_out[k] = t->exp_avg_out[k]; T.v_out[k] = t->exp_avg_sq_out[k];
        T.width[k] = t->width[k];
        if (t->width[k] < 0) return fail(-1, "dgr_mcmc_refine: negative row width");
        if (P > 0 && t->width[k] > 0 && (!T.in[k] || !T.m_in[k] || !T.v_in[k] || !T.out[k] || !T.m_out[k] || !T.v_out[k]))
            return fail(-1, "dgr_mcmc_refine: NULL tensor");
    }
    if (T.width[0] != 3 || T.width[3] != 1 || T.width[4] != 3 || T.width[5] != 4)
        return fail(-1, "dgr_mcmc_refine: row widths must be xyz 3, opacity 1, scaling 3, rotation 4");
    if (P == 0) {
        if (n_add > 0) return fail(-1, "dgr_mcmc_refine: n_add > 0 needs P > 0");
        if (n_relocated) DGR_CUDA(cudaMemsetAsync(n_relocated, 0, sizeof(int32_t), (cudaStream_t)stream));
        return 0;
    }
    if (!u_relocate || (n_add > 0 && !u_add)) return fail(-1, "dgr_mcmc_refine: NULL draws");
    const McmcLayout L(P, n_add);
    if (!scratch_v || scratch_bytes < L.total) return fail(-1, "dgr_mcmc_refine: scratch NULL or smaller than dgr_mcmc_scratch_bytes");
    cudaStream_t st = (cudaStream_t)stream;
    char *s = (char *)scratch_v;
    double *C = reinterpret_cast<double *>(s + L.off_C), *bsum = reinterpret_cast<double *>(s + L.off_bsum);
    double *boff = reinterpret_cast<double *>(s + L.off_boff);
    int *rank = reinterpret_cast<int *>(s + L.off_rank), *src = reinterpret_cast<int *>(s + L.off_src);
    int *picks = reinterpret_cast<int *>(s + L.off_picks), *gpicks = reinterpret_cast<int *>(s + L.off_gpicks);
    int *gsrc = reinterpret_cast<int *>(s + L.off_gsrc), *bdead = reinterpret_cast<int *>(s + L.off_bdead);
    int *bdoff = reinterpret_cast<int *>(s + L.off_bdoff), *ndead = reinterpret_cast<int *>(s + L.off_ndead);
    const unsigned nb = (unsigned)L.nblk;
    auto scan = [&](const float *op, int grow) -> int {
        MCMC_KERNEL(mcmc_scan_local_kernel<<<nb, kMcmcThreads, 0, st>>>(P, op, min_opacity, grow, C, rank, bsum, bdead));
        MCMC_KERNEL(mcmc_scan_blocks_kernel<<<1, kMcmcThreads, 0, st>>>(L.nblk, bsum, bdead, boff, bdoff, ndead));
        MCMC_KERNEL(mcmc_scan_add_kernel<<<nb, kMcmcThreads, 0, st>>>(P, boff, bdoff, C, rank));
        return 0;
    };
    // relocation
    DGR_CUDA(cudaMemsetAsync(picks, 0, (size_t)P * 4, st));
    if (int e = scan(T.in[3], 0)) return e;
    MCMC_KERNEL(mcmc_relocate_pick_kernel<<<nb, kMcmcThreads, 0, st>>>(P, T.in[3], min_opacity, C, rank, ndead,
                                                                                                  u_relocate, src, picks, n_relocated));
    MCMC_KERNEL(mcmc_relocate_write_kernel<<<nb, kMcmcThreads, 0, st>>>(P, T, src, picks));
    MCMC_KERNEL(mcmc_relocate_update_kernel<<<nb, kMcmcThreads, 0, st>>>(P, T.in[3], T.in[4], src, picks, min_opacity,
                                                                                                      T.out[3], T.out[4]));
    if (n_add == 0) return 0;
    // growth over the relocated rows
    const unsigned na = (unsigned)((n_add + kMcmcThreads - 1) / kMcmcThreads);
    DGR_CUDA(cudaMemsetAsync(gpicks, 0, (size_t)P * 4, st));
    if (int e = scan(T.out[3], 1)) return e;
    MCMC_KERNEL(mcmc_grow_pick_kernel<<<na, kMcmcThreads, 0, st>>>(P, n_add, C, u_add, gsrc, gpicks));
    MCMC_KERNEL(mcmc_grow_update_kernel<<<nb, kMcmcThreads, 0, st>>>(P, T, gpicks, min_opacity));
    MCMC_KERNEL(mcmc_append_kernel<<<na, kMcmcThreads, 0, st>>>(P, n_add, T, gsrc));
    return 0;
}

int dgr_mcmc_inject_noise(int32_t P, float *xyz, const float *opacity_raw, const float *scaling_raw, const float *rotation_raw,
                          const float *normals, float scale, void *stream) {
    if (P < 0) return fail(-1, "dgr_mcmc_inject_noise: P < 0");
    if (P == 0) return 0;
    if (!xyz || !opacity_raw || !scaling_raw || !rotation_raw || !normals) return fail(-1, "dgr_mcmc_inject_noise: NULL argument");
    if (!(scale >= 0.f) || isinf(scale)) return fail(-1, "dgr_mcmc_inject_noise: scale must be finite and >= 0");
    cudaStream_t st = (cudaStream_t)stream;
    MCMC_KERNEL(mcmc_noise_kernel<<<(P + kMcmcThreads - 1) / kMcmcThreads, kMcmcThreads, 0, st>>>(
                                        P, xyz, opacity_raw, scaling_raw, rotation_raw, normals, scale));
    return 0;
}

}  // extern "C"
