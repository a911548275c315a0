/*
 * dgr_mcmc.h — C ABI of the opt-in MCMC densification (libdgr_mcmc.so, built next to libdgr_b200.so from
 * dreamgaussian_b200/csrc/mcmc/).  A library of its own: the rasterizer library and its kernels are untouched by it.
 *
 * All pointers are DEVICE pointers; all work is enqueued on `stream` (a cudaStream_t passed as void*); nothing here synchronises.
 * Return value: 0 on success, otherwise a cudaError_t / negative error code; dgr_mcmc_last_error() has the text.
 */
#ifndef DGR_MCMC_H
#define DGR_MCMC_H

#include "dgr_b200.h"          /* DgrDensifyTensors */

#ifdef __cplusplus
extern "C" {
#endif

/* Opt-in MCMC densification (Kheradmand et al., NeurIPS 2024; gsplat's MCMCStrategy); constants DGR_MCMC_* in dgr_constants.h.
 *   dgr_mcmc_relocation    the relocation formula alone (gsplat's `relocation` op) on ACTIVATED values, one thread per entry, float64
 *                          inside: n = ratio clamped to [1, DGR_MCMC_N_MAX], new_opacity = 1 - (1 - o)^(1/n) (as -expm1(log1p(-o)/n)),
 *                          new_scale = scale * o / D, D = sum_{m=1..n} C(n,m) (-1)^(m-1) new_opacity^m / sqrt(m) (1 where D = 0).
 *                          No clamp.  scale / new_scale [n,3].
 *   dgr_mcmc_refine        relocation, then growth, of P rows into P + n_add rows (t: in / moments P rows, out / out moments P + n_add
 *                          rows, must not alias the inputs; f_rest width may be 0).  o = sigmoid(opacity) in float64 rounded to float.
 *                          Sampling: weights w_i = o_i of the eligible rows (0 for the rest), C_i their float64 inclusive prefix sum;
 *                          draw u picks the smallest i with C_i > u C_last (none: the last eligible row).  Relocation: rows with
 *                          o <= min_opacity are dead, the others live and eligible; the j-th dead row in index order draws
 *                          u_relocate[j] (device, [P]) when some row is alive.  Each picked source, n = 1 + its pick count (clamped to
 *                          DGR_MCMC_N_MAX), stores logit(clamp(o', min_opacity, DGR_MCMC_OPACITY_MAX)) and scaling + log(o / D) (o', D
 *                          as above, D from the unclamped o'), zero Adam moments; each dead row that picked it becomes a copy of its
 *                          updated row in all six tensors and keeps its own moments.  Growth (n_add > 0): every row of the relocated
 *                          output is eligible; u_add[j] (device, [n_add]) picks a row, the picked rows get the same update (n = 1 +
 *                          picks) and zero moments, row P + j is a copy of the j-th pick with zero moments.  n_add is the caller's
 *                          (min(cap, floor(1.05 P)) - P for the published rule), so nothing is read back to the host.  n_relocated
 *                          (device int32, may be NULL) receives the number of dead rows moved.  Integer atomics only: bit-reproducible.
 *                          Refused before any device work, each with its own dgr_mcmc_last_error text: negative P / n_add, t NULL,
 *                          min_opacity outside [0, 1), a negative width, a NULL tensor of a non-empty row, widths other than xyz 3 /
 *                          opacity 1 / scaling 3 / rotation 4, n_add > 0 with P == 0, NULL draws, scratch NULL or scratch_bytes below
 *                          dgr_mcmc_scratch_bytes(P, n_add).
 *   dgr_mcmc_inject_noise  in place: xyz += scale g(o) R diag(s^2) R^T z, g(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995))), o =
 *                          sigmoid(opacity_raw), s = exp(scaling_raw), R of rotation_raw / |rotation_raw| (w, x, y, z); normals z
 *                          [P,3] standard normals (device).  Refused: P < 0, a NULL pointer (P > 0), scale negative, infinite or NaN. */
int dgr_mcmc_relocation(int32_t n, const float *opacity, const float *scale, const int32_t *ratio, float *new_opacity, float *new_scale,
                        void *stream);
size_t dgr_mcmc_scratch_bytes(int32_t P, int32_t n_add);
int dgr_mcmc_refine(int32_t P, int32_t n_add, const DgrDensifyTensors *t, const float *u_relocate, const float *u_add, float min_opacity,
                    void *scratch, size_t scratch_bytes, int32_t *n_relocated, void *stream);
int dgr_mcmc_inject_noise(int32_t P, float *xyz, const float *opacity_raw, const float *scaling_raw, const float *rotation_raw,
                          const float *normals, float scale, void *stream);

const char *dgr_mcmc_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* DGR_MCMC_H */
