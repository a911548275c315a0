/*
 * dgr_constants.h — every threshold of the Gaussian-splat rasterizer path in ONE place.
 *
 * All of these are recalled from the public diff-gaussian-rasterization behaviour (ashawkey fork,
 * depth+alpha outputs); that package is NOT vendored in the reference (SURVEY.md §8c), so each value is
 * tagged UNVERIFIED-EXT: a later correction is a one-line change here, picked up by the CUDA kernels
 * (dreamgaussian_b200/csrc) and by the CPU oracle (oracle/dgr_oracle.c) alike.
 *
 * In-tree anchors that DO pin values: SH constants = /root/reference/sh_utils.py:26-43,
 * SH offset +0.5 / clamp >= 0 = /root/reference/gs_renderer.py:793.
 */
#ifndef DGR_CONSTANTS_H
#define DGR_CONSTANTS_H

#define DGR_TILE            16          /* UNVERIFIED-EXT tile edge in pixels (BLOCK_X = BLOCK_Y)            */
#define DGR_NEAR_CULL_Z     0.2f        /* UNVERIFIED-EXT view-space z at or below which a Gaussian is culled */
#define DGR_W_EPS           1e-7f       /* UNVERIFIED-EXT added to clip-space w before the divide             */
#define DGR_COV2D_LOWPASS   0.3f        /* UNVERIFIED-EXT added to cov2D xx, yy                               */
#define DGR_EIG_FLOOR       0.1f        /* UNVERIFIED-EXT floor under the eigenvalue discriminant             */
#define DGR_RADIUS_SIGMAS   3.0f        /* UNVERIFIED-EXT radius = ceil(3 sqrt(lambda_max))                   */
#define DGR_FOV_CLAMP       1.3f        /* UNVERIFIED-EXT tx/tz, ty/tz clamped to +-1.3 tan(fov/2) inside J   */
#define DGR_ALPHA_MAX       0.99f       /* UNVERIFIED-EXT alpha = min(0.99, o * G)                            */
#define DGR_ALPHA_MIN       (1.0f / 255.0f) /* UNVERIFIED-EXT contributions below this are skipped           */
#define DGR_T_STOP          1e-4f       /* UNVERIFIED-EXT stop when T * (1 - alpha) < 1e-4                    */
#define DGR_SH_OFFSET       0.5f        /* gs_renderer.py:793                                                 */
#define DGR_AA_RATIO_FLOOR  2.5e-5f     /* UNVERIFIED-EXT anti-aliased mode: floor under det(cov2D) / det(cov2D + lowpass) */

/* MCMC densification (Kheradmand et al., NeurIPS 2024; gsplat MCMCStrategy), recalled from the published code */
#define DGR_MCMC_N_MAX         51       /* UNVERIFIED-EXT size of the published binomial table: copies per source clamp here   */
#define DGR_MCMC_MIN_OPACITY   0.005f   /* UNVERIFIED-EXT dead at or below this opacity; floor of the relocated opacity        */
#define DGR_MCMC_OPACITY_MAX   (1.0 - 1.0 / 8388608.0) /* UNVERIFIED-EXT 1 - 2^-23: ceiling of the relocated opacity        */
#define DGR_MCMC_GROW_PERCENT  105      /* UNVERIFIED-EXT target count floor(1.05 P) per refinement, up to the cap             */
#define DGR_MCMC_NOISE_K       100.0f   /* UNVERIFIED-EXT noise gate 1 / (1 + exp(-k ((1 - o) - x0)))                          */
#define DGR_MCMC_NOISE_X0      0.995f   /* UNVERIFIED-EXT                                                                      */
#define DGR_MCMC_NOISE_LR      5e5f     /* UNVERIFIED-EXT noise scale = lr_xyz(step) * noise_lr                                */
#define DGR_MCMC_OPACITY_REG   0.01f    /* UNVERIFIED-EXT loss += opacity_reg * mean(sigmoid(opacity))                         */
#define DGR_MCMC_SCALE_REG     0.01f    /* UNVERIFIED-EXT loss += scale_reg * mean(exp(scaling))                               */

/* sh_utils.py:26-43 */
#define DGR_SH_C0   0.28209479177387814f
#define DGR_SH_C1   0.4886025119029199f
#define DGR_SH_C2_0 1.0925484305920792f
#define DGR_SH_C2_1 -1.0925484305920792f
#define DGR_SH_C2_2 0.31539156525252005f
#define DGR_SH_C2_3 -1.0925484305920792f
#define DGR_SH_C2_4 0.5462742152960396f
#define DGR_SH_C3_0 -0.5900435899266435f
#define DGR_SH_C3_1 2.890611442640554f
#define DGR_SH_C3_2 -0.4570457994644658f
#define DGR_SH_C3_3 0.3731763325901154f
#define DGR_SH_C3_4 -0.4570457994644658f
#define DGR_SH_C3_5 1.445305721320277f
#define DGR_SH_C3_6 -0.5900435899266435f

#endif /* DGR_CONSTANTS_H */
