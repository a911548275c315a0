// dgr_mesh_api.cu — the C ABI of include/dgr_mesh.h over the kernels of dgr_mesh.cuh (libdgr_mesh.so).
#include <cuda_runtime.h>

#include <cmath>
#include <string>

#include "../../../include/dgr_mesh.h"
#include "dgr_mesh.cuh"

using namespace dgr;

namespace {
thread_local std::string g_err;

int fail(int code, const char *what, const char *detail = nullptr) {
    g_err = what;
    if (detail) { g_err += ": "; g_err += detail; }
    return code;
}

constexpr long long kLimit = 2147483648LL;               // 2^31: ids and counts are int32

bool misaligned(const void *p, size_t a) { return ((uintptr_t)p) % a != 0; }

// grid shape -> point count, or -1 when refused
long long grid_points(int32_t NX, int32_t NY, int32_t NZ) {
    if (NX < 2 || NY < 2 || NZ < 2) return -1;
    const long long N = (long long)NX * NY * NZ;
    return N < kLimit ? N : -1;
}
}  // namespace

#define DGR_CUDA(call)                                                                         \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess) return fail((int)e_, #call, cudaGetErrorString(e_));            \
    } while (0)
#define MESH_KERNEL(...)                                                                       \
    do {                                                                                       \
        __VA_ARGS__;                                                                           \
        cudaError_t e_ = cudaGetLastError();                                                   \
        if (e_ != cudaSuccess) return fail((int)e_, "kernel launch", cudaGetErrorString(e_));  \
    } while (0)

extern "C" {

const char *dgr_mesh_last_error(void) { return g_err.c_str(); }

size_t dgr_mesh_scratch_bytes(int32_t NX, int32_t NY, int32_t NZ) {
    const long long N = grid_points(NX, NY, NZ);
    return N < 0 ? 0 : McLayout(N).total;
}

static int mc_check(const char *who, const float *occ, int32_t NX, int32_t NY, int32_t NZ, float thr, const void *scratch,
                    size_t scratch_bytes) {
    std::string w(who);
    if (NX < 2 || NY < 2 || NZ < 2) return fail(-1, (w + ": every grid side must be >= 2").c_str());
    if (grid_points(NX, NY, NZ) < 0) return fail(-1, (w + ": grids of 2^31 points or more are refused").c_str());
    if (!occ) return fail(-1, (w + ": NULL occ").c_str());
    if (misaligned(occ, 4)) return fail(-1, (w + ": occ is not 4-byte aligned").c_str());
    if (std::isnan(thr)) return fail(-1, (w + ": thr is NaN").c_str());
    if (!scratch || scratch_bytes < dgr_mesh_scratch_bytes(NX, NY, NZ))
        return fail(-1, (w + ": scratch NULL or smaller than dgr_mesh_scratch_bytes").c_str());
    if (misaligned(scratch, 16)) return fail(-1, (w + ": scratch is not 16-byte aligned").c_str());
    return 0;
}

int dgr_mesh_marching_cubes_count(const float *occ, int32_t NX, int32_t NY, int32_t NZ, float thr, void *scratch, size_t scratch_bytes,
                                  int64_t *counts, void *stream) {
    if (int e = mc_check("dgr_mesh_marching_cubes_count", occ, NX, NY, NZ, thr, scratch, scratch_bytes)) return e;
    if (!counts) return fail(-1, "dgr_mesh_marching_cubes_count: NULL counts");
    const int N = (int)grid_points(NX, NY, NZ);
    const McLayout L(N);
    cudaStream_t st = (cudaStream_t)stream;
    char *s = (char *)scratch;
    MeshMisc *misc = reinterpret_cast<MeshMisc *>(s + L.off_misc);
    int *bt = reinterpret_cast<int *>(s + L.off_bt);
    DGR_CUDA(cudaMemsetAsync(misc, 0, sizeof(MeshMisc), st));
    MESH_KERNEL(mesh_classify_kernel<<<L.nblk, kMeshThreads, 0, st>>>(occ, NX, NY, NZ, thr, N, (unsigned char *)(s + L.off_code), bt, misc));
    MESH_KERNEL(mesh_scan_blocks_kernel<<<1, kMeshScanThreads, 0, st>>>(L.nblk, bt, reinterpret_cast<long long *>(s + L.off_bo), misc));
    MeshMisc h;
    DGR_CUDA(cudaMemcpyAsync(&h, misc, sizeof(MeshMisc), cudaMemcpyDeviceToHost, st));
    DGR_CUDA(cudaStreamSynchronize(st));
    if (h.err) return fail(-2, "dgr_mesh_marching_cubes_count: occ holds a non-finite value");
    if (h.counts[0] >= kLimit || h.counts[1] >= kLimit) return fail(-3, "dgr_mesh_marching_cubes_count: 2^31 vertices or faces or more");
    counts[0] = h.counts[0];
    counts[1] = h.counts[1];
    return 0;
}

int dgr_mesh_marching_cubes_emit(const float *occ, int32_t NX, int32_t NY, int32_t NZ, float thr, void *scratch, size_t scratch_bytes,
                                 int64_t Nv, int64_t Nf, float *vertices, int32_t *faces, void *stream) {
    if (int e = mc_check("dgr_mesh_marching_cubes_emit", occ, NX, NY, NZ, thr, scratch, scratch_bytes)) return e;
    if (Nv < 0 || Nf < 0 || Nv >= kLimit || Nf >= kLimit) return fail(-1, "dgr_mesh_marching_cubes_emit: counts outside [0, 2^31)");
    if ((Nv > 0 && !vertices) || (Nf > 0 && !faces)) return fail(-1, "dgr_mesh_marching_cubes_emit: NULL output");
    if (misaligned(vertices, 4) || misaligned(faces, 4)) return fail(-1, "dgr_mesh_marching_cubes_emit: output is not 4-byte aligned");
    if (Nf > 0 && Nv == 0) return fail(-1, "dgr_mesh_marching_cubes_emit: faces without vertices");
    if (Nv == 0) return 0;
    const int N = (int)grid_points(NX, NY, NZ);
    const McLayout L(N);
    cudaStream_t st = (cudaStream_t)stream;
    char *s = (char *)scratch;
    const unsigned char *code = (const unsigned char *)(s + L.off_code);
    const int *bt = reinterpret_cast<const int *>(s + L.off_bt);
    const long long *bo = reinterpret_cast<const long long *>(s + L.off_bo);
    int *vofs = reinterpret_cast<int *>(s + L.off_vofs);
    MESH_KERNEL(mesh_vertices_kernel<<<L.nblk, kMeshThreads, 0, st>>>(occ, NY, NZ, thr, N, code, bt, bo, vofs, vertices));
    if (Nf > 0) MESH_KERNEL(mesh_faces_kernel<<<L.nblk, kMeshThreads, 0, st>>>(NX, NY, NZ, N, code, bt, bo, vofs, faces));
    return 0;
}

size_t dgr_mesh_components_scratch_bytes(int32_t Nv, int32_t Nf) {
    if (Nv < 0 || Nf < 0) return 0;
    return CcLayout(Nv, Nf).total;
}

static int cc_check(const char *who, const float *vertices, int32_t Nv, const int32_t *faces, int32_t Nf, const void *scratch,
                    size_t scratch_bytes) {
    std::string w(who);
    if (Nv < 0 || Nf < 0) return fail(-1, (w + ": negative Nv or Nf").c_str());
    if ((Nv > 0 && !vertices) || (Nf > 0 && !faces)) return fail(-1, (w + ": NULL vertices or faces").c_str());
    if (misaligned(vertices, 4) || misaligned(faces, 4)) return fail(-1, (w + ": vertices or faces not 4-byte aligned").c_str());
    if (!scratch || scratch_bytes < dgr_mesh_components_scratch_bytes(Nv, Nf))
        return fail(-1, (w + ": scratch NULL or smaller than dgr_mesh_components_scratch_bytes").c_str());
    if (misaligned(scratch, 16)) return fail(-1, (w + ": scratch is not 16-byte aligned").c_str());
    return 0;
}

int dgr_mesh_remove_components_count(const float *vertices, int32_t Nv, const int32_t *faces, int32_t Nf, int32_t min_faces,
                                     double min_diag_pct, void *scratch, size_t scratch_bytes, int64_t *counts, void *stream) {
    if (int e = cc_check("dgr_mesh_remove_components_count", vertices, Nv, faces, Nf, scratch, scratch_bytes)) return e;
    if (!counts) return fail(-1, "dgr_mesh_remove_components_count: NULL counts");
    if (min_faces < 0 || !(min_diag_pct >= 0.0 && min_diag_pct <= 100.0))
        return fail(-1, "dgr_mesh_remove_components_count: min_faces < 0 or min_diag_pct outside [0, 100]");
    if (Nv == 0 || Nf == 0) {                             // no face: nothing is kept
        counts[0] = counts[1] = 0;
        return 0;
    }
    const CcLayout L(Nv, Nf);
    cudaStream_t st = (cudaStream_t)stream;
    char *s = (char *)scratch;
    int *parent = reinterpret_cast<int *>(s + L.off_parent), *fcount = reinterpret_cast<int *>(s + L.off_fcount);
    int *box = reinterpret_cast<int *>(s + L.off_box), *bt = reinterpret_cast<int *>(s + L.off_bt);
    unsigned char *ref = (unsigned char *)(s + L.off_ref), *flags = (unsigned char *)(s + L.off_flags);
    MeshMisc *misc = reinterpret_cast<MeshMisc *>(s + L.off_misc);
    const int E = Nv > Nf ? Nv : Nf;
    const unsigned gv = (unsigned)((Nv + kMeshThreads - 1) / kMeshThreads), gf = (unsigned)((Nf + kMeshThreads - 1) / kMeshThreads);
    const unsigned ge = (unsigned)((E + kMeshThreads - 1) / kMeshThreads);
    MESH_KERNEL(mesh_cc_init_kernel<<<gv, kMeshThreads, 0, st>>>(Nv, parent, fcount, box, ref, misc));
    MESH_KERNEL(mesh_cc_link_kernel<<<gf, kMeshThreads, 0, st>>>(Nv, Nf, faces, parent, ref, misc));
    MESH_KERNEL(mesh_cc_label_kernel<<<gv, kMeshThreads, 0, st>>>(Nv, parent));
    MESH_KERNEL(mesh_cc_stats_kernel<<<ge, kMeshThreads, 0, st>>>(Nv, Nf, vertices, faces, parent, ref, fcount, box, misc));
    MESH_KERNEL(mesh_cc_count_kernel<<<L.nblk, kMeshThreads, 0, st>>>(Nv, Nf, faces, parent, ref, fcount, box, min_faces, min_diag_pct,
                                                                      misc, flags, bt));
    MESH_KERNEL(mesh_scan_blocks_kernel<<<1, kMeshScanThreads, 0, st>>>(L.nblk, bt, reinterpret_cast<long long *>(s + L.off_bo), misc));
    MeshMisc h;
    DGR_CUDA(cudaMemcpyAsync(&h, misc, sizeof(MeshMisc), cudaMemcpyDeviceToHost, st));
    DGR_CUDA(cudaStreamSynchronize(st));
    if (h.err) return fail(-2, "dgr_mesh_remove_components_count: a face index is outside [0, Nv)");
    counts[0] = h.counts[0];
    counts[1] = h.counts[1];
    return 0;
}

int dgr_mesh_remove_components_emit(const float *vertices, int32_t Nv, const int32_t *faces, int32_t Nf, void *scratch,
                                    size_t scratch_bytes, int64_t kept_nv, int64_t kept_nf, float *vertices_out, int32_t *faces_out,
                                    void *stream) {
    if (int e = cc_check("dgr_mesh_remove_components_emit", vertices, Nv, faces, Nf, scratch, scratch_bytes)) return e;
    if (misaligned(vertices_out, 4) || misaligned(faces_out, 4))
        return fail(-1, "dgr_mesh_remove_components_emit: output is not 4-byte aligned");
    if (kept_nv < 0 || kept_nf < 0 || kept_nv > Nv || kept_nf > Nf)
        return fail(-1, "dgr_mesh_remove_components_emit: kept counts outside [0, Nv] x [0, Nf]");
    if ((kept_nv > 0 && !vertices_out) || (kept_nf > 0 && !faces_out)) return fail(-1, "dgr_mesh_remove_components_emit: NULL output");
    if (kept_nf == 0) return 0;
    const CcLayout L(Nv, Nf);
    cudaStream_t st = (cudaStream_t)stream;
    char *s = (char *)scratch;
    const unsigned char *flags = (const unsigned char *)(s + L.off_flags);
    const int *bt = reinterpret_cast<const int *>(s + L.off_bt);
    const long long *bo = reinterpret_cast<const long long *>(s + L.off_bo);
    int *vmap = reinterpret_cast<int *>(s + L.off_vmap);
    MESH_KERNEL(mesh_cc_vertices_kernel<<<L.nblk, kMeshThreads, 0, st>>>(vertices, flags, bt, bo, vmap, vertices_out));
    MESH_KERNEL(mesh_cc_faces_kernel<<<L.nblk, kMeshThreads, 0, st>>>(faces, flags, bt, bo, vmap, faces_out));
    return 0;
}

}  // extern "C"
