// dgr_mesh.cuh — mesh export kernels (include/dgr_mesh.h): marching cubes over the extract_fields grid and small-component removal.
//
// Both run as count -> (one host read-back) -> emit over tiles of kMeshTile consecutive elements in C order:
//   mesh_classify_kernel     one pass over occ: each grid point's corner code (inside bits of the cell it is the origin of, with the
//                            corners past the grid clamped onto it), the error flag of a non-finite value, per-tile vertex / face counts
//   mesh_scan_blocks_kernel  one CTA: exclusive 64-bit scan of the per-tile (vertex, face) counts, the totals
//   mesh_vertices_kernel     tiles with vertices: tile-local scan + tile offset -> vertex ids in (point, axis) order, positions,
//                            and each point's first vertex id
//   mesh_faces_kernel        tiles with faces: tile-local scan -> face ids in (cell, table) order, corners' vertex ids
//   mesh_cc_init_kernel      union-find parents, component counters and boxes
//   mesh_cc_link_kernel      per face: index check, referenced-vertex marks, union of its edges linking to the smaller root
//   mesh_cc_label_kernel     pointer jumping: every vertex's parent becomes its root (the component's least vertex id)
//   mesh_cc_stats_kernel     per face: integer face count of its component; per referenced vertex: ordered-int min / max boxes
//   mesh_cc_count_kernel     keep decisions (diagonals in float64) of vertices and faces, per-tile kept counts
//   mesh_cc_vertices_kernel  order-preserving compaction of the kept vertices, old -> new ids
//   mesh_cc_faces_kernel     order-preserving compaction of the kept faces, re-indexed
// The only atomics are on integers, and every scan has a fixed order: outputs are bit-reproducible.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dgr_mc_table.h"

namespace dgr {

constexpr int kMeshThreads = 256;
constexpr int kMeshItems = 4;                              // consecutive elements per thread
constexpr int kMeshTile = kMeshThreads * kMeshItems;
constexpr int kMeshScanThreads = 1024;

// read back once per count call: the output sizes, the error flag, the mesh's box (ordered ints)
struct MeshMisc {
    long long counts[2];
    int err;
    int box[6];
};

__host__ __device__ __forceinline__ size_t mesh_up(size_t o) { return (o + 255) / 256 * 256; }

// marching-cubes scratch: [corner code u8 x tiles*kMeshTile][first vertex id i32 x N][tile counts i32 x 2 tiles]
// [tile offsets i64 x 2 tiles][MeshMisc]
struct McLayout {
    size_t off_code, off_vofs, off_bt, off_bo, off_misc, total;
    int nblk;
    __host__ McLayout(long long N) {
        nblk = (int)((N + kMeshTile - 1) / kMeshTile);
        size_t o = 0;
        off_code = o; o = mesh_up(o + (size_t)nblk * kMeshTile);
        off_vofs = o; o = mesh_up(o + 4 * (size_t)N);
        off_bt = o;   o = mesh_up(o + 8 * (size_t)nblk);
        off_bo = o;   o = mesh_up(o + 16 * (size_t)nblk);
        off_misc = o; o = mesh_up(o + sizeof(MeshMisc));
        total = o;
    }
};

// component-removal scratch over E = max(Nv, Nf) elements: [parent i32 x Nv][fcount i32 x Nv][box i32 x 6 Nv][vmap i32 x Nv]
// [referenced u8 x Nv][keep flags u8 x tiles*kMeshTile][tile counts][tile offsets][MeshMisc]
struct CcLayout {
    size_t off_parent, off_fcount, off_box, off_vmap, off_ref, off_flags, off_bt, off_bo, off_misc, total;
    int nblk;
    __host__ CcLayout(int Nv, int Nf) {
        const size_t V = Nv > 0 ? (size_t)Nv : 1, E = (size_t)(Nv > Nf ? Nv : Nf) > 0 ? (size_t)(Nv > Nf ? Nv : Nf) : 1;
        nblk = (int)((E + kMeshTile - 1) / kMeshTile);
        size_t o = 0;
        off_parent = o; o = mesh_up(o + 4 * V);
        off_fcount = o; o = mesh_up(o + 4 * V);
        off_box = o;    o = mesh_up(o + 24 * V);
        off_vmap = o;   o = mesh_up(o + 4 * V);
        off_ref = o;    o = mesh_up(o + V);
        off_flags = o;  o = mesh_up(o + (size_t)nblk * kMeshTile);
        off_bt = o;     o = mesh_up(o + 8 * (size_t)nblk);
        off_bo = o;     o = mesh_up(o + 16 * (size_t)nblk);
        off_misc = o;   o = mesh_up(o + sizeof(MeshMisc));
        total = o;
    }
};

// exclusive scan of (a, b) over the CTA in thread order; returns the CTA totals through ta / tb
template <typename T, int THREADS>
__device__ __forceinline__ void mesh_block_scan2(T &a, T &b, T &ta, T &tb) {
    __shared__ T s_a[THREADS / 32], s_b[THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T x = a, y = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T nx = __shfl_up_sync(0xffffffffu, x, o), ny = __shfl_up_sync(0xffffffffu, y, o);
        if (lane >= o) { x += nx; y += ny; }
    }
    if (lane == 31) { s_a[warp] = x; s_b[warp] = y; }
    __syncthreads();
    if (warp == 0) {
        T u = lane < THREADS / 32 ? s_a[lane] : T(0), v = lane < THREADS / 32 ? s_b[lane] : T(0);
#pragma unroll
        for (int o = 1; o < THREADS / 32; o <<= 1) {
            const T nu = __shfl_up_sync(0xffffffffu, u, o), nv = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) { u += nu; v += nv; }
        }
        if (lane < THREADS / 32) { s_a[lane] = u; s_b[lane] = v; }
    }
    __syncthreads();
    const T wa = warp ? s_a[warp - 1] : T(0), wb = warp ? s_b[warp - 1] : T(0);
    ta = s_a[THREADS / 32 - 1];
    tb = s_b[THREADS / 32 - 1];
    a = wa + x - a;
    b = wb + y - b;
}

// bit a set: the grid edge from this point along axis a is cut (corner 0 vs corner 1 << a of the code)
__device__ __forceinline__ int mc_cut_mask(int code) {
    const int c0 = code & 1;
    return (c0 ^ ((code >> 1) & 1)) | ((c0 ^ ((code >> 2) & 1)) << 1) | ((c0 ^ ((code >> 4) & 1)) << 2);
}

__device__ __forceinline__ void mc_decode(int p, int NY, int NZ, int &i, int &j, int &k) {
    const int row = p / NZ;
    k = p - row * NZ;
    i = row / NY;
    j = row - i * NY;
}

__device__ __forceinline__ int mc_faces_of(int code, int i, int j, int k, int NX, int NY, int NZ) {
    return (i < NX - 1 && j < NY - 1 && k < NZ - 1) ? (int)kMcTriCount[code] : 0;
}

// the four codes of a thread's consecutive points (the code array is padded to whole tiles)
__device__ __forceinline__ uint32_t mc_codes4(const unsigned char *code, int p0) {
    return *reinterpret_cast<const uint32_t *>(code + p0);
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_classify_kernel(const float *__restrict__ occ, int NX, int NY, int NZ, float thr, int N, unsigned char *__restrict__ code,
                     int *__restrict__ bt, MeshMisc *__restrict__ misc) {
    const int sx = NY * NZ, sy = NZ;
    int nv = 0, nf = 0;
    bool bad = false;
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) {
        const long long pl = (long long)blockIdx.x * kMeshTile + u * kMeshThreads + threadIdx.x;
        if (pl >= N) {                                   // the padding of the last tile
            code[pl] = 0;
            continue;
        }
        const int p = (int)pl;
        int i, j, k;
        mc_decode(p, NY, NZ, i, j, k);
        const int dx = i + 1 < NX ? sx : 0, dy = j + 1 < NY ? sy : 0, dz = k + 1 < NZ ? 1 : 0;
        const float v0 = __ldg(occ + p);
        bad |= !isfinite(v0);
        int c = v0 > thr;
        c |= (__ldg(occ + p + dx) > thr) << 1;
        c |= (__ldg(occ + p + dy) > thr) << 2;
        c |= (__ldg(occ + p + dx + dy) > thr) << 3;
        c |= (__ldg(occ + p + dz) > thr) << 4;
        c |= (__ldg(occ + p + dx + dz) > thr) << 5;
        c |= (__ldg(occ + p + dy + dz) > thr) << 6;
        c |= (__ldg(occ + p + dx + dy + dz) > thr) << 7;
        code[p] = (unsigned char)c;
        nv += __popc(mc_cut_mask(c));
        nf += mc_faces_of(c, i, j, k, NX, NY, NZ);
    }
    if (bad) misc->err = 1;
    int ta, tb;
    mesh_block_scan2<int, kMeshThreads>(nv, nf, ta, tb);
    if (threadIdx.x == 0) { bt[2 * blockIdx.x] = ta; bt[2 * blockIdx.x + 1] = tb; }
}

// one CTA: bo[2b + c] = sum of bt[2b' + c] over b' < b, misc->counts[c] = the total (64-bit: no wrap)
__global__ void __launch_bounds__(kMeshScanThreads)
mesh_scan_blocks_kernel(int nblk, const int *__restrict__ bt, long long *__restrict__ bo, MeshMisc *__restrict__ misc) {
    const int chunk = (nblk + kMeshScanThreads - 1) / kMeshScanThreads;
    const int s = min(nblk, (int)threadIdx.x * chunk), e = min(nblk, s + chunk);
    long long a = 0, b = 0, ta, tb;
    for (int x = s; x < e; x++) { a += bt[2 * x]; b += bt[2 * x + 1]; }
    mesh_block_scan2<long long, kMeshScanThreads>(a, b, ta, tb);
    for (int x = s; x < e; x++) {
        bo[2 * x] = a; bo[2 * x + 1] = b;
        a += bt[2 * x]; b += bt[2 * x + 1];
    }
    if (threadIdx.x == 0) { misc->counts[0] = ta; misc->counts[1] = tb; }
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_vertices_kernel(const float *__restrict__ occ, int NY, int NZ, float thr, int N, const unsigned char *__restrict__ code,
                     const int *__restrict__ bt, const long long *__restrict__ bo, int *__restrict__ vofs, float *__restrict__ vert) {
    if (bt[2 * blockIdx.x] == 0) return;                 // uniform over the CTA
    const int p0 = blockIdx.x * kMeshTile + threadIdx.x * kMeshItems;
    const uint32_t c4 = mc_codes4(code, p0);
    int n = 0, dummy = 0, ta, tb;
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) n += __popc(mc_cut_mask((c4 >> (8 * u)) & 255));
    mesh_block_scan2<int, kMeshThreads>(n, dummy, ta, tb);
    int vid = (int)bo[2 * blockIdx.x] + n;
    const int stride[3] = {NY * NZ, NZ, 1};
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) {
        const int m = mc_cut_mask((c4 >> (8 * u)) & 255), p = p0 + u;
        if (!m || p >= N) continue;
        int ijk[3];
        mc_decode(p, NY, NZ, ijk[0], ijk[1], ijk[2]);
        vofs[p] = vid;
        const float v0 = occ[p];
#pragma unroll
        for (int a = 0; a < 3; a++) {
            if (!((m >> a) & 1)) continue;
            const float v1 = occ[p + stride[a]];
            const float t = __fdiv_rn(__fsub_rn(thr, v0), __fsub_rn(v1, v0));
            float *o = vert + 3 * (size_t)vid;
#pragma unroll
            for (int b = 0; b < 3; b++) o[b] = b == a ? __fadd_rn((float)ijk[b], t) : (float)ijk[b];
            vid++;
        }
    }
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_faces_kernel(int NX, int NY, int NZ, int N, const unsigned char *__restrict__ code, const int *__restrict__ bt,
                  const long long *__restrict__ bo, const int *__restrict__ vofs, int *__restrict__ faces) {
    if (bt[2 * blockIdx.x + 1] == 0) return;             // uniform over the CTA
    const int p0 = blockIdx.x * kMeshTile + threadIdx.x * kMeshItems;
    const uint32_t c4 = mc_codes4(code, p0);
    int cnt[kMeshItems], n = 0, dummy = 0, ta, tb;
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) {
        cnt[u] = 0;
        if (p0 + u < N) {
            int i, j, k;
            mc_decode(p0 + u, NY, NZ, i, j, k);
            cnt[u] = mc_faces_of((c4 >> (8 * u)) & 255, i, j, k, NX, NY, NZ);
        }
        n += cnt[u];
    }
    mesh_block_scan2<int, kMeshThreads>(n, dummy, ta, tb);
    int fid = (int)bo[2 * blockIdx.x + 1] + n;
    const int sx = NY * NZ, sy = NZ;
    for (int u = 0; u < kMeshItems; u++) {
        if (!cnt[u]) continue;
        const int c = (c4 >> (8 * u)) & 255, p = p0 + u;
        for (int t = 0; t < cnt[u]; t++, fid++) {
#pragma unroll
            for (int m = 0; m < 3; m++) {
                const int e = kMcTris[c][3 * t + m], corner = kMcEdgeCorner[e], a = kMcEdgeAxis[e];
                const int q = p + ((corner & 1) ? sx : 0) + ((corner & 2) ? sy : 0) + ((corner & 4) ? 1 : 0);
                faces[3 * (size_t)fid + m] = vofs[q] + __popc(mc_cut_mask(code[q]) & ((1 << a) - 1));
            }
        }
    }
}

// ---- small-component removal -------------------------------------------------------------------------------------------------------
// float -> int with the same order (min / max by integer atomics)
__device__ __forceinline__ int mesh_ordered(float f) {
    const int b = __float_as_int(f);
    return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float mesh_unordered(int o) { return __int_as_float(o >= 0 ? o : o ^ 0x7fffffff); }

__global__ void __launch_bounds__(kMeshThreads)
mesh_cc_init_kernel(int Nv, int *__restrict__ parent, int *__restrict__ fcount, int *__restrict__ box, unsigned char *__restrict__ ref,
                    MeshMisc *__restrict__ misc) {
    const int i = blockIdx.x * kMeshThreads + threadIdx.x;
    if (i == 0) {
        misc->err = 0;
        for (int a = 0; a < 3; a++) { misc->box[a] = 0x7fffffff; misc->box[3 + a] = (int)0x80000000; }
    }
    if (i >= Nv) return;
    parent[i] = i;
    fcount[i] = 0;
    ref[i] = 0;
#pragma unroll
    for (int a = 0; a < 3; a++) { box[6 * i + a] = 0x7fffffff; box[6 * i + 3 + a] = (int)0x80000000; }
}

// parents change under the linking kernel's atomics: read them past L1 so a retry sees the new root
__device__ __forceinline__ int mesh_find(const volatile int *parent, int x) {
    int p = parent[x];
    while (p != x) { x = p; p = parent[x]; }
    return x;
}

// link the roots of a and b, the larger under the smaller: a component's final root is its least vertex id, in any atomic order
__device__ __forceinline__ void mesh_union(int *parent, int a, int b) {
    while (true) {
        a = mesh_find(parent, a);
        b = mesh_find(parent, b);
        if (a == b) return;
        const int lo = min(a, b), hi = max(a, b);
        if (atomicCAS(parent + hi, hi, lo) == hi) return;
        a = lo; b = hi;                                   // hi got a parent meanwhile: retry from the new roots
    }
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_cc_link_kernel(int Nv, int Nf, const int *__restrict__ faces, int *parent, unsigned char *__restrict__ ref, MeshMisc *__restrict__ misc) {
    const int i = blockIdx.x * kMeshThreads + threadIdx.x;
    if (i >= Nf) return;
    const int a = faces[3 * (size_t)i], b = faces[3 * (size_t)i + 1], c = faces[3 * (size_t)i + 2];
    if (a < 0 || b < 0 || c < 0 || a >= Nv || b >= Nv || c >= Nv) { misc->err = 1; return; }
    ref[a] = ref[b] = ref[c] = 1;
    mesh_union(parent, a, b);
    mesh_union(parent, a, c);
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_cc_label_kernel(int Nv, int *parent) {
    const int i = blockIdx.x * kMeshThreads + threadIdx.x;
    if (i >= Nv) return;
    parent[i] = mesh_find(parent, i);                    // roots never move, so concurrent jumps stay inside the tree
}

// one lane per group of lanes with the same root applies the group's reduction: most lanes of a warp share a component, so the
// integer atomics stay uncontended
__global__ void __launch_bounds__(kMeshThreads)
mesh_cc_stats_kernel(int Nv, int Nf, const float *__restrict__ vert, const int *__restrict__ faces, const int *__restrict__ parent,
                     const unsigned char *__restrict__ ref, int *__restrict__ fcount, int *__restrict__ box, MeshMisc *__restrict__ misc) {
    const int i = blockIdx.x * kMeshThreads + threadIdx.x, lane = threadIdx.x & 31;
    const bool face = i < Nf && !misc->err;
    const int froot = face ? parent[faces[3 * (size_t)i]] : -1;
    for (unsigned pending = __ballot_sync(0xffffffffu, face); pending;) {
        const int r = __shfl_sync(0xffffffffu, froot, __ffs(pending) - 1);
        const unsigned grp = __ballot_sync(0xffffffffu, face && froot == r);
        if (lane == __ffs(grp) - 1) atomicAdd(fcount + r, __popc(grp));
        pending &= ~grp;
    }
    const bool live = i < Nv && ref[i];
    const int vroot = live ? parent[i] : -1;
    int o[3];
#pragma unroll
    for (int a = 0; a < 3; a++) o[a] = live ? mesh_ordered(vert[3 * (size_t)i + a]) : 0;
    const unsigned any = __ballot_sync(0xffffffffu, live);
    for (unsigned pending = any; pending;) {
        const int r = __shfl_sync(0xffffffffu, vroot, __ffs(pending) - 1);
        const bool in = live && vroot == r;
        const unsigned grp = __ballot_sync(0xffffffffu, in);
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const int mn = __reduce_min_sync(0xffffffffu, in ? o[a] : 0x7fffffff);
            const int mx = __reduce_max_sync(0xffffffffu, in ? o[a] : (int)0x80000000);
            if (lane == __ffs(grp) - 1) { atomicMin(box + 6 * (size_t)r + a, mn); atomicMax(box + 6 * (size_t)r + 3 + a, mx); }
        }
        pending &= ~grp;
    }
    if (!any) return;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const int mn = __reduce_min_sync(0xffffffffu, live ? o[a] : 0x7fffffff);
        const int mx = __reduce_max_sync(0xffffffffu, live ? o[a] : (int)0x80000000);
        if (lane == 0) { atomicMin(misc->box + a, mn); atomicMax(misc->box + 3 + a, mx); }
    }
}

__device__ __forceinline__ double mesh_diag(const int *b) {
    double s = 0.0;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double d = __dsub_rn((double)mesh_unordered(b[3 + a]), (double)mesh_unordered(b[a]));
        s = __dadd_rn(s, __dmul_rn(d, d));
    }
    return __dsqrt_rn(s);
}

__device__ __forceinline__ bool mesh_cc_keep(int root, const int *fcount, const int *box, int min_faces, double min_diag, bool use_diag) {
    if (min_faces > 0 && fcount[root] < min_faces) return false;
    return !(use_diag && mesh_diag(box + 6 * (size_t)root) < min_diag);
}

// flags bit 0: vertex i kept, bit 1: face i kept; per-tile counts of both
__global__ void __launch_bounds__(kMeshThreads)
mesh_cc_count_kernel(int Nv, int Nf, const int *__restrict__ faces, const int *__restrict__ parent, const unsigned char *__restrict__ ref,
                     const int *__restrict__ fcount, const int *__restrict__ box, int min_faces, double min_diag_pct,
                     const MeshMisc *__restrict__ misc, unsigned char *__restrict__ flags, int *__restrict__ bt) {
    const bool use_diag = min_diag_pct > 0.0;
    const double min_diag = use_diag ? __dmul_rn(__ddiv_rn(min_diag_pct, 100.0), mesh_diag(misc->box)) : 0.0;
    const bool ok = !misc->err;                          // a face index out of range: nothing is read through the faces
    int nv = 0, nf = 0, ta, tb;
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) {
        const int i = blockIdx.x * kMeshTile + threadIdx.x * kMeshItems + u;
        const bool kv = i < Nv && ref[i] && mesh_cc_keep(parent[i], fcount, box, min_faces, min_diag, use_diag);
        const bool kf = ok && i < Nf && mesh_cc_keep(parent[faces[3 * (size_t)i]], fcount, box, min_faces, min_diag, use_diag);
        flags[i] = (unsigned char)(kv | (kf << 1));      // flags is padded to whole tiles
        nv += kv;
        nf += kf;
    }
    mesh_block_scan2<int, kMeshThreads>(nv, nf, ta, tb);
    if (threadIdx.x == 0) { bt[2 * blockIdx.x] = ta; bt[2 * blockIdx.x + 1] = tb; }
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_cc_vertices_kernel(const float *__restrict__ vert, const unsigned char *__restrict__ flags, const int *__restrict__ bt,
                        const long long *__restrict__ bo, int *__restrict__ vmap, float *__restrict__ vout) {
    if (bt[2 * blockIdx.x] == 0) return;
    const int i0 = blockIdx.x * kMeshTile + threadIdx.x * kMeshItems;
    const uint32_t f4 = mc_codes4(flags, i0);
    int n = 0, dummy = 0, ta, tb;
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) n += (f4 >> (8 * u)) & 1;
    mesh_block_scan2<int, kMeshThreads>(n, dummy, ta, tb);
    int id = (int)bo[2 * blockIdx.x] + n;
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) {
        if (!((f4 >> (8 * u)) & 1)) continue;
        const int i = i0 + u;
        vmap[i] = id;
#pragma unroll
        for (int a = 0; a < 3; a++) vout[3 * (size_t)id + a] = vert[3 * (size_t)i + a];
        id++;
    }
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_cc_faces_kernel(const int *__restrict__ faces, const unsigned char *__restrict__ flags, const int *__restrict__ bt,
                     const long long *__restrict__ bo, const int *__restrict__ vmap, int *__restrict__ fout) {
    if (bt[2 * blockIdx.x + 1] == 0) return;
    const int i0 = blockIdx.x * kMeshTile + threadIdx.x * kMeshItems;
    const uint32_t f4 = mc_codes4(flags, i0);
    int n = 0, dummy = 0, ta, tb;
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) n += (f4 >> (8 * u + 1)) & 1;
    mesh_block_scan2<int, kMeshThreads>(dummy, n, ta, tb);
    int id = (int)bo[2 * blockIdx.x + 1] + n;
#pragma unroll
    for (int u = 0; u < kMeshItems; u++) {
        if (!((f4 >> (8 * u + 1)) & 1)) continue;
        const int i = i0 + u;
#pragma unroll
        for (int m = 0; m < 3; m++) fout[3 * (size_t)id + m] = vmap[faces[3 * (size_t)i + m]];
        id++;
    }
}

}  // namespace dgr
