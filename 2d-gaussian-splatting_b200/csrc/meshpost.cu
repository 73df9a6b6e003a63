// meshpost.cu — cluster filtering of an extracted mesh (the reference's post_process_mesh, utils/mesh_utils.py:22-43,
// which `render.py` runs on every exported mesh) on the device.  DESIGN.md §7k has the rules; tests/meshpost_ref.py
// restates them.
//
//  * surfel_meshpost_clusters: connected components of the faces over shared edges, numbered as Open3D's
//    ClusterConnectedTriangles numbers them (the rank of the component's smallest face among all components'
//    smallest faces), and each component's face count.
//     - edges: one thread per face checks its indices (a bad one raises the error flag; nothing is ever addressed by
//       a face index in this call) and writes three records, key min * M + max of each edge and value the face.
//     - launch_radix_sort_pairs sorts the records by key.
//     - union: every pair of neighbouring sorted records with equal keys unions their faces in a lock-free
//       union-find that hooks the larger root under the smaller with atomicCAS and halves paths in find.  Since a
//       parent is never larger than its child, each component ends with its smallest face as its only root,
//       whatever order the races ran in.
//     - label: a pass of path halving shortens the paths; then a pass that writes only each face's own parent
//       (halving writes other faces' parents, and a stale one could overwrite a root already stored) sets parent[t]
//       to t's root and scans the root flags with the look-back of scan.cuh (the rank of a root is its cluster id);
//       a last pass writes each face's id and adds it to its cluster's count with warp-aggregated integer atomics,
//       so the counts do not depend on the order either.
//  * surfel_meshpost_compact: sorts the C counts with the same radix sort, takes the threshold max(sorted[index], 50)
//    on the device, marks the vertices of the faces that pass it (degenerate ones included), scans the marks into
//    new vertex indices and the old index of each kept vertex, and scans the kept non-degenerate faces, writing them
//    remapped.  Both scans keep order, so the output is the reference's whatever the schedule.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "kernels.h"
#include "profile.h"
#include "scan.cuh"

namespace surfel {
namespace {

constexpr int kMpThreads = 256;
constexpr long long kMpMaxVerts = 1ll << 31;      // vertex indices and counts travel in 32 bits
constexpr long long kMpMaxFaces = kRadixSortMaxPairs / 3;   // 3 F edge records go through one radix sort
constexpr uint32_t kMpMinCluster = 50;            // post_process_mesh's max(n_cluster, 50)

__device__ __forceinline__ uint32_t ld_parent(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_parent(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// root of x, halving the path on the way: every value written is an ancestor of its node, so concurrent finds and
// hooks (which only change roots) never break the forest
__device__ __forceinline__ uint32_t uf_find(uint32_t* parent, uint32_t x) {
    while (true) {
        const uint32_t p = ld_parent(parent + x);
        if (p == x) return x;
        const uint32_t gp = ld_parent(parent + p);
        if (gp == p) return p;
        st_parent(parent + x, gp);
        x = gp;
    }
}

// root of x without writing: once no union is running, the only stores are each node's own root, so this is exact
__device__ __forceinline__ uint32_t uf_root(const uint32_t* parent, uint32_t x) {
    uint32_t p;
    while ((p = ld_parent(parent + x)) != x) x = p;
    return x;
}

__device__ __forceinline__ void uf_union(uint32_t* parent, uint32_t a, uint32_t b) {
    while (true) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        if (a > b) { const uint32_t t = a; a = b; b = t; }
        if (atomicCAS(parent + b, b, a) == b) return;       // b was still a root: hooked under the smaller a
    }
}

__global__ void __launch_bounds__(kMpThreads) mp_edges_kernel(long long F, long long M,
                                                              const long long* __restrict__ faces,
                                                              uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                              uint32_t* __restrict__ parent, uint32_t* err) {
    const long long f = (long long)blockIdx.x * kMpThreads + threadIdx.x;
    if (f >= F) return;
    long long v[3];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 3; j++) {
        v[j] = faces[3 * f + j];
        ok &= v[j] >= 0 && v[j] < M;
    }
    if (!ok) atomicOr(err, 1u);
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const long long a = v[j], b = v[(j + 1) % 3];
        keys[3 * f + j] = ok ? (uint64_t)(a < b ? a : b) * (uint64_t)M + (uint64_t)(a < b ? b : a) : 0ull;
        vals[3 * f + j] = (uint32_t)f;
    }
    parent[f] = (uint32_t)f;
}

__global__ void __launch_bounds__(kMpThreads) mp_union_kernel(long long n, const uint64_t* __restrict__ keys,
                                                              const uint32_t* __restrict__ vals, uint32_t* parent) {
    const long long i = (long long)blockIdx.x * kMpThreads + threadIdx.x + 1;
    if (i >= n || keys[i] != keys[i - 1]) return;
    uf_union(parent, vals[i - 1], vals[i]);
}

// shortens every path after the unions, with the halving of uf_find.  A halving write may land on a node after
// that node stored its root, so this pass leaves short paths, not roots; mp_roots_kernel finishes them.
__global__ void __launch_bounds__(kMpThreads) mp_compress_kernel(long long F, uint32_t* parent) {
    const long long t = (long long)blockIdx.x * kMpThreads + threadIdx.x;
    if (t < F) st_parent(parent + t, uf_find(parent, (uint32_t)t));
}

// parent[t] = root of t (each thread writes only its own node); the rank of each root among the roots (its cluster
// id) into rank[root]; the last block writes C and the error flag to info
__global__ void __launch_bounds__(kMpThreads) mp_roots_kernel(long long F, uint32_t* parent, uint32_t* __restrict__ rank,
                                                              uint32_t* ctrl, unsigned long long* status,
                                                              long long* info) {
    const uint32_t bid = block_ticket(&ctrl[0]);
    const long long t = (long long)bid * kMpThreads + threadIdx.x;
    bool root = false;
    if (t < F) {
        const uint32_t r = uf_root(parent, (uint32_t)t);
        st_parent(parent + t, r);
        root = r == (uint32_t)t;
    }
    const GridScan s = grid_exclusive_scan<kMpThreads>(root ? 1u : 0u, bid, status);
    if (root) rank[t] = s.rank;
    if (s.last && threadIdx.x == 0) {
        info[0] = (long long)s.base + s.total;
        info[1] = ctrl[4];
    }
}

__global__ void __launch_bounds__(kMpThreads) mp_label_kernel(long long F, const uint32_t* __restrict__ parent,
                                                              const uint32_t* __restrict__ rank,
                                                              int* __restrict__ face_cluster, int* cluster_count) {
    const long long t = (long long)blockIdx.x * kMpThreads + threadIdx.x;
    const uint32_t c = t < F ? rank[parent[t]] : 0xffffffffu;
    if (t < F) face_cluster[t] = (int)c;
    const unsigned peers = __match_any_sync(0xffffffffu, c);   // a component's faces are often neighbours
    if (t < F && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(cluster_count + c, __popc(peers));
}

__global__ void mp_count_keys_kernel(long long C, const int* __restrict__ cluster_count, uint64_t* __restrict__ keys,
                                     uint32_t* __restrict__ vals) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C) return;
    keys[i] = (uint64_t)(uint32_t)cluster_count[i];
    vals[i] = (uint32_t)i;
}

__device__ __forceinline__ bool mp_kept(long long f, const int* face_cluster, const int* cluster_count,
                                        const uint64_t* kth) {
    const uint64_t k = *kth, thr = k > kMpMinCluster ? k : kMpMinCluster;
    return (uint64_t)(uint32_t)cluster_count[face_cluster[f]] >= thr;
}

__global__ void __launch_bounds__(kMpThreads) mp_mark_kernel(long long F, long long M, const long long* __restrict__ faces,
                                                             const int* __restrict__ face_cluster,
                                                             const int* __restrict__ cluster_count,
                                                             const uint64_t* kth, uint32_t* vnew) {
    const long long f = (long long)blockIdx.x * kMpThreads + threadIdx.x;
    if (f >= F || !mp_kept(f, face_cluster, cluster_count, kth)) return;
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const long long v = faces[3 * f + j];
        if (v >= 0 && v < M) vnew[v] = 1u;
    }
}

// in place: the mark of each vertex becomes its new index; kept vertices write their old index to vert_map
__global__ void __launch_bounds__(kMpThreads) mp_vscan_kernel(long long M, uint32_t* vnew, long long* __restrict__ vert_map,
                                                              uint32_t* ctrl, unsigned long long* status,
                                                              long long* info) {
    const uint32_t bid = block_ticket(&ctrl[1]);
    const long long v = (long long)bid * kMpThreads + threadIdx.x;
    const bool marked = v < M && vnew[v] != 0;
    const GridScan s = grid_exclusive_scan<kMpThreads>(marked ? 1u : 0u, bid, status);
    if (marked) {
        vnew[v] = s.rank;
        vert_map[s.rank] = v;
    }
    if (s.last && threadIdx.x == 0) info[0] = (long long)s.base + s.total;
}

__global__ void __launch_bounds__(kMpThreads) mp_fscan_kernel(long long F, long long M, const long long* __restrict__ faces,
                                                              const int* __restrict__ face_cluster,
                                                              const int* __restrict__ cluster_count,
                                                              const uint64_t* kth, const uint32_t* __restrict__ vnew,
                                                              long long* __restrict__ out_faces, uint32_t* ctrl,
                                                              unsigned long long* status, long long* info) {
    const uint32_t bid = block_ticket(&ctrl[2]);
    const long long f = (long long)bid * kMpThreads + threadIdx.x;
    long long v[3] = {0, 0, 0};
    bool keep = false;
    if (f < F && mp_kept(f, face_cluster, cluster_count, kth)) {
        keep = true;
#pragma unroll
        for (int j = 0; j < 3; j++) {
            v[j] = faces[3 * f + j];
            keep &= v[j] >= 0 && v[j] < M;
        }
        keep &= v[0] != v[1] && v[1] != v[2] && v[0] != v[2];
    }
    const GridScan s = grid_exclusive_scan<kMpThreads>(keep ? 1u : 0u, bid, status);
    if (keep) {
#pragma unroll
        for (int j = 0; j < 3; j++) out_faces[3 * (long long)s.rank + j] = vnew[v[j]];
    }
    if (s.last && threadIdx.x == 0) info[1] = (long long)s.base + s.total;
}

struct MpLayout {
    size_t ctrl, status_f, status_m, status_c, sort, parent, rank, vnew, total;
};

// ctrl: [0..2] tickets of the three scans, [4] error flag
MpLayout mp_layout(long long M, long long F) {
    MpLayout L;
    const size_t f = (size_t)std::max<long long>(F, 1), m = (size_t)std::max<long long>(M, 1), r = 3 * f;
    size_t o = 0;
    L.ctrl = o;     o = align_up(o + 64, 256);
    L.status_f = o; o = align_up(o + (size_t)grid_blocks(F, kMpThreads) * 8, 256);
    L.status_m = o; o = align_up(o + (size_t)grid_blocks(M, kMpThreads) * 8, 256);
    L.status_c = o; o = align_up(o + (size_t)grid_blocks(F, kMpThreads) * 8, 256);
    L.sort = o;     o = align_up(o + radix_sort_workspace_bytes(r), 256);
    L.parent = o;   o = align_up(o + f * 4, 256);
    L.rank = o;     o = align_up(o + f * 4, 256);
    L.vnew = o;     o = align_up(o + m * 4, 256);
    L.total = o;
    return L;
}

bool sizes_ok(const char* who, long long M, long long F) {
    if (M < 0 || F < 0) { surfel_set_error("%s: negative size (%lld vertices, %lld faces)", who, M, F); return false; }
    if (M >= kMpMaxVerts) {
        surfel_set_error("%s: %lld vertices; fewer than 2^31 are supported", who, M);
        return false;
    }
    if (F > kMpMaxFaces) {
        surfel_set_error("%s: %lld faces give %lld edge records; the radix sort takes fewer than 2^30", who, F, 3 * F);
        return false;
    }
    return true;
}

}  // namespace
}  // namespace surfel

using namespace surfel;

extern "C" {

size_t surfel_meshpost_workspace_bytes(long long n_verts, long long n_faces) {
    if (n_verts < 0 || n_faces < 0 || n_verts >= kMpMaxVerts || n_faces > kMpMaxFaces) return 0;
    return mp_layout(n_verts, n_faces).total;
}

int surfel_meshpost_clusters(long long n_verts, long long n_faces, const long long* faces, void* workspace,
                             size_t workspace_bytes, int* face_cluster, int* cluster_count, long long* info,
                             void* stream) {
    const char* who = "surfel_meshpost_clusters";
    if (!sizes_ok(who, n_verts, n_faces)) return 1;
    if (!info || (n_faces > 0 && (!faces || !face_cluster || !cluster_count))) {
        surfel_set_error("%s: NULL faces, cluster ids, cluster counts or info", who);
        return 1;
    }
    const MpLayout L = mp_layout(n_verts, n_faces);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (n_faces == 0) {
        SURFEL_CUDA_OK(cudaMemsetAsync(info, 0, 2 * sizeof(long long), st));
        return 0;
    }
    char* w = (char*)workspace;
    uint32_t* ctrl = (uint32_t*)(w + L.ctrl);
    const unsigned long long M = (unsigned long long)n_verts;
    const RadixSortWs sort = radix_sort_ws(w + L.sort, 3 * (size_t)n_faces, radix_key_bits(M > 0 ? M * M - 1 : 0));
    uint32_t *parent = (uint32_t*)(w + L.parent), *rank = (uint32_t*)(w + L.rank);
    SURFEL_CUDA_OK(cudaMemsetAsync(ctrl, 0, 64, st));
    const unsigned nb_f = grid_blocks(n_faces, kMpThreads);
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status_f, 0, (size_t)nb_f * 8, st));
    SURFEL_CUDA_OK(cudaMemsetAsync(cluster_count, 0, (size_t)n_faces * sizeof(int), st));
    const long long n_rec = 3 * n_faces;
    {
        LaunchScope scope(kStMeshpostEdges, st);
        mp_edges_kernel<<<nb_f, kMpThreads, 0, st>>>(n_faces, n_verts, faces, sort.in.keys, sort.in.vals, parent,
                                                     ctrl + 4);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    if (launch_radix_sort_pairs(sort, (size_t)n_rec, st)) return 1;
    {
        LaunchScope scope(kStMeshpostUnion, st);
        mp_union_kernel<<<grid_blocks(n_rec - 1, kMpThreads), kMpThreads, 0, st>>>(n_rec, sort.out.keys, sort.out.vals,
                                                                                    parent);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    {
        LaunchScope scope(kStMeshpostUnion, st);
        mp_compress_kernel<<<nb_f, kMpThreads, 0, st>>>(n_faces, parent);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    {
        LaunchScope scope(kStMeshpostLabel, st);
        mp_roots_kernel<<<nb_f, kMpThreads, 0, st>>>(n_faces, parent, rank, ctrl,
                                                     (unsigned long long*)(w + L.status_f), info);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    {
        LaunchScope scope(kStMeshpostLabel, st);
        mp_label_kernel<<<nb_f, kMpThreads, 0, st>>>(n_faces, parent, rank, face_cluster, cluster_count);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int surfel_meshpost_compact(long long n_verts, long long n_faces, const long long* faces, const int* face_cluster,
                            const int* cluster_count, long long n_clusters, long long index, void* workspace,
                            size_t workspace_bytes, long long* out_faces, long long* vert_map, long long* info,
                            void* stream) {
    const char* who = "surfel_meshpost_compact";
    if (!sizes_ok(who, n_verts, n_faces)) return 1;
    if (n_clusters < 1 || n_clusters > n_faces) {
        surfel_set_error("%s: %lld clusters for %lld faces", who, n_clusters, n_faces);
        return 1;
    }
    if (index < 0 || index >= n_clusters) {
        surfel_set_error("%s: index %lld outside [0, %lld)", who, index, n_clusters);
        return 1;
    }
    if (!faces || !face_cluster || !cluster_count || !out_faces || !info || (n_verts > 0 && !vert_map)) {
        surfel_set_error("%s: NULL faces, cluster ids, cluster counts, output or info", who);
        return 1;
    }
    const MpLayout L = mp_layout(n_verts, n_faces);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    uint32_t* ctrl = (uint32_t*)(w + L.ctrl);
    const RadixSortWs sort = radix_sort_ws(w + L.sort, 3 * (size_t)n_faces, radix_key_bits((unsigned long long)n_faces));
    uint32_t* vnew = (uint32_t*)(w + L.vnew);
    SURFEL_CUDA_OK(cudaMemsetAsync(ctrl, 0, 64, st));
    const unsigned nb_m = grid_blocks(n_verts, kMpThreads), nb_f = grid_blocks(n_faces, kMpThreads);
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status_m, 0, (size_t)nb_m * 8, st));
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status_c, 0, (size_t)nb_f * 8, st));
    SURFEL_CUDA_OK(cudaMemsetAsync(vnew, 0, (size_t)std::max<long long>(n_verts, 1) * 4, st));
    {
        LaunchScope scope(kStMeshpostCompact, st);
        mp_count_keys_kernel<<<grid_blocks(n_clusters, kMpThreads), kMpThreads, 0, st>>>(n_clusters, cluster_count,
                                                                                          sort.in.keys, sort.in.vals);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    if (launch_radix_sort_pairs(sort, (size_t)n_clusters, st)) return 1;
    const uint64_t* kth = sort.out.keys + index;
    {
        LaunchScope scope(kStMeshpostCompact, st);
        mp_mark_kernel<<<nb_f, kMpThreads, 0, st>>>(n_faces, n_verts, faces, face_cluster, cluster_count, kth, vnew);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    {
        LaunchScope scope(kStMeshpostCompact, st);
        mp_vscan_kernel<<<nb_m, kMpThreads, 0, st>>>(n_verts, vnew, vert_map, ctrl,
                                                     (unsigned long long*)(w + L.status_m), info);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    {
        LaunchScope scope(kStMeshpostCompact, st);
        mp_fscan_kernel<<<nb_f, kMpThreads, 0, st>>>(n_faces, n_verts, faces, face_cluster, cluster_count, kth, vnew,
                                                     out_faces, ctrl, (unsigned long long*)(w + L.status_c), info);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

}  // extern "C"
