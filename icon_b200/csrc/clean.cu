// clean_mesh on the device: keep the connected component with the most vertices.
//
// Replaces lib/dataset/mesh_util.py:778-791 (trimesh: Trimesh(verts, faces).split(only_watertight=False), component
// with the most vertices), the step apps/ICON.py:755-756 runs right after export_mesh -- the marching-cubes output
// never has to leave the GPU just to be split on the CPU.
//
// trimesh's relation, for any triangle mesh: two FACES are adjacent when they share an edge that is used by exactly
// two faces (an edge counted once per face corner pair, so a face [a, a, b] uses (a, b) twice); a component's size is
// its number of distinct vertices (a vertex can belong to several components: bow ties, edges of 3+ faces); the first
// largest component in smallest-face-index order is kept.  Computed with a lock-free union-find over the face ids:
//   k_cc_edges     every face corner pair (min, max vertex) into an open-addressing hash table: use count and the
//                  XOR of the using face ids (for an edge of two faces, my id ^ xor = the other face)
//   k_cc_union     for every edge used by exactly two faces: unite(f, other)   (atomicMin hooks: roots only decrease,
//                  so every root is its component's smallest face index, whatever order the blocks run in)
//   k_cc_flatten   parent[f] = root(f)
//   k_cc_vcount    distinct (root, vertex) pairs through a second table: count[root] += 1 per new pair
//   k_cc_best      arg max of count (ties: smallest root)
//   k_cc_flag      kept faces; their vertices; scans -> ascending original order (trimesh's submesh re-indexing)
//   k_cc_emit      compacted float32 vertices and int32 faces (the reference returns .float() / .int())
// Every step is exact integer work, so the result does not depend on scheduling.
#include "common.cuh"

namespace icon {

constexpr unsigned long long CC_EMPTY = ~0ull;          // no key: vertex / face ids are < 2^31

__device__ __forceinline__ int cc_find(const int *parent_, int v) {
    const volatile int *parent = parent_;                // other threads hook roots concurrently: always re-read
    int p = parent[v];
    while (p != v) { v = p; p = parent[v]; }
    return v;
}

__device__ __forceinline__ void cc_unite(int *parent, int a, int b) {
    while (true) {
        a = cc_find(parent, a);
        b = cc_find(parent, b);
        if (a == b) return;
        if (a > b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(&parent[b], a);        // hook the larger root under the smaller one
        if (old == b) return;
        b = old;                                         // somebody hooked b first: continue from where it points
    }
}

// insert `key` (linear probing, splitmix64 slot); returns the slot, *fresh = this call claimed it
__device__ __forceinline__ unsigned cc_insert(unsigned long long *keys, unsigned mask, unsigned long long key, bool *fresh) {
    unsigned long long h = key;
    h = (h ^ (h >> 30)) * 0xbf58476d1ce4e5b9ull;
    h = (h ^ (h >> 27)) * 0x94d049bb133111ebull;
    h ^= h >> 31;
    unsigned s = (unsigned)h & mask;
    while (true) {
        const unsigned long long prev = atomicCAS(&keys[s], CC_EMPTY, key);
        if (prev == CC_EMPTY || prev == key) { *fresh = prev == CC_EMPTY; return s; }
        s = (s + 1) & mask;                              // the table is at most half full: a free slot exists
    }
}

__global__ void k_cc_init(int *parent, int *count, int32_t *vflag, int nv, int nf) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nf) { parent[i] = i; count[i] = 0; }
    if (i < nv) vflag[i] = 0;
}

// one thread per face corner pair e = 3 f + c: edge (faces[f][c], faces[f][(c + 1) % 3])
__global__ void k_cc_edges(const int64_t *__restrict__ faces, int64_t ne, unsigned long long *keys, unsigned mask,
                           int *ecount, unsigned *exor, int32_t *slot_of) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne) return;
    const int64_t f = e / 3, c = e - 3 * f;
    const unsigned a = (unsigned)faces[e], b = (unsigned)faces[3 * f + (c == 2 ? 0 : c + 1)];
    const unsigned long long key = a < b ? ((unsigned long long)a << 32 | b) : ((unsigned long long)b << 32 | a);
    bool fresh;
    const unsigned s = cc_insert(keys, mask, key, &fresh);
    atomicAdd(&ecount[s], 1);
    atomicXor(&exor[s], (unsigned)f);
    slot_of[e] = (int32_t)s;
}

__global__ void k_cc_union(int64_t ne, const int *__restrict__ ecount, const unsigned *__restrict__ exor,
                           const int32_t *__restrict__ slot_of, int *parent) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne) return;
    const int s = slot_of[e];
    if (ecount[s] != 2) return;
    const int f = (int)(e / 3), other = (int)(exor[s] ^ (unsigned)f);
    if (f < other) cc_unite(parent, f, other);           // the pair's other corner sees f > other; f == other: a loop
}

__global__ void k_cc_flatten(int *parent, int nf) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nf) parent[i] = cc_find(parent, i);          // other threads may still walk through i: r is on their path
}

__global__ void k_cc_vcount(const int64_t *__restrict__ faces, int64_t ne, const int *__restrict__ parent,
                            unsigned long long *keys, unsigned mask, int *count) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne) return;
    const int r = parent[e / 3];
    bool fresh;
    cc_insert(keys, mask, (unsigned long long)(unsigned)r << 32 | (unsigned)faces[e], &fresh);
    if (fresh) atomicAdd(&count[r], 1);
}

__global__ void k_cc_best(const int *__restrict__ count, int nf, unsigned long long *best) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long key = 0;
    if (i < nf && count[i] > 0) key = ((unsigned long long)(unsigned)count[i] << 32) | (unsigned)(0x7fffffff - i);
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
        key = other > key ? other : key;
    }
    if ((threadIdx.x & 31) == 0 && key) atomicMax(best, key);
}

__device__ __forceinline__ int cc_best_root(const unsigned long long *best) {
    return 0x7fffffff - (int)(unsigned)(*best & 0xffffffffull);
}

__global__ void k_cc_flag(const int *__restrict__ parent, const int64_t *__restrict__ faces, int nf,
                          const unsigned long long *__restrict__ best, int32_t *vflag, int32_t *fflag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    const bool keep = parent[i] == cc_best_root(best);
    fflag[i] = keep ? 1 : 0;
    if (keep) {                                          // every writer stores the same 1
        vflag[faces[3 * (size_t)i]] = 1;
        vflag[faces[3 * (size_t)i + 1]] = 1;
        vflag[faces[3 * (size_t)i + 2]] = 1;
    }
}

template <typename VT>
__global__ void k_cc_emit(const VT *__restrict__ verts, const int64_t *__restrict__ faces, int nv, int nf,
                          const int *__restrict__ parent, const unsigned long long *__restrict__ best,
                          const int32_t *__restrict__ vflag, const int32_t *__restrict__ vpos,
                          const int32_t *__restrict__ fpos, float *__restrict__ out_v, int32_t *__restrict__ out_f) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nv && vflag[i]) {
        const int d = vpos[i];
        out_v[3 * (size_t)d] = (float)verts[3 * (size_t)i];
        out_v[3 * (size_t)d + 1] = (float)verts[3 * (size_t)i + 1];
        out_v[3 * (size_t)d + 2] = (float)verts[3 * (size_t)i + 2];
    }
    if (i < nf && parent[i] == cc_best_root(best)) {
        const int d = fpos[i];
        out_f[3 * (size_t)d] = vpos[(int)faces[3 * (size_t)i]];
        out_f[3 * (size_t)d + 1] = vpos[(int)faces[3 * (size_t)i + 1]];
        out_f[3 * (size_t)d + 2] = vpos[(int)faces[3 * (size_t)i + 2]];
    }
}

// hash table slots: a power of two >= 2 x (3 nf) keys, so that linear probing always finds a free slot quickly
static int64_t clean_slots(int64_t nf) {
    int64_t s = 1024;
    while (s < 6 * nf) s *= 2;
    return s;
}

struct CleanWs {
    int *parent, *count;                                 // per face
    int32_t *vflag, *vpos, *fpos;
    int32_t *slot_of;                                    // per face corner pair
    unsigned long long *keys;                            // per slot
    int *ecount;
    unsigned *exor;
    unsigned long long *best;
    void *scan;
};
static size_t clean_carve(void *ws, int64_t nv, int64_t nf, CleanWs *o) {
    Carver c(ws);
    CleanWs w;
    const int64_t ns = clean_slots(nf);
    w.parent = c.take<int>(nf);
    w.count = c.take<int>(nf);
    w.vflag = c.take<int32_t>(nv);
    w.vpos = c.take<int32_t>(nv);
    w.fpos = c.take<int32_t>(nf);
    w.slot_of = c.take<int32_t>(3 * nf);
    w.keys = c.take<unsigned long long>(ns);
    w.ecount = c.take<int>(ns);
    w.exor = c.take<unsigned>(ns);
    w.best = c.take<unsigned long long>(1);
    w.scan = c.take<char>(scan_ws_bytes(nv > nf ? nv : nf));
    if (o) *o = w;
    return c.total();
}

}  // namespace icon

using namespace icon;

extern "C" size_t icon_clean_mesh_workspace_bytes(int64_t nv, int64_t nf) { return clean_carve(nullptr, nv, nf, nullptr); }

extern "C" int icon_clean_mesh_count(const int64_t *faces, int64_t nv, int64_t nf, void *ws, size_t ws_bytes,
                                     int64_t *d_counts /* [2]: vertices, faces kept */, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(faces && ws && d_counts && nv > 0 && nf > 0 && nv < 0x7fffffff && nf < ((int64_t)1 << 28),
                   "icon_clean_mesh_count: bad argument");
    if (ws_bytes < icon_clean_mesh_workspace_bytes(nv, nf)) { set_error("icon_clean_mesh_count: workspace too small"); return ICON_ENOSPC; }
    CleanWs w;
    clean_carve(ws, nv, nf, &w);
    const int64_t ne = 3 * nf, ns = clean_slots(nf);
    const unsigned mask = (unsigned)(ns - 1);
    const unsigned gv = (unsigned)((nv + 255) / 256), gf = (unsigned)((nf + 255) / 256), gm = gv > gf ? gv : gf;
    const unsigned ge = (unsigned)((ne + 255) / 256);
    k_cc_init<<<gm, 256, 0, stream>>>(w.parent, w.count, w.vflag, (int)nv, (int)nf);
    ICON_LAUNCHED();
    ICON_CUDA(cudaMemsetAsync(w.keys, 0xff, ns * sizeof(unsigned long long), stream));
    ICON_CUDA(cudaMemsetAsync(w.ecount, 0, ns * sizeof(int), stream));
    ICON_CUDA(cudaMemsetAsync(w.exor, 0, ns * sizeof(unsigned), stream));
    ICON_CUDA(cudaMemsetAsync(w.best, 0, sizeof(unsigned long long), stream));
    k_cc_edges<<<ge, 256, 0, stream>>>(faces, ne, w.keys, mask, w.ecount, w.exor, w.slot_of);
    ICON_LAUNCHED();
    k_cc_union<<<ge, 256, 0, stream>>>(ne, w.ecount, w.exor, w.slot_of, w.parent);
    ICON_LAUNCHED();
    k_cc_flatten<<<gf, 256, 0, stream>>>(w.parent, (int)nf);
    ICON_LAUNCHED();
    ICON_CUDA(cudaMemsetAsync(w.keys, 0xff, ns * sizeof(unsigned long long), stream));   // second table: (root, vertex)
    k_cc_vcount<<<ge, 256, 0, stream>>>(faces, ne, w.parent, w.keys, mask, w.count);
    ICON_LAUNCHED();
    k_cc_best<<<gf, 256, 0, stream>>>(w.count, (int)nf, w.best);
    ICON_LAUNCHED();
    k_cc_flag<<<gf, 256, 0, stream>>>(w.parent, faces, (int)nf, w.best, w.vflag, w.fpos);
    ICON_LAUNCHED();
    int rc = scan_exclusive_i32(w.vflag, w.vpos, nv, d_counts, w.scan, stream);
    if (rc) return rc;
    return scan_exclusive_i32(w.fpos, w.fpos, nf, d_counts + 1, w.scan, stream);
}

extern "C" int icon_clean_mesh_emit(const void *verts, int verts_f64, const int64_t *faces, int64_t nv, int64_t nf,
                                    const void *ws, float *out_verts, int32_t *out_faces, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(verts && faces && ws && out_verts && out_faces && nv > 0 && nf > 0, "icon_clean_mesh_emit: bad argument");
    CleanWs w;
    clean_carve(const_cast<void *>(ws), nv, nf, &w);
    const unsigned gm = (unsigned)(((nv > nf ? nv : nf) + 255) / 256);
    if (verts_f64)
        k_cc_emit<double><<<gm, 256, 0, stream>>>((const double *)verts, faces, (int)nv, (int)nf, w.parent, w.best, w.vflag,
                                                  w.vpos, w.fpos, out_verts, out_faces);
    else
        k_cc_emit<float><<<gm, 256, 0, stream>>>((const float *)verts, faces, (int)nv, (int)nf, w.parent, w.best, w.vflag,
                                                 w.vpos, w.fpos, out_verts, out_faces);
    ICON_LAUNCHED();
    return ICON_OK;
}
