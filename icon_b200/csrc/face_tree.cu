// The one builder of the face tree (face_tree.cuh), for icon_smpl_prepare and icon_mesh_prepare.  Compiled with
// -fmad=false.  One launch per step: the faces' bounding box; per face the key morton << 32 | face id (Morton code of
// the centroid in the caller's TreeFrame) and its bucket's count (top 18 code bits); the bucket scan; the scatter; each
// key's rank in its bucket -- keys are unique, so that is the order of a full sort by (code, face id).  Then the sorted
// records and spheres straight from verts / faces, and the boxes level by level.  A fixed frame clamps the codes of a
// mesh that leaves its cube, so one bucket may hold many faces and rank in O(n^2) of its size.
#include <float.h>

#include "common.cuh"
#include "face_tree.cuh"
#include "geom.cuh"

namespace icon {

constexpr int TREE_BUCKET_BITS = 18;
constexpr int TREE_NBUCKET = 1 << TREE_BUCKET_BITS;

TreeWs face_tree_carve(Carver &c, int F) {
    TreeWs w{};
    const size_t total_nodes = tree_levels(w.t, F);
    w.t.tri_s = c.take<float4>((size_t)F * 3);
    w.t.sph_s = c.take<float4>((size_t)F);
    w.t.order = c.take<int32_t>((size_t)F);
    w.t.nodes = c.take<float4>(total_nodes * 2);
    w.t.bounds = c.take<TreeBounds>(1);
    w.keys = c.take<unsigned long long>((size_t)F);
    w.keys_b = c.take<unsigned long long>((size_t)F);
    w.bcount = c.take<int32_t>(TREE_NBUCKET + 1);
    w.boff = c.take<int32_t>(TREE_NBUCKET + 1);
    w.scan_ws = c.take<char>(scan_ws_bytes(TREE_NBUCKET + 1));
    return w;
}

FaceTree face_tree_view(const void *ws, int F) {
    Carver c((void *)ws);
    return face_tree_carve(c, F).t;
}

// ---------------------------------------------------------------- kernels
__device__ __forceinline__ unsigned f2ord(float v) {
    const unsigned b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__global__ void __launch_bounds__(256) k_tree_bounds(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                                     int F, TreeBounds *b) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
    if (f < F) {
        V3 v[3];
        load_face(verts, faces, f, v[0], v[1], v[2]);
        for (int j = 0; j < 3; ++j) {
            const float xs[3] = {v[j].x, v[j].y, v[j].z};
            for (int k = 0; k < 3; ++k) { lo[k] = min(lo[k], f2ord(xs[k])); hi[k] = max(hi[k], f2ord(xs[k])); }
        }
    }
    for (int o = 16; o; o >>= 1)
        for (int k = 0; k < 3; ++k) {
            lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
            hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
        }
    if ((threadIdx.x & 31) == 0)
        for (int k = 0; k < 3; ++k) { atomicMin(&b->lo[k], lo[k]); atomicMax(&b->hi[k], hi[k]); }
}

__global__ void __launch_bounds__(256) k_tree_keys(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                                   TreeFrame fr, TreeWs w) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= w.t.F) return;
    TreeBounds *bd = w.t.bounds;
    const V3 blo = mk3(ord2f(bd->lo[0]), ord2f(bd->lo[1]), ord2f(bd->lo[2]));
    const V3 bhi = mk3(ord2f(bd->hi[0]), ord2f(bd->hi[1]), ord2f(bd->hi[2]));
    if (f == 0)
        bd->absmax = fmaxf(fmaxf(fmaxf(fabsf(blo.x), fabsf(blo.y)), fabsf(blo.z)),
                           fmaxf(fmaxf(fabsf(bhi.x), fabsf(bhi.y)), fabsf(bhi.z)));
    V3 lo = mk3(fr.lo, fr.lo, fr.lo);
    float s = fr.scale;
    if (fr.fit) {
        const float ext = fmaxf(fmaxf(bhi.x - blo.x, bhi.y - blo.y), bhi.z - blo.z);
        lo = blo;
        s = ext > 0.f ? 1024.f / ext : 0.f;
    }
    V3 a, b, c;
    load_face(verts, faces, f, a, b, c);
    const unsigned code = morton30(centroid(a, b, c), lo, s);
    w.keys[f] = ((unsigned long long)code << 32) | (unsigned)f;
    atomicAdd(&w.bcount[code >> (30 - TREE_BUCKET_BITS)], 1);
}

__global__ void __launch_bounds__(256) k_tree_scatter(TreeWs w, int32_t *__restrict__ cursor) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= w.t.F) return;
    const unsigned long long k = w.keys[f];
    const int b = (int)(k >> (62 - TREE_BUCKET_BITS));
    w.keys_b[w.boff[b] + atomicAdd(&cursor[b], 1)] = k;
}

__global__ void __launch_bounds__(256) k_tree_rank(TreeWs w) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w.t.F) return;
    const unsigned long long k = w.keys_b[i];
    const int b = (int)(k >> (62 - TREE_BUCKET_BITS));
    const int o0 = w.boff[b], o1 = w.boff[b + 1];
    int r = 0;
    for (int j = o0; j < o1; ++j) r += w.keys_b[j] < k;
    w.t.order[o0 + r] = (int32_t)(k & 0xffffffffull);
}

// record (a, ab, ac) and bounding sphere (centroid, largest corner distance inflated by 1.0001 and the slack: only a
// conservative lower bound for pruning, never a reported distance) of the face at each sorted position
__global__ void __launch_bounds__(256) k_tree_records(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                                      TreeFrame fr, FaceTree t) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= t.F) return;
    V3 a, b, c;
    load_face(verts, faces, t.order[p], a, b, c);
    write_tri(a, b, c, t.tri_s + 3 * (size_t)p);
    const V3 sc = centroid(a, b, c);
    const float ra = dot3(sub3(a, sc), sub3(a, sc)), rb = dot3(sub3(b, sc), sub3(b, sc)),
                rc = dot3(sub3(c, sc), sub3(c, sc));
    const float slack = fr.scaled_slack ? 1e-7f * fmaxf(1.f, t.bounds->absmax) : 1e-7f;
    t.sph_s[p] = make_float4(sc.x, sc.y, sc.z, sqrtf(fmaxf(ra, fmaxf(rb, rc))) * 1.0001f + slack);
}

// the boxes of level l (0: leaves); a launch of one CTA goes on through the root
__global__ void __launch_bounds__(1024) k_tree_levels(FaceTree t, int l) {
    for (;;) {
        for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < t.lvl_cnt[l]; n += gridDim.x * blockDim.x) {
            if (l == 0) write_leaf_box(t, n);
            else write_parent_box(t, l, n);
        }
        if (gridDim.x > 1 || ++l == t.nlevels) return;
        __threadfence_block();
        __syncthreads();
    }
}

int face_tree_build(void *ws, const float *verts, const int64_t *faces, int F, TreeFrame frame, cudaStream_t stream) {
    Carver c(ws);
    const TreeWs w = face_tree_carve(c, F);
    const unsigned nb = (unsigned)((F + 255) / 256);
    ICON_CUDA(cudaMemsetAsync(w.t.bounds->lo, 0xff, sizeof(w.t.bounds->lo), stream));
    ICON_CUDA(cudaMemsetAsync(w.t.bounds->hi, 0, sizeof(w.t.bounds->hi), stream));
    k_tree_bounds<<<nb, 256, 0, stream>>>(verts, faces, F, w.t.bounds);
    ICON_LAUNCHED();
    ICON_CUDA(cudaMemsetAsync(w.bcount, 0, sizeof(int32_t) * (TREE_NBUCKET + 1), stream));
    k_tree_keys<<<nb, 256, 0, stream>>>(verts, faces, frame, w);
    ICON_LAUNCHED();
    const int rc = scan_exclusive_i32(w.bcount, w.boff, TREE_NBUCKET + 1, nullptr, w.scan_ws, stream);
    if (rc) return rc;
    ICON_CUDA(cudaMemsetAsync(w.bcount, 0, sizeof(int32_t) * (TREE_NBUCKET + 1), stream));   // reuse as cursor
    k_tree_scatter<<<nb, 256, 0, stream>>>(w, w.bcount);
    ICON_LAUNCHED();
    k_tree_rank<<<nb, 256, 0, stream>>>(w);
    ICON_LAUNCHED();
    k_tree_records<<<nb, 256, 0, stream>>>(verts, faces, frame, w.t);
    ICON_LAUNCHED();
    for (int l = 0; l < w.t.nlevels; ++l) {
        const unsigned nl = (unsigned)((w.t.lvl_cnt[l] + 1023) / 1024);
        k_tree_levels<<<nl, 1024, 0, stream>>>(w.t, l);
        ICON_LAUNCHED();
        if (nl == 1) break;
    }
    return ICON_OK;
}

}  // namespace icon

using namespace icon;

extern "C" int icon_face_tree_read(const void *mesh_ws, int V, int F, int32_t *order, float *tri_s, float *sph_s,
                                   float *nodes) {
    ICON_CHECK_ARG(mesh_ws && V > 0 && F > 0 && order && tri_s && sph_s && nodes, "icon_face_tree_read: bad argument");
    const FaceTree t = face_tree_view(mesh_ws, F);
    const size_t total_nodes = (size_t)t.lvl_off[t.nlevels - 1] + 1;
    ICON_CUDA(cudaDeviceSynchronize());
    ICON_CUDA(cudaMemcpy(order, t.order, sizeof(int32_t) * F, cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(tri_s, t.tri_s, sizeof(float4) * 3 * (size_t)F, cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(sph_s, t.sph_s, sizeof(float4) * (size_t)F, cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(nodes, t.nodes, sizeof(float4) * 2 * total_nodes, cudaMemcpyDeviceToHost));
    return ICON_OK;
}
