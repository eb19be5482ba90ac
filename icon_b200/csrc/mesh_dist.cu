// Distance-only mesh workspace, unsigned nearest-face query and even surface sampler: the two trimesh calls of the
// benchmark's Chamfer / P2S metric (reference: Evaluator.calculate_chamfer_p2s, lib/dataset/Evaluator.py:200-230).
// Compiled with -fmad=false.
//
//   trimesh.proximity.closest_point  -> icon_mesh_distance: exact squared distance + lowest-index nearest face
//   trimesh.sample.sample_surface_even -> icon_mesh_sample: area-weighted candidates, greedy radius removal
//
// Any triangle mesh (no cmap / vis / normals, no sign): icon_mesh_prepare builds the face tree with the same builder
// as icon_smpl_prepare (face_tree.cu), over the mesh's own bounding cube and with the sphere slack scaled by its
// largest |coordinate|; the walk uses 32-bit ids, so F is bounded by memory only.  The rest of the prepare is the
// sampler's: the largest face area, the fixed-point area weights and their uint64 prefix sum.
//
// k_mesh_dist runs face_tree.cuh's walk at one query point per warp (PPW = 1): the query sets are sparse (1000 samples
// on a mesh), so the warp box is the point and the 32 lanes split the candidate faces.  The frontier holds 1024
// 32-bit ids; the slacks scale with the largest coordinate in play.  Results equal the brute-force scan
// (oracle_mesh_distance in oracle/mesh_oracle.c) bit for bit.
//
// Resources (nvcc 12.9 -Xptxas -v, sm_90a): k_mesh_dist 56 registers, 41472 bytes static shared memory per
// 128-thread block (4 warps x (2 x 1024 frontier ids + 32 staged faces)), no spills; shared memory bounds residency at
// 5 blocks = 20 warps per SM.  k_gm_select 32 registers, no spills.
#include <float.h>

#include "common.cuh"
#include "face_tree.cuh"
#include "geom.cuh"

namespace icon {

constexpr int GM_T = 128;                    // 4 warps per block, one query point per warp
constexpr int GM_FR_CAP = 1024;              // frontier capacity per warp (node / leaf ids)
constexpr int GM_SAMPLE_MAX = 8192;          // most samples icon_mesh_sample keeps (shared memory of the removal pass)
constexpr int S64_T = 256, S64_I = 8, S64_B = S64_T * S64_I;   // uint64 inclusive scan: elements per block

struct GMeshHeader {                         // device-resident, written by icon_mesh_prepare
    unsigned long long amax;                 // largest face area (fp64 bits; areas are >= 0 so bits order like values)
    unsigned long long total;                // sum of the fixed-point face weights (sampler)
    int wbits;                               // weight_f = floor(area_f / amax * 2^wbits)
};

struct GMesh : FaceTree {
    unsigned long long *wcum;                // [F] inclusive prefix sum of the face weights, original face order
    GMeshHeader *hdr;
    unsigned long long *s64_ws;              // block totals of the uint64 scan
    int V;
};

static size_t s64_ws_elems(int64_t n) {
    size_t tot = 0;
    while (n > 1) {
        n = (n + S64_B - 1) / S64_B;
        tot += (size_t)n + 32;
    }
    return tot + 32;
}

static GMesh carve_gmesh(Carver &c, int V, int F) {
    GMesh m{};
    static_cast<FaceTree &>(m) = face_tree_carve(c, F).t;     // first: icon_face_tree_read finds it there
    m.V = V;
    m.wcum = c.take<unsigned long long>((size_t)F);
    m.hdr = c.take<GMeshHeader>(1);
    m.s64_ws = c.take<unsigned long long>(s64_ws_elems(F));
    return m;
}

static size_t gmesh_ws_bytes(int V, int F) {
    Carver c(nullptr);
    carve_gmesh(c, V, F);
    return c.total();
}

// ---------------------------------------------------------------- prepare: the sampler's area weights
__global__ void k_gm_init(GMeshHeader *h, int wbits) {
    h->amax = 0ull;
    h->total = 0ull;
    h->wbits = wbits;
}

// trimesh's area_faces: |(b - a) x (c - a)| / 2 in fp64
__device__ __forceinline__ double face_area(V3 a, V3 b, V3 c) {
    const double abx = (double)b.x - (double)a.x, aby = (double)b.y - (double)a.y, abz = (double)b.z - (double)a.z;
    const double acx = (double)c.x - (double)a.x, acy = (double)c.y - (double)a.y, acz = (double)c.z - (double)a.z;
    const double cx = aby * acz - abz * acy, cy = abz * acx - abx * acz, cz = abx * acy - aby * acx;
    return sqrt(cx * cx + cy * cy + cz * cz) * 0.5;
}

// largest face area
__global__ void __launch_bounds__(256) k_gm_area(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                                 int F, GMeshHeader *h) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    double area = 0.0;
    if (f < F) {
        V3 a, b, c;
        load_face(verts, faces, f, a, b, c);
        area = face_area(a, b, c);
    }
    for (int o = 16; o; o >>= 1) area = fmax(area, __shfl_xor_sync(0xffffffffu, area, o));
    if ((threadIdx.x & 31) == 0) atomicMax(&h->amax, (unsigned long long)__double_as_longlong(area));
}

// per face: the fixed-point sampling weight, the area relative to the largest in wbits bits
__global__ void __launch_bounds__(256) k_gm_weights(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                                    GMesh m) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.F) return;
    const GMeshHeader *h = m.hdr;
    V3 a, b, c;
    load_face(verts, faces, f, a, b, c);
    const double amax = __longlong_as_double((long long)h->amax);
    m.wcum[f] = amax > 0.0 ? (unsigned long long)ldexp(face_area(a, b, c) / amax, h->wbits) : 0ull;
}

// ---- inclusive uint64 prefix sum (the weights' cumulative sum): integer, so exact and independent of block order
__global__ void __launch_bounds__(S64_T) k_scan64_block(unsigned long long *__restrict__ x, int64_t n,
                                                        unsigned long long *__restrict__ sums) {
    __shared__ unsigned long long s_w[S64_T / 32];
    const int64_t base = (int64_t)blockIdx.x * S64_B + (int64_t)threadIdx.x * S64_I;
    unsigned long long v[S64_I], t = 0;
#pragma unroll
    for (int i = 0; i < S64_I; ++i) { v[i] = base + i < n ? x[base + i] : 0ull; t += v[i]; v[i] = t; }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned long long inc = t;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
    }
    if (lane == 31) s_w[w] = inc;
    __syncthreads();
    unsigned long long off = inc - t;
    for (int k = 0; k < w; ++k) off += s_w[k];
#pragma unroll
    for (int i = 0; i < S64_I; ++i)
        if (base + i < n) x[base + i] = v[i] + off;
    if (threadIdx.x == S64_T - 1) sums[blockIdx.x] = off + t;
}

__global__ void __launch_bounds__(S64_T) k_scan64_add(unsigned long long *__restrict__ x, int64_t n,
                                                      const unsigned long long *__restrict__ sums) {
    if (blockIdx.x == 0) return;
    const unsigned long long o = sums[blockIdx.x - 1];
    const int64_t base = (int64_t)blockIdx.x * S64_B + (int64_t)threadIdx.x * S64_I;
#pragma unroll
    for (int i = 0; i < S64_I; ++i)
        if (base + i < n) x[base + i] += o;
}

static int scan64_inclusive(unsigned long long *x, int64_t n, unsigned long long *ws, cudaStream_t stream) {
    const int64_t nb = (n + S64_B - 1) / S64_B;
    k_scan64_block<<<(unsigned)nb, S64_T, 0, stream>>>(x, n, ws);
    ICON_LAUNCHED();
    if (nb == 1) return ICON_OK;
    int rc = scan64_inclusive(ws, nb, ws + nb + 32, stream);
    if (rc) return rc;
    k_scan64_add<<<(unsigned)nb, S64_T, 0, stream>>>(x, n, ws);
    ICON_LAUNCHED();
    return ICON_OK;
}

__global__ void k_gm_total(GMesh m) { m.hdr->total = m.wcum[m.F - 1]; }

// ---------------------------------------------------------------- nearest face, one point per warp
using MeshDistSmem = WalkSmem<int32_t, GM_FR_CAP>;

__global__ void __launch_bounds__(GM_T) k_mesh_dist(const float *__restrict__ pts, int64_t N, GMesh m,
                                                    float *__restrict__ out_d, int32_t *__restrict__ out_f) {
    __shared__ MeshDistSmem smem[GM_T / 32];
    const int64_t i = (int64_t)blockIdx.x * (GM_T / 32) + (threadIdx.x >> 5);
    if (i >= N) return;                                          // whole warp
    const V3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
    // the SMPL path's additive slacks (1e-6 on lengths, 1e-7 on the support bound) are sized for coordinates of
    // magnitude <= 1; a general mesh may be in any unit, so they scale with the largest coordinate in play (the leaf
    // boxes are built from a + ab, which may sit an ulp of that magnitude away from the vertex)
    const float sc = fmaxf(fmaxf(1.f, m.bounds->absmax), fmaxf(fmaxf(fabsf(p.x), fabsf(p.y)), fabsf(p.z)));
    const float tol = 1e-6f * sc;
    NearestFace<1> nf(p, tol, 1e-7f * sc * sc);
    // one point: the warp's box is the point inflated by tol, its radius tol
    tree_nearest(m, smem[threadIdx.x >> 5], nf, p, tol, make_float4(p.x - tol, p.y - tol, p.z - tol, 0.f),
                 make_float4(p.x + tol, p.y + tol, p.z + tol, 0.f));
    if ((threadIdx.x & 31) == 0) {
        out_d[i] = nf.best;
        if (out_f) out_f[i] = nf.bi;
    }
}

// ---------------------------------------------------------------- even surface sampler (trimesh 3.9.35 semantics)
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {       // splitmix64 finaliser
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
// uniform double in [0, 1) with 53 random bits: draw k of candidate i
__device__ __forceinline__ double uniform01(unsigned long long key, long long i, int k) {
    return (double)(mix64(key + 3ull * (unsigned long long)i + (unsigned long long)k) >> 11) * 0x1.0p-53;
}

// candidate i: face by inverse CDF of the area weights, uniform point of the face by the folded parallelogram draw
__global__ void __launch_bounds__(256) k_gm_candidates(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                                       GMesh m, int M, unsigned long long key, float4 *__restrict__ cand,
                                                       int32_t *__restrict__ cface) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    const unsigned long long total = m.hdr->total;
    unsigned long long r = (unsigned long long)(uniform01(key, i, 0) * (double)total);
    if (r >= total) r = total - 1;
    int lo = 0, hi = m.F - 1;                                    // first face with wcum > r
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (m.wcum[mid] > r) hi = mid; else lo = mid + 1;
    }
    V3 a, b, c;
    load_face(verts, faces, lo, a, b, c);
    double u1 = uniform01(key, i, 1), u2 = uniform01(key, i, 2);
    if (u1 + u2 > 1.0) { u1 = 1.0 - u1; u2 = 1.0 - u2; }
    const double x = (((double)b.x - (double)a.x) * u1 + ((double)c.x - (double)a.x) * u2) + (double)a.x;
    const double y = (((double)b.y - (double)a.y) * u1 + ((double)c.y - (double)a.y) * u2) + (double)a.y;
    const double z = (((double)b.z - (double)a.z) * u1 + ((double)c.z - (double)a.z) * u2) + (double)a.z;
    cand[i] = make_float4((float)x, (float)y, (float)z, 0.f);
    cface[i] = lo;
}

__device__ __forceinline__ bool gm_near(float4 p, float4 q, double r2) {
    const double dx = (double)p.x - (double)q.x, dy = (double)p.y - (double)q.y, dz = (double)p.z - (double)q.z;
    return dx * dx + dy * dy + dz * dz <= r2;
}

// greedy removal in candidate order: a candidate is kept unless a kept one lies within the radius; stops at `count`.
// One CTA, 32 candidates per step: every warp tests the step's candidates against its share of the kept points, then
// warp 0 settles the step's own conflicts in order.
__global__ void __launch_bounds__(1024) k_gm_select(GMesh m, int M, int count, const float4 *__restrict__ cand,
                                                    const int32_t *__restrict__ cface, float *__restrict__ out_p,
                                                    int32_t *__restrict__ out_f, int32_t *__restrict__ out_n) {
    extern __shared__ float4 s_kept[];                           // [count]
    __shared__ unsigned s_block;
    __shared__ int s_nk;
    const GMeshHeader *h = m.hdr;
    const double area = ldexp((double)h->total, -h->wbits) * __longlong_as_double((long long)h->amax);
    const double r2 = area / (3.0 * (double)count);              // radius^2 = area / (3 count)
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_nk = 0;
    int nk = 0;
    for (int j0 = 0; j0 < M && nk < count; j0 += 32) {
        if (threadIdx.x == 0) s_block = 0u;
        __syncthreads();
        const int j = j0 + lane;
        const bool valid = j < M;
        const float4 p = valid ? cand[j] : make_float4(0.f, 0.f, 0.f, 0.f);
        bool hit = false;
        for (int k = w; k < nk && !hit; k += 32) hit = gm_near(p, s_kept[k], r2);
        const unsigned hm = __ballot_sync(0xffffffffu, valid && hit);
        if (lane == 0 && hm) atomicOr(&s_block, hm);
        __syncthreads();
        if (w == 0) {
            unsigned intra = 0u;                                 // earlier candidates of this step within the radius
            for (int i = 0; i < 32; ++i) {
                float4 q;
                q.x = __shfl_sync(0xffffffffu, p.x, i); q.y = __shfl_sync(0xffffffffu, p.y, i);
                q.z = __shfl_sync(0xffffffffu, p.z, i); q.w = 0.f;
                if (i < lane && gm_near(p, q, r2)) intra |= 1u << i;
            }
            const unsigned blocked = s_block | ~__ballot_sync(0xffffffffu, valid);
            unsigned keep = 0u;
            for (int i = 0; i < 32; ++i) {
                const unsigned ii = __shfl_sync(0xffffffffu, intra, i);
                if (!((blocked >> i) & 1u) && !(ii & keep)) keep |= 1u << i;
            }
            const int at = nk + __popc(keep & ((1u << lane) - 1u));
            if (((keep >> lane) & 1u) && at < count) {
                s_kept[at] = p;
                out_p[3 * (size_t)at] = p.x; out_p[3 * (size_t)at + 1] = p.y; out_p[3 * (size_t)at + 2] = p.z;
                out_f[at] = cface[j];
            }
            if (lane == 0) s_nk = min(count, nk + __popc(keep));
        }
        __syncthreads();
        nk = s_nk;
    }
    if (threadIdx.x == 0) *out_n = nk;
}

}  // namespace icon

using namespace icon;

extern "C" size_t icon_mesh_workspace_bytes(int V, int F) {
    if (V <= 0 || F <= 0) return 0;
    return gmesh_ws_bytes(V, F);
}

extern "C" int icon_mesh_prepare(const float *verts, const int64_t *faces, int V, int F, void *mesh_ws,
                                 size_t mesh_ws_bytes_, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(V > 0 && F > 0, "icon_mesh_prepare: empty mesh (V=%d F=%d)", V, F);
    ICON_CHECK_ARG(verts && faces && mesh_ws, "icon_mesh_prepare: null pointer");
    if (mesh_ws_bytes_ < gmesh_ws_bytes(V, F)) {
        set_error("icon_mesh_prepare: workspace %zu < %zu", mesh_ws_bytes_, gmesh_ws_bytes(V, F));
        return ICON_ENOSPC;
    }
    Carver c(mesh_ws);
    GMesh m = carve_gmesh(c, V, F);
    int rc = face_tree_build(mesh_ws, verts, faces, F, TreeFrame{true, 0.f, 0.f, true}, stream);
    if (rc) return rc;
    const unsigned nb = (unsigned)((F + 255) / 256);
    int wbits = 62;                                              // F * 2^wbits < 2^62: the weight sum fits
    for (int f = F; f; f >>= 1) --wbits;
    k_gm_init<<<1, 1, 0, stream>>>(m.hdr, wbits);
    ICON_LAUNCHED();
    k_gm_area<<<nb, 256, 0, stream>>>(verts, faces, F, m.hdr);
    ICON_LAUNCHED();
    k_gm_weights<<<nb, 256, 0, stream>>>(verts, faces, m);
    ICON_LAUNCHED();
    rc = scan64_inclusive(m.wcum, F, m.s64_ws, stream);
    if (rc) return rc;
    k_gm_total<<<1, 1, 0, stream>>>(m);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_mesh_distance(const float *points, int64_t N, const void *mesh_ws, int V, int F, float *out_sqdist,
                                  int32_t *out_face, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(N >= 0 && V > 0 && F > 0, "icon_mesh_distance: bad sizes (N=%lld V=%d F=%d)", (long long)N, V, F);
    if (N == 0) return ICON_OK;
    ICON_CHECK_ARG(points && mesh_ws && out_sqdist, "icon_mesh_distance: null pointer");
    Carver mc((void *)mesh_ws);
    GMesh m = carve_gmesh(mc, V, F);
    const int64_t nblk = (N + GM_T / 32 - 1) / (GM_T / 32);
    ICON_CHECK_ARG(nblk <= INT32_MAX, "icon_mesh_distance: N=%lld too large", (long long)N);
    k_mesh_dist<<<(unsigned)nblk, GM_T, 0, stream>>>(points, N, m, out_sqdist, out_face);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_mesh_sample(const float *verts, const int64_t *faces, int V, int F, const void *mesh_ws, int count,
                                uint64_t seed, float *out_points, int32_t *out_face, int32_t *out_count, void *ws,
                                size_t ws_bytes, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(V > 0 && F > 0 && count > 0 && count <= GM_SAMPLE_MAX,
                   "icon_mesh_sample: bad sizes (V=%d F=%d count=%d, at most %d samples)", V, F, count, GM_SAMPLE_MAX);
    ICON_CHECK_ARG(verts && faces && mesh_ws && out_points && out_face && out_count && ws, "icon_mesh_sample: null pointer");
    const int M = 3 * count;
    Carver c(ws);
    float4 *cand = c.take<float4>((size_t)M);
    int32_t *cface = c.take<int32_t>((size_t)M);
    if (ws_bytes < c.total()) {
        set_error("icon_mesh_sample: workspace %zu < %zu", ws_bytes, c.total());
        return ICON_ENOSPC;
    }
    Carver mc((void *)mesh_ws);
    GMesh m = carve_gmesh(mc, V, F);
    // the sampler's key: a function of the seed only, so a seed draws the same candidates on every mesh
    const unsigned long long key = (unsigned long long)seed * 0xD1B54A32D192ED03ull;
    k_gm_candidates<<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(verts, faces, m, M, key, cand, cface);
    ICON_LAUNCHED();
    const int smem = (int)(sizeof(float4) * (size_t)count);
    static bool attr_set[ICON_MAX_DEVICES] = {};
    if (device_needs_setup(attr_set))
        ICON_CUDA(cudaFuncSetAttribute(k_gm_select, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(sizeof(float4) * GM_SAMPLE_MAX)));
    k_gm_select<<<1, 1024, smem, stream>>>(m, M, count, cand, cface, out_points, out_face, out_count);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" size_t icon_mesh_sample_workspace_bytes(int count) {
    if (count <= 0) return 0;
    Carver c(nullptr);
    c.take<float4>((size_t)3 * count);
    c.take<int32_t>((size_t)3 * count);
    return c.total();
}
