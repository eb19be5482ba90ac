// Precomputed radiance transfer of a scan: the dataset renderer's computePRT (reference: lib/renderer/prt_util.py:
// 115-182, called by scripts/render_single.py:118 with n = 10, order 2).  Compiled with -fmad=false.
//
// For vertex v (origin o_v, unit normal n_v) and direction d of the caller's D sphere samples:
//   dot = d.n_v (fp64), front = dot > 0, hit = any face met by the ray o_v + delta n_v + t d, t > 0,
//   PRT[v, k] = w * sum_d front (1 - hit) dot SH[d, k].
//
// The faces are those of a workspace icon_mesh_prepare filled: its Morton-sorted 4-ary AABB tree (face_tree.cuh) is
// walked as it is, there is no second builder.
//   k_prt_hits  one warp per vertex, lanes over directions, 32 rays per round sharing one origin.  Each lane walks the
//               tree depth-first without a stack (a node's children are 4n..4n+3 of the level below, so the next
//               node is found by arithmetic) and stops at its first hit.  Boxes are tested with a slab test padded
//               outward (prt_box); faces with geom.cuh's ray_hit_tri, whose convention is written there.  The
//               verdicts land as a bit per ray, ballot words [V, ceil(D / 32)].  With no hit_bits requested only
//               front-facing rays are cast (the others weigh nothing); with hit_bits every ray is.
//   k_prt_sum   one thread per (vertex, coefficient), fp64: the terms in direction order, summed in blocks of n
//               directions when D = n^2 (else one block), the block sums added in order, then times w: the order of
//               the reference's loop (its numpy block sum is sequential for K >= 2 coefficients).
// Origins o + delta n and directions are formed in fp64 and rounded to fp32 once; dot, SH and the sums stay fp64, so
// the only fp32 decisions are hit / miss.  Vertices go in chunks of the caller's workspace, so memory does not grow
// with V D.  No atomics: results are bitwise reproducible and independent of the chunking.
//
// Resources (nvcc 12.9 -Xptxas -v, sm_90a): k_prt_hits 46 registers, k_prt_sum 48, no stack frame, no spills.
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "face_tree.cuh"
#include "geom.cuh"

namespace icon {

constexpr int PRT_T = 128;                  // k_prt_hits: 4 warps per block, one vertex per warp
constexpr int PRT_SUM_T = 128;              // k_prt_sum: threads per block
constexpr int PRT_CHUNK = 65536;            // vertices per chunk of the default workspace
// box padding: PRT_PAD_ABS * max(1, largest |coordinate|) covers the fp32 rounding of the leaf corners a + ab, a + ac;
// PRT_PAD_REL * (largest offset of a box corner from the origin) covers the rounding of the slab test's t values and
// the fp32 error of Moller-Trumbore's barycentrics, which grows with the distance to the face (~1e-7 |o - a| / sin of
// the ray's angle to the face's plane: the pad covers rays more than ~1e-3 rad off the plane; closer to parallel
// the fp32 verdict is itself rounding noise, see DESIGN.md 4.14)
constexpr float PRT_PAD_ABS = 0x1.0p-20f;
constexpr float PRT_PAD_REL = 0x1.0p-10f;

// can the ray o + t inv^-1, t >= 0, meet the box [lo, hi] padded outward?  A zero direction component gives an
// infinite inv; the NaN of 0 * inf (origin on a padded face) is dropped by fminf / fmaxf, which culls that axis' slab
// only for an origin a whole pad away from the box.
__device__ __forceinline__ bool prt_box(V3 o, V3 inv, float4 lo, float4 hi, float tol) {
    const float far = fmaxf(fmaxf(fmaxf(fabsf(lo.x - o.x), fabsf(hi.x - o.x)), fmaxf(fabsf(lo.y - o.y), fabsf(hi.y - o.y))),
                            fmaxf(fabsf(lo.z - o.z), fabsf(hi.z - o.z)));
    const float pad = fmaf(PRT_PAD_REL, far, tol);
    const float x0 = (lo.x - pad - o.x) * inv.x, x1 = (hi.x + pad - o.x) * inv.x;
    const float y0 = (lo.y - pad - o.y) * inv.y, y1 = (hi.y + pad - o.y) * inv.y;
    const float z0 = (lo.z - pad - o.z) * inv.z, z1 = (hi.z + pad - o.z) * inv.z;
    const float tn = fmaxf(fmaxf(fminf(x0, x1), fminf(y0, y1)), fminf(z0, z1));
    const float tf = fminf(fminf(fmaxf(x0, x1), fmaxf(y0, y1)), fmaxf(z0, z1));
    return tn <= tf && tf >= 0.f;
}

// does the ray o + t d, t > 0, meet any face?  Depth-first over the implicit 4-ary tree, first hit wins.
__device__ __forceinline__ bool prt_any_hit(const FaceTree &t, V3 o, V3 d, float tol) {
    // approximate reciprocals (~2 ulp): the slab test only culls, and its pad is far larger than their error
    const V3 inv = mk3(__fdividef(1.f, d.x), __fdividef(1.f, d.y), __fdividef(1.f, d.z));
    const int top = t.nlevels - 1;
    int l = top, n = 0;
    while (true) {
        const float4 *nb = t.nodes + 2 * ((size_t)t.lvl_off[l] + n);
        if (prt_box(o, inv, __ldg(nb), __ldg(nb + 1), tol)) {
            if (l > 0) {                                          // first child
                --l;
                n *= 4;
                continue;
            }
            for (int k = 4 * n; k < min(4 * n + 4, t.F); ++k) {
                const Tri tr = load_tri(t.tri_s + 3 * (size_t)k);
                if (ray_hit_tri(o, d, tr.a, tr.ab, tr.ac)) return true;
            }
        }
        // next node: up while this is the last child of its parent, then the next sibling
        while (l < top && ((n & 3) == 3 || n + 1 == t.lvl_cnt[l])) {
            n >>= 2;
            ++l;
        }
        if (l == top) return false;
        ++n;
    }
}

__global__ void __launch_bounds__(PRT_T) k_prt_hits(FaceTree t, const float *__restrict__ absmax,
                                                   const double *__restrict__ origins, const double *__restrict__ normals,
                                                   double delta, const double *__restrict__ dirs, int D, int W, int v0,
                                                   int nv, int all, uint32_t *__restrict__ bits) {
    const int wi = blockIdx.x * (PRT_T / 32) + (threadIdx.x >> 5);
    if (wi >= nv) return;                                         // whole warp
    const int lane = threadIdx.x & 31;
    const int64_t v = (int64_t)v0 + wi;
    const double nx = normals[3 * v], ny = normals[3 * v + 1], nz = normals[3 * v + 2];
    const V3 o = mk3((float)(origins[3 * v] + delta * nx), (float)(origins[3 * v + 1] + delta * ny),
                     (float)(origins[3 * v + 2] + delta * nz));
    const float sc = fmaxf(fmaxf(1.f, *absmax), fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fabsf(o.z)));
    const float tol = PRT_PAD_ABS * sc;
    uint32_t *row = bits + (size_t)wi * W;
    for (int r = 0; r < W; ++r) {
        const int j = 32 * r + lane;
        bool hit = false;
        if (j < D) {
            const double dx = dirs[3 * j], dy = dirs[3 * j + 1], dz = dirs[3 * j + 2];
            if (all || (dx * nx + dy * ny) + dz * nz > 0.0)
                hit = prt_any_hit(t, o, mk3((float)dx, (float)dy, (float)dz), tol);
        }
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) row[r] = b;
    }
}

__global__ void __launch_bounds__(PRT_SUM_T) k_prt_sum(const double *__restrict__ normals,
                                                      const double *__restrict__ dirs, const double *__restrict__ sh,
                                                      int D, int K, int B, double w, int W, int v0, int nv,
                                                      const uint32_t *__restrict__ bits, double *__restrict__ prt) {
    const int64_t i = (int64_t)blockIdx.x * PRT_SUM_T + threadIdx.x;
    if (i >= (int64_t)nv * K) return;
    const int wi = (int)(i / K), k = (int)(i % K);
    const int64_t v = (int64_t)v0 + wi;
    const double nx = normals[3 * v], ny = normals[3 * v + 1], nz = normals[3 * v + 2];
    const uint32_t *row = bits + (size_t)wi * W;
    double acc = 0.0;
    for (int b0 = 0; b0 < D; b0 += B) {
        const int b1 = min(b0 + B, D);
        double s = 0.0;
        for (int j = b0; j < b1; ++j) {
            const double dot = (dirs[3 * j] * nx + dirs[3 * j + 1] * ny) + dirs[3 * j + 2] * nz;
            const double lit = (dot > 0.0 && !((row[j >> 5] >> (j & 31)) & 1u)) ? 1.0 : 0.0;
            const double term = (lit * dot) * sh[(size_t)j * K + k];
            s = j == b0 ? term : s + term;
        }
        acc = b0 == 0 ? s : acc + s;
    }
    prt[v * K + k] = w * acc;
}

static size_t prt_row_bytes(int D) { return sizeof(uint32_t) * (size_t)((D + 31) / 32); }

}  // namespace icon

using namespace icon;

extern "C" size_t icon_prt_workspace_bytes(int V, int D, int K) {
    if (V <= 0 || D <= 0 || K <= 0) return 0;
    Carver c(nullptr);
    c.take<char>(prt_row_bytes(D) * (size_t)min(V, PRT_CHUNK));
    return c.total();
}

extern "C" int icon_prt(const void *mesh_ws, int Vm, int F, const double *origins, const double *normals, int V,
                        double delta, const double *dirs, const double *sh, int D, int K, double w, double *prt_out,
                        uint32_t *hit_bits, void *ws, size_t ws_bytes, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(Vm > 0 && F > 0 && V > 0 && D > 0 && K > 0,
                   "icon_prt: bad sizes (mesh V=%d F=%d, vertices %d, directions %d, coefficients %d)", Vm, F, V, D, K);
    ICON_CHECK_ARG(mesh_ws && origins && normals && dirs && sh && prt_out && ws, "icon_prt: null pointer");
    ICON_CHECK_ARG(isfinite(delta) && isfinite(w), "icon_prt: delta / w not finite");
    const size_t row = prt_row_bytes(D);
    if (ws_bytes < row) {
        set_error("icon_prt: workspace %zu < %zu (one vertex's hit bits)", ws_bytes, row);
        return ICON_ENOSPC;
    }
    const int chunk = (int)std::min<size_t>((size_t)V, ws_bytes / row);
    const int W = (D + 31) / 32;
    const int n = (int)llround(sqrt((double)D));
    const int B = n * n == D ? n : D;                            // the reference's block of n directions
    const FaceTree t = face_tree_view(mesh_ws, F);
    const float *absmax = &t.bounds->absmax;
    for (int v0 = 0; v0 < V; v0 += chunk) {
        const int nv = std::min(chunk, V - v0);
        uint32_t *bits = hit_bits ? hit_bits + (size_t)v0 * W : (uint32_t *)ws;
        k_prt_hits<<<(unsigned)((nv + PRT_T / 32 - 1) / (PRT_T / 32)), PRT_T, 0, stream>>>(
            t, absmax, origins, normals, delta, dirs, D, W, v0, nv, hit_bits != nullptr, bits);
        ICON_LAUNCHED();
        const int64_t nt = (int64_t)nv * K;
        k_prt_sum<<<(unsigned)((nt + PRT_SUM_T - 1) / PRT_SUM_T), PRT_SUM_T, 0, stream>>>(
            normals, dirs, sh, D, K, B, w, W, v0, nv, bits, prt_out);
        ICON_LAUNCHED();
    }
    return ICON_OK;
}
