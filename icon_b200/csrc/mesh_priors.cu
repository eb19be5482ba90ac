// Cloth-refinement geometry of apps/infer.py:435-476: the mesh topology and the three shape priors of
// update_mesh_shape_prior_losses (lib/dataset/mesh_util.py:168-176), and LocalAffine (lib/net/local_affine.py), forward
// and backward.  Restated by oracle/mesh_priors.py (float64 torch, autograd for the gradients).
//
// PARITY UNPINNED: pytorch3d is not a dependency of this project.  The rules below are this file's contract.  Inputs
// are fp32; unless a rule says fp32, every term is evaluated in fp64 from the fp32 inputs, summed in fp64 in the fixed
// order given, and rounded to fp32 once.  No float atomics anywhere: values and gradients are bitwise reproducible.
// -fmad=false (the fp32 rules are restated operation for operation).
//
// Topology (icon_mesh_topology_count / _build), of faces [F,3] with every index in [0, V) (else ICON_EINVAL):
//   edges         the distinct (min, max) pairs of each face's corner pairs (v1,v2), (v2,v0), (v0,v1), ascending by
//                 (min, max) (pytorch3d's edges_packed); a face [a,a,b] gives the self-loop (a,a).
//   face_to_edge  [F,3], columns e12, e20, e01.
//   vert_edges    per vertex, the ids of the edges it is an endpoint of, ascending; a self-loop is listed twice, so
//                 deg_i = the row length = the count of edge endpoints at i.
//   edge_entries  per edge, the face-corner entries 3 f + col (col of face_to_edge) that map to it, ascending.
//   vert_corners  per vertex, the corners 3 f + c with faces[f][c] = i, ascending (common.cu's vertex_corners).
//   Construction: every list comes from common.cu's row-list builder (csr_build).  Each corner pair (min, max) is
//   listed under min; each list is heap-sorted and de-duplicated in place, and a scan of the unique counts gives edge
//   ids in (min, max) order with no global sort.  The edge count is read back to the host once per build (the caller
//   caches the topology: the faces do not change across the loop).
//
// Priors (icon_mesh_priors_forward / _backward), for one mesh:
//   edge = (1/E) sum_e (L_e - 0)^2, L_e = sqrt(d.d), d = v_a - v_b.  Backward: 2 d (g/E) to a, -2 d (g/E) to b; at
//     L = 0 torch's norm passes 0 (d = 0 there, so the formula already does; a self-loop has d = 0).
//   lap = (1/V) sum_i |l_i|, l_i = (sum over vert_edges of i of v_other / deg_i) - v_i, other = the edge's other
//     endpoint (a self-loop gives v_a twice); deg_i = 0 (an unreferenced vertex included) gives l_i = -v_i; V counts
//     every vertex.  Backward: u_i = (g/V) l_i / |l_i| (0 where |l_i| = 0); grad_j = (sum over vert_edges of j of
//     u_other / deg_other) - u_j.
//   nc = (1/P) sum over pairs (1 - cos(n_i, -n_j)); the pairs are all unordered pairs i < j of an edge's entries (k
//     entries give C(k,2) pairs), P their count; P = 0 gives 0.  An entry's n = sum_{k=0..2} (v1 - v0) x (f_k - v0)
//     over its face's corners in order, (v0, v1) = the edge's (min, max): the terms on the edge's own vertices are
//     exactly 0, so a degenerate face gives n = 0.  cos is torch 2.x cosine_similarity(eps = 1e-8):
//     sum_c (x_c / Nx) (y_c / Ny), Nx = max(|x|, eps); its gradient flows through the unclamped norm:
//     dcos/dx_c = y_c / (Nx Ny) - ((x.y) / (Nx Nx Ny)) (x_c / |x|), the last term 0 at |x| = 0.
//     The backward of an entry's n: gu = sum_k (f_k - v0) x gn, gw_k = gn x u (u = v1 - v0): v1 += gu,
//     v0 -= gu + 3 gw, corner k += gw.
//   The three scalars come from fixed-order per-block partials (256-thread tree) and one fixed-order final sum.
//   Backward: g_edge, g_nc, g_lap are device pointers (no host sync); a NULL one skips its term.  Per vertex the
//   gradient is ((edge part) + (lap part)) + (nc part), each summed over the vertex's rows in ascending order.
//
// LocalAffine (icon_local_affine_forward / _backward), B = 1, N vertices, A [N,3,3], b [N,3], W = [A | b] [N,3,4]:
//   out_r = ((A_r0 x + A_r1 y) + A_r2 z) + b_r in fp32;
//   w_diff[e] = (W_i - W_j)^2 per element in fp32 (subtract, then square: torch's own fp32 result), (i, j) = edges[e];
//   w_rigid = (det A - 1)^2, det A = A00 C00 + A01 C01 + A02 C02 with the cofactors
//     C00 = A11 A22 - A12 A21, C01 = -(A10 A22 - A12 A20), C02 = A10 A21 - A11 A20 (all in fp64; rounded once).
//   Backward per vertex, summed in this order: g_out (grad_A = g x^T, grad_b = g); then over vert_edges ascending,
//   +-2 (W_i - W_j) g_e (+ at i, - at j; a self-loop's difference is 0); then 2 (det - 1) g_rigid C (C = adj(A)^T,
//   the cofactor matrix).  grad_x = A^T g_out.  The vertex-to-edge lists are the topology's vert_edges construction,
//   applied to the caller's edges.
#include <math.h>

#include "common.cuh"

namespace icon {

constexpr int PR_T = 256;

__device__ __forceinline__ double pr_block_sum(double x, double *sh) {
    sh[threadIdx.x] = x;
    __syncthreads();
    for (int h = PR_T / 2; h > 0; h >>= 1) {
        if ((int)threadIdx.x < h) sh[threadIdx.x] = sh[threadIdx.x] + sh[threadIdx.x + h];
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}

// ---------------------------------------------------------------- topology

// corner pair col of a face: col 0 = (v1, v2), 1 = (v2, v0), 2 = (v0, v1)
__device__ __forceinline__ int tp_c1(int col) { return (col + 1) % 3; }
__device__ __forceinline__ int tp_c2(int col) { return (col + 2) % 3; }

// item 3 f + col: owner min, key max; a face with an index outside [0, V) raises *bad and lists nothing
__global__ void k_tp_pairs(const int64_t *__restrict__ faces, int F, int V, int32_t *__restrict__ own,
                           int32_t *__restrict__ key, int32_t *__restrict__ bad) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    int id[3];
    if (!face_ids(faces, f, V, id)) {
        *bad = 1;
#pragma unroll
        for (int col = 0; col < 3; ++col) own[3 * f + col] = -1;
        return;
    }
#pragma unroll
    for (int col = 0; col < 3; ++col) {
        const int a = id[tp_c1(col)], b = id[tp_c2(col)];
        own[3 * f + col] = min(a, b);
        key[3 * f + col] = max(a, b);
    }
}

__global__ void k_tp_edges(const int32_t *__restrict__ poff, const int32_t *__restrict__ plist,
                           const int32_t *__restrict__ eoff, int V, int64_t *__restrict__ edges,
                           int32_t *__restrict__ own, int32_t *__restrict__ key) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= V) return;
    const int e0 = eoff[a], n = eoff[a + 1] - e0;
    for (int r = 0; r < n; ++r) {
        const int e = e0 + r, b = plist[poff[a] + r];
        edges[2 * (int64_t)e] = a;
        edges[2 * (int64_t)e + 1] = b;
        own[2 * (int64_t)e] = a; key[2 * (int64_t)e] = e;          // vert_edges items
        own[2 * (int64_t)e + 1] = b; key[2 * (int64_t)e + 1] = e;
    }
}

// face_to_edge by binary search in min's unique list; edge_entries items (own = edge, key = 3 f + col)
__global__ void k_tp_f2e(const int64_t *__restrict__ faces, int F, const int32_t *__restrict__ poff,
                         const int32_t *__restrict__ plist, const int32_t *__restrict__ eoff,
                         int64_t *__restrict__ f2e, int32_t *__restrict__ own, int32_t *__restrict__ key) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
#pragma unroll
    for (int col = 0; col < 3; ++col) {
        const int p = (int)faces[3 * (int64_t)f + tp_c1(col)], q = (int)faces[3 * (int64_t)f + tp_c2(col)];
        const int a = min(p, q), b = max(p, q);
        const int32_t *l = plist + poff[a];
        int lo = 0, hi = eoff[a + 1] - eoff[a] - 1;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (l[mid] < b) lo = mid + 1; else hi = mid;
        }
        const int e = eoff[a] + lo;
        f2e[3 * (int64_t)f + col] = e;
        own[3 * f + col] = e;
        key[3 * f + col] = 3 * f + col;
    }
}

struct TpWs {
    int32_t *own, *key;       // [6F] items
    int32_t *poff, *plist;    // pair lists: [V+1], [3F]
    int32_t *ucnt, *eoff;     // [V+1] unique counts, their scan (edge offsets)
    int64_t *d_E;
    int32_t *bad;
    CsrWs csr;               // rows up to max(V, 3F)
};

static size_t tp_carve(void *ws, int V, int F, TpWs *o) {
    Carver c(ws);
    TpWs w{};
    w.own = c.take<int32_t>(6 * (size_t)F);
    w.key = c.take<int32_t>(6 * (size_t)F);
    w.poff = c.take<int32_t>((size_t)V + 1);
    w.plist = c.take<int32_t>(3 * (size_t)F);
    w.ucnt = c.take<int32_t>((size_t)V + 1);
    w.eoff = c.take<int32_t>((size_t)V + 1);
    w.d_E = c.take<int64_t>(1);
    w.bad = c.take<int32_t>(1);
    w.csr = csr_take(c, (int64_t)(V > 3 * F ? V : 3 * F));
    if (o) *o = w;
    const size_t vc = vertex_corners_ws_bytes(V, F);    // the corner lists are built last, over the whole workspace
    return c.total() > vc ? c.total() : vc;
}

// vert_edges of `edges` [E,2] (every index in [0, V), checked by the caller): the own/key items, then the lists
__global__ void k_ve_items(const int64_t *__restrict__ edges, int E, int32_t *__restrict__ own,
                           int32_t *__restrict__ key) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * E) return;
    own[i] = (int)edges[i];
    key[i] = i >> 1;
}

// ---------------------------------------------------------------- priors

struct Topo {
    int V, F, E;
    const int64_t *faces, *edges;
    const int32_t *voff, *vedge, *eoff, *eent, *coff, *vcorner;
};

static Topo topo_of(const icon_mesh_topology *t) {
    return Topo{t->V, t->F, t->E, t->faces, t->edges, t->vert_off, t->vert_edges, t->edge_off, t->edge_entries,
                t->corner_off, t->vert_corners};
}

__device__ __forceinline__ void ld3(const float *v, int64_t i, double p[3]) {
    p[0] = v[3 * i]; p[1] = v[3 * i + 1]; p[2] = v[3 * i + 2];
}

__device__ __forceinline__ void cross(const double a[3], const double b[3], double o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// the normal of entry key = 3 f + col of an edge (a, b); u = v_b - v_a and w_k = f_k - v_a for the backward
__device__ __forceinline__ void nc_normal(const float *verts, const int64_t *faces, int key, int a, int b, double n[3],
                                          double u[3], double w[3][3]) {
    const int f = key / 3;
    double p0[3], p1[3];
    ld3(verts, a, p0);
    ld3(verts, b, p1);
#pragma unroll
    for (int c = 0; c < 3; ++c) u[c] = p1[c] - p0[c];
    n[0] = n[1] = n[2] = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double q[3], t[3];
        ld3(verts, faces[3 * (int64_t)f + k], q);
#pragma unroll
        for (int c = 0; c < 3; ++c) w[k][c] = q[c] - p0[c];
        cross(u, w[k], t);
#pragma unroll
        for (int c = 0; c < 3; ++c) n[c] = n[c] + t[c];
    }
}

// torch's cosine_similarity(x, y, eps = 1e-8) and, when gx / gy are given, its gradients
__device__ __forceinline__ double cos_sim(const double x[3], const double y[3], double *gx, double *gy) {
    const double lx = sqrt((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]);
    const double ly = sqrt((y[0] * y[0] + y[1] * y[1]) + y[2] * y[2]);
    const double nx = lx > 1e-8 ? lx : 1e-8, ny = ly > 1e-8 ? ly : 1e-8;
    double s = 0.0, xy = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        s = s + (x[c] / nx) * (y[c] / ny);
        xy = xy + x[c] * y[c];
    }
    if (gx) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            gx[c] = y[c] / (nx * ny) - (lx > 0.0 ? (xy / (nx * nx * ny)) * (x[c] / lx) : 0.0);
            gy[c] = x[c] / (nx * ny) - (ly > 0.0 ? (xy / (nx * ny * ny)) * (y[c] / ly) : 0.0);
        }
    }
    return s;
}

// per edge: edge term, nc pair sum and pair count -> block partials part[0 .. 3 nb)
__global__ void k_pr_edge_terms(Topo t, const float *__restrict__ verts, double *__restrict__ part, int nb,
                                int want_terms) {
    __shared__ double sh[PR_T];
    const int e = blockIdx.x * PR_T + threadIdx.x;
    double te = 0.0, tn = 0.0, tp = 0.0;
    if (e < t.E) {
        const int a = (int)t.edges[2 * (int64_t)e], b = (int)t.edges[2 * (int64_t)e + 1];
        const int e0 = t.eoff[e], k = t.eoff[e + 1] - e0;
        tp = 0.5 * (double)k * (double)(k - 1);
        if (want_terms) {
            double pa[3], pb[3];
            ld3(verts, a, pa);
            ld3(verts, b, pb);
            const double d0 = pa[0] - pb[0], d1 = pa[1] - pb[1], d2 = pa[2] - pb[2];
            const double L = sqrt((d0 * d0 + d1 * d1) + d2 * d2);
            te = L * L;
            for (int i = 0; i < k; ++i) {
                double ni[3], u[3], w[3][3];
                nc_normal(verts, t.faces, t.eent[e0 + i], a, b, ni, u, w);
                for (int j = i + 1; j < k; ++j) {
                    double nj[3];
                    nc_normal(verts, t.faces, t.eent[e0 + j], a, b, nj, u, w);
                    nj[0] = -nj[0]; nj[1] = -nj[1]; nj[2] = -nj[2];
                    tn = tn + (1.0 - cos_sim(ni, nj, nullptr, nullptr));
                }
            }
        }
    }
    te = pr_block_sum(te, sh);
    tn = pr_block_sum(tn, sh);
    tp = pr_block_sum(tp, sh);
    if (threadIdx.x == 0) {
        part[blockIdx.x] = te;
        part[nb + blockIdx.x] = tn;
        part[2 * nb + blockIdx.x] = tp;
    }
}

// l_i into lap [V,3] (fp64); block partials of |l_i|
__global__ void k_pr_lap(Topo t, const float *__restrict__ verts, double *__restrict__ lap, double *__restrict__ part) {
    __shared__ double sh[PR_T];
    const int i = blockIdx.x * PR_T + threadIdx.x;
    double len = 0.0;
    if (i < t.V) {
        const int r0 = t.voff[i], deg = t.voff[i + 1] - r0;
        double s[3] = {0.0, 0.0, 0.0}, p[3];
        for (int r = 0; r < deg; ++r) {
            const int e = t.vedge[r0 + r];
            const int a = (int)t.edges[2 * (int64_t)e], b = (int)t.edges[2 * (int64_t)e + 1];
            ld3(verts, a == i ? b : a, p);
#pragma unroll
            for (int c = 0; c < 3; ++c) s[c] = s[c] + p[c] / (double)deg;
        }
        ld3(verts, i, p);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            s[c] = s[c] - p[c];
            lap[3 * (int64_t)i + c] = s[c];
        }
        len = sqrt((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2]);
    }
    len = pr_block_sum(len, sh);
    if (threadIdx.x == 0) part[blockIdx.x] = len;
}

// one block: fixed-order sums of n partial arrays of length m each -> sums[n]
__global__ void k_pr_reduce(const double *__restrict__ part, int n, int m, double *__restrict__ sums) {
    __shared__ double sh[PR_T];
    for (int q = 0; q < n; ++q) {
        double s = 0.0;
        for (int i = threadIdx.x; i < m; i += PR_T) s = s + part[(int64_t)q * m + i];
        s = pr_block_sum(s, sh);
        if (threadIdx.x == 0) sums[q] = s;
    }
}

// sums: edge, nc, pairs, lap
__global__ void k_pr_out(const double *__restrict__ sums, int V, int E, float *out_edge, float *out_nc,
                         float *out_lap) {
    if (threadIdx.x != 0) return;
    *out_edge = (float)(sums[0] / (double)E);
    *out_nc = sums[2] > 0.0 ? (float)(sums[1] / sums[2]) : 0.f;
    *out_lap = (float)(sums[3] / (double)V);
}

// backward: u_i = (g/V) l_i / |l_i| in place
__global__ void k_pr_lap_u(int V, const float *__restrict__ g_lap, double *__restrict__ lap) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    double *l = lap + 3 * (int64_t)i;
    const double len = sqrt((l[0] * l[0] + l[1] * l[1]) + l[2] * l[2]);
    const double s = len > 0.0 ? ((double)*g_lap / (double)V) / len : 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) l[c] = len > 0.0 ? l[c] * s : 0.0;
}

// backward of nc, per edge: each entry's d/dn, then through n to its face's corners: fc [3F][3] (entry 3 f + col
// holds the contributions of that entry to corners 0, 1, 2 of f in fc[3 f + c] -- summed per face below)
__global__ void k_pr_nc_entry(Topo t, const float *__restrict__ verts, const float *__restrict__ g_nc,
                              const double *__restrict__ sums, double *__restrict__ ent) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.E) return;
    const int a = (int)t.edges[2 * (int64_t)e], b = (int)t.edges[2 * (int64_t)e + 1];
    const int e0 = t.eoff[e], k = t.eoff[e + 1] - e0;
    const double scale = sums[2] > 0.0 ? (double)*g_nc / sums[2] : 0.0;
    for (int i = 0; i < k; ++i) {
        const int key = t.eent[e0 + i];
        double ni[3], u[3], w[3][3], gn[3] = {0.0, 0.0, 0.0};
        nc_normal(verts, t.faces, key, a, b, ni, u, w);
        for (int j = 0; j < k; ++j) {
            if (j == i) continue;
            double nj[3], uj[3], wj[3][3], gx[3], gy[3];
            nc_normal(verts, t.faces, t.eent[e0 + j], a, b, nj, uj, wj);
            if (i < j) {            // term 1 - cos(n_i, -n_j): d/dn_i = -dcos/dx
                nj[0] = -nj[0]; nj[1] = -nj[1]; nj[2] = -nj[2];
                cos_sim(ni, nj, gx, gy);
#pragma unroll
                for (int c = 0; c < 3; ++c) gn[c] = gn[c] - gx[c];
            } else {                // term 1 - cos(n_j, -n_i): d/dn_i = +dcos/dy
                double mi[3] = {-ni[0], -ni[1], -ni[2]};
                cos_sim(nj, mi, gx, gy);
#pragma unroll
                for (int c = 0; c < 3; ++c) gn[c] = gn[c] + gy[c];
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) gn[c] = gn[c] * scale;
        // gu = sum_k w_k x gn, gw = gn x u; v_b += gu, v_a -= gu + 3 gw, corner k += gw
        double gu[3] = {0.0, 0.0, 0.0}, gw[3], t3[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            cross(w[q], gn, t3);
#pragma unroll
            for (int c = 0; c < 3; ++c) gu[c] = gu[c] + t3[c];
        }
        cross(gn, u, gw);
        const int f = key / 3, col = key % 3;
        const int c1 = (col + 1) % 3, c2 = (col + 2) % 3;
        const bool first_min = t.faces[3 * (int64_t)f + c1] <= t.faces[3 * (int64_t)f + c2];
        const int ca = first_min ? c1 : c2, cb = first_min ? c2 : c1;     // corners holding v_a, v_b
        double *o = ent + 9 * (int64_t)key;
#pragma unroll
        for (int q = 0; q < 3; ++q)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                double x = gw[c];
                if (q == ca) x = x - (gu[c] + 3.0 * gw[c]);
                if (q == cb) x = x + gu[c];
                o[3 * q + c] = x;
            }
    }
}

// per face corner: the sum over the face's three entries, col 0, 1, 2
__global__ void k_pr_nc_face(int F, const double *__restrict__ ent, double *__restrict__ fc) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * F) return;
    const int f = i / 3, q = i % 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        double s = 0.0;
#pragma unroll
        for (int col = 0; col < 3; ++col) s = s + ent[9 * (int64_t)(3 * f + col) + 3 * q + c];
        fc[3 * (int64_t)i + c] = s;
    }
}

__global__ void k_pr_vertex(Topo t, const float *__restrict__ verts, const float *__restrict__ g_edge,
                            const double *__restrict__ u, const double *__restrict__ fc, float *__restrict__ grad) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= t.V) return;
    double ge[3] = {0.0, 0.0, 0.0}, gl[3] = {0.0, 0.0, 0.0}, gn[3] = {0.0, 0.0, 0.0}, pj[3], po[3];
    const int r0 = t.voff[j], deg = t.voff[j + 1] - r0;
    ld3(verts, j, pj);
    const double se = g_edge ? 2.0 * ((double)*g_edge / (double)t.E) : 0.0;
    for (int r = 0; r < deg; ++r) {
        const int e = t.vedge[r0 + r];
        const int a = (int)t.edges[2 * (int64_t)e], b = (int)t.edges[2 * (int64_t)e + 1];
        const int o = a == j ? b : a;
        if (g_edge) {
            ld3(verts, o, po);
#pragma unroll
            for (int c = 0; c < 3; ++c) ge[c] = ge[c] + se * (pj[c] - po[c]);
        }
        if (u) {
            const double dego = (double)(t.voff[o + 1] - t.voff[o]);
#pragma unroll
            for (int c = 0; c < 3; ++c) gl[c] = gl[c] + u[3 * (int64_t)o + c] / dego;
        }
    }
    if (u)
#pragma unroll
        for (int c = 0; c < 3; ++c) gl[c] = gl[c] - u[3 * (int64_t)j + c];
    if (fc) {
        const int c0 = t.coff[j], nc = t.coff[j + 1] - c0;
        for (int r = 0; r < nc; ++r) {
            const double *x = fc + 3 * (int64_t)t.vcorner[c0 + r];
#pragma unroll
            for (int c = 0; c < 3; ++c) gn[c] = gn[c] + x[c];
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) grad[3 * (int64_t)j + c] = (float)((ge[c] + gl[c]) + gn[c]);
}

struct PrWs {
    double *part, *sums, *lap, *ent, *fc;
    int nbE, nbV;
};

static size_t pr_carve(void *ws, int V, int F, int E, bool bwd, PrWs *o) {
    Carver c(ws);
    PrWs w{};
    w.nbE = (E + PR_T - 1) / PR_T;
    w.nbV = (V + PR_T - 1) / PR_T;
    w.part = c.take<double>(3 * (size_t)w.nbE + (size_t)w.nbV);
    w.sums = c.take<double>(4);
    w.lap = c.take<double>(3 * (size_t)V);
    if (bwd) {
        w.ent = c.take<double>(27 * (size_t)F);
        w.fc = c.take<double>(9 * (size_t)F);
    }
    if (o) *o = w;
    return c.total();
}

static bool topo_ok(const icon_mesh_topology *t) {
    return t && t->V > 0 && t->F > 0 && t->E > 0 && t->faces && t->edges && t->vert_off && t->vert_edges &&
           t->edge_off && t->edge_entries && t->corner_off && t->vert_corners;
}

// ---------------------------------------------------------------- LocalAffine

__device__ __forceinline__ void la_cof(const float *A, double C[9]) {
    double a[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) a[k] = A[k];
    C[0] = a[4] * a[8] - a[5] * a[7];
    C[1] = -(a[3] * a[8] - a[5] * a[6]);
    C[2] = a[3] * a[7] - a[4] * a[6];
    C[3] = -(a[1] * a[8] - a[2] * a[7]);
    C[4] = a[0] * a[8] - a[2] * a[6];
    C[5] = -(a[0] * a[7] - a[1] * a[6]);
    C[6] = a[1] * a[5] - a[2] * a[4];
    C[7] = -(a[0] * a[5] - a[2] * a[3]);
    C[8] = a[0] * a[4] - a[1] * a[3];
}

__device__ __forceinline__ double la_det(const float *A, const double C[9]) {
    return ((double)A[0] * C[0] + (double)A[1] * C[1]) + (double)A[2] * C[2];
}

__global__ void k_la_vertex(int N, const float *__restrict__ A, const float *__restrict__ b,
                            const float *__restrict__ x, float *__restrict__ out, float *__restrict__ w_rigid) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float *a = A + 9 * (int64_t)i;
    const float px = x[3 * (int64_t)i], py = x[3 * (int64_t)i + 1], pz = x[3 * (int64_t)i + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        out[3 * (int64_t)i + r] = ((a[3 * r] * px + a[3 * r + 1] * py) + a[3 * r + 2] * pz) + b[3 * (int64_t)i + r];
    double C[9];
    la_cof(a, C);
    const double d = la_det(a, C) - 1.0;
    w_rigid[i] = (float)(d * d);
}

__device__ __forceinline__ float la_w(const float *A, const float *b, int64_t i, int rc) {
    const int r = rc >> 2, c = rc & 3;
    return c < 3 ? A[9 * i + 3 * r + c] : b[3 * i + r];
}

__global__ void k_la_diff(int E, const int64_t *__restrict__ edges, const float *__restrict__ A,
                          const float *__restrict__ b, float *__restrict__ w_diff) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= 12 * (int64_t)E) return;
    const int64_t e = q / 12;
    const int rc = (int)(q % 12);
    const float d = la_w(A, b, edges[2 * e], rc) - la_w(A, b, edges[2 * e + 1], rc);
    w_diff[q] = d * d;
}

__global__ void k_la_backward(int N, const float *__restrict__ A, const float *__restrict__ b,
                              const float *__restrict__ x, const int64_t *__restrict__ edges,
                              const int32_t *__restrict__ voff, const int32_t *__restrict__ vedge,
                              const float *__restrict__ g_out, const float *__restrict__ g_diff,
                              const float *__restrict__ g_rigid, float *__restrict__ gA, float *__restrict__ gb,
                              float *__restrict__ gx) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    double s[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) s[k] = 0.0;
    if (g_out) {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const double g = g_out[3 * (int64_t)i + r];
#pragma unroll
            for (int c = 0; c < 3; ++c) s[4 * r + c] = g * (double)x[3 * (int64_t)i + c];
            s[4 * r + 3] = g;
        }
    }
    if (g_diff) {
        for (int r = voff[i]; r < voff[i + 1]; ++r) {
            const int e = vedge[r];
            const int64_t p = edges[2 * (int64_t)e], q = edges[2 * (int64_t)e + 1];
            const double sg = p == i ? 2.0 : -2.0;
#pragma unroll
            for (int rc = 0; rc < 12; ++rc)
                s[rc] = s[rc] + sg * ((double)la_w(A, b, p, rc) - (double)la_w(A, b, q, rc)) *
                                    (double)g_diff[12 * (int64_t)e + rc];
        }
    }
    const float *a = A + 9 * (int64_t)i;
    if (g_rigid) {
        double C[9];
        la_cof(a, C);
        const double k = 2.0 * (la_det(a, C) - 1.0) * (double)g_rigid[i];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) s[4 * r + c] = s[4 * r + c] + k * C[3 * r + c];
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) gA[9 * (int64_t)i + 3 * r + c] = (float)s[4 * r + c];
        gb[3 * (int64_t)i + r] = (float)s[4 * r + 3];
    }
    if (gx) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            double t = 0.0;
            if (g_out)
#pragma unroll
                for (int r = 0; r < 3; ++r) t = t + (double)a[3 * r + c] * (double)g_out[3 * (int64_t)i + r];
            gx[3 * (int64_t)i + c] = (float)t;
        }
    }
}

}  // namespace icon

// ---------------------------------------------------------------- C ABI

extern "C" size_t icon_mesh_topology_workspace_bytes(int V, int F) {
    if (V <= 0 || F <= 0 || F > INT32_MAX / 6) return 0;
    return icon::tp_carve(nullptr, V, F, nullptr);
}

extern "C" int icon_mesh_topology_count(const int64_t *faces, int V, int F, int64_t *h_E, void *ws, size_t ws_bytes,
                                        icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(faces && h_E && ws, "icon_mesh_topology_count: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && F <= INT32_MAX / 6, "icon_mesh_topology_count: bad sizes V=%d F=%d", V, F);
    ICON_CHECK_ARG(ws_bytes >= icon_mesh_topology_workspace_bytes(V, F), "icon_mesh_topology_count: workspace too small");
    TpWs w;
    tp_carve(ws, V, F, &w);
    ICON_CUDA(cudaMemsetAsync(w.bad, 0, sizeof(int32_t), stream));
    ICON_CUDA(cudaMemsetAsync(w.ucnt + V, 0, sizeof(int32_t), stream));      // the scan's last input
    k_tp_pairs<<<(unsigned)((F + 255) / 256), 256, 0, stream>>>(faces, F, V, w.own, w.key, w.bad);
    ICON_LAUNCHED();
    int rc = csr_build(w.own, w.key, 3 * (int64_t)F, V, w.poff, w.plist, w.ucnt, w.csr, stream);
    if (rc) return rc;
    rc = scan_exclusive_i32(w.ucnt, w.eoff, (int64_t)V + 1, w.d_E, w.csr.scan_ws, stream);
    if (rc) return rc;
    int32_t bad = 0;
    int64_t E = 0;
    ICON_CUDA(cudaMemcpyAsync(&bad, w.bad, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    ICON_CUDA(cudaMemcpyAsync(&E, w.d_E, sizeof(int64_t), cudaMemcpyDeviceToHost, stream));
    ICON_CUDA(cudaStreamSynchronize(stream));
    ICON_CHECK_ARG(!bad, "icon_mesh_topology_count: a face index is outside [0, %d)", V);
    *h_E = E;
    return ICON_OK;
}

extern "C" int icon_mesh_topology_build(const icon_mesh_topology *t, void *ws, size_t ws_bytes,
                                        icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(topo_ok(t) && ws, "icon_mesh_topology_build: null pointer or empty topology");
    ICON_CHECK_ARG(t->F <= INT32_MAX / 6, "icon_mesh_topology_build: bad sizes F=%d", t->F);
    ICON_CHECK_ARG(ws_bytes >= icon_mesh_topology_workspace_bytes(t->V, t->F),
                   "icon_mesh_topology_build: workspace too small");
    const int V = t->V, F = t->F, E = t->E;
    TpWs w;
    tp_carve(ws, V, F, &w);
    k_tp_edges<<<(unsigned)((V + 255) / 256), 256, 0, stream>>>(w.poff, w.plist, w.eoff, V, t->edges, w.own,
                                                                 w.key);
    ICON_LAUNCHED();
    int rc = csr_build(w.own, w.key, 2 * (int64_t)E, V, t->vert_off, t->vert_edges, nullptr, w.csr, stream);
    if (rc) return rc;
    k_tp_f2e<<<(unsigned)((F + 255) / 256), 256, 0, stream>>>(t->faces, F, w.poff, w.plist, w.eoff,
                                                               t->face_to_edge, w.own, w.key);
    ICON_LAUNCHED();
    rc = csr_build(w.own, w.key, 3 * (int64_t)F, E, t->edge_off, t->edge_entries, nullptr, w.csr, stream);
    if (rc) return rc;
    return vertex_corners(t->faces, F, V, t->corner_off, t->vert_corners, ws, stream);
}

extern "C" size_t icon_vertex_edges_workspace_bytes(int V, int E) {
    if (V <= 0 || E <= 0 || E > INT32_MAX / 2) return 0;
    icon::Carver c(nullptr);
    c.take<int32_t>(2 * (size_t)E);
    c.take<int32_t>(2 * (size_t)E);
    icon::csr_take(c, V);
    return c.total();
}

extern "C" int icon_vertex_edges(const int64_t *edges, int E, int V, int32_t *vert_off, int32_t *vert_edges, void *ws,
                                 size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(edges && vert_off && vert_edges && ws, "icon_vertex_edges: null pointer");
    ICON_CHECK_ARG(V > 0 && E > 0 && E <= INT32_MAX / 2, "icon_vertex_edges: bad sizes V=%d E=%d", V, E);
    ICON_CHECK_ARG(ws_bytes >= icon_vertex_edges_workspace_bytes(V, E), "icon_vertex_edges: workspace too small");
    Carver c(ws);
    int32_t *own = c.take<int32_t>(2 * (size_t)E), *key = c.take<int32_t>(2 * (size_t)E);
    CsrWs w = csr_take(c, V);
    k_ve_items<<<(unsigned)((2 * (int64_t)E + 255) / 256), 256, 0, stream>>>(edges, E, own, key);
    ICON_LAUNCHED();
    return csr_build(own, key, 2 * (int64_t)E, V, vert_off, vert_edges, nullptr, w, stream);
}

extern "C" size_t icon_mesh_priors_workspace_bytes(int V, int F, int E, int backward) {
    if (V <= 0 || F <= 0 || E <= 0) return 0;
    return icon::pr_carve(nullptr, V, F, E, backward != 0, nullptr);
}

extern "C" int icon_mesh_priors_forward(const icon_mesh_topology *t, const float *verts, float *out_edge,
                                        float *out_nc, float *out_lap, void *ws, size_t ws_bytes,
                                        icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(topo_ok(t) && verts && out_edge && out_nc && out_lap && ws, "icon_mesh_priors_forward: null pointer");
    ICON_CHECK_ARG(ws_bytes >= icon_mesh_priors_workspace_bytes(t->V, t->F, t->E, 0),
                   "icon_mesh_priors_forward: workspace too small");
    PrWs w;
    pr_carve(ws, t->V, t->F, t->E, false, &w);
    const Topo T = topo_of(t);
    k_pr_edge_terms<<<(unsigned)w.nbE, PR_T, 0, stream>>>(T, verts, w.part, w.nbE, 1);
    ICON_LAUNCHED();
    k_pr_lap<<<(unsigned)w.nbV, PR_T, 0, stream>>>(T, verts, w.lap, w.part + 3 * (int64_t)w.nbE);
    ICON_LAUNCHED();
    k_pr_reduce<<<1, PR_T, 0, stream>>>(w.part, 3, w.nbE, w.sums);
    ICON_LAUNCHED();
    k_pr_reduce<<<1, PR_T, 0, stream>>>(w.part + 3 * (int64_t)w.nbE, 1, w.nbV, w.sums + 3);
    ICON_LAUNCHED();
    k_pr_out<<<1, 32, 0, stream>>>(w.sums, t->V, t->E, out_edge, out_nc, out_lap);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_mesh_priors_backward(const icon_mesh_topology *t, const float *verts, const float *g_edge,
                                         const float *g_nc, const float *g_lap, float *grad_verts, void *ws,
                                         size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(topo_ok(t) && verts && grad_verts && ws, "icon_mesh_priors_backward: null pointer");
    ICON_CHECK_ARG(ws_bytes >= icon_mesh_priors_workspace_bytes(t->V, t->F, t->E, 1),
                   "icon_mesh_priors_backward: workspace too small");
    PrWs w;
    pr_carve(ws, t->V, t->F, t->E, true, &w);
    const Topo T = topo_of(t);
    const unsigned vb = (unsigned)((t->V + 255) / 256), eb = (unsigned)((t->E + 255) / 256);
    if (g_lap) {
        k_pr_lap<<<(unsigned)w.nbV, PR_T, 0, stream>>>(T, verts, w.lap, w.part + 3 * (int64_t)w.nbE);
        ICON_LAUNCHED();
        k_pr_lap_u<<<vb, 256, 0, stream>>>(t->V, g_lap, w.lap);
        ICON_LAUNCHED();
    }
    if (g_nc) {
        k_pr_edge_terms<<<(unsigned)w.nbE, PR_T, 0, stream>>>(T, verts, w.part, w.nbE, 0);     // pair count only
        ICON_LAUNCHED();
        k_pr_reduce<<<1, PR_T, 0, stream>>>(w.part, 3, w.nbE, w.sums);
        ICON_LAUNCHED();
        k_pr_nc_entry<<<eb, 256, 0, stream>>>(T, verts, g_nc, w.sums, w.ent);
        ICON_LAUNCHED();
        k_pr_nc_face<<<(unsigned)((3 * (int64_t)t->F + 255) / 256), 256, 0, stream>>>(t->F, w.ent, w.fc);
        ICON_LAUNCHED();
    }
    k_pr_vertex<<<vb, 256, 0, stream>>>(T, verts, g_edge, g_lap ? w.lap : nullptr, g_nc ? w.fc : nullptr,
                                        grad_verts);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_local_affine_forward(const float *A, const float *b, const float *x, int N, const int64_t *edges,
                                         int E, float *out, float *w_diff, float *w_rigid, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(A && b && x && out && w_rigid && (E == 0 || (edges && w_diff)),
                   "icon_local_affine_forward: null pointer");
    ICON_CHECK_ARG(N > 0 && E >= 0, "icon_local_affine_forward: bad sizes N=%d E=%d", N, E);
    k_la_vertex<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(N, A, b, x, out, w_rigid);
    ICON_LAUNCHED();
    if (E > 0) {
        k_la_diff<<<(unsigned)((12 * (int64_t)E + 255) / 256), 256, 0, stream>>>(E, edges, A, b, w_diff);
        ICON_LAUNCHED();
    }
    return ICON_OK;
}

extern "C" int icon_local_affine_backward(const float *A, const float *b, const float *x, int N, const int64_t *edges,
                                          int E, const int32_t *vert_off, const int32_t *vert_edges,
                                          const float *g_out, const float *g_diff, const float *g_rigid, float *grad_A,
                                          float *grad_b, float *grad_x, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(A && b && x && grad_A && grad_b && (!g_diff || (edges && vert_off && vert_edges)),
                   "icon_local_affine_backward: null pointer");
    ICON_CHECK_ARG(N > 0 && E >= 0, "icon_local_affine_backward: bad sizes N=%d E=%d", N, E);
    k_la_backward<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(N, A, b, x, edges, vert_off, vert_edges, g_out,
                                                                    g_diff, g_rigid, grad_A, grad_b, grad_x);
    ICON_LAUNCHED();
    return ICON_OK;
}
