// Self-rotation video of the demo: replaces the per-frame pytorch3d renders of Render.get_rendered_video
// (lib/common/render.py:327-374): MeshRasterizer + cleanShader at the settings of get_camera and
// init_renderer(camera, "clean_mesh", "gray") (render.py:136-235), A views of one mesh per call.  Also the colours
// VF2Mesh gives a mesh (render.py:237-258): (Meshes.verts_normals_padded() + 1) / 2.
//
// PARITY UNPINNED: pytorch3d is not a dependency of this project.  The rules below are this file's contract, restated
// operation for operation by oracle/mesh_views.py (hence -fmad=false for this file).  All arithmetic is fp32, one
// rounding per operation, in the order written; "e(p, a, b)" is (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x).
//
// Vertex normals (icon_area_vertex_normals), pytorch3d's verts_normals_packed as oracle_vertex_normals restates it:
//   three passes (corner 1, 2, 0), each in face order, add n = (p1 - p0) x (p2 - p0) to vertex p0, where p1, p2 are
//   the next two corners of the face; then n / max(sqrt((x x + y y) + z z), 1e-6).  Each vertex's contributions are
//   sorted by (pass, face) and summed in that order: no float atomics, bitwise reproducible.  Faces with an index
//   outside [0, V) contribute nothing.
//   Backward (icon_area_vertex_normals_backward; restated by oracle/mesh_priors.py with float64 autograd): the
//   gradient of F.normalize(s, eps = 1e-6) with torch's semantics, from the fp32 s of the forward, in fp64:
//   (g - n (n.g)) / |s| with n = s / |s| when the fp32 norm is >= 1e-6, else g / 1e-6 (clamp_min passes g there);
//   then through each corner product n = u x w (u = p1 - p0, w = p2 - p0): p1 += w x G, p2 += G x u,
//   p0 -= both.  Each vertex sums its contributions over the same sorted (pass, face) lists in fp64 (its own position
//   in each listed face, all three products of that face) and rounds once.
//
// Views (icon_mesh_views).  Cameras: view a has eye = (100 cos t, y_c, 100 sin t), at = (0, y_c, 0), up = +y;
//   look_at_view_transform's basis z = unit(at - eye), x = unit(up x z), y = unit(z x x), and FoVOrthographicCameras
//   (x / y in +-100, scale_xyz = s) give x_ndc = s x_view / 100, y_ndc likewise, depth = z_view (what
//   MeshRasterizer leaves in zbuf).  The host builds M = [diag(s/100, s/100, 1) R | T] (3 x 4, rows) in float64 and
//   rounds it to fp32; the device computes each row as ((m0 x + m1 y) + m2 z) + m3.
//   Pixel grid: pixel (row i, col j) of an S x S image is centred at p = (1 - (2j+1)/S, 1 - (2i+1)/S).
//   Faces: a face is not drawn when an index is outside [0, V), a projected coordinate is not finite, all three
//   depths are < 0, or |e(v0, v1, v2)| <= 1e-8.  Both windings are drawn (no back-face culling).
//   Fragment of face (v0, v1, v2) at pixel p, with r = sqrt(blur), blur = fp32(ln(1e4) 1e-7):
//     skipped when p.x > xmax + r, p.x < xmin - r, p.y > ymax + r or p.y < ymin - r (the face's box);
//     den = e(v2, v0, v1) + 1e-8; w0 = e(p, v1, v2) / den, w1 = e(p, v2, v0) / den, w2 = e(p, v0, v1) / den;
//     inside = w0 > 0 and w1 > 0 and w2 > 0; d = min(min(d(v0,v1), d(v0,v2)), d(v1,v2)), the squared distance to a
//     segment a b being: u = b - a, q = p - a, l = u.x u.x + u.y u.y; q.q if l <= 1e-8, else with
//     t = clamp((u.x q.x + u.y q.y) / l, 0, 1) the squared length of p - (a + t u) (per component);
//     skipped when not inside and d >= blur;
//     clipped barycentrics c_k = max(w_k, 0) / max((c0 + c1) + c2, 1e-5); z = (c0 z0 + c1 z1) + c2 z2, skipped
//     when z < 0; dist = -d inside, d outside; colour = (c0 C0 + c1 C1) + c2 C2 per channel.
//   Per pixel the K = 30 nearest fragments by (z, face index) are kept and blended in that ascending order with
//   softmax_rgb_blend (sigma 1e-4, gamma 1e-8, background 0.5, znear -256, zfar 256, eps 1e-10):
//     zinv_k = (256 - z_k) / 512; zmax = max(zinv of the nearest fragment, 1e-10) (1e-10 for an empty pixel);
//     w_k = (1 / (1 + exp(dist_k / sigma))) exp((zinv_k - zmax) / gamma); delta = max(exp((1e-10 - zmax) / gamma), 1e-10);
//     rgb = (sum_k w_k colour_k + delta 0.5) / (sum_k w_k + delta), each sum accumulated from 0 in fragment order.
//   Output uint8 = trunc(min(max(rgb 255, 0), 255)) (NaN -> 0), RGB, [A, S, S, 3] with row 0 at the top.
//
// Kernel structure, per call (one chunk of A views; the mesh is read once per chunk):
//   k_mv_vertex   projects every vertex into every view;
//   pass 1        one thread per face rasterises it in each view (faces whose pixel box exceeds MV_SMALL pixels are
//                 listed and drawn by a block each, as in normal_render.cu), 64-bit atomicMin of (z bits, face):
//                 the nearest fragment, hence zmax;
//   pass 2        the same traversal keeps only fragments with (zinv - zmax) / gamma > -MV_CUT: exp of anything at
//                 or below -MV_CUT is 0 in fp32, so every fragment it drops has weight exactly 0 and lies behind all
//                 that it keeps.  The kept keys enter K per-pixel slots by an atomicMin insertion chain, which leaves
//                 the K smallest keys sorted whatever the arrival order;
//   k_mv_shade    one thread per pixel recomputes its slots' fragments and blends them.
// No float atomics: the result is bitwise reproducible and independent of the chunking.
//
// Differentiable renders of the fitting loops (icon_mesh_render_forward / _backward; restated by oracle/fit_render.py):
// Render.get_rgb_image and
// Render.get_silhouette_image (render.py:296-325, 376-387) at the cameras load_meshes sets (render.py:260-287: eyes
// (0, 0, 100), (100, 0, 0), (0, 0, -100), (-100, 0, 0), y_c = 0, s = 100; matrices from the eye tuples as above).
//   Mode NORMAL (init_renderer(camera, "clean_mesh", "gray")): the forward is exactly the rules above; its rgb equals
//     icon_mesh_views' rgb_out bit for bit.
//   Mode SILHOUETTE (init_renderer(camera, "silhouette")): blur = fp32(ln(1/1e-4 - 1) 5e-5), the K = 50 nearest
//     fragments by (z, face), cull_backfaces: a face is also not drawn when e(v0, v1, v2) < 0; SoftSilhouetteShader's
//     sigmoid_alpha_blend at sigma 1e-4: prob_k = 1 / (1 + exp(dist_k / sigma)), out = 1 - prod_k (1 - prob_k), the
//     product accumulated from 1 in fragment order (1 - 1 = 0 for an empty pixel).
//   The backward is the derivative of these formulas with the fragment set and every branch of the forward fixed
//   (pytorch3d's rasteriser passes no gradient through the selection), in fp32 per fragment:
//     NORMAL, per pixel (D = sum_k w_k + delta, rgb as above, g = upstream gradient of rgb):
//       Gw_k = (((g0 X_k0 + g1 X_k1) + g2 X_k2) / D) / D with X_kc = (sum_j w_j (col_kc - col_jc)) + delta (col_kc - 0.5),
//       the sum from 0 over the pixel's fragments in order (D (col_kc - rgb_c) without its cancellation: neighbouring
//       faces' colours nearly agree at their shared edge); Gcol_kc = (g_c w_k) / D;
//       Gprob_k = Gw_k e_k, Ge_k = Gw_k prob_k with e_k = exp((zinv_k - zmax) / gamma);
//       zmax = max over the fragments' zinv goes to slot 0 (the first in (z, face) order), so
//       Gzinv_k = (Ge_k e_k) / gamma for k >= 1 and Gzinv_0 = -(sum_{k>=1} Gzinv_k) (e_0 = 1: the two terms of slot 0
//       cancel exactly and are not formed); Gz_k = -(Gzinv_k / 512); Gdist_k = -((Gprob_k (prob_k q_k)) / sigma), where
//       the backward forms 1 - prob_k as q_k = u_k / (1 + u_k), u_k = exp(dist_k / sigma) (prob_k = 1 / (1 + u_k)): the
//       same value without the cancellation of 1 - prob_k near prob_k = 1.
//       clamp(min = eps) passes no gradient when clamped (delta is clamped on every covered pixel), and every clamp
//       passes it when its input is >= the bound.
//     SILHOUETTE: Gprob_k = g (P_k Q_k) with P_k = prod_{j<k} q_j accumulated forward, Q_k = prod_{j>k} q_j
//       accumulated from the last fragment (no division: prob = 1 exactly for a face that
//       covers a pixel deep inside); Gdist_k as above.  Only the distance carries gradient: x and y, not z.
//     Per fragment: Gc_k = ((Gcol_0 C_k0 + Gcol_1 C_k1) + Gcol_2 C_k2) + Gz z_k (colour interpolation and z),
//       GC_kc = Gcol_c c_k, Gz_k(vertex) = Gz c_k; clip c = m / s, m_k = max(w_k, 0), s = max((m0 + m1) + m2, 1e-5):
//       Gm_k = (Gc_k - sum_i Gc_i c_i) / s, formed as ((c_0 D_k0 + c_1 D_k1) + c_2 D_k2) / s from the corner differences
//       D_ki = ((Gcol_0 (C_k0 - C_i0) + Gcol_1 (C_k1 - C_i1)) + Gcol_2 (C_k2 - C_i2)) + Gz (z_k - z_i) (the same value as
//       sum_i c_i = 1; it avoids cancelling Gz z ~ 100 Gz), and Gm_k = Gc_k / s when s is clamped; Gw_k = Gm_k when
//       w_k >= 0, else 0; w_k = n_k / den: Gn_k = Gw_k / den, Gden = -(((Gw_0 w_0 + Gw_1 w_1) + Gw_2 w_2) / den), and
//       each edge function e(p, a, b) passes (p.y - b.y, b.x - p.x) to a, (a.y - p.y, p.x - a.x) to b (p = v2 for den);
//       dist: Gd = -Gdist inside, Gdist outside, to the minimising edge (ties: the first of v0v1, v0v2, v1v2); its
//       squared distance gives a -2 r (1 - t), b -2 r t, r = p - (a + t u), plus, when 0 <= t_raw <= 1 (the clamp
//       uses the side it is on), -2 (r.u) times dt/da = ((2 t u - q) - u) / l, dt/db = (q - 2 t u) / l; a segment with
//       l <= 1e-8 gives a -2 q.  The camera row takes (Gx, Gy, Gz) to the world by M^T.
//   Fragments that pass 2 drops have weight exactly 0 (e_k = 0): Gcol, Gprob and Gzinv of such a fragment are exactly
//   0 in fp32, so the cut is exact for the gradients too.
//   Kernel structure of the backward (no float atomics; bitwise reproducible): the forward leaves each pixel's K slot
//   keys in the caller's state buffer; k_mr_pixel turns the upstream gradient into per-slot partials (NORMAL: Gcol,
//   Gz, Gdist, with the slots' weights, colours and Gw parked there first; SILHOUETTE: Gdist); k_mr_face_small / _big re-traverse each (face, view)'s pixel box in a fixed order,
//   find the face's own key among the pixel's slots and sum its three corners' (Gx, Gy, Gz, GC) in fp64 (big boxes: a
//   block per face, fixed-order tree reduction); k_mr_vertex sums each vertex's corner contributions in the sorted
//   (pass, face) order of k_an_*, view after view, applies M^T in fp64 and rounds to fp32 once.
#include <math.h>

#include "common.cuh"

namespace icon {

constexpr int MV_K = 30;                          // faces_per_pixel
constexpr int MV_SMALL = 64;                      // pixel boxes up to this size: one thread per face and view
constexpr int MV_BIG_BLOCKS = 2048;
constexpr float MV_CUT = 120.f;                   // expf(x) == 0 for x <= -MV_CUT (e^-120 < 2^-150)
constexpr unsigned long long MV_EMPTY = 0xffffffffffffffffull;
constexpr float MV_SIGMA = 1e-4f, MV_GAMMA = 1e-8f, MV_EPS = 1e-10f, MV_BG = 0.5f;
constexpr float MV_KEPS = 1e-8f;                  // pytorch3d's kEpsilon
constexpr float MV_BLUR = 9.210340371976183e-07f; // ln(1e4) 1e-7

// render modes: the passes below are templates on one of these
struct MvNormal {                                 // clean_mesh: softmax_rgb_blend of 30 fragments
    static constexpr int K = MV_K, SMALL = MV_SMALL, NP = 6, NG = 6;   // per-slot partials, per-corner gradients
    static constexpr bool CULL = false, CUT = true;
    static constexpr float BLUR = MV_BLUR;
};
struct MvSilhouette {                             // silhouette: sigmoid_alpha_blend of 50 back-face-culled fragments
    static constexpr int K = 50, SMALL = 512, NP = 1, NG = 2;          // r ~ 5.5 px at 512^2: boxes are >= 11 x 11
    static constexpr bool CULL = true, CUT = false;
    static constexpr float BLUR = 4.605120047926903e-04f;              // ln(1/1e-4 - 1) 5e-5
};

// ---------------------------------------------------------------- area-weighted vertex normals

__device__ __forceinline__ bool mv_face_ids(const int64_t *faces, int f, int V, int id[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int64_t x = faces[3 * (int64_t)f + k];
        if (x < 0 || x >= V) return false;
        id[k] = (int)x;
    }
    return true;
}

__global__ void k_an_count(const int64_t *__restrict__ faces, int F, int V, int32_t *__restrict__ cnt) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    int id[3];
    if (f >= F || !mv_face_ids(faces, f, V, id)) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) atomicAdd(&cnt[id[k]], 1);
}

// contribution keys pass * F + f (pass 0, 1, 2 = corner 1, 2, 0), in arrival order; k_an_sum sorts each list
__global__ void k_an_fill(const int64_t *__restrict__ faces, int F, int V, const int32_t *__restrict__ off,
                          int32_t *__restrict__ cursor, int32_t *__restrict__ keys) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    int id[3];
    if (f >= F || !mv_face_ids(faces, f, V, id)) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) keys[off[id[k]] + atomicAdd(&cursor[id[k]], 1)] = ((k + 2) % 3) * F + f;
}

__global__ void k_an_sum(const float *__restrict__ verts, const int64_t *__restrict__ faces, int F,
                         const int32_t *__restrict__ off, int32_t *__restrict__ keys, int V, float *__restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    int32_t *a = keys + off[v];
    const int n = off[v + 1] - off[v];
    heap_sort_i32(a, n);
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int i = 0; i < n; ++i) {
        const int pass = a[i] / F, f = a[i] % F;
        const int c = pass == 0 ? 1 : (pass == 1 ? 2 : 0);
        const int64_t i0 = faces[3 * (int64_t)f + c], i1 = faces[3 * (int64_t)f + (c + 1) % 3];
        const int64_t i2 = faces[3 * (int64_t)f + (c + 2) % 3];
        const float p0x = verts[3 * i0], p0y = verts[3 * i0 + 1], p0z = verts[3 * i0 + 2];
        const float ux = verts[3 * i1] - p0x, uy = verts[3 * i1 + 1] - p0y, uz = verts[3 * i1 + 2] - p0z;
        const float wx = verts[3 * i2] - p0x, wy = verts[3 * i2 + 1] - p0y, wz = verts[3 * i2 + 2] - p0z;
        sx = sx + (uy * wz - uz * wy);
        sy = sy + (uz * wx - ux * wz);
        sz = sz + (ux * wy - uy * wx);
    }
    float nrm = sqrtf((sx * sx + sy * sy) + sz * sz);
    if (nrm < 1e-6f) nrm = 1e-6f;
    out[3 * (int64_t)v] = sx / nrm; out[3 * (int64_t)v + 1] = sy / nrm; out[3 * (int64_t)v + 2] = sz / nrm;
}

// backward, 1: sort the vertex's list, recompute s as k_an_sum does, then the normalize gradient (fp64) into gs
__global__ void k_an_grad_s(const float *__restrict__ verts, const int64_t *__restrict__ faces, int F,
                            const int32_t *__restrict__ off, int32_t *__restrict__ keys, int V,
                            const float *__restrict__ gn, double *__restrict__ gs) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    int32_t *a = keys + off[v];
    const int n = off[v + 1] - off[v];
    heap_sort_i32(a, n);
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int i = 0; i < n; ++i) {
        const int pass = a[i] / F, f = a[i] % F;
        const int c = pass == 0 ? 1 : (pass == 1 ? 2 : 0);
        const int64_t i0 = faces[3 * (int64_t)f + c], i1 = faces[3 * (int64_t)f + (c + 1) % 3];
        const int64_t i2 = faces[3 * (int64_t)f + (c + 2) % 3];
        const float p0x = verts[3 * i0], p0y = verts[3 * i0 + 1], p0z = verts[3 * i0 + 2];
        const float ux = verts[3 * i1] - p0x, uy = verts[3 * i1 + 1] - p0y, uz = verts[3 * i1 + 2] - p0z;
        const float wx = verts[3 * i2] - p0x, wy = verts[3 * i2 + 1] - p0y, wz = verts[3 * i2 + 2] - p0z;
        sx = sx + (uy * wz - uz * wy);
        sy = sy + (uz * wx - ux * wz);
        sz = sz + (ux * wy - uy * wx);
    }
    const double s[3] = {sx, sy, sz};
    const double g[3] = {gn[3 * (int64_t)v], gn[3 * (int64_t)v + 1], gn[3 * (int64_t)v + 2]};
    const double len = sqrt((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2]);
    const float nrm = sqrtf((sx * sx + sy * sy) + sz * sz);
    if (nrm < 1e-6f) {                                    // the clamp: g / eps
#pragma unroll
        for (int k = 0; k < 3; ++k) gs[3 * (int64_t)v + k] = g[k] / 1e-6;
        return;
    }
    const double d = ((s[0] * g[0] + s[1] * g[1]) + s[2] * g[2]) / len;
#pragma unroll
    for (int k = 0; k < 3; ++k) gs[3 * (int64_t)v + k] = (g[k] - (s[k] / len) * d) / len;
}

// backward, 2: per vertex, over its sorted (pass, face) entries, the derivative of the entry face's three corner
// products n_k = (p_{k+1} - p_k) x (p_{k+2} - p_k) with respect to the vertex's own position in the face
__global__ void k_an_grad_v(const float *__restrict__ verts, const int64_t *__restrict__ faces, int F,
                            const int32_t *__restrict__ off, const int32_t *__restrict__ keys, int V,
                            const double *__restrict__ gs, float *__restrict__ gv) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const int32_t *a = keys + off[v];
    const int n = off[v + 1] - off[v];
    double acc[3] = {0.0, 0.0, 0.0};
    for (int i = 0; i < n; ++i) {
        const int pass = a[i] / F, f = a[i] % F;
        const int c = pass == 0 ? 1 : (pass == 1 ? 2 : 0);              // the vertex's corner in face f
        double p[3][3];
        int64_t id[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            id[k] = faces[3 * (int64_t)f + k];
#pragma unroll
            for (int q = 0; q < 3; ++q) p[k][q] = (double)verts[3 * id[k] + q];
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {                                   // corner k's product, added to vertex id[k]
            const double *G = gs + 3 * id[k];
            double u[3], w[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                u[q] = p[(k + 1) % 3][q] - p[k][q];
                w[q] = p[(k + 2) % 3][q] - p[k][q];
            }
            const double gu[3] = {w[1] * G[2] - w[2] * G[1], w[2] * G[0] - w[0] * G[2], w[0] * G[1] - w[1] * G[0]};
            const double gw[3] = {G[1] * u[2] - G[2] * u[1], G[2] * u[0] - G[0] * u[2], G[0] * u[1] - G[1] * u[0]};
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                if (c == k) acc[q] -= gu[q] + gw[q];
                else if (c == (k + 1) % 3) acc[q] += gu[q];
                else acc[q] += gw[q];
            }
        }
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) gv[3 * (int64_t)v + q] = (float)acc[q];
}

struct AnWs {
    int32_t *cnt, *off, *cursor, *keys;
    void *scan_ws;
};

static size_t an_carve(void *ws, int V, int F, AnWs *o) {
    Carver c(ws);
    AnWs w;
    w.cnt = c.take<int32_t>((size_t)V + 1);
    w.off = c.take<int32_t>((size_t)V + 1);
    w.cursor = c.take<int32_t>((size_t)V);
    w.keys = c.take<int32_t>(3 * (size_t)F);
    w.scan_ws = c.take<char>(scan_ws_bytes((int64_t)V + 1));
    if (o) *o = w;
    return c.total();
}

// ---------------------------------------------------------------- views

__device__ __forceinline__ float mv_e(float px, float py, float ax, float ay, float bx, float by) {
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax);
}

__device__ __forceinline__ float mv_seg(float px, float py, float ax, float ay, float bx, float by) {
    const float ux = bx - ax, uy = by - ay, qx = px - ax, qy = py - ay;
    const float l = ux * ux + uy * uy;
    if (l <= MV_KEPS) return qx * qx + qy * qy;
    const float t = fmaxf(fminf((ux * qx + uy * qy) / l, 1.f), 0.f);
    const float rx = px - (ax + t * ux), ry = py - (ay + t * uy);
    return rx * rx + ry * ry;
}

__device__ __forceinline__ float mv_pix(int j, int S) { return 1.f - (float)(2 * j + 1) / (float)S; }

// one face in one view, set up for its fragments
struct MvTri {
    float x[3], y[3], z[3];
    float den, bx0, bx1, by0, by1;   // barycentric denominator, the face's box widened by sqrt(blur)
    int j0, j1, i0, i1;              // candidate pixel columns / rows (conservative; may be empty)
};

// conservative pixel range whose centres can lie in [lo, hi]: centre(k) = 1 - (2k+1)/S decreases with k
__device__ __forceinline__ void mv_range(float lo, float hi, int S, int &k0, int &k1) {
    const double a = floor(((1.0 - (double)hi) * S - 1.0) * 0.5) - 1.0;
    const double b = ceil(((1.0 - (double)lo) * S - 1.0) * 0.5) + 1.0;
    k0 = (int)fmax(a, 0.0);
    k1 = (int)fmin(b, (double)(S - 1));
}

template <class M>
__device__ __forceinline__ bool mv_setup(const int64_t *__restrict__ faces, const float4 *__restrict__ vrec, int f,
                                         int V, int S, MvTri &t) {
    int id[3];
    if (!mv_face_ids(faces, f, V, id)) return false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float4 r = vrec[id[k]];
        if (!(isfinite(r.x) && isfinite(r.y) && isfinite(r.z))) return false;
        t.x[k] = r.x; t.y[k] = r.y; t.z[k] = r.z;
    }
    if (fmaxf(fmaxf(t.z[0], t.z[1]), t.z[2]) < 0.f) return false;
    const float area = mv_e(t.x[0], t.y[0], t.x[1], t.y[1], t.x[2], t.y[2]);
    if (area <= MV_KEPS && area >= -MV_KEPS) return false;
    if (M::CULL && area < 0.f) return false;
    t.den = mv_e(t.x[2], t.y[2], t.x[0], t.y[0], t.x[1], t.y[1]) + MV_KEPS;
    const float r = sqrtf(M::BLUR);
    t.bx0 = fminf(fminf(t.x[0], t.x[1]), t.x[2]) - r; t.bx1 = fmaxf(fmaxf(t.x[0], t.x[1]), t.x[2]) + r;
    t.by0 = fminf(fminf(t.y[0], t.y[1]), t.y[2]) - r; t.by1 = fmaxf(fmaxf(t.y[0], t.y[1]), t.y[2]) + r;
    mv_range(t.bx0, t.bx1, S, t.j0, t.j1);
    mv_range(t.by0, t.by1, S, t.i0, t.i1);
    return t.j0 <= t.j1 && t.i0 <= t.i1;
}

struct MvFrag {
    float z, dist, c[3];
    float w[3], sum, d[3];           // for the backward: raw barycentrics, clip sum, squared edge distances
    bool inside;
};

template <class M>
__device__ __forceinline__ bool mv_fragment(const MvTri &t, float px, float py, MvFrag &o) {
    if (px > t.bx1 || px < t.bx0 || py > t.by1 || py < t.by0) return false;
    const float w0 = mv_e(px, py, t.x[1], t.y[1], t.x[2], t.y[2]) / t.den;
    const float w1 = mv_e(px, py, t.x[2], t.y[2], t.x[0], t.y[0]) / t.den;
    const float w2 = mv_e(px, py, t.x[0], t.y[0], t.x[1], t.y[1]) / t.den;
    const bool inside = w0 > 0.f && w1 > 0.f && w2 > 0.f;
    const float d01 = mv_seg(px, py, t.x[0], t.y[0], t.x[1], t.y[1]);
    const float d02 = mv_seg(px, py, t.x[0], t.y[0], t.x[2], t.y[2]);
    const float d12 = mv_seg(px, py, t.x[1], t.y[1], t.x[2], t.y[2]);
    const float d = fminf(fminf(d01, d02), d12);
    if (!inside && d >= M::BLUR) return false;
    float c0 = fmaxf(w0, 0.f), c1 = fmaxf(w1, 0.f), c2 = fmaxf(w2, 0.f);
    const float sum = (c0 + c1) + c2;
    const float s = fmaxf(sum, 1e-5f);
    c0 = c0 / s; c1 = c1 / s; c2 = c2 / s;
    const float z = (c0 * t.z[0] + c1 * t.z[1]) + c2 * t.z[2];
    if (z < 0.f) return false;
    o.z = z; o.dist = inside ? -d : d;
    o.c[0] = c0; o.c[1] = c1; o.c[2] = c2;
    o.w[0] = w0; o.w[1] = w1; o.w[2] = w2; o.sum = sum;
    o.d[0] = d01; o.d[1] = d02; o.d[2] = d12; o.inside = inside;
    return true;
}

__device__ __forceinline__ unsigned long long mv_key(float z, int f) {
    return ((unsigned long long)(__float_as_uint(z) & 0x7fffffffu) << 32) | (unsigned)f;   // z >= 0 (-0 -> +0)
}

__device__ __forceinline__ float mv_zmax(unsigned long long nearest) {
    return nearest == MV_EMPTY ? MV_EPS : fmaxf((256.f - __uint_as_float((unsigned)(nearest >> 32))) / 512.f, MV_EPS);
}

// pass 1: nearest fragment; pass 2: the fragments of non-zero weight (M::CUT) or all of them into the K sorted slots
template <int PASS, class M>
__device__ __forceinline__ void mv_pixel(const MvTri &t, int f, int i, int j, int S, int64_t pix,
                                         unsigned long long *__restrict__ near, unsigned long long *__restrict__ slots) {
    MvFrag fr;
    if (!mv_fragment<M>(t, mv_pix(j, S), mv_pix(i, S), fr)) return;
    unsigned long long key = mv_key(fr.z, f);
    if (PASS == 1) {
        atomicMin(&near[pix], key);
        return;
    }
    if (M::CUT) {
        const float zmax = mv_zmax(near[pix]);
        if (!(((256.f - fr.z) / 512.f - zmax) / MV_GAMMA > -MV_CUT)) return;
    }
    unsigned long long *s = slots + pix * M::K;
    for (int k = 0; k < M::K; ++k) {
        const unsigned long long old = atomicMin(&s[k], key);
        if (old == MV_EMPTY) return;
        key = old > key ? old : key;              // the larger one moves on to the next slot
    }
}

__global__ void k_mv_vertex(const float *__restrict__ verts, int V, const float *__restrict__ mats,
                            float4 *__restrict__ vrec) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int a = blockIdx.y;
    if (i >= V) return;
    const float *m = mats + 12 * a;
    const float x = verts[3 * (int64_t)i], y = verts[3 * (int64_t)i + 1], z = verts[3 * (int64_t)i + 2];
    vrec[(int64_t)a * V + i] = make_float4(((m[0] * x + m[1] * y) + m[2] * z) + m[3],
                                           ((m[4] * x + m[5] * y) + m[6] * z) + m[7],
                                           ((m[8] * x + m[9] * y) + m[10] * z) + m[11], 0.f);
}

// one thread per face, looping over the chunk's views; pass 1 lists the (face, view) pairs with a large box (and,
// with a cut only, finds the nearest fragments)
template <int PASS, class M>
__global__ void k_mv_small(const int64_t *__restrict__ faces, int F, int V, int A, int S,
                           const float4 *__restrict__ vrec, unsigned long long *__restrict__ near,
                           unsigned long long *__restrict__ slots, int2 *__restrict__ big, int32_t *__restrict__ nbig) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    for (int a = 0; a < A; ++a) {
        MvTri t;
        if (!mv_setup<M>(faces, vrec + (int64_t)a * V, f, V, S, t)) continue;
        const int nj = t.j1 - t.j0 + 1, ni = t.i1 - t.i0 + 1;
        if (nj * ni > M::SMALL) {
            if (PASS == 1) big[atomicAdd(nbig, 1)] = make_int2(f, a);
            continue;
        }
        if (PASS == 1 && !M::CUT) continue;
        const int64_t base = (int64_t)a * S * S;
        for (int i = t.i0; i <= t.i1; ++i)
            for (int j = t.j0; j <= t.j1; ++j)
                mv_pixel<PASS, M>(t, f, i, j, S, base + (int64_t)i * S + j, near, slots);
    }
}

// one block per listed (face, view) pair; the block's threads stride over the face's pixel box
template <int PASS, class M>
__global__ void __launch_bounds__(256) k_mv_big(const int64_t *__restrict__ faces, int V, int S,
                                                const float4 *__restrict__ vrec, unsigned long long *__restrict__ near,
                                                unsigned long long *__restrict__ slots, const int2 *__restrict__ big,
                                                const int32_t *__restrict__ nbig) {
    const int n = *nbig;
    for (int b = blockIdx.x; b < n; b += gridDim.x) {
        const int f = big[b].x, a = big[b].y;
        MvTri t;
        if (!mv_setup<M>(faces, vrec + (int64_t)a * V, f, V, S, t)) continue;
        const int nj = t.j1 - t.j0 + 1;
        const int np = nj * (t.i1 - t.i0 + 1);
        const int64_t base = (int64_t)a * S * S;
        for (int p = threadIdx.x; p < np; p += blockDim.x) {
            const int i = t.i0 + p / nj, j = t.j0 + p % nj;
            mv_pixel<PASS, M>(t, f, i, j, S, base + (int64_t)i * S + j, near, slots);
        }
    }
}

// the fragment of slot key `key` at pixel (px, py) of view a (it was drawn by the raster passes, so both succeed)
template <class M>
__device__ __forceinline__ int mv_slot_fragment(const int64_t *__restrict__ faces, const float4 *__restrict__ vrec,
                                                int V, int S, unsigned long long key, float px, float py, MvFrag &fr) {
    const int f = (int)(key & 0xffffffffull);
    MvTri t;
    mv_setup<M>(faces, vrec, f, V, S, t);
    mv_fragment<M>(t, px, py, fr);
    return f;
}

__device__ __forceinline__ void mv_colour(const int64_t *__restrict__ faces, const float *__restrict__ colors, int f,
                                          const MvFrag &fr, float col[3]) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const int64_t c0 = 3 * faces[3 * (int64_t)f], c1 = 3 * faces[3 * (int64_t)f + 1];
        const int64_t c2 = 3 * faces[3 * (int64_t)f + 2];
        col[ch] = (fr.c[0] * colors[c0 + ch] + fr.c[1] * colors[c1 + ch]) + fr.c[2] * colors[c2 + ch];
    }
}

__device__ __forceinline__ float mv_prob(float dist) { return 1.f / (1.f + expf(dist / MV_SIGMA)); }

// the backward's prob and 1 - prob, the latter as u / (1 + u), u = exp(dist / sigma): no cancellation near prob = 1
__device__ __forceinline__ void mv_prob_q(float dist, float &prob, float &q) {
    const float u = expf(dist / MV_SIGMA);
    prob = 1.f / (1.f + u);
    q = u / (1.f + u);
}

// one thread per (view, pixel): blend the slots' fragments in ascending (z, face) order
__global__ void k_mv_shade(const int64_t *__restrict__ faces, int V, int A, int S, const float4 *__restrict__ vrec,
                           const float *__restrict__ colors, const unsigned long long *__restrict__ slots,
                           uint8_t *__restrict__ out, int32_t *__restrict__ face_out, float *__restrict__ rgb_out) {
    const int64_t npix = (int64_t)S * S;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)A * npix) return;
    const int a = (int)(p / npix);
    const int i = (int)((p % npix) / S), j = (int)(p % S);
    const unsigned long long *s = slots + p * MV_K;
    const float zmax = mv_zmax(s[0]);
    const float px = mv_pix(j, S), py = mv_pix(i, S);
    float nr = 0.f, ng = 0.f, nb = 0.f, den = 0.f;
    for (int k = 0; k < MV_K; ++k) {
        const unsigned long long key = s[k];
        if (key == MV_EMPTY) break;
        MvFrag fr;
        const int f = mv_slot_fragment<MvNormal>(faces, vrec + (int64_t)a * V, V, S, key, px, py, fr);
        const float w = mv_prob(fr.dist) * expf(((256.f - fr.z) / 512.f - zmax) / MV_GAMMA);
        float col[3];
        mv_colour(faces, colors, f, fr, col);
        nr = nr + w * col[0]; ng = ng + w * col[1]; nb = nb + w * col[2];
        den = den + w;
    }
    const float delta = fmaxf(expf((MV_EPS - zmax) / MV_GAMMA), MV_EPS);
    den = den + delta;
    const float rgb[3] = {(nr + delta * MV_BG) / den, (ng + delta * MV_BG) / den, (nb + delta * MV_BG) / den};
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float v = rgb[ch] * 255.f;
        if (out) out[3 * p + ch] = v >= 255.f ? (uint8_t)255 : (v > 0.f ? (uint8_t)v : (uint8_t)0);
        if (rgb_out) rgb_out[3 * p + ch] = rgb[ch];
    }
    if (face_out) face_out[p] = s[0] == MV_EMPTY ? -1 : (int)(s[0] & 0xffffffffull);
}

// one thread per (view, pixel): the silhouette, 1 - prod_k (1 - prob_k) in slot order
__global__ void k_mv_silhouette(const int64_t *__restrict__ faces, int V, int A, int S,
                                const float4 *__restrict__ vrec, const unsigned long long *__restrict__ slots,
                                float *__restrict__ out) {
    const int64_t npix = (int64_t)S * S;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)A * npix) return;
    const int a = (int)(p / npix);
    const int i = (int)((p % npix) / S), j = (int)(p % S);
    const unsigned long long *s = slots + p * MvSilhouette::K;
    const float px = mv_pix(j, S), py = mv_pix(i, S);
    float prod = 1.f;
    for (int k = 0; k < MvSilhouette::K; ++k) {
        if (s[k] == MV_EMPTY) break;
        MvFrag fr;
        mv_slot_fragment<MvSilhouette>(faces, vrec + (int64_t)a * V, V, S, s[k], px, py, fr);
        prod = prod * (1.f - mv_prob(fr.dist));
    }
    out[p] = 1.f - prod;
}

// ---------------------------------------------------------------- backward

// per-slot partials of one pixel: NORMAL (Gcol r, g, b, Gz, Gdist; the sixth float is scratch), SILHOUETTE (Gdist);
// header formulas
__global__ void k_mr_pixel_normal(const int64_t *__restrict__ faces, int V, int A, int S,
                                  const float4 *__restrict__ vrec, const float *__restrict__ colors,
                                  const unsigned long long *__restrict__ slots, const float *__restrict__ gout,
                                  float *__restrict__ part) {
    constexpr int K = MvNormal::K, NP = MvNormal::NP;
    const int64_t npix = (int64_t)S * S;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)A * npix) return;
    const unsigned long long *s = slots + p * K;
    if (s[0] == MV_EMPTY) return;                 // no key of this pixel is ever looked up
    const int a = (int)(p / npix);
    const int i = (int)((p % npix) / S), j = (int)(p % S);
    const float4 *vr = vrec + (int64_t)a * V;
    const float zmax = mv_zmax(s[0]);
    const float px = mv_pix(j, S), py = mv_pix(i, S);
    float *q = part + p * K * NP;
    float den = 0.f;
    int n = 0;
    for (; n < K && s[n] != MV_EMPTY; ++n) {      // the forward's weights and colours, parked in the slots
        MvFrag fr;
        const int f = mv_slot_fragment<MvNormal>(faces, vr, V, S, s[n], px, py, fr);
        const float w = mv_prob(fr.dist) * expf(((256.f - fr.z) / 512.f - zmax) / MV_GAMMA);
        mv_colour(faces, colors, f, fr, q + NP * n);
        q[NP * n + 3] = w;
        den = den + w;
    }
    const float delta = fmaxf(expf((MV_EPS - zmax) / MV_GAMMA), MV_EPS);
    den = den + delta;
    const float g[3] = {gout[3 * p], gout[3 * p + 1], gout[3 * p + 2]};
    for (int k = 0; k < n; ++k) {                 // Gw_k from colour differences, parked in slot k
        float x[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) x[ch] = 0.f;
        for (int m = 0; m < n; ++m) {
            const float wm = q[NP * m + 3];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) x[ch] = x[ch] + wm * (q[NP * k + ch] - q[NP * m + ch]);
        }
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) x[ch] = x[ch] + delta * (q[NP * k + ch] - MV_BG);
        q[NP * k + 5] = (((g[0] * x[0] + g[1] * x[1]) + g[2] * x[2]) / den) / den;
    }
    float zsum = 0.f;                             // sum_{k>=1} Gzinv_k
    for (int k = 0; k < n; ++k) {
        MvFrag fr;
        mv_slot_fragment<MvNormal>(faces, vr, V, S, s[k], px, py, fr);
        float prob, qb;
        mv_prob_q(fr.dist, prob, qb);
        const float e = expf(((256.f - fr.z) / 512.f - zmax) / MV_GAMMA);
        const float w = prob * e;
        const float gw = q[NP * k + 5];
        const float gprob = gw * e, ge = gw * prob;
        const float gzinv = k == 0 ? 0.f : (ge * e) / MV_GAMMA;
        zsum = zsum + gzinv;
        q[NP * k] = (g[0] * w) / den; q[NP * k + 1] = (g[1] * w) / den; q[NP * k + 2] = (g[2] * w) / den;
        q[NP * k + 3] = -(gzinv / 512.f);
        q[NP * k + 4] = -((gprob * (prob * qb)) / MV_SIGMA);
    }
    q[3] = -(-zsum / 512.f);                      // slot 0: Gzinv_0 = -zsum
}

__global__ void k_mr_pixel_silhouette(const int64_t *__restrict__ faces, int V, int A, int S,
                                      const float4 *__restrict__ vrec, const unsigned long long *__restrict__ slots,
                                      const float *__restrict__ gout, float *__restrict__ part) {
    constexpr int K = MvSilhouette::K;
    const int64_t npix = (int64_t)S * S;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)A * npix) return;
    const unsigned long long *s = slots + p * K;
    const int a = (int)(p / npix);
    const int i = (int)((p % npix) / S), j = (int)(p % S);
    const float4 *vr = vrec + (int64_t)a * V;
    const float px = mv_pix(j, S), py = mv_pix(i, S);
    float *q = part + p * K;
    float pre = 1.f;
    int n = 0;
    for (; n < K && s[n] != MV_EMPTY; ++n) {      // P_k parked in the partial slots
        MvFrag fr;
        mv_slot_fragment<MvSilhouette>(faces, vr, V, S, s[n], px, py, fr);
        float prob, qb;
        mv_prob_q(fr.dist, prob, qb);
        q[n] = pre;
        pre = pre * qb;
    }
    const float g = gout[p];
    float suf = 1.f;
    for (int k = n - 1; k >= 0; --k) {
        MvFrag fr;
        mv_slot_fragment<MvSilhouette>(faces, vr, V, S, s[k], px, py, fr);
        float prob, qb;
        mv_prob_q(fr.dist, prob, qb);
        const float gprob = g * (q[k] * suf);
        q[k] = -((gprob * (prob * qb)) / MV_SIGMA);
        suf = suf * qb;
    }
}

// squared distance to segment a b: adds its gradient times g to (ga, gb)
__device__ __forceinline__ void mv_seg_grad(float px, float py, float ax, float ay, float bx, float by, float g,
                                            float &gax, float &gay, float &gbx, float &gby) {
    const float ux = bx - ax, uy = by - ay, qx = px - ax, qy = py - ay;
    const float l = ux * ux + uy * uy;
    if (l <= MV_KEPS) {
        gax = gax + g * (-2.f * qx); gay = gay + g * (-2.f * qy);
        return;
    }
    const float tr = (ux * qx + uy * qy) / l;
    const float t = fmaxf(fminf(tr, 1.f), 0.f);
    const float rx = px - (ax + t * ux), ry = py - (ay + t * uy);
    float dax = -2.f * rx * (1.f - t), day = -2.f * ry * (1.f - t), dbx = -2.f * rx * t, dby = -2.f * ry * t;
    if (tr >= 0.f && tr <= 1.f) {
        const float gt = -2.f * (rx * ux + ry * uy);
        dax = dax + gt * (((2.f * t * ux - qx) - ux) / l); day = day + gt * (((2.f * t * uy - qy) - uy) / l);
        dbx = dbx + gt * ((qx - 2.f * t * ux) / l); dby = dby + gt * ((qy - 2.f * t * uy) / l);
    }
    gax = gax + g * dax; gay = gay + g * day; gbx = gbx + g * dbx; gby = gby + g * dby;
}

// e(p, a, b) times g: (p.y - b.y, b.x - p.x) to a, (a.y - p.y, p.x - a.x) to b
__device__ __forceinline__ void mv_e_grad(float px, float py, float ax, float ay, float bx, float by, float g,
                                          float &gax, float &gay, float &gbx, float &gby) {
    gax = gax + g * (py - by); gay = gay + g * (bx - px);
    gbx = gbx + g * (ay - py); gby = gby + g * (px - ax);
}

// one fragment's gradient to its face's corners, added to acc[corner * NG + (x, y[, z, r, g, b])] in fp64
template <class M>
__device__ __forceinline__ void mv_frag_grad(const MvTri &t, const MvFrag &fr, float px, float py,
                                             const float *__restrict__ q, const float C[9], double *acc) {
    float gx[3] = {0.f, 0.f, 0.f}, gy[3] = {0.f, 0.f, 0.f};
    const float gdist = q[M::NP == 1 ? 0 : 4];
    if constexpr (M::NP == 6) {
        const float gcol[3] = {q[0], q[1], q[2]}, gz = q[3];
        float gc[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            gc[k] = ((gcol[0] * C[3 * k] + gcol[1] * C[3 * k + 1]) + gcol[2] * C[3 * k + 2]) + gz * t.z[k];
            acc[M::NG * k + 2] += (double)(gz * fr.c[k]);
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) acc[M::NG * k + 3 + ch] += (double)(gcol[ch] * fr.c[k]);
        }
        const float s = fmaxf(fr.sum, 1e-5f);
        float gw[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float gm = gc[k] / s;                    // s clamped: no gradient through s
            if (fr.sum >= 1e-5f) {                   // sum_i c_i (Gc_k - Gc_i) from corner differences
                float acc = 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    const float dki = ((gcol[0] * (C[3 * k] - C[3 * i]) + gcol[1] * (C[3 * k + 1] - C[3 * i + 1])) +
                                       gcol[2] * (C[3 * k + 2] - C[3 * i + 2])) + gz * (t.z[k] - t.z[i]);
                    acc = acc + fr.c[i] * dki;
                }
                gm = acc / s;
            }
            gw[k] = fr.w[k] >= 0.f ? gm : 0.f;
        }
        const float gden = -(((gw[0] * fr.w[0] + gw[1] * fr.w[1]) + gw[2] * fr.w[2]) / t.den);
        mv_e_grad(px, py, t.x[1], t.y[1], t.x[2], t.y[2], gw[0] / t.den, gx[1], gy[1], gx[2], gy[2]);
        mv_e_grad(px, py, t.x[2], t.y[2], t.x[0], t.y[0], gw[1] / t.den, gx[2], gy[2], gx[0], gy[0]);
        mv_e_grad(px, py, t.x[0], t.y[0], t.x[1], t.y[1], gw[2] / t.den, gx[0], gy[0], gx[1], gy[1]);
        // den = e(v2, v0, v1): v2 is its point
        gx[2] = gx[2] + gden * (t.y[1] - t.y[0]); gy[2] = gy[2] + gden * (t.x[0] - t.x[1]);
        mv_e_grad(t.x[2], t.y[2], t.x[0], t.y[0], t.x[1], t.y[1], gden, gx[0], gy[0], gx[1], gy[1]);
    }
    const float gd = fr.inside ? -gdist : gdist;
    const int e = (fr.d[0] <= fr.d[1] && fr.d[0] <= fr.d[2]) ? 0 : (fr.d[1] <= fr.d[2] ? 1 : 2);
    const int ea = e == 2 ? 1 : 0, eb = e == 0 ? 1 : 2;
    float gax = 0.f, gay = 0.f, gbx = 0.f, gby = 0.f;
    const float ax = ea == 0 ? t.x[0] : t.x[1], ay = ea == 0 ? t.y[0] : t.y[1];
    const float bx = eb == 1 ? t.x[1] : t.x[2], by = eb == 1 ? t.y[1] : t.y[2];
    mv_seg_grad(px, py, ax, ay, bx, by, gd, gax, gay, gbx, gby);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float ux = k == ea ? gax : (k == eb ? gbx : 0.f), uy = k == ea ? gay : (k == eb ? gby : 0.f);
        acc[M::NG * k] += (double)(gx[k] + ux);
        acc[M::NG * k + 1] += (double)(gy[k] + uy);
    }
}

// the slot of `key` among a pixel's K sorted keys, or -1
template <int K>
__device__ __forceinline__ int mv_find(const unsigned long long *__restrict__ s, unsigned long long key) {
    int lo = 0, hi = K;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo < K && s[lo] == key ? lo : -1;
}

template <class M>
__device__ __forceinline__ void mv_face_pixel(const MvTri &t, int f, int i, int j, int S, int64_t pix,
                                              const unsigned long long *__restrict__ slots,
                                              const float *__restrict__ part, const float C[9], double *acc) {
    const float px = mv_pix(j, S), py = mv_pix(i, S);
    MvFrag fr;
    if (!mv_fragment<M>(t, px, py, fr)) return;
    const int k = mv_find<M::K>(slots + pix * M::K, mv_key(fr.z, f));
    if (k < 0) return;                            // not kept: weight exactly 0 (NORMAL) or beyond the K nearest
    mv_frag_grad<M>(t, fr, px, py, part + (pix * M::K + k) * M::NP, C, acc);
}

template <class M>
__device__ __forceinline__ void mv_face_colours(const int64_t *__restrict__ faces, const float *__restrict__ colors,
                                                int f, float C[9]) {
#pragma unroll
    for (int k = 0; k < 9; ++k) C[k] = 0.f;
    if constexpr (M::NP == 6) {
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) C[3 * k + ch] = colors[3 * faces[3 * (int64_t)f + k] + ch];
    }
}

// one thread per face looping over the views: the corner gradients of (face, view) -> fgrad[a][f][corner][NG]
template <class M>
__global__ void k_mr_face_small(const int64_t *__restrict__ faces, int F, int V, int A, int S,
                                const float4 *__restrict__ vrec, const float *__restrict__ colors,
                                const unsigned long long *__restrict__ slots, const float *__restrict__ part,
                                double *__restrict__ fgrad, int2 *__restrict__ big, int32_t *__restrict__ nbig) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    for (int a = 0; a < A; ++a) {
        MvTri t;
        if (!mv_setup<M>(faces, vrec + (int64_t)a * V, f, V, S, t)) continue;
        const int nj = t.j1 - t.j0 + 1, ni = t.i1 - t.i0 + 1;
        if (nj * ni > M::SMALL) {
            big[atomicAdd(nbig, 1)] = make_int2(f, a);
            continue;
        }
        float C[9];
        mv_face_colours<M>(faces, colors, f, C);
        double acc[3 * M::NG];
#pragma unroll
        for (int k = 0; k < 3 * M::NG; ++k) acc[k] = 0.0;
        const int64_t base = (int64_t)a * S * S;
        for (int i = t.i0; i <= t.i1; ++i)
            for (int j = t.j0; j <= t.j1; ++j)
                mv_face_pixel<M>(t, f, i, j, S, base + (int64_t)i * S + j, slots, part, C, acc);
        double *o = fgrad + ((int64_t)a * F + f) * 3 * M::NG;
#pragma unroll
        for (int k = 0; k < 3 * M::NG; ++k) o[k] = acc[k];
    }
}

// one block per listed (face, view): threads stride over the box, then a fixed-order tree reduction
template <class M>
__global__ void __launch_bounds__(256, 1) k_mr_face_big(const int64_t *__restrict__ faces, int F, int V, int S,
                                                     const float4 *__restrict__ vrec, const float *__restrict__ colors,
                                                     const unsigned long long *__restrict__ slots,
                                                     const float *__restrict__ part, double *__restrict__ fgrad,
                                                     const int2 *__restrict__ big, const int32_t *__restrict__ nbig) {
    constexpr int NG3 = 3 * M::NG;
    __shared__ double red[NG3][256];
    const int n = *nbig;
    for (int b = blockIdx.x; b < n; b += gridDim.x) {
        const int f = big[b].x, a = big[b].y;
        MvTri t;
        mv_setup<M>(faces, vrec + (int64_t)a * V, f, V, S, t);       // succeeded when listed
        float C[9];
        mv_face_colours<M>(faces, colors, f, C);
        double acc[NG3];
#pragma unroll
        for (int k = 0; k < NG3; ++k) acc[k] = 0.0;
        const int nj = t.j1 - t.j0 + 1;
        const int np = nj * (t.i1 - t.i0 + 1);
        const int64_t base = (int64_t)a * S * S;
        for (int p = threadIdx.x; p < np; p += blockDim.x) {
            const int i = t.i0 + p / nj, j = t.j0 + p % nj;
            mv_face_pixel<M>(t, f, i, j, S, base + (int64_t)i * S + j, slots, part, C, acc);
        }
#pragma unroll
        for (int k = 0; k < NG3; ++k) red[k][threadIdx.x] = acc[k];
        __syncthreads();
        for (int h = 128; h > 0; h >>= 1) {
            if ((int)threadIdx.x < h)
#pragma unroll
                for (int k = 0; k < NG3; ++k) red[k][threadIdx.x] = red[k][threadIdx.x] + red[k][threadIdx.x + h];
            __syncthreads();
        }
        if (threadIdx.x < NG3) fgrad[((int64_t)a * F + f) * NG3 + threadIdx.x] = red[threadIdx.x][0];
        __syncthreads();
    }
}

// one thread per vertex: its corners in sorted (pass, face) order, view after view, M^T in fp64
template <class M>
__global__ void k_mr_vertex(const int64_t *__restrict__ faces, int F, int V, int A, const float *__restrict__ mats,
                            const int32_t *__restrict__ off, int32_t *__restrict__ keys,
                            const double *__restrict__ fgrad, float *__restrict__ gverts, float *__restrict__ gcolors) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    int32_t *kl = keys + off[v];
    const int n = off[v + 1] - off[v];
    heap_sort_i32(kl, n);
    double gv[3] = {0.0, 0.0, 0.0}, gc[3] = {0.0, 0.0, 0.0};
    for (int a = 0; a < A; ++a) {
        double s[M::NG];
#pragma unroll
        for (int q = 0; q < M::NG; ++q) s[q] = 0.0;
        for (int i = 0; i < n; ++i) {
            const int pass = kl[i] / F, f = kl[i] % F;
            const int c = pass == 0 ? 1 : (pass == 1 ? 2 : 0);
            const double *g = fgrad + (((int64_t)a * F + f) * 3 + c) * M::NG;
#pragma unroll
            for (int q = 0; q < M::NG; ++q) s[q] += g[q];
        }
        const float *m = mats + 12 * a;
        if constexpr (M::NG == 6) {
#pragma unroll
            for (int r = 0; r < 3; ++r)
                gv[r] += ((double)m[r] * s[0] + (double)m[4 + r] * s[1]) + (double)m[8 + r] * s[2];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) gc[ch] += s[3 + ch];
        } else {
#pragma unroll
            for (int r = 0; r < 3; ++r) gv[r] += (double)m[r] * s[0] + (double)m[4 + r] * s[1];
        }
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) gverts[3 * (int64_t)v + r] = (float)gv[r];
    if (gcolors)
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) gcolors[3 * (int64_t)v + ch] = (float)gc[ch];
}

struct MvWs {
    float *mats;
    float4 *vrec;
    unsigned long long *near, *slots;
    int2 *big;
    int32_t *nbig;
    float *part;                     // backward: per-slot partials
    double *fgrad;                   // backward: per (view, face, corner) gradients
    AnWs an;                         // backward: per-vertex corner lists
};

// slots == false: the caller keeps them (icon_mesh_render_*'s state); bwd: the backward's buffers too
static size_t mv_carve(void *ws, int V, int F, int S, int A, int K, bool slots, int NP, int NG, bool bwd, MvWs *o) {
    Carver c(ws);
    MvWs w{};
    const size_t npix = (size_t)A * S * S;
    w.mats = c.take<float>(12 * (size_t)A);
    w.vrec = c.take<float4>((size_t)A * V);
    w.near = c.take<unsigned long long>(npix);
    if (slots) w.slots = c.take<unsigned long long>(npix * K);
    w.big = c.take<int2>((size_t)A * F);
    w.nbig = c.take<int32_t>(1);
    if (bwd) {
        w.part = c.take<float>(npix * K * NP);
        w.fgrad = c.take<double>((size_t)A * F * 3 * NG);
        void *an = c.take<char>(an_carve(nullptr, V, F, nullptr));
        if (ws) an_carve(an, V, F, &w.an);
    }
    if (o) *o = w;
    return c.total();
}

// project, then the two raster passes: each pixel's slots hold its kept keys, sorted
template <class M>
static int mv_raster(const float *verts, int V, const int64_t *faces, int F, const float *h_view_mats, int A, int S,
                     const MvWs &w, cudaStream_t stream) {
    const int64_t npix = (int64_t)A * S * S;
    ICON_CUDA(cudaMemcpyAsync(w.mats, h_view_mats, sizeof(float) * 12 * (size_t)A, cudaMemcpyHostToDevice, stream));
    if (M::CUT) ICON_CUDA(cudaMemsetAsync(w.near, 0xff, sizeof(unsigned long long) * (size_t)npix, stream));
    ICON_CUDA(cudaMemsetAsync(w.slots, 0xff, sizeof(unsigned long long) * (size_t)npix * M::K, stream));
    ICON_CUDA(cudaMemsetAsync(w.nbig, 0, sizeof(int32_t), stream));
    k_mv_vertex<<<dim3((unsigned)((V + 255) / 256), (unsigned)A), 256, 0, stream>>>(verts, V, w.mats, w.vrec);
    ICON_LAUNCHED();
    const unsigned fb = (unsigned)((F + 127) / 128);
    k_mv_small<1, M><<<fb, 128, 0, stream>>>(faces, F, V, A, S, w.vrec, w.near, w.slots, w.big, w.nbig);
    ICON_LAUNCHED();
    if (M::CUT) {
        k_mv_big<1, M><<<MV_BIG_BLOCKS, 256, 0, stream>>>(faces, V, S, w.vrec, w.near, w.slots, w.big, w.nbig);
        ICON_LAUNCHED();
    }
    k_mv_small<2, M><<<fb, 128, 0, stream>>>(faces, F, V, A, S, w.vrec, w.near, w.slots, w.big, w.nbig);
    ICON_LAUNCHED();
    k_mv_big<2, M><<<MV_BIG_BLOCKS, 256, 0, stream>>>(faces, V, S, w.vrec, w.near, w.slots, w.big, w.nbig);
    ICON_LAUNCHED();
    return ICON_OK;
}

template <class M>
static int mr_backward(const float *verts, const float *colors, int V, const int64_t *faces, int F,
                       const float *h_view_mats, int A, int S, const float *gout, const unsigned long long *slots,
                       float *gverts, float *gcolors, const MvWs &w, cudaStream_t stream) {
    const int64_t npix = (int64_t)A * S * S;
    ICON_CUDA(cudaMemcpyAsync(w.mats, h_view_mats, sizeof(float) * 12 * (size_t)A, cudaMemcpyHostToDevice, stream));
    ICON_CUDA(cudaMemsetAsync(w.nbig, 0, sizeof(int32_t), stream));
    ICON_CUDA(cudaMemsetAsync(w.fgrad, 0, sizeof(double) * (size_t)A * F * 3 * M::NG, stream));
    ICON_CUDA(cudaMemsetAsync(w.an.cnt, 0, sizeof(int32_t) * ((size_t)V + 1), stream));
    ICON_CUDA(cudaMemsetAsync(w.an.cursor, 0, sizeof(int32_t) * (size_t)V, stream));
    k_mv_vertex<<<dim3((unsigned)((V + 255) / 256), (unsigned)A), 256, 0, stream>>>(verts, V, w.mats, w.vrec);
    ICON_LAUNCHED();
    const unsigned pb = (unsigned)((npix + 255) / 256);
    if constexpr (M::NP == 6)
        k_mr_pixel_normal<<<pb, 256, 0, stream>>>(faces, V, A, S, w.vrec, colors, slots, gout, w.part);
    else
        k_mr_pixel_silhouette<<<pb, 256, 0, stream>>>(faces, V, A, S, w.vrec, slots, gout, w.part);
    ICON_LAUNCHED();
    const unsigned fb = (unsigned)((F + 127) / 128);
    k_mr_face_small<M><<<fb, 128, 0, stream>>>(faces, F, V, A, S, w.vrec, colors, slots, w.part, w.fgrad, w.big,
                                                 w.nbig);
    ICON_LAUNCHED();
    k_mr_face_big<M><<<MV_BIG_BLOCKS, 256, 0, stream>>>(faces, F, V, S, w.vrec, colors, slots, w.part, w.fgrad, w.big,
                                                         w.nbig);
    ICON_LAUNCHED();
    const unsigned fb2 = (unsigned)((F + 255) / 256), vb = (unsigned)((V + 255) / 256);
    k_an_count<<<fb2, 256, 0, stream>>>(faces, F, V, w.an.cnt);
    ICON_LAUNCHED();
    int rc = scan_exclusive_i32(w.an.cnt, w.an.off, (int64_t)V + 1, nullptr, w.an.scan_ws, stream);
    if (rc) return rc;
    k_an_fill<<<fb2, 256, 0, stream>>>(faces, F, V, w.an.off, w.an.cursor, w.an.keys);
    ICON_LAUNCHED();
    k_mr_vertex<M><<<vb, 256, 0, stream>>>(faces, F, V, A, w.mats, w.an.off, w.an.keys, w.fgrad, gverts, gcolors);
    ICON_LAUNCHED();
    return ICON_OK;
}

}  // namespace icon

extern "C" size_t icon_area_vertex_normals_workspace_bytes(int V, int F) {
    if (V <= 0 || F <= 0) return 0;
    return icon::an_carve(nullptr, V, F, nullptr);
}

extern "C" int icon_area_vertex_normals(const float *verts, int V, const int64_t *faces, int F, float *out, void *ws,
                                        size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(verts && faces && out && ws, "icon_area_vertex_normals: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && F <= (INT32_MAX - 2) / 3, "icon_area_vertex_normals: bad sizes V=%d F=%d", V, F);
    ICON_CHECK_ARG(ws_bytes >= icon_area_vertex_normals_workspace_bytes(V, F),
                   "icon_area_vertex_normals: workspace too small");
    AnWs w;
    an_carve(ws, V, F, &w);
    ICON_CUDA(cudaMemsetAsync(w.cnt, 0, sizeof(int32_t) * ((size_t)V + 1), stream));
    ICON_CUDA(cudaMemsetAsync(w.cursor, 0, sizeof(int32_t) * (size_t)V, stream));
    const unsigned fb = (unsigned)((F + 255) / 256), vb = (unsigned)((V + 255) / 256);
    k_an_count<<<fb, 256, 0, stream>>>(faces, F, V, w.cnt);
    ICON_LAUNCHED();
    int rc = scan_exclusive_i32(w.cnt, w.off, (int64_t)V + 1, nullptr, w.scan_ws, stream);
    if (rc) return rc;
    k_an_fill<<<fb, 256, 0, stream>>>(faces, F, V, w.off, w.cursor, w.keys);
    ICON_LAUNCHED();
    k_an_sum<<<vb, 256, 0, stream>>>(verts, faces, F, w.off, w.keys, V, out);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" size_t icon_area_vertex_normals_backward_workspace_bytes(int V, int F) {
    if (V <= 0 || F <= 0) return 0;
    icon::Carver c(nullptr);
    c.take<char>(icon::an_carve(nullptr, V, F, nullptr));
    c.take<double>(3 * (size_t)V);
    return c.total();
}

extern "C" int icon_area_vertex_normals_backward(const float *verts, int V, const int64_t *faces, int F,
                                                 const float *grad_normals, float *grad_verts, void *ws,
                                                 size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(verts && faces && grad_normals && grad_verts && ws, "icon_area_vertex_normals_backward: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && F <= (INT32_MAX - 2) / 3, "icon_area_vertex_normals_backward: bad sizes V=%d F=%d",
                   V, F);
    ICON_CHECK_ARG(ws_bytes >= icon_area_vertex_normals_backward_workspace_bytes(V, F),
                   "icon_area_vertex_normals_backward: workspace too small");
    Carver c(ws);
    AnWs w;
    an_carve(c.take<char>(an_carve(nullptr, V, F, nullptr)), V, F, &w);
    double *gs = c.take<double>(3 * (size_t)V);
    ICON_CUDA(cudaMemsetAsync(w.cnt, 0, sizeof(int32_t) * ((size_t)V + 1), stream));
    ICON_CUDA(cudaMemsetAsync(w.cursor, 0, sizeof(int32_t) * (size_t)V, stream));
    const unsigned fb = (unsigned)((F + 255) / 256), vb = (unsigned)((V + 255) / 256);
    k_an_count<<<fb, 256, 0, stream>>>(faces, F, V, w.cnt);
    ICON_LAUNCHED();
    int rc = scan_exclusive_i32(w.cnt, w.off, (int64_t)V + 1, nullptr, w.scan_ws, stream);
    if (rc) return rc;
    k_an_fill<<<fb, 256, 0, stream>>>(faces, F, V, w.off, w.cursor, w.keys);
    ICON_LAUNCHED();
    k_an_grad_s<<<vb, 256, 0, stream>>>(verts, faces, F, w.off, w.keys, V, grad_normals, gs);
    ICON_LAUNCHED();
    k_an_grad_v<<<vb, 256, 0, stream>>>(verts, faces, F, w.off, w.keys, V, gs, grad_verts);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" size_t icon_mesh_views_workspace_bytes(int V, int F, int S, int A) {
    if (V <= 0 || F <= 0 || S <= 0 || A <= 0) return 0;
    return icon::mv_carve(nullptr, V, F, S, A, icon::MV_K, true, 0, 0, false, nullptr);
}

extern "C" int icon_mesh_views(const float *verts, const float *colors, int V, const int64_t *faces, int F,
                               const float *h_view_mats, int A, int S, uint8_t *out, int32_t *face_out, float *rgb_out,
                               void *ws, size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(verts && colors && faces && h_view_mats && out && ws, "icon_mesh_views: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && A > 0 && S > 0 && S <= 4096 && (int64_t)A * F <= INT32_MAX,
                   "icon_mesh_views: bad sizes V=%d F=%d A=%d S=%d", V, F, A, S);
    ICON_CHECK_ARG(ws_bytes >= icon_mesh_views_workspace_bytes(V, F, S, A), "icon_mesh_views: workspace too small");
    MvWs w;
    mv_carve(ws, V, F, S, A, MV_K, true, 0, 0, false, &w);
    const int64_t npix = (int64_t)A * S * S;
    int rc = mv_raster<MvNormal>(verts, V, faces, F, h_view_mats, A, S, w, stream);
    if (rc) return rc;
    k_mv_shade<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(faces, V, A, S, w.vrec, colors, w.slots, out,
                                                                     face_out, rgb_out);
    ICON_LAUNCHED();
    return ICON_OK;
}

// ---------------------------------------------------------------- differentiable renders of the fitting loops

static bool mr_mode(int mode, int &K, int &NP, int &NG) {
    if (mode == ICON_RENDER_NORMAL) { K = icon::MvNormal::K; NP = icon::MvNormal::NP; NG = icon::MvNormal::NG; return true; }
    if (mode == ICON_RENDER_SILHOUETTE) {
        K = icon::MvSilhouette::K; NP = icon::MvSilhouette::NP; NG = icon::MvSilhouette::NG;
        return true;
    }
    return false;
}

extern "C" size_t icon_mesh_render_state_bytes(int mode, int S, int A) {
    int K, NP, NG;
    if (!mr_mode(mode, K, NP, NG) || S <= 0 || A <= 0) return 0;
    return sizeof(unsigned long long) * (size_t)A * S * S * K;
}

extern "C" size_t icon_mesh_render_workspace_bytes(int mode, int backward, int V, int F, int S, int A) {
    int K, NP, NG;
    if (!mr_mode(mode, K, NP, NG) || V <= 0 || F <= 0 || S <= 0 || A <= 0) return 0;
    return icon::mv_carve(nullptr, V, F, S, A, K, false, NP, NG, backward != 0, nullptr);
}

extern "C" int icon_mesh_render_forward(int mode, const float *verts, const float *colors, int V, const int64_t *faces,
                                        int F, const float *h_view_mats, int A, int S, float *out, void *state,
                                        size_t state_bytes, void *ws, size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    int K, NP, NG;
    ICON_CHECK_ARG(mr_mode(mode, K, NP, NG), "icon_mesh_render_forward: bad mode %d", mode);
    ICON_CHECK_ARG(verts && faces && h_view_mats && out && state && ws && (colors || mode != ICON_RENDER_NORMAL),
                   "icon_mesh_render_forward: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && A > 0 && S > 0 && S <= 4096 && (int64_t)A * F <= INT32_MAX,
                   "icon_mesh_render_forward: bad sizes V=%d F=%d A=%d S=%d", V, F, A, S);
    ICON_CHECK_ARG(state_bytes >= icon_mesh_render_state_bytes(mode, S, A), "icon_mesh_render_forward: state too small");
    ICON_CHECK_ARG(ws_bytes >= icon_mesh_render_workspace_bytes(mode, 0, V, F, S, A),
                   "icon_mesh_render_forward: workspace too small");
    MvWs w;
    mv_carve(ws, V, F, S, A, K, false, NP, NG, false, &w);
    w.slots = (unsigned long long *)state;
    const int64_t npix = (int64_t)A * S * S;
    const unsigned pb = (unsigned)((npix + 255) / 256);
    if (mode == ICON_RENDER_NORMAL) {
        int rc = mv_raster<MvNormal>(verts, V, faces, F, h_view_mats, A, S, w, stream);
        if (rc) return rc;
        k_mv_shade<<<pb, 256, 0, stream>>>(faces, V, A, S, w.vrec, colors, w.slots, nullptr, nullptr, out);
    } else {
        int rc = mv_raster<MvSilhouette>(verts, V, faces, F, h_view_mats, A, S, w, stream);
        if (rc) return rc;
        k_mv_silhouette<<<pb, 256, 0, stream>>>(faces, V, A, S, w.vrec, w.slots, out);
    }
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_mesh_render_backward(int mode, const float *verts, const float *colors, int V,
                                         const int64_t *faces, int F, const float *h_view_mats, int A, int S,
                                         const float *grad_out, const void *state, size_t state_bytes,
                                         float *grad_verts, float *grad_colors, void *ws, size_t ws_bytes,
                                         icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    int K, NP, NG;
    ICON_CHECK_ARG(mr_mode(mode, K, NP, NG), "icon_mesh_render_backward: bad mode %d", mode);
    ICON_CHECK_ARG(verts && faces && h_view_mats && grad_out && state && grad_verts && ws &&
                       (mode != ICON_RENDER_NORMAL || colors),
                   "icon_mesh_render_backward: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && A > 0 && S > 0 && S <= 4096 && (int64_t)A * F <= INT32_MAX &&
                       F <= (INT32_MAX - 2) / 3,
                   "icon_mesh_render_backward: bad sizes V=%d F=%d A=%d S=%d", V, F, A, S);
    ICON_CHECK_ARG(state_bytes >= icon_mesh_render_state_bytes(mode, S, A), "icon_mesh_render_backward: state too small");
    ICON_CHECK_ARG(ws_bytes >= icon_mesh_render_workspace_bytes(mode, 1, V, F, S, A),
                   "icon_mesh_render_backward: workspace too small");
    MvWs w;
    mv_carve(ws, V, F, S, A, K, false, NP, NG, true, &w);
    const unsigned long long *slots = (const unsigned long long *)state;
    if (mode == ICON_RENDER_NORMAL)
        return mr_backward<MvNormal>(verts, colors, V, faces, F, h_view_mats, A, S, grad_out, slots, grad_verts,
                                     grad_colors, w, stream);
    return mr_backward<MvSilhouette>(verts, nullptr, V, faces, F, h_view_mats, A, S, grad_out, slots, grad_verts,
                                     nullptr, w, stream);
}
