// Vertex normals of a triangle mesh, two rules.  Both sum each vertex's contributions over its vertex_corners list
// (common.cu: the corners 3 f + k of the vertex, ascending) in a fixed order: no float atomics, bitwise reproducible.
// Faces with an index outside [0, V) are not listed and contribute nothing.
//
// PARITY UNPINNED: trimesh and pytorch3d are not dependencies of this project.  The rules below are this file's
// contract, restated operation for operation by the oracles named with them (hence -fmad=false for this file).
//
// Angle-weighted (icon_vertex_normals): trimesh 3.9.35's `vertex_normals`, restated by oracle/normal_render.py; fp64,
// rounded to fp32 at the end:
//   unit(v) = v / |v| if |v| > 1e-13 (trimesh's tol.zero) else 0, |v| = sqrt((x x + y y) + z z);
//   face normal n_f = unit((b - a) x (c - a)); corner angles a0 = acos(clamp(u.v)), a1 = acos(clamp((-u).w)),
//   a2 = (pi - a0) - a1 with u = unit(b - a), v = unit(c - a), w = unit(c - b);
//   vertex normal = unit(sum of a_k n_f over its corners, added in corner order 3 f + k).
//   Unreferenced vertices and degenerate faces get / contribute zero.
//
// Area-weighted (icon_area_vertex_normals, and area_vertex_normals for the SMPL body): pytorch3d's
// verts_normals_packed as oracle.query.vertex_normals restates it; fp32:
//   three passes (corner 1, 2, 0), each in face order, add n = (p1 - p0) x (p2 - p0) to vertex p0, where p1, p2 are
//   the next two corners of the face; then n / max(sqrt((x x + y y) + z z), 1e-6).  Pass p of a vertex reads the
//   corners 3 f + (p + 1) % 3 of its list, in list order, so each vertex adds its own contributions in exactly the
//   order of the sequential passes.
//   Backward (icon_area_vertex_normals_backward; restated by oracle/mesh_priors.py with float64 autograd): the
//   gradient of F.normalize(s, eps = 1e-6) with torch's semantics, from the fp32 s of the forward, in fp64:
//   (g - n (n.g)) / |s| with n = s / |s| when the fp32 norm is >= 1e-6, else g / 1e-6 (clamp_min passes g there);
//   then through each corner product n = u x w (u = p1 - p0, w = p2 - p0): p1 += w x G, p2 += G x u, p0 -= both.
//   Each vertex sums its contributions over the same three passes in fp64 (its own position in each listed face,
//   all three products of that face) and rounds once.
#include "common.cuh"
#include "geom.cuh"

namespace icon {

// a vertex_corners list and its builder's scratch
struct Corners {
    int32_t *off, *list;
    void *ws;
};

static Corners corners_take(Carver &c, int V, int F) {
    Corners k;
    k.off = c.take<int32_t>((size_t)V + 1);
    k.list = c.take<int32_t>(3 * (size_t)F);
    k.ws = c.take<char>(vertex_corners_ws_bytes(V, F));
    return k;
}

// ---------------------------------------------------------------- angle-weighted (trimesh)

constexpr double VN_TOL_ZERO = 1e-13;

__device__ __forceinline__ double3 d3_sub(double3 a, double3 b) { return make_double3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double d3_dot(double3 a, double3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__device__ __forceinline__ double3 d3_unit(double3 v) {
    const double n = sqrt(d3_dot(v, v));
    if (!(n > VN_TOL_ZERO)) return make_double3(0.0, 0.0, 0.0);
    return make_double3(v.x / n, v.y / n, v.z / n);
}
__device__ __forceinline__ double clamp_acos(double c) { return acos(fmin(fmax(c, -1.0), 1.0)); }

// per face: unit normal and the three corner angles (a face with a bad index is not listed: left unwritten)
__global__ void k_vn_face(const double *__restrict__ verts, const int64_t *__restrict__ faces, int F, int V,
                          double *__restrict__ fdata) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    int id[3];
    if (f >= F || !face_ids(faces, f, V, id)) return;
    double3 p[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int64_t i = id[k];
        p[k] = make_double3(verts[3 * i], verts[3 * i + 1], verts[3 * i + 2]);
    }
    const double3 e1 = d3_sub(p[1], p[0]), e2 = d3_sub(p[2], p[0]);
    const double3 n = d3_unit(make_double3(e1.y * e2.z - e1.z * e2.y, e1.z * e2.x - e1.x * e2.z,
                                           e1.x * e2.y - e1.y * e2.x));
    const double3 u = d3_unit(e1), v = d3_unit(e2), w = d3_unit(d3_sub(p[2], p[1]));
    const double a0 = clamp_acos(d3_dot(u, v));
    const double a1 = clamp_acos(d3_dot(make_double3(-u.x, -u.y, -u.z), w));
    double *o = fdata + 6 * (int64_t)f;
    o[0] = n.x; o[1] = n.y; o[2] = n.z;
    o[3] = a0; o[4] = a1; o[5] = (3.141592653589793 - a0) - a1;
}

// per vertex: sum a_k n_f in corner order, unit
__global__ void k_vn_sum(const int32_t *__restrict__ off, const int32_t *__restrict__ corners,
                         const double *__restrict__ fdata, int V, float *__restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    double3 s = make_double3(0.0, 0.0, 0.0);
    for (int i = off[v]; i < off[v + 1]; ++i) {
        const int c = corners[i];
        const double *fd = fdata + 6 * (int64_t)(c / 3);
        const double w = fd[3 + c % 3];
        s.x = s.x + w * fd[0]; s.y = s.y + w * fd[1]; s.z = s.z + w * fd[2];
    }
    s = d3_unit(s);
    out[3 * (int64_t)v] = (float)s.x; out[3 * (int64_t)v + 1] = (float)s.y; out[3 * (int64_t)v + 2] = (float)s.z;
}

static size_t vn_carve(void *ws, int V, int F, Corners *k, double **fdata) {
    Carver c(ws);
    const Corners kk = corners_take(c, V, F);
    double *fd = c.take<double>(6 * (size_t)F);
    if (k) *k = kk, *fdata = fd;
    return c.total();
}

// ---------------------------------------------------------------- area-weighted (pytorch3d)

__device__ __forceinline__ V3 an_vert(const float *verts, int64_t i) {
    return mk3(verts[3 * i], verts[3 * i + 1], verts[3 * i + 2]);
}

// the fp32 sum s of one vertex's corner products, in pass order
__device__ __forceinline__ V3 an_sum(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                                     const int32_t *corners, int n) {
    V3 s = mk3(0.f, 0.f, 0.f);
    for_each_pass_corner(corners, n, [&](int f, int c) {
        const int64_t *fc = faces + 3 * (int64_t)f;
        const V3 p0 = an_vert(verts, fc[c]);
        const V3 t = cross3(sub3(an_vert(verts, fc[(c + 1) % 3]), p0), sub3(an_vert(verts, fc[(c + 2) % 3]), p0));
        s.x = s.x + t.x; s.y = s.y + t.y; s.z = s.z + t.z;
    });
    return s;
}

__global__ void k_an_sum(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                         const int32_t *__restrict__ off, const int32_t *__restrict__ corners, int V,
                         float *__restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const V3 s = an_sum(verts, faces, corners + off[v], off[v + 1] - off[v]);
    float nrm = sqrtf((s.x * s.x + s.y * s.y) + s.z * s.z);
    if (nrm < 1e-6f) nrm = 1e-6f;
    out[3 * (int64_t)v] = s.x / nrm; out[3 * (int64_t)v + 1] = s.y / nrm; out[3 * (int64_t)v + 2] = s.z / nrm;
}

// backward, 1: s as k_an_sum forms it, then the normalize gradient (fp64) into gs
__global__ void k_an_grad_s(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                            const int32_t *__restrict__ off, const int32_t *__restrict__ corners, int V,
                            const float *__restrict__ gn, double *__restrict__ gs) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const V3 sf = an_sum(verts, faces, corners + off[v], off[v + 1] - off[v]);
    const double s[3] = {sf.x, sf.y, sf.z};
    const double g[3] = {gn[3 * (int64_t)v], gn[3 * (int64_t)v + 1], gn[3 * (int64_t)v + 2]};
    const double len = sqrt((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2]);
    const float nrm = sqrtf((sf.x * sf.x + sf.y * sf.y) + sf.z * sf.z);
    if (nrm < 1e-6f) {                                    // the clamp: g / eps
#pragma unroll
        for (int k = 0; k < 3; ++k) gs[3 * (int64_t)v + k] = g[k] / 1e-6;
        return;
    }
    const double d = ((s[0] * g[0] + s[1] * g[1]) + s[2] * g[2]) / len;
#pragma unroll
    for (int k = 0; k < 3; ++k) gs[3 * (int64_t)v + k] = (g[k] - (s[k] / len) * d) / len;
}

// backward, 2: per vertex, in pass order, the derivative of each listed face's three corner products
// n_k = (p_{k+1} - p_k) x (p_{k+2} - p_k) with respect to the vertex's own position c in the face
__global__ void k_an_grad_v(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                            const int32_t *__restrict__ off, const int32_t *__restrict__ corners, int V,
                            const double *__restrict__ gs, float *__restrict__ gv) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    double acc[3] = {0.0, 0.0, 0.0};
    for_each_pass_corner(corners + off[v], off[v + 1] - off[v], [&](int f, int c) {
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
    });
#pragma unroll
    for (int q = 0; q < 3; ++q) gv[3 * (int64_t)v + q] = (float)acc[q];
}

size_t area_vertex_normals_ws_bytes(int V, int F) {
    Carver c(nullptr);
    corners_take(c, V, F);
    return c.total();
}

int area_vertex_normals(const float *verts, int V, const int64_t *faces, int F, float *out, void *ws,
                        cudaStream_t stream) {
    Carver c(ws);
    const Corners k = corners_take(c, V, F);
    if (int rc = vertex_corners(faces, F, V, k.off, k.list, k.ws, stream)) return rc;
    k_an_sum<<<(unsigned)((V + 255) / 256), 256, 0, stream>>>(verts, faces, k.off, k.list, V, out);
    ICON_LAUNCHED();
    return ICON_OK;
}

static size_t an_backward_carve(void *ws, int V, int F, Corners *k, double **gs) {
    Carver c(ws);
    const Corners kk = corners_take(c, V, F);
    double *g = c.take<double>(3 * (size_t)V);
    if (k) *k = kk, *gs = g;
    return c.total();
}

}  // namespace icon

// ---------------------------------------------------------------- C ABI

extern "C" size_t icon_vertex_normals_workspace_bytes(int V, int F) {
    if (V <= 0 || F <= 0) return 0;
    return icon::vn_carve(nullptr, V, F, nullptr, nullptr);
}

extern "C" int icon_vertex_normals(const double *verts, int V, const int64_t *faces, int F, float *out, void *ws,
                                   size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(verts && faces && out && ws, "icon_vertex_normals: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && F <= (INT32_MAX - 2) / 3, "icon_vertex_normals: bad sizes V=%d F=%d", V, F);
    ICON_CHECK_ARG(ws_bytes >= icon_vertex_normals_workspace_bytes(V, F), "icon_vertex_normals: workspace too small");
    Corners k;
    double *fdata;
    vn_carve(ws, V, F, &k, &fdata);
    if (int rc = vertex_corners(faces, F, V, k.off, k.list, k.ws, stream)) return rc;
    k_vn_face<<<(unsigned)((F + 255) / 256), 256, 0, stream>>>(verts, faces, F, V, fdata);
    ICON_LAUNCHED();
    k_vn_sum<<<(unsigned)((V + 255) / 256), 256, 0, stream>>>(k.off, k.list, fdata, V, out);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" size_t icon_area_vertex_normals_workspace_bytes(int V, int F) {
    if (V <= 0 || F <= 0) return 0;
    return icon::area_vertex_normals_ws_bytes(V, F);
}

extern "C" int icon_area_vertex_normals(const float *verts, int V, const int64_t *faces, int F, float *out, void *ws,
                                        size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    ICON_CHECK_ARG(verts && faces && out && ws, "icon_area_vertex_normals: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && F <= (INT32_MAX - 2) / 3, "icon_area_vertex_normals: bad sizes V=%d F=%d", V, F);
    ICON_CHECK_ARG(ws_bytes >= icon_area_vertex_normals_workspace_bytes(V, F),
                   "icon_area_vertex_normals: workspace too small");
    return area_vertex_normals(verts, V, faces, F, out, ws, (cudaStream_t)stream_);
}

extern "C" size_t icon_area_vertex_normals_backward_workspace_bytes(int V, int F) {
    if (V <= 0 || F <= 0) return 0;
    return icon::an_backward_carve(nullptr, V, F, nullptr, nullptr);
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
    Corners k;
    double *gs;
    an_backward_carve(ws, V, F, &k, &gs);
    if (int rc = vertex_corners(faces, F, V, k.off, k.list, k.ws, stream)) return rc;
    const unsigned vb = (unsigned)((V + 255) / 256);
    k_an_grad_s<<<vb, 256, 0, stream>>>(verts, faces, k.off, k.list, V, grad_normals, gs);
    ICON_LAUNCHED();
    k_an_grad_v<<<vb, 256, 0, stream>>>(verts, faces, k.off, k.list, V, gs, grad_verts);
    ICON_LAUNCHED();
    return ICON_OK;
}
