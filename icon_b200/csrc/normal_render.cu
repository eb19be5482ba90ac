// Normal images of the benchmark's evaluation: replaces lib.renderer.gl.normal_render.NormalRender as
// Evaluator._render_normal drives it (lib/dataset/Evaluator.py:58-73; shaders lib/renderer/gl/data/normal.{vs,fs}),
// and trimesh's `vertex_normals` it draws by default.  The reference needs an OpenGL context; this does not.
//
// PARITY UNPINNED: the GL rasteriser and trimesh are not dependencies of this project.  The rules below are this file's contract,
// restated operation for operation by oracle/normal_render.py, and the images are compared bit for bit (hence
// -fmad=false for this file).
//
// The default vertex normals (trimesh's `vertex_normals`, icon_vertex_normals) are normals.cu's angle-weighted rule.
//
// Normal image (icon_normal_render), NormalRender(W, H) with ModelMat M (3x4 rows, fp32, passed on the host) and the
// projection diag(1, 1, -1, 1) (orthographic), all fp32 in the order written:
//   p' = M p (each row ((m0 x + m1 y) + m2 z) + m3); x_ndc = p'.x, y_ndc = p'.y, z_ndc = -p'.z;
//   viewport x_w = x_ndc (W/2) + W/2, y_w likewise with H (y up, window row 0 at the bottom);
//   snapped X = rint(256 x_w), Y = rint(256 y_w) (1/256 pixel).  EXACT RANGE: |x_w|, |y_w| <= 65536 pixels, so every
//   edge function below is an exact int64 (< 2^51).  A face with a vertex outside that range, a non-finite vertex or
//   an index outside [0, V) is not drawn (clipped whole; no wrap-around).
//   Coverage: pixel (px, py) is sampled at its centre (256 px + 128, 256 py + 128).  Both windings are drawn: a face
//   of negative snapped area is traversed with corners 1 and 2 swapped, a face of zero snapped area is drawn nowhere.
//   With the face counter-clockwise, edge a->b has E = (Xb - Xa)(Py - Ya) - (Yb - Ya)(Px - Xa); the pixel is covered
//   when every edge has E > 0, or E == 0 on a top-left edge (dy < 0, or dy == 0 and dx < 0; y up), so a pixel on an
//   edge shared by two faces is covered by exactly one of them.
//   Depth: l_k = float(E_k) / float(2 area) for the edge opposite ORIGINAL corner k; z_w,k = (z_ndc,k + 1) 0.5;
//   z = (l0 z_w,0 + l1 z_w,1) + l2 z_w,2.  Fragments with z outside [0, 1] are dropped (near/far clipping).  The depth
//   buffer is assumed 24-bit: q = rint(z (2^24 - 1)), cleared to 2^24 - 1 and tested with GL_LESS, so q = 2^24 - 1
//   never passes.  Nearest q wins, then the lowest face index (draw order): a 64-bit atomicMin of (q << 32 | face).
//   Colour: n = (l0 n'0 + l1 n'1) + l2 n'2 per component with n'k = M3x3 n_k (no translation); r = sqrt((n.x n.x +
//   n.y n.y) + n.z n.z); rgb = (n / r + 1) 0.5, alpha 1.  A zero interpolated normal (r == 0, which GLSL's normalize
//   leaves undefined) is written as rgb (0.5, 0.5, 0.5).
//   Output [H, W, 4] f32 in get_color's order: image row r is window row H - 1 - r; background (1, 1, 1, 0).
#include "common.cuh"

namespace icon {

constexpr unsigned long long NR_EMPTY = 0xffffffffffffffffull;
constexpr float NR_RANGE = 65536.f;          // |x_w|, |y_w| limit of the exact fixed-point path (pixels)
constexpr int NR_SMALL = 64;                 // faces whose pixel box has at most this many pixels: one thread each
constexpr int NR_BIG_BLOCKS = 1024;          // grid of the cooperative pass (one block per listed face, grid-stride)

struct NrModel {
    float m[12];
};

__device__ __forceinline__ float row3(const float *r, float x, float y, float z) { return (r[0] * x + r[1] * y) + r[2] * z; }

__global__ void k_nr_vertex(const float *__restrict__ verts, const float *__restrict__ norms, int V, NrModel M,
                            int W, int H, int4 *__restrict__ vrec, float4 *__restrict__ nrot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    const float x = verts[3 * (int64_t)i], y = verts[3 * (int64_t)i + 1], z = verts[3 * (int64_t)i + 2];
    const float px = row3(M.m, x, y, z) + M.m[3], py = row3(M.m + 4, x, y, z) + M.m[7];
    const float pz = row3(M.m + 8, x, y, z) + M.m[11];
    const float hw = (float)W * 0.5f, hh = (float)H * 0.5f;
    const float xw = px * hw + hw, yw = py * hh + hh;
    const float zw = (-pz + 1.f) * 0.5f;
    // vertex record: snapped window x, y (1/256 px), z_w (float bits), 1 = drawable
    const int ok = fabsf(xw) <= NR_RANGE && fabsf(yw) <= NR_RANGE && isfinite(zw);
    vrec[i] = make_int4(ok ? (int)rintf(xw * 256.f) : 0, ok ? (int)rintf(yw * 256.f) : 0, __float_as_int(zw), ok);
    const float nx = norms[3 * (int64_t)i], ny = norms[3 * (int64_t)i + 1], nz = norms[3 * (int64_t)i + 2];
    nrot[i] = make_float4(row3(M.m, nx, ny, nz), row3(M.m + 4, nx, ny, nz), row3(M.m + 8, nx, ny, nz), 0.f);
}

// one face, set up for coverage: internal corner order (0, 1, 2) or (0, 2, 1) so that the face is counter-clockwise
struct NrTri {
    int X[3], Y[3];      // internal order
    long long area;      // > 0
    bool swapped;
    int bx0, bx1, by0, by1;   // pixel box clamped to the viewport (empty when bx0 > bx1 or by0 > by1)
};

__device__ __forceinline__ bool tri_setup(const int64_t *__restrict__ faces, const int4 *__restrict__ vrec, int f,
                                          int V, int W, int H, NrTri &t, float zw[3]) {
    int id[3];
    if (!face_ids(faces, f, V, id)) return false;
    int4 r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        r[k] = vrec[id[k]];
        if (!r[k].w) return false;
        zw[k] = __int_as_float(r[k].z);
    }
    long long area = (long long)(r[1].x - r[0].x) * (r[2].y - r[0].y) - (long long)(r[1].y - r[0].y) * (r[2].x - r[0].x);
    if (area == 0) return false;
    t.swapped = area < 0;
    t.area = t.swapped ? -area : area;
    const int4 ra = t.swapped ? r[2] : r[1], rb = t.swapped ? r[1] : r[2];
    t.X[0] = r[0].x; t.Y[0] = r[0].y; t.X[1] = ra.x; t.Y[1] = ra.y; t.X[2] = rb.x; t.Y[2] = rb.y;
    const int xmin = min(min(t.X[0], t.X[1]), t.X[2]), xmax = max(max(t.X[0], t.X[1]), t.X[2]);
    const int ymin = min(min(t.Y[0], t.Y[1]), t.Y[2]), ymax = max(max(t.Y[0], t.Y[1]), t.Y[2]);
    // pixels whose centre 256 p + 128 lies in [min, max]; >> is a floor division
    t.bx0 = max(-((128 - xmin) >> 8), 0); t.bx1 = min((xmax - 128) >> 8, W - 1);
    t.by0 = max(-((128 - ymin) >> 8), 0); t.by1 = min((ymax - 128) >> 8, H - 1);
    return t.bx0 <= t.bx1 && t.by0 <= t.by1;
}

// edge functions at pixel (px, py), indexed by ORIGINAL corner; false when the pixel is not covered
__device__ __forceinline__ bool tri_cover(const NrTri &t, int px, int py, long long e[3]) {
    const int Px = px * 256 + 128, Py = py * 256 + 128;
    long long ei[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int a = (k + 1) % 3, b = (k + 2) % 3;
        const int dx = t.X[b] - t.X[a], dy = t.Y[b] - t.Y[a];
        ei[k] = (long long)dx * (Py - t.Y[a]) - (long long)dy * (Px - t.X[a]);
        const bool top_left = dy < 0 || (dy == 0 && dx < 0);
        if (ei[k] < 0 || (ei[k] == 0 && !top_left)) return false;
    }
    e[0] = ei[0];
    e[1] = t.swapped ? ei[2] : ei[1];
    e[2] = t.swapped ? ei[1] : ei[2];
    return true;
}

__device__ __forceinline__ void tri_weights(const NrTri &t, const long long e[3], float l[3]) {
    const float fa = __ll2float_rn(t.area);
#pragma unroll
    for (int k = 0; k < 3; ++k) l[k] = __ll2float_rn(e[k]) / fa;
}

__device__ __forceinline__ void tri_fragment(const NrTri &t, const float zw[3], int f, int px, int py, int W,
                                             unsigned long long *__restrict__ zbuf) {
    long long e[3];
    if (!tri_cover(t, px, py, e)) return;
    float l[3];
    tri_weights(t, e, l);
    const float z = (l[0] * zw[0] + l[1] * zw[1]) + l[2] * zw[2];
    if (!(z >= 0.f && z <= 1.f)) return;
    const unsigned q = (unsigned)rintf(z * 16777215.f);
    if (q >= 16777215u) return;                  // GL_LESS against the cleared depth 1.0
    atomicMin(&zbuf[(size_t)py * W + px], ((unsigned long long)q << 32) | (unsigned)f);
}

// one thread per face: small faces rasterise here, faces with a larger pixel box go to the cooperative list
__global__ void k_nr_small(const int64_t *__restrict__ faces, int F, int V, const int4 *__restrict__ vrec, int W, int H,
                           unsigned long long *__restrict__ zbuf, int32_t *__restrict__ big, int32_t *__restrict__ nbig) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    NrTri t;
    float zw[3];
    if (!tri_setup(faces, vrec, f, V, W, H, t, zw)) return;
    const int nx = t.bx1 - t.bx0 + 1, ny = t.by1 - t.by0 + 1;
    if ((long long)nx * ny > NR_SMALL) {
        big[atomicAdd(nbig, 1)] = f;
        return;
    }
    for (int py = t.by0; py <= t.by1; ++py)
        for (int px = t.bx0; px <= t.bx1; ++px) tri_fragment(t, zw, f, px, py, W, zbuf);
}

// one block per listed face (grid-stride over the list); the block's threads stride over the face's pixel box
__global__ void __launch_bounds__(256) k_nr_big(const int64_t *__restrict__ faces, int V, const int4 *__restrict__ vrec,
                                                int W, int H, unsigned long long *__restrict__ zbuf,
                                                const int32_t *__restrict__ big, const int32_t *__restrict__ nbig) {
    const int n = *nbig;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const int f = big[i];
        NrTri t;
        float zw[3];
        if (!tri_setup(faces, vrec, f, V, W, H, t, zw)) continue;
        const int nx = t.bx1 - t.bx0 + 1;
        const long long np = (long long)nx * (t.by1 - t.by0 + 1);
        for (long long p = threadIdx.x; p < np; p += blockDim.x)
            tri_fragment(t, zw, f, t.bx0 + (int)(p % nx), t.by0 + (int)(p / nx), W, zbuf);
    }
}

// one thread per pixel: the winning face's barycentrics at the pixel centre -> interpolated normal -> RGBA
__global__ void k_nr_shade(const unsigned long long *__restrict__ zbuf, const int64_t *__restrict__ faces, int V,
                           const int4 *__restrict__ vrec, const float4 *__restrict__ nrot, int W, int H,
                           float4 *__restrict__ rgba, int32_t *__restrict__ face_out) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)W * H) return;
    const int px = (int)(p % W), py = (int)(p / W);
    const int64_t o = (int64_t)(H - 1 - py) * W + px;          // get_color flips the rows
    const unsigned long long key = zbuf[p];
    float4 c = make_float4(1.f, 1.f, 1.f, 0.f);
    int f = -1;
    if (key != NR_EMPTY) {
        f = (int)(key & 0xffffffffull);
        NrTri t;
        float zw[3];
        long long e[3];
        tri_setup(faces, vrec, f, V, W, H, t, zw);                 // succeeded in the raster pass
        tri_cover(t, px, py, e);
        float l[3];
        tri_weights(t, e, l);
        float4 nk[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) nk[k] = nrot[faces[3 * (int64_t)f + k]];
        const float nx = (l[0] * nk[0].x + l[1] * nk[1].x) + l[2] * nk[2].x;
        const float ny = (l[0] * nk[0].y + l[1] * nk[1].y) + l[2] * nk[2].y;
        const float nz = (l[0] * nk[0].z + l[1] * nk[1].z) + l[2] * nk[2].z;
        const float r = sqrtf((nx * nx + ny * ny) + nz * nz);
        if (r == 0.f) {
            c = make_float4(0.5f, 0.5f, 0.5f, 1.f);
        } else {
            c = make_float4((nx / r + 1.f) * 0.5f, (ny / r + 1.f) * 0.5f, (nz / r + 1.f) * 0.5f, 1.f);
        }
    }
    rgba[o] = c;
    if (face_out) face_out[o] = f;
}

struct NrWs {
    unsigned long long *zbuf;
    int4 *vrec;
    float4 *nrot;
    int32_t *big, *nbig;
};

static size_t nr_carve(void *ws, int V, int F, int W, int H, NrWs *o) {
    Carver c(ws);
    NrWs w;
    w.zbuf = c.take<unsigned long long>((size_t)W * H);
    w.vrec = c.take<int4>((size_t)V);
    w.nrot = c.take<float4>((size_t)V);
    w.big = c.take<int32_t>((size_t)F);
    w.nbig = c.take<int32_t>(1);
    if (o) *o = w;
    return c.total();
}

}  // namespace icon

extern "C" size_t icon_normal_render_workspace_bytes(int V, int F, int width, int height) {
    if (V <= 0 || F <= 0 || width <= 0 || height <= 0) return 0;
    return icon::nr_carve(nullptr, V, F, width, height, nullptr);
}

extern "C" int icon_normal_render(const float *verts, const float *norms, int V, const int64_t *faces, int F,
                                  const float *h_model, int width, int height, float *out_rgba, int32_t *out_face,
                                  void *ws, size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(verts && norms && faces && h_model && out_rgba && ws, "icon_normal_render: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && width > 0 && height > 0 && width <= 16384 && height <= 16384,
                   "icon_normal_render: bad sizes V=%d F=%d %dx%d", V, F, width, height);
    ICON_CHECK_ARG(ws_bytes >= icon_normal_render_workspace_bytes(V, F, width, height),
                   "icon_normal_render: workspace too small");
    NrWs w;
    nr_carve(ws, V, F, width, height, &w);
    NrModel M;
    for (int k = 0; k < 12; ++k) M.m[k] = h_model[k];
    const int64_t npix = (int64_t)width * height;
    ICON_CUDA(cudaMemsetAsync(w.zbuf, 0xff, (size_t)npix * sizeof(unsigned long long), stream));
    ICON_CUDA(cudaMemsetAsync(w.nbig, 0, sizeof(int32_t), stream));
    k_nr_vertex<<<(unsigned)((V + 255) / 256), 256, 0, stream>>>(verts, norms, V, M, width, height, w.vrec, w.nrot);
    ICON_LAUNCHED();
    k_nr_small<<<(unsigned)((F + 255) / 256), 256, 0, stream>>>(faces, F, V, w.vrec, width, height, w.zbuf, w.big,
                                                                   w.nbig);
    ICON_LAUNCHED();
    k_nr_big<<<NR_BIG_BLOCKS, 256, 0, stream>>>(faces, V, w.vrec, width, height, w.zbuf, w.big, w.nbig);
    ICON_LAUNCHED();
    k_nr_shade<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(w.zbuf, faces, V, w.vrec, w.nrot, width, height,
                                                                     (float4 *)out_rgba, out_face);
    ICON_LAUNCHED();
    return ICON_OK;
}
