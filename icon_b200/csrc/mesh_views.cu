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
    t.den = mv_e(t.x[2], t.y[2], t.x[0], t.y[0], t.x[1], t.y[1]) + MV_KEPS;
    const float r = sqrtf(MV_BLUR);
    t.bx0 = fminf(fminf(t.x[0], t.x[1]), t.x[2]) - r; t.bx1 = fmaxf(fmaxf(t.x[0], t.x[1]), t.x[2]) + r;
    t.by0 = fminf(fminf(t.y[0], t.y[1]), t.y[2]) - r; t.by1 = fmaxf(fmaxf(t.y[0], t.y[1]), t.y[2]) + r;
    mv_range(t.bx0, t.bx1, S, t.j0, t.j1);
    mv_range(t.by0, t.by1, S, t.i0, t.i1);
    return t.j0 <= t.j1 && t.i0 <= t.i1;
}

struct MvFrag {
    float z, dist, c[3];
};

__device__ __forceinline__ bool mv_fragment(const MvTri &t, float px, float py, MvFrag &o) {
    if (px > t.bx1 || px < t.bx0 || py > t.by1 || py < t.by0) return false;
    const float w0 = mv_e(px, py, t.x[1], t.y[1], t.x[2], t.y[2]) / t.den;
    const float w1 = mv_e(px, py, t.x[2], t.y[2], t.x[0], t.y[0]) / t.den;
    const float w2 = mv_e(px, py, t.x[0], t.y[0], t.x[1], t.y[1]) / t.den;
    const bool inside = w0 > 0.f && w1 > 0.f && w2 > 0.f;
    const float d = fminf(fminf(mv_seg(px, py, t.x[0], t.y[0], t.x[1], t.y[1]),
                                mv_seg(px, py, t.x[0], t.y[0], t.x[2], t.y[2])),
                          mv_seg(px, py, t.x[1], t.y[1], t.x[2], t.y[2]));
    if (!inside && d >= MV_BLUR) return false;
    float c0 = fmaxf(w0, 0.f), c1 = fmaxf(w1, 0.f), c2 = fmaxf(w2, 0.f);
    const float s = fmaxf((c0 + c1) + c2, 1e-5f);
    c0 = c0 / s; c1 = c1 / s; c2 = c2 / s;
    const float z = (c0 * t.z[0] + c1 * t.z[1]) + c2 * t.z[2];
    if (z < 0.f) return false;
    o.z = z; o.dist = inside ? -d : d;
    o.c[0] = c0; o.c[1] = c1; o.c[2] = c2;
    return true;
}

__device__ __forceinline__ unsigned long long mv_key(float z, int f) {
    return ((unsigned long long)(__float_as_uint(z) & 0x7fffffffu) << 32) | (unsigned)f;   // z >= 0 (-0 -> +0)
}

__device__ __forceinline__ float mv_zmax(unsigned long long nearest) {
    return nearest == MV_EMPTY ? MV_EPS : fmaxf((256.f - __uint_as_float((unsigned)(nearest >> 32))) / 512.f, MV_EPS);
}

// pass 1: nearest fragment; pass 2: the fragments of non-zero weight into the K sorted slots
template <int PASS>
__device__ __forceinline__ void mv_pixel(const MvTri &t, int f, int i, int j, int S, int64_t pix,
                                         unsigned long long *__restrict__ near, unsigned long long *__restrict__ slots) {
    MvFrag fr;
    if (!mv_fragment(t, mv_pix(j, S), mv_pix(i, S), fr)) return;
    unsigned long long key = mv_key(fr.z, f);
    if (PASS == 1) {
        atomicMin(&near[pix], key);
        return;
    }
    const float zmax = mv_zmax(near[pix]);
    if (!(((256.f - fr.z) / 512.f - zmax) / MV_GAMMA > -MV_CUT)) return;
    unsigned long long *s = slots + pix * MV_K;
    for (int k = 0; k < MV_K; ++k) {
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

// one thread per face, looping over the chunk's views; pass 1 lists the (face, view) pairs with a large box
template <int PASS>
__global__ void k_mv_small(const int64_t *__restrict__ faces, int F, int V, int A, int S,
                           const float4 *__restrict__ vrec, unsigned long long *__restrict__ near,
                           unsigned long long *__restrict__ slots, int2 *__restrict__ big, int32_t *__restrict__ nbig) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    for (int a = 0; a < A; ++a) {
        MvTri t;
        if (!mv_setup(faces, vrec + (int64_t)a * V, f, V, S, t)) continue;
        const int nj = t.j1 - t.j0 + 1, ni = t.i1 - t.i0 + 1;
        if (nj * ni > MV_SMALL) {
            if (PASS == 1) big[atomicAdd(nbig, 1)] = make_int2(f, a);
            continue;
        }
        const int64_t base = (int64_t)a * S * S;
        for (int i = t.i0; i <= t.i1; ++i)
            for (int j = t.j0; j <= t.j1; ++j) mv_pixel<PASS>(t, f, i, j, S, base + (int64_t)i * S + j, near, slots);
    }
}

// one block per listed (face, view) pair; the block's threads stride over the face's pixel box
template <int PASS>
__global__ void __launch_bounds__(256) k_mv_big(const int64_t *__restrict__ faces, int V, int S,
                                                const float4 *__restrict__ vrec, unsigned long long *__restrict__ near,
                                                unsigned long long *__restrict__ slots, const int2 *__restrict__ big,
                                                const int32_t *__restrict__ nbig) {
    const int n = *nbig;
    for (int b = blockIdx.x; b < n; b += gridDim.x) {
        const int f = big[b].x, a = big[b].y;
        MvTri t;
        if (!mv_setup(faces, vrec + (int64_t)a * V, f, V, S, t)) continue;
        const int nj = t.j1 - t.j0 + 1;
        const int np = nj * (t.i1 - t.i0 + 1);
        const int64_t base = (int64_t)a * S * S;
        for (int p = threadIdx.x; p < np; p += blockDim.x) {
            const int i = t.i0 + p / nj, j = t.j0 + p % nj;
            mv_pixel<PASS>(t, f, i, j, S, base + (int64_t)i * S + j, near, slots);
        }
    }
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
        const int f = (int)(key & 0xffffffffull);
        MvTri t;
        MvFrag fr;
        mv_setup(faces, vrec + (int64_t)a * V, f, V, S, t);      // both succeeded in the raster passes
        mv_fragment(t, px, py, fr);
        const float prob = 1.f / (1.f + expf(fr.dist / MV_SIGMA));
        const float w = prob * expf(((256.f - fr.z) / 512.f - zmax) / MV_GAMMA);
        float col[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const int64_t c0 = 3 * faces[3 * (int64_t)f], c1 = 3 * faces[3 * (int64_t)f + 1];
            const int64_t c2 = 3 * faces[3 * (int64_t)f + 2];
            col[ch] = (fr.c[0] * colors[c0 + ch] + fr.c[1] * colors[c1 + ch]) + fr.c[2] * colors[c2 + ch];
        }
        nr = nr + w * col[0]; ng = ng + w * col[1]; nb = nb + w * col[2];
        den = den + w;
    }
    const float delta = fmaxf(expf((MV_EPS - zmax) / MV_GAMMA), MV_EPS);
    den = den + delta;
    const float rgb[3] = {(nr + delta * MV_BG) / den, (ng + delta * MV_BG) / den, (nb + delta * MV_BG) / den};
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float v = rgb[ch] * 255.f;
        out[3 * p + ch] = v >= 255.f ? (uint8_t)255 : (v > 0.f ? (uint8_t)v : (uint8_t)0);
        if (rgb_out) rgb_out[3 * p + ch] = rgb[ch];
    }
    if (face_out) face_out[p] = s[0] == MV_EMPTY ? -1 : (int)(s[0] & 0xffffffffull);
}

struct MvWs {
    float *mats;
    float4 *vrec;
    unsigned long long *near, *slots;
    int2 *big;
    int32_t *nbig;
};

static size_t mv_carve(void *ws, int V, int F, int S, int A, MvWs *o) {
    Carver c(ws);
    MvWs w;
    const size_t npix = (size_t)A * S * S;
    w.mats = c.take<float>(12 * (size_t)A);
    w.vrec = c.take<float4>((size_t)A * V);
    w.near = c.take<unsigned long long>(npix);
    w.slots = c.take<unsigned long long>(npix * MV_K);
    w.big = c.take<int2>((size_t)A * F);
    w.nbig = c.take<int32_t>(1);
    if (o) *o = w;
    return c.total();
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

extern "C" size_t icon_mesh_views_workspace_bytes(int V, int F, int S, int A) {
    if (V <= 0 || F <= 0 || S <= 0 || A <= 0) return 0;
    return icon::mv_carve(nullptr, V, F, S, A, nullptr);
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
    mv_carve(ws, V, F, S, A, &w);
    const int64_t npix = (int64_t)A * S * S;
    ICON_CUDA(cudaMemcpyAsync(w.mats, h_view_mats, sizeof(float) * 12 * (size_t)A, cudaMemcpyHostToDevice, stream));
    ICON_CUDA(cudaMemsetAsync(w.near, 0xff, sizeof(unsigned long long) * (size_t)npix, stream));
    ICON_CUDA(cudaMemsetAsync(w.slots, 0xff, sizeof(unsigned long long) * (size_t)npix * MV_K, stream));
    ICON_CUDA(cudaMemsetAsync(w.nbig, 0, sizeof(int32_t), stream));
    k_mv_vertex<<<dim3((unsigned)((V + 255) / 256), (unsigned)A), 256, 0, stream>>>(verts, V, w.mats, w.vrec);
    ICON_LAUNCHED();
    const unsigned fb = (unsigned)((F + 127) / 128);
    k_mv_small<1><<<fb, 128, 0, stream>>>(faces, F, V, A, S, w.vrec, w.near, w.slots, w.big, w.nbig);
    ICON_LAUNCHED();
    k_mv_big<1><<<MV_BIG_BLOCKS, 256, 0, stream>>>(faces, V, S, w.vrec, w.near, w.slots, w.big, w.nbig);
    ICON_LAUNCHED();
    k_mv_small<2><<<fb, 128, 0, stream>>>(faces, F, V, A, S, w.vrec, w.near, w.slots, w.big, w.nbig);
    ICON_LAUNCHED();
    k_mv_big<2><<<MV_BIG_BLOCKS, 256, 0, stream>>>(faces, V, S, w.vrec, w.near, w.slots, w.big, w.nbig);
    ICON_LAUNCHED();
    k_mv_shade<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(faces, V, A, S, w.vrec, colors, w.slots, out,
                                                                     face_out, rgb_out);
    ICON_LAUNCHED();
    return ICON_OK;
}
