// Vertex visibility of the fitted body: replaces get_visibility (lib/dataset/mesh_util.py:280-316), the producer of
// the `smpl_vis` input of the query path (TestDataset.compute_vis_cmap, lib/dataset/TestDataset.py:134-148).
//
// The reference rasterises the mesh with pytorch3d.rasterize_meshes (image 4096^2, blur 0, 1 face per pixel,
// perspective_correct = True, cull_backfaces = True; settings at lib/common/render_utils.py:178-186) and marks the
// vertices of every face that owns at least one pixel.  PARITY UNPINNED: pytorch3d is not installable here and its
// source is not in the reference tree; the rasterisation rules below restate its documented / published kernel
//   * pixel (yi, xi) has NDC centre (1 - (2 xi + 1) / S, 1 - (2 yi + 1) / S)  (+X left, +Y up);
//   * a face is skipped when max z < 0, when its signed area e(v0, v1, v2) is < 0 (back face) or |area| <= 1e-8;
//     e(p, a, b) = (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x);
//   * barycentrics w0 = e(p, v1, v2) / (area + 1e-8), w1 = e(p, v2, v0) / .., w2 = e(p, v0, v1) / ..; the pixel is
//     covered when all three are > 0; depth uses the perspective-corrected weights
//     (w0 z1 z2, z0 w1 z2, z0 z1 w2) / (their sum + 1e-8), pz = sum w_i z_i, pixels with pz < 0 are dropped;
//   * the nearest pz wins, ties go to the lowest face index (scan order of the naive rasteriser); -0 ties with +0,
//     and pz = +inf (the background's depth) or NaN never takes a pixel.
// Bug-compatibility: `faces[torch.unique(pix_to_face)]` also indexes with the background value -1, i.e. the LAST
// face, whenever some pixel is empty (mesh_util.py:310) -- its three vertices are then marked visible too.
// pix_to_face, the depth of every pixel (read back from the workspace, include/icon_b200.h) and the mask are compared
// bit for bit with oracle/visibility.py, hence -fmad=false for this file.
#include "common.cuh"

namespace icon {

constexpr unsigned long long VIS_EMPTY = 0xffffffffffffffffull;

__device__ __forceinline__ float edge_fn(float px, float py, float ax, float ay, float bx, float by) {
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax);
}

// one warp per face; lanes stride over the pixels of its bounding box
__global__ void k_vis_raster(const float *__restrict__ xyz, const int64_t *__restrict__ faces, int F, int V, int S,
                             unsigned long long *__restrict__ zbuf) {
    const int f = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (f >= F) return;
    float v[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        int64_t id = faces[3 * (int64_t)f + k];
        id = id < 0 ? 0 : (id >= V ? V - 1 : id);
        v[k][0] = xyz[3 * id]; v[k][1] = xyz[3 * id + 1]; v[k][2] = xyz[3 * id + 2];
    }
    const float zmax = fmaxf(fmaxf(v[0][2], v[1][2]), v[2][2]);
    const float area = edge_fn(v[0][0], v[0][1], v[1][0], v[1][1], v[2][0], v[2][1]);
    if (zmax < 0.f || area < 0.f || (area <= 1e-8f && area >= -1e-8f)) return;
    const float xmin = fminf(fminf(v[0][0], v[1][0]), v[2][0]), xmax = fmaxf(fmaxf(v[0][0], v[1][0]), v[2][0]);
    const float ymin = fminf(fminf(v[0][1], v[1][1]), v[2][1]), ymax = fmaxf(fmaxf(v[0][1], v[1][1]), v[2][1]);
    // pixel index ranges whose centres can fall inside [min, max]: x_ndc = 1 - (2 xi + 1) / S (conservative by 1),
    // clamped in float before the int conversion -- a vertex far off screen must not saturate it and wrap the count
    // -- and so that a NaN bound (all three coordinates NaN) spans the whole image, as the oracle evaluates it
    const float Sf = (float)S;
    const int xi0 = (int)fminf(fmaxf(floorf(((1.f - xmax) * Sf - 1.f) * 0.5f) - 1.f, 0.f), Sf);
    const int xi1 = (int)fmaxf(fminf(ceilf(((1.f - xmin) * Sf - 1.f) * 0.5f) + 1.f, Sf - 1.f), -1.f);
    const int yi0 = (int)fminf(fmaxf(floorf(((1.f - ymax) * Sf - 1.f) * 0.5f) - 1.f, 0.f), Sf);
    const int yi1 = (int)fmaxf(fminf(ceilf(((1.f - ymin) * Sf - 1.f) * 0.5f) + 1.f, Sf - 1.f), -1.f);
    const int nx = xi1 - xi0 + 1, ny = yi1 - yi0 + 1;
    if (nx <= 0 || ny <= 0) return;
    const float den = area + 1e-8f;
    const float z0 = v[0][2], z1 = v[1][2], z2 = v[2][2];
    for (int t = lane; t < nx * ny; t += 32) {
        const int xi = xi0 + t % nx, yi = yi0 + t / nx;
        const float px = 1.f - (float)(2 * xi + 1) / Sf, py = 1.f - (float)(2 * yi + 1) / Sf;
        if (px < xmin || px > xmax || py < ymin || py > ymax) continue;
        const float w0 = edge_fn(px, py, v[1][0], v[1][1], v[2][0], v[2][1]) / den;
        const float w1 = edge_fn(px, py, v[2][0], v[2][1], v[0][0], v[0][1]) / den;
        const float w2 = edge_fn(px, py, v[0][0], v[0][1], v[1][0], v[1][1]) / den;
        if (!(w0 > 0.f && w1 > 0.f && w2 > 0.f)) continue;
        const float t0 = w0 * z1 * z2, t1 = z0 * w1 * z2, t2 = z0 * z1 * w2;
        const float dsum = (t0 + t1 + t2) + 1e-8f;
        const float pz = (t0 / dsum) * z0 + (t1 / dsum) * z1 + (t2 / dsum) * z2;
        // the oracle takes a pixel on a strictly nearer depth only: NaN, pz < 0 and pz = +inf (the background's
        // depth) never take one
        if (!(pz >= 0.f && pz < INFINITY)) continue;
        // pz is +0 .. +FLT_MAX or -0 here: clearing the sign makes -0 the key of +0, so -0 ties with +0 (lowest face
        // wins) and is nearer than every positive depth, as `pz < zbuf` orders them
        const unsigned long long key = ((unsigned long long)(__float_as_uint(pz) & 0x7fffffffu) << 32) | (unsigned)f;
        atomicMin(&zbuf[(size_t)yi * S + xi], key);
    }
}

__global__ void k_vis_mark(const unsigned long long *__restrict__ zbuf, int64_t npix, const int64_t *__restrict__ faces,
                           int V, float *__restrict__ vis, int *__restrict__ any_empty) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool empty = false;
    if (p < npix) {
        const unsigned long long key = zbuf[p];
        if (key == VIS_EMPTY) {
            empty = true;
        } else {
            const int64_t f = (int64_t)(key & 0xffffffffull);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int64_t id = faces[3 * f + k];
                if (id >= 0 && id < V) vis[id] = 1.0f;
            }
        }
    }
    if (__syncthreads_or(empty) && threadIdx.x == 0) *any_empty = 1;
}

// torch.unique(pix_to_face) contains -1 when a pixel is empty, and faces[-1] is the last face
__global__ void k_vis_background(const int *__restrict__ any_empty, const int64_t *__restrict__ faces, int F, int V,
                                 float *__restrict__ vis) {
    if (threadIdx.x < 3 && *any_empty) {
        const int64_t id = faces[3 * (int64_t)(F - 1) + threadIdx.x];
        if (id >= 0 && id < V) vis[id] = 1.0f;
    }
}

}  // namespace icon

extern "C" size_t icon_visibility_workspace_bytes(int image_size) {
    if (image_size <= 0) return 0;
    return (size_t)image_size * image_size * sizeof(unsigned long long) + 256;
}

extern "C" int icon_visibility(const float *xyz, int V, const int64_t *faces, int F, int image_size, float *vis,
                               void *ws, size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(xyz && faces && vis && ws, "icon_visibility: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0 && image_size > 0 && image_size <= 16384, "icon_visibility: bad sizes");
    ICON_CHECK_ARG(ws_bytes >= icon_visibility_workspace_bytes(image_size), "icon_visibility: workspace too small");
    const int64_t npix = (int64_t)image_size * image_size;
    unsigned long long *zbuf = (unsigned long long *)ws;
    int *any_empty = (int *)((char *)ws + (size_t)npix * sizeof(unsigned long long));
    ICON_CUDA(cudaMemsetAsync(zbuf, 0xff, (size_t)npix * sizeof(unsigned long long), stream));
    ICON_CUDA(cudaMemsetAsync(any_empty, 0, sizeof(int), stream));
    ICON_CUDA(cudaMemsetAsync(vis, 0, sizeof(float) * (size_t)V, stream));
    k_vis_raster<<<(unsigned)(((int64_t)F * 32 + 255) / 256), 256, 0, stream>>>(xyz, faces, F, V, image_size, zbuf);
    ICON_LAUNCHED();
    k_vis_mark<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(zbuf, npix, faces, V, vis, any_empty);
    ICON_LAUNCHED();
    k_vis_background<<<1, 32, 0, stream>>>(any_empty, faces, F, V, vis);
    ICON_LAUNCHED();
    return ICON_OK;
}
