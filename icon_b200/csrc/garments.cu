// Garment extraction of the demo (lib/common/cloth_extraction.py:extract_cloth, called from apps/infer.py:566-605):
// the per-vertex body-part labels and the per-face keep mask.  The polygon mapping and the trimesh steps stay on the
// host (icon_b200/garments.py).
//
// Labels: each reconstruction vertex takes the part of its nearest SMPL vertex, nearest in the float64 squared
// distance ((x0-y0)^2 + (x1-y1)^2) + (x2-y2)^2 (the order of sklearn's kd_tree rdist), exact ties to the lowest
// SMPL index.  Brute force over all SMPL vertices, staged through shared memory in tiles.
//
// Face mask: a vertex is kept when it lies inside any of the garment's polygons (matplotlib's point_in_path crossings
// rule, DESIGN.md 4.16) and its part is not in the removal set; a face is kept when any of its corners is kept.  A
// vertex pass and then a face pass: every vertex is tested against the polygons once, where a face-only kernel would
// test each vertex about six times (once per incident face).
//
// Every float64 decision expression is written with __dsub_rn / __dmul_rn / __dadd_rn, so no multiply-add can be
// contracted into a fused one whatever the flags; the unit is compiled with -fmad=false like the other geometry units.
#include "common.cuh"

namespace icon {

constexpr int GL_T = 256;        // labels: threads per block = SMPL vertices per shared-memory tile
constexpr int GM_T = 256;        // face mask: threads per block
constexpr int GM_CHUNK = 1024;   // polygon vertices per shared-memory stage

// validation word (bit per failure), in the face-mask workspace
constexpr int GERR_PART = 1, GERR_FACE = 2;

__global__ void __launch_bounds__(GL_T) k_garment_labels(const double *__restrict__ recon, int V,
                                                         const double *__restrict__ smpl, int S,
                                                         const uint8_t *__restrict__ parts,
                                                         uint8_t *__restrict__ labels) {
    __shared__ double s_x[GL_T], s_y[GL_T], s_z[GL_T];
    const int v = blockIdx.x * GL_T + threadIdx.x;
    double px = 0.0, py = 0.0, pz = 0.0;
    if (v < V) {
        px = recon[3 * (size_t)v];
        py = recon[3 * (size_t)v + 1];
        pz = recon[3 * (size_t)v + 2];
    }
    double best = 0.0;
    int bi = -1;
    for (int base = 0; base < S; base += GL_T) {
        const int n = min(GL_T, S - base);
        __syncthreads();
        if (threadIdx.x < n) {
            const size_t j = (size_t)(base + threadIdx.x);
            s_x[threadIdx.x] = smpl[3 * j];
            s_y[threadIdx.x] = smpl[3 * j + 1];
            s_z[threadIdx.x] = smpl[3 * j + 2];
        }
        __syncthreads();
        for (int k = 0; k < n; ++k) {
            const double dx = __dsub_rn(px, s_x[k]), dy = __dsub_rn(py, s_y[k]), dz = __dsub_rn(pz, s_z[k]);
            const double d = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
            // ascending index and a strict comparison: the lowest index wins an exact tie
            if (bi < 0 || d < best) {
                best = d;
                bi = base + k;
            }
        }
    }
    if (v < V) labels[v] = parts[bi];
}

// matplotlib's crossing test of the point (tx, ty) against the edge (x0, y0) -> (x1, y1): does it flip the parity?
__device__ __forceinline__ bool edge_flips(double x0, double y0, double x1, double y1, double tx, double ty) {
    const bool f0 = y0 >= ty, f1 = y1 >= ty;
    if (f0 == f1) return false;
    const double lhs = __dmul_rn(__dsub_rn(y1, ty), __dsub_rn(x0, x1));
    const double rhs = __dmul_rn(__dsub_rn(x1, tx), __dsub_rn(y0, y1));
    return (lhs >= rhs) == f1;
}

// keep[v] = inside any polygon && part not removed.  Every thread of a block walks the same polygon edges (staged
// through shared memory), so the loop and its barriers are block-uniform; threads past V only help stage.
__global__ void __launch_bounds__(GM_T) k_garment_keep(const double *__restrict__ verts, int V,
                                                       const uint8_t *__restrict__ labels, uint32_t remove_parts,
                                                       const double *__restrict__ poly_xy,
                                                       const int32_t *__restrict__ poly_off, int npoly,
                                                       uint8_t *__restrict__ keep, int32_t *__restrict__ err) {
    __shared__ double2 s_xy[GM_CHUNK];
    const int v = blockIdx.x * GM_T + threadIdx.x;
    double tx = 0.0, ty = 0.0;
    if (v < V) {
        tx = verts[3 * (size_t)v];
        ty = verts[3 * (size_t)v + 1];
    }
    // a point with a non-finite coordinate is never inside
    const bool finite = isfinite(tx) && isfinite(ty);
    bool inside = false;
    for (int p = 0; p < npoly; ++p) {
        const int s = poly_off[p], e = poly_off[p + 1];
        if (e - s < 3) continue;                        // fewer than three vertices enclose nothing
        bool par = false;
        double fx = 0.0, fy = 0.0, qx = 0.0, qy = 0.0;  // first and previous vertex
        for (int c = s; c < e; c += GM_CHUNK) {
            const int n = min(GM_CHUNK, e - c);
            __syncthreads();
            for (int i = threadIdx.x; i < n; i += GM_T)
                s_xy[i] = make_double2(poly_xy[2 * (size_t)(c + i)], poly_xy[2 * (size_t)(c + i) + 1]);
            __syncthreads();
            for (int k = 0; k < n; ++k) {
                const double2 w = s_xy[k];
                if (c + k == s) {
                    fx = w.x;
                    fy = w.y;
                } else {
                    par ^= edge_flips(qx, qy, w.x, w.y, tx, ty);
                }
                qx = w.x;
                qy = w.y;
            }
        }
        par ^= edge_flips(qx, qy, fx, fy, tx, ty);      // the implicit closing edge
        inside |= par;
    }
    if (v >= V) return;
    const unsigned part = labels[v];
    if (part >= 32) {
        atomicOr(err, GERR_PART);
        return;
    }
    keep[v] = (finite && inside && !((remove_parts >> part) & 1u)) ? 1 : 0;
}

__global__ void __launch_bounds__(GM_T) k_garment_faces(const int64_t *__restrict__ faces, int F, int V,
                                                        const uint8_t *__restrict__ keep,
                                                        uint8_t *__restrict__ face_mask, int32_t *__restrict__ count,
                                                        int32_t *__restrict__ err) {
    const int f = blockIdx.x * GM_T + threadIdx.x;
    bool kept = false;
    if (f < F) {
        bool ok = true;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int64_t id = faces[3 * (size_t)f + c];
            if (id < 0 || id >= V) {
                ok = false;
            } else {
                kept |= keep[id] != 0;
            }
        }
        if (!ok) {
            atomicOr(err, GERR_FACE);
            kept = false;
        }
        face_mask[f] = kept ? 1 : 0;
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, kept);
    if ((threadIdx.x & 31) == 0 && ballot) atomicAdd(count, __popc(ballot));
}

}  // namespace icon

using namespace icon;

extern "C" size_t icon_garment_labels_workspace_bytes(int S) { return S > 0 ? align_up((size_t)S, 256) : 0; }

extern "C" int icon_garment_labels(const double *recon_verts, int V, const double *smpl_verts, int S,
                                   const uint8_t *h_smpl_parts, uint8_t *labels, void *ws, size_t ws_bytes,
                                   icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(V >= 0 && S > 0, "icon_garment_labels: bad sizes (reconstruction V=%d, SMPL S=%d)", V, S);
    ICON_CHECK_ARG(recon_verts && smpl_verts && h_smpl_parts && labels && ws, "icon_garment_labels: null pointer");
    for (int j = 0; j < S; ++j)
        ICON_CHECK_ARG(h_smpl_parts[j] < 32, "icon_garment_labels: SMPL vertex %d has part id %d (at most 31)", j,
                       (int)h_smpl_parts[j]);
    const size_t need = icon_garment_labels_workspace_bytes(S);
    if (ws_bytes < need) {
        set_error("icon_garment_labels: workspace %zu < %zu bytes", ws_bytes, need);
        return ICON_ENOSPC;
    }
    if (V == 0) return ICON_OK;
    uint8_t *parts = (uint8_t *)ws;
    ICON_CUDA(cudaMemcpyAsync(parts, h_smpl_parts, (size_t)S, cudaMemcpyHostToDevice, stream));
    k_garment_labels<<<(unsigned)((V + GL_T - 1) / GL_T), GL_T, 0, stream>>>(recon_verts, V, smpl_verts, S, parts,
                                                                             labels);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" size_t icon_garment_face_mask_workspace_bytes(int V, int npoly) {
    if (V <= 0 || npoly < 0) return 0;
    Carver c(nullptr);
    c.take<uint8_t>((size_t)V);
    c.take<int32_t>((size_t)npoly + 1);
    c.take<int32_t>(1);
    return c.total();
}

extern "C" int icon_garment_face_mask(const double *verts, int V, const int64_t *faces, int F, const uint8_t *labels,
                                      uint32_t remove_parts, const double *poly_xy, int NP, const int32_t *h_poly_off,
                                      int npoly, uint8_t *face_mask, int32_t *kept_count, void *ws, size_t ws_bytes,
                                      icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(V > 0 && F >= 0 && NP >= 0 && npoly >= 0,
                   "icon_garment_face_mask: bad sizes (V=%d, F=%d, polygon vertices %d, polygons %d)", V, F, NP,
                   npoly);
    ICON_CHECK_ARG(verts && labels && kept_count && ws && h_poly_off && ((faces && face_mask) || F == 0) &&
                       (poly_xy || NP == 0),
                   "icon_garment_face_mask: null pointer");
    for (int p = 0; p <= npoly; ++p)
        ICON_CHECK_ARG(h_poly_off[p] >= (p ? h_poly_off[p - 1] : 0) && h_poly_off[p] <= NP,
                       "icon_garment_face_mask: polygon offset %d = %d: offsets must not decrease and must lie in "
                       "[0, %d]", p, h_poly_off[p], NP);
    const size_t need = icon_garment_face_mask_workspace_bytes(V, npoly);
    if (ws_bytes < need) {
        set_error("icon_garment_face_mask: workspace %zu < %zu bytes", ws_bytes, need);
        return ICON_ENOSPC;
    }
    Carver c(ws);
    uint8_t *keep = c.take<uint8_t>((size_t)V);
    int32_t *off = c.take<int32_t>((size_t)npoly + 1);
    int32_t *err = c.take<int32_t>(1);
    ICON_CUDA(cudaMemcpyAsync(off, h_poly_off, sizeof(int32_t) * ((size_t)npoly + 1), cudaMemcpyHostToDevice, stream));
    ICON_CUDA(cudaMemsetAsync(err, 0, sizeof(int32_t), stream));
    ICON_CUDA(cudaMemsetAsync(kept_count, 0, sizeof(int32_t), stream));
    k_garment_keep<<<(unsigned)((V + GM_T - 1) / GM_T), GM_T, 0, stream>>>(verts, V, labels, remove_parts, poly_xy,
                                                                           off, npoly, keep, err);
    ICON_LAUNCHED();
    if (F > 0) {
        k_garment_faces<<<(unsigned)((F + GM_T - 1) / GM_T), GM_T, 0, stream>>>(faces, F, V, keep, face_mask,
                                                                                kept_count, err);
        ICON_LAUNCHED();
    }
    // labels and faces live on the device: the kernels flag bad ones and the verdict is read back
    int32_t h_err = 0;
    ICON_CUDA(cudaMemcpyAsync(&h_err, err, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    ICON_CUDA(cudaStreamSynchronize(stream));
    ICON_CHECK_ARG(!(h_err & GERR_PART), "icon_garment_face_mask: a vertex label is a part id of 32 or more");
    ICON_CHECK_ARG(!(h_err & GERR_FACE), "icon_garment_face_mask: a face index is outside [0, %d)", V);
    return ICON_OK;
}
