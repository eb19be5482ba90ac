// SMPL body preparation: vertex normals (normals.cu's area-weighted rule), per-face records in original order, the
// face tree (face_tree.cu, over the fixed cube [-1.5, 1.5)^3 of a body in the query frame) and the yz ray grid.
// Compiled with -fmad=false.
//
// Replaces the per-query preamble of cal_sdf_batch (lib/dataset/mesh_util.py:367-372):
//   normals = Meshes(verts, faces).verts_normals_padded()          (pytorch3d)
//   triangles / normals / cmaps / vis = face_vertices(., faces)    (render_utils.py:149-163)
// which the reference recomputes on every query() call; here it runs once per body.  The
// acceleration structures only decide WHICH faces a query point looks at; distances, signs and
// attributes always come from the per-face records in original face order.
#include <float.h>

#include "common.cuh"
#include "face_tree.cuh"
#include "geom.cuh"

namespace icon {

static MeshView carve_mesh(Carver &c, int V, int F) {
    MeshView m{};
    static_cast<FaceTree &>(m) = face_tree_carve(c, F).t;     // first: icon_face_tree_read finds it there
    m.V = V;
    m.tri = c.take<float4>((size_t)F * 3);
    m.attr = c.take<float4>((size_t)F * 6);
    m.rbox = c.take<float4>((size_t)F * 2);
    m.rcount = c.take<int32_t>(RAY_GRID * RAY_GRID + 1);
    m.roff = c.take<int32_t>(RAY_GRID * RAY_GRID + 1);
    m.rlist = c.take<int32_t>((size_t)F * RAY_LIST_PER_FACE);
    m.hdr = c.take<MeshHeader>(1);
    m.scan_ws = c.take<char>(scan_ws_bytes(RAY_GRID * RAY_GRID + 1));
    m.bxyz = c.take<float4>(NBRICK);
    m.bperm = c.take<int32_t>(NBRICK);
    m.brec = c.take<float>((size_t)NBRICK * 8);
    m.bface = c.take<int32_t>(NBRICK);
    m.bub = c.take<float>(NBRICK);
    m.foff = c.take<int32_t>(NBRICK + 1);
    m.face_cap = brick_face_cap(F);
    m.flist = c.take<unsigned short>((size_t)m.face_cap);
    m.fkey = c.take<float>((size_t)m.face_cap);
    m.vn_ws = c.take<char>(area_vertex_normals_ws_bytes(V, F));
    m.vnormals = c.take<float>((size_t)V * 3);      // last: tests read it from the tail
    return m;
}

size_t mesh_ws_bytes(int V, int F) {
    Carver c(nullptr);
    carve_mesh(c, V, F);
    return c.total();
}

MeshView mesh_view(const void *ws, int V, int F) {
    Carver c((void *)ws);
    return carve_mesh(c, V, F);
}

__global__ void k_face_records(const float *__restrict__ verts, const int64_t *__restrict__ faces,
                               const float *__restrict__ vnormals, const float *__restrict__ cmap,
                               const float *__restrict__ vis, int F, float4 *__restrict__ tri,
                               float4 *__restrict__ attr, float4 *__restrict__ rbox) {
    int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    int64_t i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
    V3 a, b, c;
    load_face(verts, faces, f, a, b, c);
    write_tri(a, b, c, tri + 3 * f);
    const float *n0 = vnormals + 3 * i0, *n1 = vnormals + 3 * i1, *n2 = vnormals + 3 * i2;
    const float *m0 = cmap + 3 * i0, *m1 = cmap + 3 * i1, *m2 = cmap + 3 * i2;
    attr[6 * f + 0] = make_float4(n0[0], n0[1], n0[2], n1[0]);
    attr[6 * f + 1] = make_float4(n1[1], n1[2], n2[0], n2[1]);
    attr[6 * f + 2] = make_float4(n2[2], m0[0], m0[1], m0[2]);
    attr[6 * f + 3] = make_float4(m1[0], m1[1], m1[2], m2[0]);
    attr[6 * f + 4] = make_float4(m2[1], m2[2], vis[i0], vis[i1]);
    attr[6 * f + 5] = make_float4(vis[i2], 0.f, 0.f, 0.f);
    rbox[2 * f + 0] = make_float4(fminf(a.y, fminf(b.y, c.y)), fmaxf(a.y, fmaxf(b.y, c.y)),
                                  fminf(a.z, fminf(b.z, c.z)), fmaxf(a.z, fmaxf(b.z, c.z)));
    rbox[2 * f + 1] = make_float4(fmaxf(a.x, fmaxf(b.x, c.x)), fminf(a.x, fminf(b.x, c.x)), 0.f, 0.f);
}

// ray grid frame from the tree's root box
__global__ void k_ray_header(MeshView m) {
    const size_t root = (size_t)m.lvl_off[m.nlevels - 1];
    float4 lo = m.nodes[2 * root], hi = m.nodes[2 * root + 1];
    const float pad = 1e-3f;
    MeshHeader h;
    h.y0 = lo.y - pad; h.z0 = lo.z - pad;
    h.inv_cy = (float)RAY_GRID / ((hi.y + pad) - h.y0);
    h.inv_cz = (float)RAY_GRID / ((hi.z + pad) - h.z0);
    h.ray_overflow = 0;
    h.brick_built = h.brick_overflow = h.pad = 0;
    *m.hdr = h;
}

// ---- yz cell lists for the +x ray: a face is listed in every cell its (inflated) yz box overlaps
__device__ __forceinline__ void cell_range(const MeshHeader &h, float4 rb, int &cy0, int &cy1, int &cz0, int &cz1) {
    const float e = 1e-4f;
    cy0 = max(0, min(RAY_GRID - 1, (int)floorf((rb.x - e - h.y0) * h.inv_cy)));
    cy1 = max(0, min(RAY_GRID - 1, (int)floorf((rb.y + e - h.y0) * h.inv_cy)));
    cz0 = max(0, min(RAY_GRID - 1, (int)floorf((rb.z - e - h.z0) * h.inv_cz)));
    cz1 = max(0, min(RAY_GRID - 1, (int)floorf((rb.w + e - h.z0) * h.inv_cz)));
}

__global__ void k_ray_count(MeshView m) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.F) return;
    const MeshHeader h = *m.hdr;
    int cy0, cy1, cz0, cz1;
    cell_range(h, m.rbox[2 * (size_t)f], cy0, cy1, cz0, cz1);
    for (int cz = cz0; cz <= cz1; ++cz)
        for (int cy = cy0; cy <= cy1; ++cy) atomicAdd(&m.rcount[cz * RAY_GRID + cy], 1);
}

__global__ void k_ray_fill(MeshView m, int32_t *__restrict__ cursor) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.F) return;
    const MeshHeader h = *m.hdr;
    int cy0, cy1, cz0, cz1;
    cell_range(h, m.rbox[2 * (size_t)f], cy0, cy1, cz0, cz1);
    const int cap = m.F * RAY_LIST_PER_FACE;
    for (int cz = cz0; cz <= cz1; ++cz)
        for (int cy = cy0; cy <= cy1; ++cy) {
            const int c = cz * RAY_GRID + cy;
            const int pos = m.roff[c] + atomicAdd(&cursor[c], 1);
            if (pos < cap) m.rlist[pos] = f;
            else m.hdr->ray_overflow = 1;
        }
}

}  // namespace icon

using namespace icon;

extern "C" size_t icon_smpl_workspace_bytes(int V, int F) { return mesh_ws_bytes(V, F); }

extern "C" int icon_smpl_prepare(const float *verts, const int64_t *faces, const float *cmap,
                                 const float *vis, int V, int F, void *mesh_ws, size_t mesh_ws_bytes_,
                                 icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(V > 0 && F > 0, "icon_smpl_prepare: empty mesh (V=%d F=%d)", V, F);
    ICON_CHECK_ARG(F <= 4 * 65535, "icon_smpl_prepare: F=%d too large (leaf ids are 16-bit)", F);
    ICON_CHECK_ARG(verts && faces && cmap && vis && mesh_ws, "icon_smpl_prepare: null pointer");
    if (mesh_ws_bytes_ < mesh_ws_bytes(V, F)) {
        set_error("icon_smpl_prepare: workspace %zu < %zu", mesh_ws_bytes_, mesh_ws_bytes(V, F));
        return ICON_ENOSPC;
    }
    Carver c(mesh_ws);
    MeshView m = carve_mesh(c, V, F);
    bricks_forget(m);
    void *scan_ws = m.scan_ws;
    int rc = area_vertex_normals(verts, V, faces, F, m.vnormals, m.vn_ws, stream);
    if (rc) return rc;
    k_face_records<<<(F + 127) / 128, 128, 0, stream>>>(verts, faces, m.vnormals, cmap, vis, F, (float4 *)m.tri,
                                                        (float4 *)m.attr, (float4 *)m.rbox);
    ICON_LAUNCHED();
    rc = face_tree_build(mesh_ws, verts, faces, F, TreeFrame{false, -1.5f, 1024.f / 3.f, false}, stream);
    if (rc) return rc;
    k_ray_header<<<1, 1, 0, stream>>>(m);
    ICON_LAUNCHED();
    ICON_CUDA(cudaMemsetAsync(m.rcount, 0, sizeof(int32_t) * (RAY_GRID * RAY_GRID + 1), stream));
    k_ray_count<<<(F + 127) / 128, 128, 0, stream>>>(m);
    ICON_LAUNCHED();
    rc = scan_exclusive_i32(m.rcount, m.roff, RAY_GRID * RAY_GRID + 1, nullptr, scan_ws, stream);
    if (rc) return rc;
    ICON_CUDA(cudaMemsetAsync(m.rcount, 0, sizeof(int32_t) * (RAY_GRID * RAY_GRID + 1), stream));   // reuse as cursor
    k_ray_fill<<<(F + 127) / 128, 128, 0, stream>>>(m, m.rcount);
    ICON_LAUNCHED();
    return ICON_OK;
}
