// Marching cubes with shared (edge-owned) vertices.
//
// Replaces Seg3dLossless.export_mesh (lib/common/seg3d_lossless.py:583-604): the
// occupancys[1:,1:,1:] crop, kaolin voxelgrids_to_trianglemeshes (zero pad, iso 0.5) or
// PyMCubes marching_cubes, and the [:, [2,1,0]] / [:, [0,2,1]] permutations -- everything
// stays on the device; only the finished vertex / face arrays travel to the host.
//
// Indexing contract (oracle/mcubes.py restates it; DESIGN.md "marching cubes"):
//   * working grid g[i][j][k] (i = z, j = y, k = x of the occupancy frame); padded branch:
//     G = R+1, g = occ for 1 <= i,j,k <= R-1 and 0 on the two outer shells (crop + zero pad);
//     plain branch: G = R-1, g[i][j][k] = occ[i+1][j+1][k+1];
//   * a vertex lives on a grid edge, owned by the edge's lower voxel; id order = ascending
//     3*linear(owner)+axis (axis 0 = i, 1 = j, 2 = k); position = owner + t along the axis,
//     t = (iso - f_lo) / (f_hi - f_lo); output column order (k, j, i) = (x, y, z);
//   * triangles: cells in linear order, table order inside a cell, corners (0, 2, 1).
// The surface touches only a few percent of the voxels, so the passes are organised around blocks of 1024
// consecutive voxels (in the linear order that defines the ids):
//   count : classify every voxel (the only pass that reads the whole grid: 4 B per voxel), reduce the block's
//           vertex / triangle totals; blocks that own something also store 2 B of flags per voxel;
//   scans : over the per-block totals only (n / 1024 entries);
//   verts : active blocks: block-local scan -> global vertex id of every owning voxel, interpolate, write;
//   faces : active blocks: block-local scan -> triangle slots; vertex ids through the owners' ids.
#include "common.cuh"

namespace icon {

#include "mc_tables.inc"   // __constant__ c_num_verts[256], c_tri_table[256][16], c_edge_owner[12][4]

struct McGrid {
    const float *occ;
    int R, G, shift;   // g[i][j][k] = inside ? occ[i+shift][j+shift][k+shift] : 0
    int lo, hi;        // inside when lo <= i,j,k <= hi
    __device__ __forceinline__ float at(int i, int j, int k) const {
        bool in = i >= lo && i <= hi && j >= lo && j <= hi && k >= lo && k <= hi;
        return in ? occ[((size_t)(i + shift) * R + (j + shift)) * R + (k + shift)] : 0.f;
    }
};

static McGrid make_grid(const float *occ, int R, int padded) {
    McGrid g;
    g.occ = occ; g.R = R;
    if (padded) { g.G = R + 1; g.shift = 0; g.lo = 1; g.hi = R - 1; }
    else        { g.G = R - 1; g.shift = 1; g.lo = 0; g.hi = R - 2; }
    return g;
}

constexpr int MC_T = 256;      // threads per block; every thread owns 4 consecutive voxels of one grid row
constexpr int MC_VPT = 4;

struct McGeom {
    int G, Q;                  // grid size, quads (4 voxels) per row = ceil(G / 4)
    int64_t nquads;            // G * G * Q
};
static McGeom make_geom(int G) {
    McGeom q;
    q.G = G; q.Q = (G + MC_VPT - 1) / MC_VPT; q.nquads = (int64_t)G * G * q.Q;
    return q;
}

// pointer to the occupancy row (i, j, :) already shifted so that [k] addresses grid column k, or null outside
__device__ __forceinline__ const float *mc_row(const McGrid &g, int i, int j) {
    const bool in = i >= g.lo && i <= g.hi && j >= g.lo && j <= g.hi;
    return in ? g.occ + ((size_t)(i + g.shift) * g.R + (j + g.shift)) * g.R + g.shift : nullptr;
}

// classification of the 4 voxels (i, j, k0 .. k0+3): fl = edge-ownership bits (i, j, k axis), cs = cube case.
// CT = the branch's precision (float padded, double plain): a node is below iso iff (CT)f < iso, so NaN never is
template <typename CT>
__device__ __forceinline__ void mc_classify4(const McGrid &g, CT iso, int i, int j, int k0, unsigned fl[4], int cs[4]) {
    const int G = g.G;
    const float *rows[4] = {mc_row(g, i, j), i + 1 < G ? mc_row(g, i + 1, j) : nullptr,
                            (i + 1 < G && j + 1 < G) ? mc_row(g, i + 1, j + 1) : nullptr,
                            j + 1 < G ? mc_row(g, i, j + 1) : nullptr};       // corner order 0, 1, 2, 3 (dk = 0)
    unsigned nib[5];                                                         // bit c: corner c of column k0 + m below iso
#pragma unroll
    for (int m = 0; m < 5; ++m) nib[m] = 0;
    if (rows[0] && rows[1] && rows[2] && rows[3] && k0 >= g.lo && k0 + 4 <= g.hi) {   // interior: no per-load checks
#pragma unroll
        for (int r = 0; r < 4; ++r) {
#pragma unroll
            for (int m = 0; m < 5; ++m) nib[m] |= ((CT)__ldg(rows[r] + k0 + m) < iso) ? (1u << r) : 0u;
        }
    } else {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const float *p = rows[r];
#pragma unroll
            for (int m = 0; m < 5; ++m) {
                const int k = k0 + m;
                const float f = (p != nullptr && k >= g.lo && k <= g.hi) ? __ldg(p + k) : 0.f;
                nib[m] |= ((CT)f < iso) ? (1u << r) : 0u;
            }
        }
    }
    const bool i1 = i + 1 < G, j1 = j + 1 < G;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        const int k = k0 + m;
        const bool k1 = k + 1 < G;
        const unsigned a = nib[m], bnext = nib[m + 1];
        unsigned f = 0;
        if (i1 && (((a >> 1) ^ a) & 1u)) f |= 1;                  // corner 1 vs corner 0
        if (j1 && (((a >> 3) ^ a) & 1u)) f |= 2;                  // corner 3 vs corner 0
        if (k1 && ((bnext ^ a) & 1u)) f |= 4;                     // corner 4 vs corner 0
        const bool valid = k < G;
        fl[m] = valid ? f : 0u;
        cs[m] = (valid && i1 && j1 && k1) ? (int)(a | (bnext << 4)) : 0;
    }
}

__device__ __forceinline__ void mc_quad_coords(const McGeom &q, int64_t u, int &i, int &j, int &k0) {
    const unsigned uu = (unsigned)u;                        // nquads < 2^31 is checked by the host
    const unsigned row = uu / (unsigned)q.Q;
    k0 = (int)(uu - row * (unsigned)q.Q) * MC_VPT;
    i = (int)(row / (unsigned)q.G);
    j = (int)(row - (unsigned)i * (unsigned)q.G);
}

// block-wide exclusive scan of one int per thread (MC_T threads); returns the exclusive prefix, total in *total
__device__ __forceinline__ int mc_block_scan(int x, int *total) {
    __shared__ int s_w[MC_T / 32];
    __shared__ int s_tot;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    __syncthreads();                        // protects s_w / s_tot between successive calls
    if (lane == 31) s_w[w] = inc;
    __syncthreads();
    if (w == 0) {
        int v = lane < MC_T / 32 ? s_w[lane] : 0;
        int vi = v;
#pragma unroll
        for (int o = 1; o < MC_T / 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, vi, o);
            if (lane >= o) vi += y;
        }
        if (lane < MC_T / 32) s_w[lane] = vi - v;
        if (lane == MC_T / 32 - 1) s_tot = vi;
    }
    __syncthreads();
    *total = s_tot;
    return s_w[w] + inc - x;
}

template <typename CT>
__global__ void __launch_bounds__(MC_T) k_mc_count(McGrid g, McGeom q, CT iso, int32_t *__restrict__ blk_v,
                                                   int32_t *__restrict__ blk_t, uint8_t *__restrict__ vflags,
                                                   uint8_t *__restrict__ vcase) {
    const int64_t u = (int64_t)blockIdx.x * MC_T + threadIdx.x;
    unsigned fl[4] = {0, 0, 0, 0};
    int cs[4] = {0, 0, 0, 0};
    int i = 0, j = 0, k0 = 0;
    const bool live = u < q.nquads;
    if (live) {
        mc_quad_coords(q, u, i, j, k0);
        mc_classify4(g, iso, i, j, k0, fl, cs);
    }
    int nv = 0, nt = 0;
#pragma unroll
    for (int m = 0; m < 4; ++m) { nv += __popc(fl[m]); nt += c_num_verts[cs[m]]; }
    // block totals (vertex count and 3 x triangle count packed: both < 2^15 per block)
    int packed = nv | (nt << 16);
#pragma unroll
    for (int o = 16; o; o >>= 1) packed += __shfl_xor_sync(0xffffffffu, packed, o);
    __shared__ int s_p[MC_T / 32];
    if ((threadIdx.x & 31) == 0) s_p[threadIdx.x >> 5] = packed;
    __syncthreads();
    int tot = 0;
#pragma unroll
    for (int w = 0; w < MC_T / 32; ++w) tot += s_p[w];
    if (threadIdx.x == 0) {
        blk_v[blockIdx.x] = tot & 0xffff;
        blk_t[blockIdx.x] = (tot >> 16) / 3;
    }
    if (tot == 0 || !live) return;
    const size_t v0 = ((size_t)i * g.G + j) * g.G + k0;
#pragma unroll
    for (int m = 0; m < 4; ++m)
        if (k0 + m < g.G) { vflags[v0 + m] = (uint8_t)fl[m]; vcase[v0 + m] = (uint8_t)cs[m]; }
}

// MC_T threads per block; the register cap replaces __launch_bounds__, under which ptxas spilled the fp32 variant
template <typename VT>
__global__ void __maxnreg__(64) k_mc_verts(McGrid g, McGeom q, VT iso, const int32_t *__restrict__ blk_v,
                                                   const int32_t *__restrict__ base_v,
                                                   const uint8_t *__restrict__ vflags, int32_t *__restrict__ voff,
                                                   VT *__restrict__ verts) {
    if (blk_v[blockIdx.x] == 0) return;
    const int64_t u = (int64_t)blockIdx.x * MC_T + threadIdx.x;
    int i = 0, j = 0, k0 = 0;
    unsigned fl[4] = {0, 0, 0, 0};
    size_t v0 = 0;
    if (u < q.nquads) {
        mc_quad_coords(q, u, i, j, k0);
        v0 = ((size_t)i * g.G + j) * g.G + k0;
#pragma unroll
        for (int m = 0; m < 4; ++m)
            if (k0 + m < g.G) fl[m] = vflags[v0 + m];
    }
    const int mine = __popc(fl[0]) + __popc(fl[1]) + __popc(fl[2]) + __popc(fl[3]);
    int total;
    int64_t id = (int64_t)base_v[blockIdx.x] + mc_block_scan(mine, &total);
    if (!mine) return;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        if (!fl[m]) continue;
        const int k = k0 + m;
        voff[v0 + m] = (int32_t)id;
        const VT f0 = (VT)g.at(i, j, k);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (!(fl[m] & (1u << a))) continue;
            const VT f1 = (VT)g.at(i + (a == 0), j + (a == 1), k + (a == 2));
            const VT t = (iso - f0) / (f1 - f0);
            VT pi = (VT)i, pj = (VT)j, pk = (VT)k;
            if (a == 0) pi += t; else if (a == 1) pj += t; else pk += t;
            verts[3 * id + 0] = pk;   // x
            verts[3 * id + 1] = pj;   // y
            verts[3 * id + 2] = pi;   // z
            ++id;
        }
    }
}

__global__ void __launch_bounds__(MC_T) k_mc_faces(McGeom q, const int32_t *__restrict__ blk_t,
                                                   const int32_t *__restrict__ base_t,
                                                   const uint8_t *__restrict__ vflags, const uint8_t *__restrict__ vcase,
                                                   const int32_t *__restrict__ voff, int64_t *__restrict__ faces) {
    if (blk_t[blockIdx.x] == 0) return;
    const int G = q.G;
    const int64_t u = (int64_t)blockIdx.x * MC_T + threadIdx.x;
    int i = 0, j = 0, k0 = 0;
    int cs[4] = {0, 0, 0, 0};
    if (u < q.nquads) {
        mc_quad_coords(q, u, i, j, k0);
        const size_t v0 = ((size_t)i * G + j) * G + k0;
#pragma unroll
        for (int m = 0; m < 4; ++m)
            if (k0 + m < G) cs[m] = vcase[v0 + m];
    }
    const int mine = (c_num_verts[cs[0]] + c_num_verts[cs[1]] + c_num_verts[cs[2]] + c_num_verts[cs[3]]) / 3;
    int total;
    int64_t t0 = (int64_t)base_t[blockIdx.x] + mc_block_scan(mine, &total);
    if (!mine) return;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        const int nv = c_num_verts[cs[m]];
        const int k = k0 + m;
        for (int t = 0; t < nv; t += 3) {
            int64_t ids[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int e = c_tri_table[cs[m]][t + c];
                const int oi = i + c_edge_owner[e][0], oj = j + c_edge_owner[e][1], ok = k + c_edge_owner[e][2];
                const int ax = c_edge_owner[e][3];
                const size_t ov = ((size_t)oi * G + oj) * G + ok;
                ids[c] = (int64_t)voff[ov] + __popc((unsigned)vflags[ov] & ((1u << ax) - 1u));
            }
            faces[3 * t0 + 0] = ids[0];
            faces[3 * t0 + 1] = ids[2];
            faces[3 * t0 + 2] = ids[1];
            ++t0;
        }
    }
}

struct McWs {
    int32_t *voff;             // global vertex id of a voxel's first owned vertex (written for owners only)
    uint8_t *vflags, *vcase;   // written for voxels of active blocks only
    int32_t *blk_v, *blk_t;    // per-block totals
    int32_t *base_v, *base_t;  // their exclusive scans
    void *scan_ws;
    int64_t nblocks;
};
static McWs carve_mc(Carver &c, int G) {
    const size_t n = (size_t)G * G * G;
    const McGeom q = make_geom(G);
    McWs w;
    w.nblocks = (q.nquads + MC_T - 1) / MC_T;
    w.voff = c.take<int32_t>(n);
    w.vflags = c.take<uint8_t>(n);
    w.vcase = c.take<uint8_t>(n);
    w.blk_v = c.take<int32_t>(w.nblocks);
    w.blk_t = c.take<int32_t>(w.nblocks);
    w.base_v = c.take<int32_t>(w.nblocks);
    w.base_t = c.take<int32_t>(w.nblocks);
    w.scan_ws = c.take<char>(scan_ws_bytes(w.nblocks));
    return w;
}

}  // namespace icon

using namespace icon;

extern "C" size_t icon_mc_workspace_bytes(int R, int padded) {
    Carver c(nullptr);
    carve_mc(c, padded ? R + 1 : R - 1);
    return c.total();
}

extern "C" int icon_mc_count(const float *occ, int R, double iso, int padded, void *ws, size_t ws_bytes,
                             int64_t *d_counts, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(occ && ws && d_counts && R >= 3 && R <= 1290, "icon_mc_count: bad argument (R=%d)", R);
    static_assert((int64_t)1291 * 1291 * 323 < (int64_t)1 << 31, "quad index must fit 32 bits");
    if (ws_bytes < icon_mc_workspace_bytes(R, padded)) {
        set_error("icon_mc_count: workspace %zu < %zu", ws_bytes, icon_mc_workspace_bytes(R, padded));
        return ICON_ENOSPC;
    }
    McGrid g = make_grid(occ, R, padded);
    Carver c(ws);
    McWs w = carve_mc(c, g.G);
    const McGeom q = make_geom(g.G);
    if (padded)
        k_mc_count<float><<<(unsigned)w.nblocks, MC_T, 0, stream>>>(g, q, (float)iso, w.blk_v, w.blk_t, w.vflags, w.vcase);
    else
        k_mc_count<double><<<(unsigned)w.nblocks, MC_T, 0, stream>>>(g, q, iso, w.blk_v, w.blk_t, w.vflags, w.vcase);
    ICON_LAUNCHED();
    int rc = scan_exclusive_i32(w.blk_v, w.base_v, w.nblocks, d_counts, w.scan_ws, stream);
    if (rc) return rc;
    return scan_exclusive_i32(w.blk_t, w.base_t, w.nblocks, d_counts + 1, w.scan_ws, stream);
}

extern "C" int icon_mc_emit(const float *occ, int R, double iso, int padded, const void *ws, void *verts,
                            int64_t *faces, int64_t n_verts, int64_t n_tris, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (n_verts == 0 && n_tris == 0) return ICON_OK;
    ICON_CHECK_ARG(occ && ws && verts && faces, "icon_mc_emit: null pointer");
    McGrid g = make_grid(occ, R, padded);
    Carver c((void *)ws);
    McWs w = carve_mc(c, g.G);
    const McGeom q = make_geom(g.G);
    if (n_verts > 0) {
        if (padded)
            k_mc_verts<float><<<(unsigned)w.nblocks, MC_T, 0, stream>>>(g, q, (float)iso, w.blk_v, w.base_v, w.vflags, w.voff,
                                                                        (float *)verts);
        else
            k_mc_verts<double><<<(unsigned)w.nblocks, MC_T, 0, stream>>>(g, q, iso, w.blk_v, w.base_v, w.vflags, w.voff,
                                                                         (double *)verts);
        ICON_LAUNCHED();
    }
    if (n_tris > 0) k_mc_faces<<<(unsigned)w.nblocks, MC_T, 0, stream>>>(q, w.blk_t, w.base_t, w.vflags, w.vcase, w.voff,
                                                                        faces);
    ICON_LAUNCHED();
    return ICON_OK;
}
