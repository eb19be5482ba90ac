// SMPL-body SDF block of the occupancy query.  Compiled with -fmad=false.
//
// Replaces, per query point (reference: cal_sdf_batch, lib/dataset/mesh_util.py:357-396):
//   kaolin point_to_mesh_distance  -> nearest face (lowest index on ties) + squared distance
//   kaolin check_sign              -> +x ray parity
//   barycentric_coordinates_of_projection + the four gathers -> cmap / normal / vis
//
// Design (DESIGN.md 4.2): one WARP per group of PPW query points (32 Morton-adjacent lattice points on the dense grid).
//   nearest face  the tree walk of face_tree.cuh over the body's tree (icon_smpl_prepare), descending towards the
//                 warp centre, with a 16-bit frontier and the fixed slacks of coordinates of magnitude ~1.
//                 Dense lattices (PPW = 32) replace its phases A and B by a per-body face list of the warp's brick
//                 (32^3 bricks over [-1,1]^3, built by the body's first dense call), sorted by distance, so phase C
//                 can stop early.
//   sign          the faces listed in the point's yz cell (256 x 256 grid over the mesh's yz
//                 box) are the only ones a +x ray can hit; each is tested with the same
//                 Moller-Trumbore code as the brute-force scan, so the hit COUNT is identical.
// Results are identical to brute force over all faces (icon_sdf_bruteforce, the CPU oracle):
// the pruning is conservative and the per-face arithmetic is the same code (geom.cuh).
#include <float.h>

#include <algorithm>
#include <mutex>
#include <type_traits>
#include <unordered_set>
#include <vector>

#include "common.cuh"
#include "face_tree.cuh"
#include "geom.cuh"

namespace icon {

struct Calib {
    float r[9];
    float t[3];
};

__device__ __forceinline__ V3 load_point(const float *__restrict__ pts, int64_t sc, int64_t sn,
                                         int64_t i, const Calib &cb) {
    float px = pts[i * sn], py = pts[sc + i * sn], pz = pts[2 * sc + i * sn];
    V3 o;
    o.x = fmaf(cb.r[2], pz, fmaf(cb.r[1], py, cb.r[0] * px)) + cb.t[0];
    o.y = fmaf(cb.r[5], pz, fmaf(cb.r[4], py, cb.r[3] * px)) + cb.t[1];
    o.z = fmaf(cb.r[8], pz, fmaf(cb.r[7], py, cb.r[6] * px)) + cb.t[2];
    return o;
}

// cmap / normal / vis of the winning face + final sdf; mirrors the tail of oracle_cal_sdf().
__device__ __forceinline__ void emit_record(V3 p, int bi, float best, int hits, const MeshView &m,
                                            float *__restrict__ rec, int32_t *__restrict__ face,
                                            int64_t idx) {
    Tri t = load_tri(m.tri + 3 * (size_t)bi);
    V3 n = cross3(t.ab, t.ac);
    float s = n.x * n.x + n.y * n.y + n.z * n.z;
    if (s == 0.f) s = 1e-6f;
    float inv = 1.0f / s;
    V3 w = sub3(p, t.a);
    V3 uw = cross3(t.ab, w), wv = cross3(w, t.ac);
    float b2 = (uw.x * n.x + uw.y * n.y + uw.z * n.z) * inv;
    float b1 = (wv.x * n.x + wv.y * n.y + wv.z * n.z) * inv;
    float b0 = 1.0f - b1 - b2;
    const float4 *at = m.attr + 6 * (size_t)bi;
    float4 a0 = __ldg(at), a1 = __ldg(at + 1), a2 = __ldg(at + 2), a3 = __ldg(at + 3),
           a4 = __ldg(at + 4), a5 = __ldg(at + 5);
    // normals n0=(a0.x,a0.y,a0.z) n1=(a0.w,a1.x,a1.y) n2=(a1.z,a1.w,a2.x)
    float nx = (a0.x * b0 + a0.w * b1 + a1.z * b2) * -1.f;
    float ny = (a0.y * b0 + a1.x * b1 + a1.w * b2) * 1.f;
    float nz = (a0.z * b0 + a1.y * b1 + a2.x * b2) * -1.f;
    // cmap m0=(a2.y,a2.z,a2.w) m1=(a3.x,a3.y,a3.z) m2=(a3.w,a4.x,a4.y)
    float cx = a2.y * b0 + a3.x * b1 + a3.w * b2;
    float cy = a2.z * b0 + a3.y * b1 + a4.x * b2;
    float cz = a2.w * b0 + a3.z * b1 + a4.y * b2;
    float vv = a4.z * b0 + a4.w * b1 + a5.x * b2;
    float vis = vv >= 0.1f ? 1.f : 0.f;
    float dist = sqrtf(best) / sqrtf(3.0f);
    float sign = 2.0f * ((float)(hits & 1) - 0.5f);
    float sdf = dist * sign;
    float4 *r = (float4 *)(rec + 8 * idx);
    r[0] = make_float4(sdf, cx, cy, cz);
    r[1] = make_float4(nx, ny, nz, vis);
    if (face) face[idx] = bi;
}

constexpr int SW_T = 128;               // 4 warps per block, one warp = 32 Morton-adjacent points
constexpr int NBIN_AX = 128;            // Morton bins per axis over [-1,1]^3 (+1 overflow bin)
constexpr int NBIN = NBIN_AX * NBIN_AX * NBIN_AX;
// frontier / leaf list capacity per warp: the fewer points a warp carries the tighter its box and the shorter the
// lists, and the smaller footprint lets more warps be resident to hide the tree walk's dependent loads
__host__ __device__ constexpr int fr_cap(int ppw) { return ppw >= 16 ? 1024 : (ppw >= 4 ? 768 : 384); }

__device__ __forceinline__ unsigned spread7(unsigned v) {      // <= 10 bits -> every third bit
    v = (v | (v << 16)) & 0x030000FFu;
    v = (v | (v << 8)) & 0x0300F00Fu;
    v = (v | (v << 4)) & 0x030C30C3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}

__device__ __forceinline__ int bin_of(V3 p) {
    const bool inside = p.x >= -1.f && p.x <= 1.f && p.y >= -1.f && p.y <= 1.f && p.z >= -1.f && p.z <= 1.f;
    if (!inside) return NBIN;
    const unsigned bx = min(NBIN_AX - 1, (int)((p.x + 1.f) * (NBIN_AX * 0.5f)));
    const unsigned by = min(NBIN_AX - 1, (int)((p.y + 1.f) * (NBIN_AX * 0.5f)));
    const unsigned bz = min(NBIN_AX - 1, (int)((p.z + 1.f) * (NBIN_AX * 0.5f)));
    return (int)(spread7(bx) | (spread7(by) << 1) | (spread7(bz) << 2));
}

// xyz4[i] = (x, y, z, in_cube); bid[i] = Morton bin; count[bin]++ (warp-aggregated atomics)
__global__ void k_points_bin(const float *__restrict__ pts, int64_t sc, int64_t sn, int64_t N, Calib cb,
                             float4 *__restrict__ xyz4, int32_t *__restrict__ bid, int32_t *__restrict__ count) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < N;
    int b = -1;
    if (live) {
        const V3 p = load_point(pts, sc, sn, i, cb);
        // HGPIFuNet.py:270-275: in_cube = all(-1 < xyz < 1), strict
        const float in_cube = (p.x > -1.f && p.x < 1.f && p.y > -1.f && p.y < 1.f && p.z > -1.f && p.z < 1.f) ? 1.f : 0.f;
        xyz4[i] = make_float4(p.x, p.y, p.z, in_cube);
        b = bin_of(p);
        bid[i] = b;
    }
    const unsigned act = __ballot_sync(0xffffffffu, live);
    if (live) {
        const unsigned peers = __match_any_sync(act, b);
        if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&count[b], __popc(peers));
    }
}

__global__ void k_points_scatter(const int32_t *__restrict__ bid, int64_t N, const int32_t *__restrict__ offset,
                                 int32_t *__restrict__ cursor, int32_t *__restrict__ perm) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < N;
    const int b = live ? bid[i] : -1;
    const unsigned act = __ballot_sync(0xffffffffu, live);
    if (live) {
        const unsigned peers = __match_any_sync(act, b);
        const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(&cursor[b], __popc(peers));
        base = __shfl_sync(peers, base, leader);
        perm[offset[b] + base + __popc(peers & ((1u << lane) - 1u))] = (int32_t)i;
    }
}

#ifdef ICON_SDF_STATS
// Diagnostics build only (tools/sdf_brick_counters.py).  g_stats: warps, overflow warps, face-list entries (brick
// path) or leaves (tree walk), faces staged, then the deferred tree walk's warps and cycles.  g_wstat: one record of
// WS_N words per brick-path warp.
__device__ unsigned long long g_stats[8];
__device__ unsigned *g_wstat;
enum { WS_DEFER, WS_ENTRIES, WS_STEPS, WS_STAGED, WS_SPH, WS_EXACT, WS_WIN, WS_RAY, WS_CYC_START, WS_CYC_C,
       WS_CYC_RAY, WS_CYC_EMIT, WS_UB0, WS_UBEND, WS_LIST, WS_IDEAL_ENTRIES, WS_IDEAL_FACES, WS_DEAD, WS_N = 20 };
#define STAT(i, v) do { if (lane == 0) atomicAdd(&g_stats[i], (unsigned long long)(v)); } while (0)
#define WSTAT(i, v) do { if (lane == 0 && g_wstat) g_wstat[(size_t)wid * WS_N + (i)] = (unsigned)(v); } while (0)
#define WCLK(t) __syncwarp(); const long long t = clock64()
#else
#define STAT(i, v) do { } while (0)
#define WSTAT(i, v) do { } while (0)
#endif

// 16-bit frontier ids: icon_smpl_prepare checks that the leaf count is <= 65535.  The brick path reads its face list
// from global memory and needs no frontier (a third of the shared memory; at 64 registers per thread, registers then
// bound residency at 32 warps per SM)
template <int PPW, bool BRICK>
using SdfSmem = typename std::conditional<BRICK, ChunkSmem, WalkSmem<unsigned short, fr_cap(PPW)>>::type;
template <int PPW, bool BRICK>
constexpr size_t sdf_smem_bytes() { return sizeof(SdfSmem<PPW, BRICK>) * (SW_T / 32); }

constexpr float BRICK_W = 2.0f / BRICK_AX;           // brick corners -1 + i / 16 are exact floats
constexpr float BRICK_HALF_DIAG = 0.0541266f;        // > BRICK_W * sqrt(3) / 2 = 0.05412659

// brick b = (bz * 32 + by) * 32 + bx covers [-1 + bx W, -1 + (bx + 1) W] x ...
__device__ __forceinline__ void brick_box(int b, float4 &lo, float4 &hi) {
    const int bx = b % BRICK_AX, by = (b / BRICK_AX) % BRICK_AX, bz = b / (BRICK_AX * BRICK_AX);
    lo = make_float4(-1.f + bx * BRICK_W, -1.f + by * BRICK_W, -1.f + bz * BRICK_W, 0.f);
    hi = make_float4(-1.f + (bx + 1) * BRICK_W, -1.f + (by + 1) * BRICK_W, -1.f + (bz + 1) * BRICK_W, 0.f);
}

// squared distance between the box of leaf l and a brick: the build's sort key, recomputed bit for bit by the kernel
__device__ __forceinline__ float leaf_key(const MeshView &m, int l, float4 lo, float4 hi) {
    const float4 a = __ldg(m.nodes + 2 * (size_t)l), z = __ldg(m.nodes + 2 * (size_t)l + 1);
    const float gx = fmaxf(fmaxf(a.x - hi.x, lo.x - z.x), 0.f);
    const float gy = fmaxf(fmaxf(a.y - hi.y, lo.y - z.y), 0.f);
    const float gz = fmaxf(fmaxf(a.z - hi.z, lo.z - z.z), 0.f);
    return fmaf(gz, gz, fmaf(gy, gy, gx * gx));
}

// PPW = query points per warp; each point is replicated on REP = 32/PPW lanes which split the candidate faces
// (and the ray list) between them and merge by shuffle.  32: one point per lane, for dense sets where 32 Morton-
// consecutive points fill a small box.  8 / 1: for the engine's sparse refinement sets, where 32 consecutive points
// span a large box and the shared candidate list explodes; with PPW = 1 the warp box is a point, the lists are the
// per-point minimum and the 32 lanes only share the work.  The kernel is bound by the latency of the dependent
// tree loads, so the shared-memory footprint (fr_cap) is kept small enough for >= 36 resident warps per SM.
// BRICK (PPW = 32, dense lattices): a warp whose box lies inside one brick skips phases A and B: its first bound is
// the brick's, its first candidate the face nearest the brick centre, and phase C scans the brick's face list.
template <int PPW, bool BRICK>
__device__ __forceinline__ void sdf_warp(int64_t wid, SdfSmem<PPW, BRICK> &S, const float4 *__restrict__ xyz4,
                                         const int32_t *__restrict__ perm, int64_t N, const MeshView &m,
                                         float *__restrict__ rec, int32_t *__restrict__ face,
                                         int32_t *__restrict__ defer, int32_t *__restrict__ ndefer) {
    constexpr int REP = 32 / PPW;
    const int lane = threadIdx.x & 31;
    const int sub = lane % PPW, rep_id = lane / PPW;           // which point of the warp, which replica
    const int64_t pos0 = wid * PPW;
    const int64_t pos = pos0 + sub;
    if (pos0 >= N) return;                                   // whole warp out of range
    const bool live = pos < N;
    const int64_t idx = perm[live ? pos : pos0];
    const float4 q = xyz4[idx];
    const V3 p = mk3(q.x, q.y, q.z);
    // warp bounding sphere (box centre, max distance)
    const V3 c = mk3(0.5f * (warp_min(p.x) + warp_max(p.x)), 0.5f * (warp_min(p.y) + warp_max(p.y)),
                     0.5f * (warp_min(p.z) + warp_max(p.z)));
    const float rw = warp_max(sqrtf(dot3(sub3(p, c), sub3(p, c)))) * 1.00001f + 1e-6f;
    // the warp's bounding box (tighter than the sphere for the flat 4x4x2 blocks of a lattice)
    const float4 wlo = make_float4(warp_min(p.x) - 1e-6f, warp_min(p.y) - 1e-6f, warp_min(p.z) - 1e-6f, 0.f);
    const float4 whi = make_float4(warp_max(p.x) + 1e-6f, warp_max(p.y) + 1e-6f, warp_max(p.z) + 1e-6f, 0.f);
    const MeshHeader h = *m.hdr;

    // the body lies in [-1.5, 1.5]^3 and the points that matter in [-1, 1]^3: the walk's fixed slacks
    NearestFace<PPW> nf(p, 1e-6f, 1e-7f);
#ifdef ICON_SDF_STATS
    WCLK(t_start);
    long long t_c = 0, t_ray = 0;
    int st_entries = 0, st_steps = 0, st_brick = -1;
    float st_ub0 = 0.f;
#endif
    if constexpr (BRICK) {
        bool ok = h.brick_built && !h.brick_overflow && c.x >= -1.f && c.x < 1.f && c.y >= -1.f && c.y < 1.f &&
                  c.z >= -1.f && c.z < 1.f;
        int b = 0;
        float4 blo, bhi;
        if (ok) {
            const int bx = min(BRICK_AX - 1, (int)((c.x + 1.f) * (BRICK_AX * 0.5f)));
            const int by = min(BRICK_AX - 1, (int)((c.y + 1.f) * (BRICK_AX * 0.5f)));
            const int bz = min(BRICK_AX - 1, (int)((c.z + 1.f) * (BRICK_AX * 0.5f)));
            b = (bz * BRICK_AX + by) * BRICK_AX + bx;
            brick_box(b, blo, bhi);
            ok = wlo.x >= blo.x && wlo.y >= blo.y && wlo.z >= blo.z && whi.x <= bhi.x && whi.y <= bhi.y && whi.z <= bhi.z;
        }
        if (!ok) {                     // straddles bricks, leaves the cube or the lists overflowed: the tree walk takes it
            if (lane == 0) defer[atomicAdd(ndefer, 1)] = (int32_t)wid;
            WSTAT(WS_DEFER, 1);
            return;
        }
        const int f = __ldg(m.bface + b);
        nf.try_face(m.tri + 3 * (size_t)f, f);                // not taken if NaN here; the brick's bound still holds
        nf.start_scan(fminf(warp_max(sqrtf(nf.best)), __ldg(m.bub + b)), wlo, whi);
        STAT(0, 1);
#ifdef ICON_SDF_STATS
        WCLK(t_c0);
        t_c = t_c0;
        st_brick = b;
        st_ub0 = nf.ub;
#endif
        // the keys bound from below every lane's distance to the face and ascend along the list: once a step's
        // first key is farther than the loosest lane bound, so is the rest of the list
        const int o1 = __ldg(m.foff + b + 1);
        for (int base = __ldg(m.foff + b); base < o1; base += 32) {
            const int slot = base + lane;
            const bool in = slot < o1;
            const int k = in ? (int)__ldg(m.flist + slot) : -1;
            const float key = in ? __ldg(m.fkey + slot) : 0.f;
            if (__shfl_sync(0xffffffffu, key, 0) > nf.ub * nf.ub) break;
            STAT(2, min(32, o1 - base));
#ifdef ICON_SDF_STATS
            st_entries += min(32, o1 - base);
            ++st_steps;
#endif
            nf.chunk(m, S, k, wlo, whi);
        }
        nf.merge();
    } else {
        const int n = tree_nearest(m, S, nf, c, rw, wlo, whi);
        STAT(0, 1); STAT(1, n > fr_cap(PPW) ? 1 : 0); STAT(2, n);
    }
    STAT(3, nf.staged);
#ifdef ICON_SDF_STATS
    WCLK(t_c1);
    int st_ray = 0;
#endif
    // ---- +x ray parity
    int hits = 0;
    if (!h.ray_overflow) {
        const float fy = (p.y - h.y0) * h.inv_cy, fz = (p.z - h.z0) * h.inv_cz;
        if (fy >= 0.f && fy < (float)RAY_GRID && fz >= 0.f && fz < (float)RAY_GRID) {
            const int cc = (int)fz * RAY_GRID + (int)fy;
            const int k0 = __ldg(m.roff + cc), k1 = __ldg(m.roff + cc + 1);
            for (int k = k0 + rep_id; k < k1; k += REP) {
                const int f = __ldg(m.rlist + k);
                if (__ldg(&m.rbox[2 * (size_t)f + 1].x) < p.x - 1e-3f) continue;     // wholly behind the ray origin
                const Tri tr = load_tri(m.tri + 3 * (size_t)f);
                hits += ray_hit_px(p, tr.a, tr.ab, tr.ac);
#ifdef ICON_SDF_STATS
                ++st_ray;
#endif
            }
        }
    } else {
        for (int f = rep_id; f < m.F; f += REP) {
            const Tri tr = load_tri(m.tri + 3 * (size_t)f);
            hits += ray_hit_px(p, tr.a, tr.ab, tr.ac);
        }
    }
    if (REP > 1) {
#pragma unroll
        for (int o = PPW; o < 32; o <<= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
    }
#ifdef ICON_SDF_STATS
    WCLK(t_ray0);
    t_ray = t_ray0;
#endif
    if (live && rep_id == 0) emit_record(p, nf.bi, nf.best, hits, m, rec, face, idx);
#ifdef ICON_SDF_STATS
    WCLK(t_end);
    if (BRICK && st_brick >= 0) {
        // at the final bound: list entries the break alone keeps, and faces whose sphere lies within it of the box
        const float ube = nf.ub;
        int il = 0, ifc = 0;
        const int o0 = __ldg(m.foff + st_brick), o1 = __ldg(m.foff + st_brick + 1);
        for (int s = o0 + lane; s < o1; s += 32) {
            il += __ldg(m.fkey + s) <= ube * ube;
            const float4 s4 = __ldg(m.sph_s + __ldg(m.flist + s));
            const float l2 = ube + s4.w;
            ifc += box_dist2(mk3(s4.x, s4.y, s4.z), wlo, whi) <= l2 * l2;
        }
        const int s_sph = __reduce_add_sync(0xffffffffu, nf.n_sph), s_exact = __reduce_add_sync(0xffffffffu, nf.n_exact);
        const int s_win = __reduce_add_sync(0xffffffffu, nf.n_win), s_ray = __reduce_add_sync(0xffffffffu, st_ray);
        const int s_il = __reduce_add_sync(0xffffffffu, il), s_if = __reduce_add_sync(0xffffffffu, ifc);
        WSTAT(WS_ENTRIES, st_entries);
        WSTAT(WS_STEPS, st_steps);
        WSTAT(WS_STAGED, nf.staged);
        WSTAT(WS_SPH, s_sph);
        WSTAT(WS_EXACT, s_exact);
        WSTAT(WS_WIN, s_win);
        WSTAT(WS_RAY, s_ray);
        WSTAT(WS_CYC_START, t_c - t_start);
        WSTAT(WS_CYC_C, t_c1 - t_c);
        WSTAT(WS_CYC_RAY, t_ray - t_c1);
        WSTAT(WS_CYC_EMIT, t_end - t_ray);
        WSTAT(WS_UB0, __float_as_uint(st_ub0));
        WSTAT(WS_UBEND, __float_as_uint(ube));
        WSTAT(WS_LIST, o1 - o0);
        WSTAT(WS_IDEAL_ENTRIES, s_il);
        WSTAT(WS_IDEAL_FACES, s_if);
        WSTAT(WS_DEAD, nf.n_dead);
    }
    if (!BRICK && defer != nullptr) { STAT(4, 1); STAT(5, t_end - t_start); }
#endif
}

// PPW = 32 is held to 64 registers (8 blocks, 32 warps per SM; about 50 bytes of spill): sdf_only on the 256^3 lattice
// measured 4.65 ms against 5.2 ms at 79 registers and 24 warps (H100 80GB HBM3, 700 W).  The other PPWs keep the
// compiler's choice (a minimum of 0 blocks is no bound).
// Without `defer`, warp i of the grid takes the points of warp i.  BRICK appends the warps it leaves to the tree walk
// to defer[] (count *ndefer); the tree walk given `defer` strides over those warps instead.
template <int PPW, bool BRICK>
__global__ void __launch_bounds__(SW_T, PPW == 32 ? 8 : 0) k_sdf_warp(const float4 *__restrict__ xyz4, const int32_t *__restrict__ perm,
                                                   int64_t N, MeshView m, float *__restrict__ rec,
                                                   int32_t *__restrict__ face, int32_t *__restrict__ defer,
                                                   int32_t *__restrict__ ndefer) {
    static_assert(!BRICK || PPW == 32, "brick lists serve dense lattices: 32 points per warp");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SdfSmem<PPW, BRICK> &S = reinterpret_cast<SdfSmem<PPW, BRICK> *>(smem_raw)[threadIdx.x >> 5];
    const bool listed = !BRICK && defer != nullptr;
    const int64_t nw = listed ? (int64_t)*ndefer : (N + PPW - 1) / PPW;
    for (int64_t i = (int64_t)blockIdx.x * (SW_T / 32) + (threadIdx.x >> 5); i < nw; i += (int64_t)gridDim.x * (SW_T / 32))
        sdf_warp<PPW, BRICK>(listed ? (int64_t)defer[i] : i, S, xyz4, perm, N, m, rec, face, defer, ndefer);
}

// ---------------------------------------------------------------- brick face lists (built once per body)
__global__ void k_brick_centres(MeshView m) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= NBRICK) return;
    float4 lo, hi;
    brick_box(b, lo, hi);
    m.bxyz[b] = make_float4(0.5f * (lo.x + hi.x), 0.5f * (lo.y + hi.y), 0.5f * (lo.z + hi.z), 0.f);
    m.bperm[b] = b;
}

// Block gather: put(at, key, tag) for the items i of [0, n) that take(i, key, tag) keeps, at = 0, 1, ... in no
// particular order (*s_n = 0 before the call, which starts with a barrier); returns how many were kept.  The order is
// restored by rank_sort, so no barrier per chunk of items is needed.
template <class Take, class Put>
__device__ __forceinline__ int block_gather(int n, int *s_n, Take &&take, Put &&put) {
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        float key;
        int tag;
        if (take(i, key, tag)) put(atomicAdd(s_n, 1), key, tag);
    }
    __syncthreads();
    return *s_n;
}

// A key >= +0 (never NaN or -0) and a distinct 16-bit tag as one word whose unsigned order is (key, tag): the bits of
// a non-negative float order like its value
__device__ __forceinline__ unsigned long long key_tag(float key, int tag) {
    return (unsigned long long)__float_as_uint(key) << 32 | (unsigned)tag;
}

// Rank sort of the distinct words s_kt[0, n), ascending: put(rank, i) for every i
template <class Put>
__device__ __forceinline__ void rank_sort(const unsigned long long *s_kt, int n, Put &&put) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long x = s_kt[i];
        int r = 0;
        for (int j = 0; j < n; ++j) r += s_kt[j] < x;
        put(r, i);
    }
}

// A bound beta + g.(p - pc) >= D(p) over the brick's box [lo, hi] (centre pc), D the distance to the mesh, for `beats`
// with the brick as the box.  The distance to the face nearest the brick centre bounds D from above and is convex (the
// face is a convex set), so on the box it lies below the trilinear blend of its corner values d_i, which lies below
// beta + g.(p - pc) once beta >= d_i - g.(c_i - pc) at every corner.  g is the least-squares slope of the corner values,
// clamped to [-1, 1] per axis like start_scan's; any finite g keeps the bound.
__device__ __forceinline__ void brick_plane(const MeshView &m, int b, float4 lo, float4 hi, NearestFace<32> &nf) {
    const Tri t = load_tri(m.tri + 3 * (size_t)__ldg(m.bface + b));
    float d[8], sx = 0.f, sy = 0.f, sz = 0.f;
    for (int i = 0; i < 8; ++i) {
        const V3 c = mk3(i & 1 ? hi.x : lo.x, i & 2 ? hi.y : lo.y, i & 4 ? hi.z : lo.z);
        d[i] = sqrtf(tri_sqdist(c, t.a, t.ab, t.ac)) * 1.00001f + 1e-6f;
        sx += i & 1 ? d[i] : -d[i];
        sy += i & 2 ? d[i] : -d[i];
        sz += i & 4 ? d[i] : -d[i];
    }
    const float h = 0.5f * BRICK_W;
    nf.g = mk3(fminf(fmaxf(sx / (8.f * h), -1.f), 1.f), fminf(fmaxf(sy / (8.f * h), -1.f), 1.f),
               fminf(fmaxf(sz / (8.f * h), -1.f), 1.f));
    float beta = -FLT_MAX;
    for (int i = 0; i < 8; ++i)
        beta = fmaxf(beta, d[i] - ((i & 1 ? nf.g.x : -nf.g.x) + (i & 2 ? nf.g.y : -nf.g.y) + (i & 4 ? nf.g.z : -nf.g.z)) * h);
    nf.beta = beta;                    // NaN (a degenerate face): beats() never culls
}

// candidate j of the brick's leaves (4 faces per leaf) if `beats` cannot rule it out for any point of the brick:
// its sorted position and key, a squared lower bound on the distance from any point of the brick to the face
__device__ __forceinline__ bool brick_face(const MeshView &m, const unsigned short *leaves, int j, float4 lo, float4 hi,
                                           const NearestFace<32> &nf, int &k, float &key) {
    k = 4 * (int)leaves[j / 4] + (j & 3);
    if (k >= m.F) return false;
    const float4 s = __ldg(m.sph_s + k);
    const float4 *tp = m.tri_s + 3 * (size_t)k;
    if (nf.beats(s, __ldg(tp), __ldg(tp + 1), __ldg(tp + 2), lo, hi)) return false;
    const float gap = sqrtf(box_dist2(mk3(s.x, s.y, s.z), lo, hi)) * 0.99999f - s.w - 1e-6f;
    key = gap > 0.f ? gap * gap : 0.f;
    return true;
}

// One CTA per brick.  The brick's leaves are those whose box lies within its bound U_b (every point of the brick is
// within sqrt(d) + half-diagonal of the face nearest its centre) of the brick's box, gathered into shared memory; its
// face list keeps the faces of those leaves that `beats` cannot rule out for any point of the brick.
// Count pass (!FILL): U_b into bub and the list's length into foff; more than BRICK_MAX_LEAVES leaves, a list past
// BRICK_MAX_FACES or more than 65535 faces (uint16 positions) marks the lists overflowed.  Fill pass, after the scan:
// the leaves rank-sorted by key (ties: leaf id), then the kept faces, tagged with their candidate position j over the
// sorted leaves, rank-sorted by key (ties: j) into flist / fkey.  Both orders are those of an in-order compaction.
template <bool FILL>
__global__ void __launch_bounds__(128) k_brick_faces(MeshView m, int64_t fcap) {
    static_assert(BRICK_MAX_FACES <= BRICK_MAX_LEAVES, "the face stage reuses the leaf array");
    static_assert(4 * BRICK_MAX_LEAVES <= 65536, "candidate positions are 16-bit tags");
    // count: the leaf ids; fill: (key, leaf id), then (key, candidate position j) of the faces, and the leaf ids in
    // key order
    __shared__ unsigned short s_leaf[BRICK_MAX_LEAVES];
    __shared__ unsigned long long s_kt[FILL ? BRICK_MAX_LEAVES : 1];
    __shared__ int s_n[2];                                // gathered leaves, faces
    if (FILL && (m.hdr->brick_overflow || m.foff[NBRICK] > fcap)) return;    // k_brick_done records the overflow
    if (threadIdx.x == 0) s_n[0] = s_n[1] = 0;
    const int b = blockIdx.x;
    float4 lo, hi;
    brick_box(b, lo, hi);
    float ub;
    if (FILL) {
        ub = m.bub[b];
    } else {
        const float4 cc = m.bxyz[b];
        const Tri t = load_tri(m.tri + 3 * (size_t)m.bface[b]);
        const float d = tri_sqdist(mk3(cc.x, cc.y, cc.z), t.a, t.ab, t.ac);
        ub = (sqrtf(d) + BRICK_HALF_DIAG) * 1.00001f + 1e-6f;
    }
    const float ub2 = ub * ub;
    const int n = block_gather(m.lvl_cnt[0], &s_n[0], [&](int l, float &key, int &tag) {
        key = leaf_key(m, l, lo, hi);
        tag = l;
        return key <= ub2;
    }, [&](int at, float key, int tag) {
        if (at >= BRICK_MAX_LEAVES) return;
        if (FILL) s_kt[at] = key_tag(key, tag);
        else s_leaf[at] = (unsigned short)tag;
    });
    NearestFace<32> nf(mk3(0.f, 0.f, 0.f), 1e-6f, 1e-7f);
    brick_plane(m, b, lo, hi, nf);
    if constexpr (!FILL) {
        const bool fits = n <= BRICK_MAX_LEAVES && m.F <= 65535;
        int cnt = 0, k;
        float key;
        if (fits)
            for (int j = threadIdx.x; j < 4 * n; j += blockDim.x) cnt += brick_face(m, s_leaf, j, lo, hi, nf, k, key);
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if ((threadIdx.x & 31) == 0) atomicAdd(&s_n[1], cnt);
        __syncthreads();
        if (threadIdx.x == 0) {
            m.bub[b] = ub;
            m.foff[b] = s_n[1];
            if (!fits || s_n[1] > BRICK_MAX_FACES) m.hdr->brick_overflow = 1;
            if (b == 0) m.foff[NBRICK] = 0;
        }
    } else {
        rank_sort(s_kt, n, [&](int r, int i) { s_leaf[r] = (unsigned short)s_kt[i]; });
        const int f0 = m.foff[b];
        const int nkept = block_gather(4 * n, &s_n[1], [&](int j, float &key, int &tag) {
            int k;
            tag = j;
            return brick_face(m, s_leaf, j, lo, hi, nf, k, key);
        }, [&](int at, float key, int tag) { if (at < BRICK_MAX_FACES) s_kt[at] = key_tag(key, tag); });
        rank_sort(s_kt, nkept, [&](int r, int i) {
            const unsigned long long x = s_kt[i];
            const int j = (int)(x & 0xffffu);
            m.flist[f0 + r] = (unsigned short)(4 * s_leaf[j / 4] + (j & 3));
            m.fkey[f0 + r] = __uint_as_float((unsigned)(x >> 32));
        });
    }
}

__global__ void k_brick_done(MeshView m, int64_t fcap) {
    if (m.foff[NBRICK] > fcap) m.hdr->brick_overflow = 1;
    m.hdr->brick_built = 1;
}

// brute force: every point against every face, faces staged through shared memory
__global__ void __launch_bounds__(256) k_sdf_brute(const float *__restrict__ pts, int64_t sc, int64_t sn,
                                                   int64_t N, Calib cb, MeshView m,
                                                   float *__restrict__ rec, int32_t *__restrict__ face) {
    __shared__ float4 tile[3 * 256];
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool live = i < N;
    V3 p = mk3(0.f, 0.f, 0.f);
    if (live) p = load_point(pts, sc, sn, i, cb);
    float best = FLT_MAX;
    int bi = 0, hits = 0;
    for (int f0 = 0; f0 < m.F; f0 += 256) {
        int nf = min(256, m.F - f0);
        __syncthreads();
        for (int k = threadIdx.x; k < 3 * nf; k += 256) tile[k] = m.tri[3 * (size_t)f0 + k];
        __syncthreads();
        if (live) {
            for (int k = 0; k < nf; ++k) {
                float4 r0 = tile[3 * k], r1 = tile[3 * k + 1], r2 = tile[3 * k + 2];
                V3 a = mk3(r0.x, r0.y, r0.z), ab = mk3(r0.w, r1.x, r1.y), ac = mk3(r1.z, r1.w, r2.x);
                float d = tri_sqdist(p, a, ab, ac);
                if (d < best) { best = d; bi = f0 + k; }
                hits += ray_hit_px(p, a, ab, ac);
            }
        }
    }
    if (live) emit_record(p, bi, best, hits, m, rec, face, i);
}

// points-per-warp policy of k_sdf_warp (see its header comment); icon_set_sdf_policy() overrides it for tuning
static int64_t g_sdf_ppw32_from = 6000000, g_sdf_ppw8_from = 300000;
static int g_sdf_ppw_force = 0;
static int g_sdf_bricks = 1;              // brick face lists on PPW = 32 calls (icon_set_sdf_bricks)
static int64_t g_brick_max_entries = 0;   // > 0: a build may use at most this many face-list entries

// Prepared bodies whose brick lists have been enqueued, by mesh header.  icon_smpl_prepare forgets its workspace, so
// a new body -- also one that reuses freed memory -- gets fresh lists.  The kernel itself only trusts the header.
static std::mutex g_brick_mu;
static std::unordered_set<const void *> g_brick_ready;
static int64_t g_brick_builds = 0;

void bricks_forget(const MeshView &m) {
    std::lock_guard<std::mutex> lk(g_brick_mu);
    g_brick_ready.erase(m.hdr);
}

// ---------------------------------------------------------------- host-side pipeline pieces
struct SdfWs {
    float4 *xyz4;
    int32_t *bid, *perm, *count, *offset;
    int32_t *defer, *ndefer;              // warps the brick path leaves to the tree walk
    void *scan_ws;
};
static SdfWs carve_sdf(Carver &c, int64_t N) {
    SdfWs w;
    w.xyz4 = c.take<float4>((size_t)N);
    w.bid = c.take<int32_t>((size_t)N);
    w.perm = c.take<int32_t>((size_t)N);
    w.count = c.take<int32_t>(NBIN + 1);
    w.offset = c.take<int32_t>(NBIN + 1);
    w.defer = c.take<int32_t>((size_t)(N + 31) / 32);
    w.ndefer = c.take<int32_t>(1);
    w.scan_ws = c.take<char>(scan_ws_bytes(NBIN + 1));
    return w;
}

// The brick lists of one body (DESIGN.md 4.2): the exact nearest face of each brick centre (the SDF kernel on the 32768
// centres) bounds the nearest distance of every point of the brick; count, scan and fill the faces that `beats`
// cannot rule out for the whole brick among the leaves within that bound, each list sorted by key.  Stream-ordered:
// the header's flag is set last.
static int build_bricks(const MeshView &m, cudaStream_t stream) {
    const int64_t fcap = g_brick_max_entries > 0 ? std::min(g_brick_max_entries, m.face_cap) : m.face_cap;
    k_brick_centres<<<NBRICK / 256, 256, 0, stream>>>(m);
    ICON_LAUNCHED();
    k_sdf_warp<1, false><<<NBRICK / (SW_T / 32), SW_T, sdf_smem_bytes<1, false>(), stream>>>(
        m.bxyz, m.bperm, NBRICK, m, m.brec, m.bface, nullptr, nullptr);
    ICON_LAUNCHED();
    k_brick_faces<false><<<NBRICK, 128, 0, stream>>>(m, fcap);
    ICON_LAUNCHED();
    const int rc = scan_exclusive_i32(m.foff, m.foff, NBRICK + 1, nullptr, m.scan_ws, stream);
    if (rc) return rc;
    k_brick_faces<true><<<NBRICK, 128, 0, stream>>>(m, fcap);
    ICON_LAUNCHED();
    k_brick_done<<<1, 1, 0, stream>>>(m, fcap);
    ICON_LAUNCHED();
    return ICON_OK;
}
size_t sdf_ws_bytes(int64_t N) {
    Carver c(nullptr);
    carve_sdf(c, N);
    return c.total();
}

Calib make_calib(const float *h) {
    Calib cb;
    for (int r = 0; r < 3; ++r) {
        for (int k = 0; k < 3; ++k) cb.r[3 * r + k] = h[4 * r + k];
        cb.t[r] = h[4 * r + 3];
    }
    return cb;
}

// orthogonal() + in_cube, Morton binning, warp-cooperative SDF.  Leaves xyz4 (in_cube in .w) in the
// workspace for the MLP stage.
int run_sdf(const float *points, int64_t sc, int64_t sn, int64_t N, const float *h_calib,
            const MeshView &m, float *rec, int32_t *face, void *ws, float4 **xyz4_out,
            cudaStream_t stream) {
    Carver c(ws);
    SdfWs w = carve_sdf(c, N);
    Calib cb = make_calib(h_calib);
    profile_mark(0, stream);
    ICON_CUDA(cudaMemsetAsync(w.count, 0, sizeof(int32_t) * (NBIN + 1), stream));
    const unsigned nblk = (unsigned)((N + 255) / 256);
    k_points_bin<<<nblk, 256, 0, stream>>>(points, sc, sn, N, cb, w.xyz4, w.bid, w.count);
    ICON_LAUNCHED();
    int rc = scan_exclusive_i32(w.count, w.offset, NBIN + 1, nullptr, w.scan_ws, stream);
    if (rc) return rc;
    ICON_CUDA(cudaMemsetAsync(w.count, 0, sizeof(int32_t) * (NBIN + 1), stream));       // reuse as cursor
    k_points_scatter<<<nblk, 256, 0, stream>>>(w.bid, N, w.offset, w.count, w.perm);
    ICON_LAUNCHED();
    static bool attr_set[ICON_MAX_DEVICES] = {};
    if (device_needs_setup(attr_set)) {
#define ICON_SDF_ATTR(P, B) ICON_CUDA(cudaFuncSetAttribute(k_sdf_warp<P, B>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                                           (int)sdf_smem_bytes<P, B>()))
        ICON_SDF_ATTR(32, true); ICON_SDF_ATTR(32, false); ICON_SDF_ATTR(16, false); ICON_SDF_ATTR(8, false);
        ICON_SDF_ATTR(4, false); ICON_SDF_ATTR(2, false); ICON_SDF_ATTR(1, false);
#undef ICON_SDF_ATTR
    }
    profile_mark(1, stream);
    // the kernel needs many warps in flight to hide the latency of its tree walk, so the fewer points a call has the
    // fewer of them a warp carries.  The thresholds are tuned on the engine's sparse refinement sets (36k / 167k
    // points -> PPW 1, 826k .. ~5M -> PPW 8: 3.6 ms of engine time per image instead of 6.6 ms with PPW 32) and the
    // dense 256^3 lattice (PPW 32).  A DENSE mid-sized call would prefer PPW 32 (2.1M-point lattice: 1.7 vs 2.4 ms);
    // the point count alone cannot tell the two apart -- callers that know can pin it (icon_set_sdf_policy).
    int ppw = N >= g_sdf_ppw32_from ? 32 : (N >= g_sdf_ppw8_from ? 8 : 1);
    if (g_sdf_ppw_force) ppw = g_sdf_ppw_force;
    const int wpb = SW_T / 32;
    const int64_t nwarps = (N + ppw - 1) / ppw;
    const unsigned nblk_w = (unsigned)((nwarps + wpb - 1) / wpb);
#define ICON_SDF_LAUNCH(P) k_sdf_warp<P, false><<<nblk_w, SW_T, sdf_smem_bytes<P, false>(), stream>>>( \
        w.xyz4, w.perm, N, m, rec, face, nullptr, nullptr)
    if (ppw == 32 && g_sdf_bricks) {
        // dense call: the brick lists of this body, built by its first dense call, then the brick path and the tree
        // walk over the warps it leaves (those straddling bricks or outside the cube; all of them if the lists
        // overflowed), on a grid that fills the GPU once
        bool build;
        {
            std::lock_guard<std::mutex> lk(g_brick_mu);
            build = g_brick_ready.insert(m.hdr).second;
        }
        if (build) {
            rc = build_bricks(m, stream);
            std::lock_guard<std::mutex> lk(g_brick_mu);
            if (rc) { g_brick_ready.erase(m.hdr); return rc; }
            ++g_brick_builds;
        }
        ICON_CUDA(cudaMemsetAsync(w.ndefer, 0, sizeof(int32_t), stream));
        k_sdf_warp<32, true><<<nblk_w, SW_T, sdf_smem_bytes<32, true>(), stream>>>(
            w.xyz4, w.perm, N, m, rec, face, w.defer, w.ndefer);
        ICON_LAUNCHED();
        const unsigned nblk_d = (unsigned)std::min<int64_t>(nblk_w, (int64_t)device_sm_count() * 16);
        k_sdf_warp<32, false><<<nblk_d, SW_T, sdf_smem_bytes<32, false>(), stream>>>(
            w.xyz4, w.perm, N, m, rec, face, w.defer, w.ndefer);
    } else {
        switch (ppw) {
            case 32: ICON_SDF_LAUNCH(32); break;
            case 16: ICON_SDF_LAUNCH(16); break;
            case 8: ICON_SDF_LAUNCH(8); break;
            case 4: ICON_SDF_LAUNCH(4); break;
            case 2: ICON_SDF_LAUNCH(2); break;
            default: ICON_SDF_LAUNCH(1); break;
        }
    }
#undef ICON_SDF_LAUNCH
    ICON_LAUNCHED();
    profile_mark(2, stream);
    if (xyz4_out) *xyz4_out = w.xyz4;
    return ICON_OK;
}

__global__ void k_points_only(const float *__restrict__ pts, int64_t sc, int64_t sn, int64_t N, Calib cb,
                              float4 *__restrict__ xyz4) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    V3 p = load_point(pts, sc, sn, i, cb);
    float in_cube = (p.x > -1.f && p.x < 1.f && p.y > -1.f && p.y < 1.f && p.z > -1.f && p.z < 1.f) ? 1.f : 0.f;
    xyz4[i] = make_float4(p.x, p.y, p.z, in_cube);
}

// orthogonal() + in_cube only (pifu / pamir priors: no body mesh)
int run_points_only(const float *points, int64_t sc, int64_t sn, int64_t N, const float *h_calib,
                    float4 *xyz4, cudaStream_t stream) {
    Calib cb = make_calib(h_calib);
    k_points_only<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(points, sc, sn, N, cb, xyz4);
    ICON_LAUNCHED();
    return ICON_OK;
}

}  // namespace icon

using namespace icon;

#ifdef ICON_SDF_STATS
extern "C" int icon_debug_sdf_stats(unsigned long long *out, int reset) {
    cudaMemcpyFromSymbol(out, icon::g_stats, sizeof(unsigned long long) * 8);
    if (reset) { unsigned long long z[8] = {0}; cudaMemcpyToSymbol(icon::g_stats, z, sizeof(z)); }
    return 0;
}

// per-warp records of the brick path: WS_N words per warp, indexed by warp; nullptr stops recording
extern "C" int icon_debug_sdf_warp_stats(unsigned *dev_buf) {
    cudaMemcpyToSymbol(icon::g_wstat, &dev_buf, sizeof(dev_buf));
    return 0;
}
#endif

extern "C" int icon_set_sdf_policy(int force_ppw, int64_t ppw8_from, int64_t ppw32_from) {
    ICON_CHECK_ARG(force_ppw >= 0 && force_ppw <= 32 && (force_ppw & (force_ppw - 1)) == 0, "icon_set_sdf_policy: ppw in {0,1,2,4,8,16,32}");
    icon::g_sdf_ppw_force = force_ppw;
    if (ppw8_from >= 0) icon::g_sdf_ppw8_from = ppw8_from;
    if (ppw32_from >= 0) icon::g_sdf_ppw32_from = ppw32_from;
    return ICON_OK;
}

extern "C" int icon_set_sdf_bricks(int enable, int64_t max_entries) {
    ICON_CHECK_ARG(enable == 0 || enable == 1, "icon_set_sdf_bricks: enable must be 0 or 1");
    icon::g_sdf_bricks = enable;
    icon::g_brick_max_entries = max_entries > 0 ? max_entries : 0;
    return ICON_OK;
}

extern "C" int icon_sdf_brick_info(const void *mesh_ws, int V, int F, int64_t *out) {
    ICON_CHECK_ARG(mesh_ws && out && V > 0 && F > 0, "icon_sdf_brick_info: bad argument");
    MeshView m = mesh_view(mesh_ws, V, F);
    MeshHeader h;
    int32_t total = 0;
    ICON_CUDA(cudaDeviceSynchronize());
    ICON_CUDA(cudaMemcpy(&h, m.hdr, sizeof(h), cudaMemcpyDeviceToHost));
    if (h.brick_built) ICON_CUDA(cudaMemcpy(&total, m.foff + NBRICK, sizeof(total), cudaMemcpyDeviceToHost));
    out[0] = h.brick_built;
    out[1] = h.brick_overflow;
    out[2] = total;
    out[3] = m.face_cap;
    {
        std::lock_guard<std::mutex> lk(icon::g_brick_mu);
        out[4] = icon::g_brick_builds;
    }
    return ICON_OK;
}

extern "C" int icon_sdf_brick_lists(const void *mesh_ws, int V, int F, int64_t *dims, int32_t *foff, int32_t *flist,
                                    float *fkey, float *bub, int32_t *bface, float *sph) {
    ICON_CHECK_ARG(mesh_ws && dims && V > 0 && F > 0, "icon_sdf_brick_lists: bad argument");
    MeshView m = mesh_view(mesh_ws, V, F);
    MeshHeader h;
    int32_t total = 0;
    ICON_CUDA(cudaDeviceSynchronize());
    ICON_CUDA(cudaMemcpy(&h, m.hdr, sizeof(h), cudaMemcpyDeviceToHost));
    ICON_CHECK_ARG(h.brick_built, "icon_sdf_brick_lists: the body's brick lists are not built");
    ICON_CHECK_ARG(!h.brick_overflow, "icon_sdf_brick_lists: the body's brick lists overflowed");
    ICON_CUDA(cudaMemcpy(&total, m.foff + NBRICK, sizeof(total), cudaMemcpyDeviceToHost));
    dims[0] = BRICK_AX;
    dims[1] = total;
    if (!foff && !flist && !fkey && !bub && !bface && !sph) return ICON_OK;
    ICON_CHECK_ARG(foff && flist && fkey && bub && bface && sph, "icon_sdf_brick_lists: null array");
    std::vector<int32_t> order((size_t)F);
    std::vector<unsigned short> pos((size_t)total);
    std::vector<float4> sph_s((size_t)F);
    ICON_CUDA(cudaMemcpy(order.data(), m.order, sizeof(int32_t) * F, cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(pos.data(), m.flist, sizeof(unsigned short) * total, cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(sph_s.data(), m.sph_s, sizeof(float4) * F, cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(foff, m.foff, sizeof(int32_t) * (NBRICK + 1), cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(fkey, m.fkey, sizeof(float) * total, cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(bub, m.bub, sizeof(float) * NBRICK, cudaMemcpyDeviceToHost));
    ICON_CUDA(cudaMemcpy(bface, m.bface, sizeof(int32_t) * NBRICK, cudaMemcpyDeviceToHost));
    for (int32_t i = 0; i < total; ++i) flist[i] = order[pos[i]];
    for (int k = 0; k < F; ++k) {
        float *s = sph + 4 * (size_t)order[k];
        s[0] = sph_s[k].x; s[1] = sph_s[k].y; s[2] = sph_s[k].z; s[3] = sph_s[k].w;
    }
    return ICON_OK;
}

extern "C" int icon_sdf_only(const float *points, int64_t stride_c, int64_t stride_n, int64_t N,
                             const float *h_calib, const void *mesh_ws, int V, int F, float *rec,
                             int32_t *face, void *ws, size_t ws_bytes, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(N >= 0 && N < (int64_t)INT32_MAX, "icon_sdf_only: N=%lld out of range", (long long)N);
    if (N == 0) return ICON_OK;
    ICON_CHECK_ARG(points && h_calib && mesh_ws && rec && ws, "icon_sdf_only: null pointer");
    if (ws_bytes < sdf_ws_bytes(N)) {
        set_error("icon_sdf_only: workspace %zu < %zu", ws_bytes, sdf_ws_bytes(N));
        return ICON_ENOSPC;
    }
    MeshView m = mesh_view(mesh_ws, V, F);
    return run_sdf(points, stride_c, stride_n, N, h_calib, m, rec, face, ws, nullptr, stream);
}

extern "C" int icon_sdf_bruteforce(const float *points, int64_t stride_c, int64_t stride_n, int64_t N,
                                   const float *h_calib, const void *mesh_ws, int V, int F, float *rec,
                                   int32_t *face, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (N == 0) return ICON_OK;
    ICON_CHECK_ARG(points && h_calib && mesh_ws && rec, "icon_sdf_bruteforce: null pointer");
    MeshView m = mesh_view(mesh_ws, V, F);
    Calib cb = make_calib(h_calib);
    k_sdf_brute<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(points, stride_c, stride_n, N, cb, m, rec, face);
    ICON_LAUNCHED();
    return ICON_OK;
}
