// The Morton-sorted 4-ary AABB tree over a mesh's faces (FaceTree, common.cuh) and the exact nearest-face walk over
// it, shared by the SMPL SDF block (sdf.cu, smpl.cu) and the distance-only mesh query (mesh_dist.cu).
//
// Like geom.cuh, this header is included only by translation units compiled with -fmad=false: the bounds below and the
// exact distance are the same fp32 operations in every caller, fused multiply-adds only where fmaf() is written.
//
// Layout: face records (a, ab, ac) and bounding spheres in Morton order of the face centroids; leaves of 4 consecutive
// faces, then parents of 4 consecutive nodes, level by level (leaves first, root last).
//
// The walk (DESIGN.md 4.2): one warp serves PPW query points, each replicated on REP = 32 / PPW lanes that split the
// candidate faces between them and merge by shuffle.
//   (A) greedy descent to the leaf nearest the descent centre c: a first bound for every lane;
//   (B) breadth-first cull of the tree, 32 child boxes per step, ballot-compacted into a frontier in shared memory,
//       against the warp's bound; the bound tightens with the nearest far corner on the way down;
//   (C) the surviving leaves' faces, 32 at a time: culled by bounding sphere against the warp's box (and, with 32
//       points per warp, by a support bound that follows the lanes' own bounds: NearestFace::beats), staged in shared
//       memory, then every lane tests them against ITS OWN best through two cheap lower bounds (sphere, support
//       function) before the exact Ericson distance (tri_sqdist).
// A node or face is skipped only when its bound is strictly farther than the current best, and every bound carries
// float slack: `tol` on lengths and `tol_sup` on the support bound, sized for the largest coordinate in play.  Ties
// resolve to the lowest ORIGINAL face id and a NaN distance (a degenerate face) is never taken, exactly like the
// brute-force scans, so the result equals them bit for bit.  A frontier overflow falls back to every face.
#pragma once
#include <float.h>

#include "common.cuh"
#include "geom.cuh"

namespace icon {

// ---------------------------------------------------------------- small helpers
__device__ __forceinline__ float box_dist2(V3 p, float4 lo, float4 hi) {   // squared distance to the box
    const float dx = fmaxf(fmaxf(lo.x - p.x, p.x - hi.x), 0.f);
    const float dy = fmaxf(fmaxf(lo.y - p.y, p.y - hi.y), 0.f);
    const float dz = fmaxf(fmaxf(lo.z - p.z, p.z - hi.z), 0.f);
    return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}
__device__ __forceinline__ float box_far2(V3 p, float4 lo, float4 hi) {    // squared distance to the farthest corner
    const float dx = fmaxf(fabsf(lo.x - p.x), fabsf(hi.x - p.x));
    const float dy = fmaxf(fabsf(lo.y - p.y), fabsf(hi.y - p.y));
    const float dz = fmaxf(fabsf(lo.z - p.z), fabsf(hi.z - p.z));
    return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}
__device__ __forceinline__ float warp_max(float v) {
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_min(float v) {
    for (int o = 16; o; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---------------------------------------------------------------- building the tree
// level sizes and offsets of a tree over F faces; returns the total node count
static inline size_t tree_levels(FaceTree &t, int F) {
    t.F = F;
    int n = (F + 3) / 4, o = 0, l = 0;
    while (true) {
        t.lvl_cnt[l] = n; t.lvl_off[l] = o; o += n; ++l;
        if (n == 1) break;
        n = (n + 3) / 4;
    }
    t.nlevels = l;
    return (size_t)o;
}

__device__ __forceinline__ unsigned expand10(unsigned v) {     // 10 bits -> every third bit
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

// 30-bit Morton code of p over the cube [lo, lo + 1024 / s)^3, coordinates clamped to it
__device__ __forceinline__ unsigned morton30(V3 p, V3 lo, float s) {
    auto qz = [s](float v, float l) { return (unsigned)fminf(fmaxf((v - l) * s, 0.f), 1023.f); };
    return (expand10(qz(p.x, lo.x)) << 2) | (expand10(qz(p.y, lo.y)) << 1) | expand10(qz(p.z, lo.z));
}

// record (a, ab, ac) and bounding sphere (centroid, largest corner distance inflated by 1.0001 and `slack`: only a
// conservative lower bound for pruning, never a reported distance) of the face (a, b, c); returns the centroid
__device__ __forceinline__ V3 write_face_record(V3 a, V3 b, V3 c, float slack, float4 *__restrict__ tri,
                                                float4 *__restrict__ sph) {
    const V3 ab = sub3(b, a), ac = sub3(c, a);
    const V3 sc = mk3((a.x + b.x + c.x) / 3.f, (a.y + b.y + c.y) / 3.f, (a.z + b.z + c.z) / 3.f);
    const float ra = dot3(sub3(a, sc), sub3(a, sc)), rb = dot3(sub3(b, sc), sub3(b, sc)),
                rc = dot3(sub3(c, sc), sub3(c, sc));
    const float sr = sqrtf(fmaxf(ra, fmaxf(rb, rc))) * 1.0001f + slack;
    tri[0] = make_float4(a.x, a.y, a.z, ab.x);
    tri[1] = make_float4(ab.y, ab.z, ac.x, ac.y);
    tri[2] = make_float4(ac.z, 0.f, 0.f, 0.f);
    *sph = make_float4(sc.x, sc.y, sc.z, sr);
    return sc;
}

// box of leaf n (its 4 sorted faces, corners a, a + ab, a + ac as the distance code forms them)
__device__ __forceinline__ void write_leaf_box(const FaceTree &t, int n) {
    float4 lo = make_float4(FLT_MAX, FLT_MAX, FLT_MAX, 0.f), hi = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, 0.f);
    for (int k = 4 * n; k < min(4 * n + 4, t.F); ++k) {
        const Tri tr = load_tri(t.tri_s + 3 * (size_t)k);
        const V3 vs[3] = {tr.a, mk3(tr.a.x + tr.ab.x, tr.a.y + tr.ab.y, tr.a.z + tr.ab.z),
                          mk3(tr.a.x + tr.ac.x, tr.a.y + tr.ac.y, tr.a.z + tr.ac.z)};
        for (int j = 0; j < 3; ++j) {
            lo.x = fminf(lo.x, vs[j].x); hi.x = fmaxf(hi.x, vs[j].x);
            lo.y = fminf(lo.y, vs[j].y); hi.y = fmaxf(hi.y, vs[j].y);
            lo.z = fminf(lo.z, vs[j].z); hi.z = fmaxf(hi.z, vs[j].z);
        }
    }
    t.nodes[2 * (size_t)n] = lo;
    t.nodes[2 * (size_t)n + 1] = hi;
}

// box of node n of level l >= 1 from its children (plain loads: the caller may have written them in this kernel)
__device__ __forceinline__ void write_parent_box(const FaceTree &t, int l, int n) {
    const float4 *child = t.nodes + 2 * (size_t)t.lvl_off[l - 1];
    float4 lo = make_float4(FLT_MAX, FLT_MAX, FLT_MAX, 0.f), hi = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, 0.f);
    for (int c = 4 * n; c < min(4 * n + 4, t.lvl_cnt[l - 1]); ++c) {
        const float4 a = child[2 * (size_t)c], b = child[2 * (size_t)c + 1];
        lo.x = fminf(lo.x, a.x); lo.y = fminf(lo.y, a.y); lo.z = fminf(lo.z, a.z);
        hi.x = fmaxf(hi.x, b.x); hi.y = fmaxf(hi.y, b.y); hi.z = fmaxf(hi.z, b.z);
    }
    t.nodes[2 * ((size_t)t.lvl_off[l] + n)] = lo;
    t.nodes[2 * ((size_t)t.lvl_off[l] + n) + 1] = hi;
}

// the tree of a workspace icon_mesh_prepare filled, and the device address of the mesh's largest |coordinate|
// (defined in mesh_dist.cu; the PRT ray walk of prt.cu reads the same tree)
FaceTree mesh_ws_tree(const void *mesh_ws, int V, int F, const float **absmax);

// ---------------------------------------------------------------- the walk
struct ChunkSmem {                     // phase C's staging area, one per warp
    float4 sph[32];                    // bounding spheres of the surviving faces of the current chunk (compacted)
    float4 tri[32][3];                 // their (a, ab, ac) records
    int kk[32];                        // their sorted positions
};
template <typename Id, int CAP>
struct WalkSmem : ChunkSmem {
    Id fr[2][CAP];                     // phase B's frontier: node / leaf ids, double-buffered
};

// One lane's query point and the nearest face found for it so far.
template <int PPW>
struct NearestFace {
    static constexpr int REP = 32 / PPW;
    // `beats` pays where 32 distinct points share the box; with fewer per warp the box is small and the lanes' own
    // support tests already cut nearly as much, and it measured slower at PPW 1 and 8 (H100 80GB HBM3, 700 W)
    static constexpr bool CULL = PPW == 32;
    const int lane;
    V3 p;
    float tol, tol_sup;                // additive slack on lengths / on the support bound
    float best = FLT_MAX;              // squared distance
    int bi = 0x7fffffff;               // original face id
    float sb = 0.f, ub = 0.f;          // phase C: ~sqrt(best) inflated (this lane), the warp's loosest bound
    V3 g;                              // phase C: slope of the lanes' bounds across the warp's box (see beats)
    float beta = 0.f;                  // max over lanes of min(sb, ub) - g.(p - box centre)
    int staged = 0;                    // faces staged by phase C (ICON_SDF_STATS)
#ifdef ICON_SDF_STATS
    int n_sph = 0, n_exact = 0, n_win = 0;   // this lane's faces past the sphere test, past the support test, taken
    int n_dead = 0;                    // staged faces no lane got past the sphere test with
    bool last_sph = false;
#define NF_STAT(x) x
#else
#define NF_STAT(x)
#endif

    __device__ __forceinline__ NearestFace(V3 p_, float tol_, float tol_sup_)
        : lane(threadIdx.x & 31), p(p_), tol(tol_), tol_sup(tol_sup_) {}

    // ~sqrt(d), inflated: a bound only.  Computed, then selected: the branching form measured 0.7 % slower at PPW 8
    // and 16 (H100 80GB HBM3, 700 W power limit)
    __device__ __forceinline__ float sphere_bound(float d) const {
        const float b = d * rsqrtf(d) * 1.00001f + tol;
        return d > 0.f ? b : tol;
    }

    // exact test of the face record `rec` with original id f
    __device__ __forceinline__ void try_face(const float4 *rec, int f) {
        const Tri tr = load_tri(rec);
        const float d = tri_sqdist(p, tr.a, tr.ab, tr.ac);
        if (d < best || (d == best && f < bi)) { best = d; bi = f; }
    }

    // phase A: greedy descent towards c, then the faces of the leaf reached
    __device__ __forceinline__ void descend(const FaceTree &t, V3 c) {
        int node = 0;
        for (int lvl = t.nlevels - 1; lvl > 0; --lvl) {
            const int ch = 4 * node + (lane & 3);
            float a = FLT_MAX;
            int ai = ch;
            if (ch < t.lvl_cnt[lvl - 1]) {
                const float4 *nb = t.nodes + 2 * ((size_t)t.lvl_off[lvl - 1] + ch);
                a = box_dist2(c, __ldg(nb), __ldg(nb + 1));
            }
            for (int o = 1; o <= 2; o <<= 1) {               // min over the 4 children (lanes 4j..4j+3)
                const float ob = __shfl_xor_sync(0xffffffffu, a, o);
                const int oi = __shfl_xor_sync(0xffffffffu, ai, o);
                if (ob < a || (ob == a && oi < ai)) { a = ob; ai = oi; }
            }
            node = __shfl_sync(0xffffffffu, ai, 0);
        }
        for (int k = 4 * node; k < min(4 * node + 4, t.F); ++k) try_face(t.tri_s + 3 * (size_t)k, __ldg(t.order + k));
    }

    __device__ __forceinline__ static float warp_sum(float v) {
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    }
    __device__ __forceinline__ V3 box_offset(float4 wlo, float4 whi) const {
        return mk3(p.x - 0.5f * (wlo.x + whi.x), p.y - 0.5f * (wlo.y + whi.y), p.z - 0.5f * (wlo.z + whi.z));
    }
    __device__ __forceinline__ void update_beta(float4 wlo, float4 whi) {
        beta = warp_max(fminf(sb, ub) - dot3(g, box_offset(wlo, whi)));
    }

    // phase C's bounds, given that every lane's nearest face is within ubw; [wlo, whi] holds every lane's point.
    // g is the least-squares slope of the lanes' first bounds over their offsets from the box centre, about the
    // gradient of the distance across the warp: it only makes `beats` tighter, any finite g keeps it a bound
    __device__ __forceinline__ void start_scan(float ubw, float4 wlo, float4 whi) {
        sb = sphere_bound(best);
        ub = ubw * 1.00001f + tol;
        if (!CULL) return;
        const V3 o = box_offset(wlo, whi);
        const float sx = warp_sum(o.x * o.x), sy = warp_sum(o.y * o.y), sz = warp_sum(o.z * o.z);
        const float bx = warp_sum(o.x * sb), by = warp_sum(o.y * sb), bz = warp_sum(o.z * sb);
        // 0 on an axis the points do not span, clamped to [-1, 1] (the distance is 1-Lipschitz)
        auto slope = [](float num, float den) { return den > 0.f ? fminf(fmaxf(num / den, -1.f), 1.f) : 0.f; };
        g = mk3(slope(bx, sx), slope(by, sy), slope(bz, sz));
        update_beta(wlo, whi);
    }

    // phase C, one lane: sorted face k with bounding sphere s and record tr (dereferenced only past the sphere test)
    __device__ __forceinline__ void test(const FaceTree &t, int k, float4 s, const float4 *tr) {
        const float dx = p.x - s.x, dy = p.y - s.y, dz = p.z - s.z;
        const float dd = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
        const float l = sb + s.w;
        NF_STAT(last_sph = false);
        if (dd > l * l) return;                                // sphere bound beats this lane's best
        NF_STAT(++n_sph; last_sph = true);
        // support-function bound d >= |w| - max_k u.(v_k - c_f), u = w/|w|, w = p - c_f: nearly exact head-on
        const float4 r0 = tr[0], r1 = tr[1], r2 = tr[2];
        const V3 ab = mk3(r0.w, r1.x, r1.y), ac = mk3(r1.z, r1.w, r2.x);
        const float S1 = fmaf(dz, ab.z, fmaf(dy, ab.y, dx * ab.x));
        const float T1 = fmaf(dz, ac.z, fmaf(dy, ac.y, dx * ac.x));
        const float M = fmaxf(fmaxf(-(S1 + T1), fmaf(2.f, S1, -T1)), fmaf(2.f, T1, -S1)) * (1.f / 3.f);
        const float g = dd - M - tol_sup;                      // |w|^2 - |w| h(u)
        if (g > 0.f && g * g > best * dd * 1.0001f) return;   // support bound beats this lane's best
        NF_STAT(++n_exact);
        const float d = tri_sqdist(p, mk3(r0.x, r0.y, r0.z), ab, ac);
        if (!(d <= best)) return;                              // also drops NaN, as the brute-force scans do
        NF_STAT(++n_win);
        const int f = __ldg(t.order + k);
        if (d < best || f < bi) { best = d; bi = f; sb = sphere_bound(d); }
    }

    // replicas of a point share their best (lowest distance, then lowest face id)
    __device__ __forceinline__ void merge() {
#pragma unroll
        for (int o = PPW; o < 32; o <<= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
    }

    // True when no lane can take the face (s: centroid, r0..r2: record): a support bound against the warp's box
    // [wlo, whi] (centre pc, half extents hb) that follows the lanes' own bounds sb_i <= beta + g.(p_i - pc).  For the
    // unit vector e from the centroid c towards pc, lane i's distance to any point q of the face is at least
    //   e.(p_i - q) >= e.(pc - c) + e.(p_i - pc) - max_k e.(v_k - c)
    //              >= sb_i + |pc - c| - max_k e.(v_k - c) - beta - sum_k |e_k - g_k| hb_k,
    // so the face is out for every lane once the last four terms are positive, with float slack.  Seen from afar the
    // lanes' distances to a flat region move with g, so the box's extent costs only where e leaves that direction.
    // False on a NaN (box centre on the centroid).
    __device__ __forceinline__ bool beats(float4 s, float4 r0, float4 r1, float4 r2, float4 wlo, float4 whi) const {
        const float vx = 0.5f * (wlo.x + whi.x) - s.x, vy = 0.5f * (wlo.y + whi.y) - s.y,
                    vz = 0.5f * (wlo.z + whi.z) - s.z;
        const float L = sqrtf(fmaf(vz, vz, fmaf(vy, vy, vx * vx)));
        const float il = 1.f / L;
        const float ex = vx * il, ey = vy * il, ez = vz * il;
        const float S1 = fmaf(ez, r1.y, fmaf(ey, r1.x, ex * r0.w));           // e.ab
        const float T1 = fmaf(ez, r2.x, fmaf(ey, r1.w, ex * r1.z));           // e.ac
        const float he = fmaxf(fmaxf(-(S1 + T1), fmaf(2.f, S1, -T1)), fmaf(2.f, T1, -S1)) * (1.f / 3.f);
        const float pr = fmaf(fabsf(ez - g.z), 0.5f * (whi.z - wlo.z),
                              fmaf(fabsf(ey - g.y), 0.5f * (whi.y - wlo.y), fabsf(ex - g.x) * (0.5f * (whi.x - wlo.x))));
        return L - he - pr - beta > tol + 1e-5f * (L + fabsf(he) + pr + fabsf(beta));
    }

    // phase C, one step: this lane's slot holds `leaf` (-1: none), 4 lanes per leaf, 8 leaves = 32 faces, culled
    // against the warp's box [wlo, whi] by bounding sphere and the loosest lane bound, then by `beats`, staged
    // compacted, then split over the replicas
    __device__ __forceinline__ void chunk(const FaceTree &t, ChunkSmem &S, int leaf, float4 wlo, float4 whi) {
        bool pass = false;
        int k = 0;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f), r0 = s, r1 = s, r2 = s;
        if (leaf >= 0) {
            k = 4 * leaf + (lane & 3);
            if (k < t.F) {
                s = __ldg(t.sph_s + k);
                const float l2 = ub + s.w;                     // sphere vs the warp's box: some lane may be that close
                pass = box_dist2(mk3(s.x, s.y, s.z), wlo, whi) <= l2 * l2;
                if (CULL && pass) {
                    const float4 *tp = t.tri_s + 3 * (size_t)k;
                    r0 = __ldg(tp); r1 = __ldg(tp + 1); r2 = __ldg(tp + 2);
                    pass = !beats(s, r0, r1, r2, wlo, whi);
                }
            }
        }
        const unsigned mask = __ballot_sync(0xffffffffu, pass);
        const int cnt = __popc(mask);
        staged += cnt;
        if (pass) {
            const int at = __popc(mask & ((1u << lane) - 1u));
            S.sph[at] = s;
            S.kk[at] = k;
            if (!CULL) {
                const float4 *tp = t.tri_s + 3 * (size_t)k;
                r0 = __ldg(tp); r1 = __ldg(tp + 1); r2 = __ldg(tp + 2);
            }
            S.tri[at][0] = r0; S.tri[at][1] = r1; S.tri[at][2] = r2;
        }
        __syncwarp();
        for (int j = lane / PPW; j < cnt; j += REP) {
            test(t, S.kk[j], S.sph[j], &S.tri[j][0]);
            NF_STAT(if (REP == 1) n_dead += !__any_sync(0xffffffffu, last_sph));
        }
        if (REP > 1) {
            merge();
            sb = sphere_bound(best);
        }
        ub = fminf(ub, warp_max(sb));                          // the lanes' bounds only shrink: cull the next chunk harder
        if (CULL) update_beta(wlo, whi);
        __syncwarp();
    }

    // phase C over n leaves
    template <typename Id>
    __device__ __forceinline__ void scan_leaves(const FaceTree &t, ChunkSmem &S, const Id *leaves, int n, float4 wlo,
                                                float4 whi) {
        for (int base = 0; base < n; base += 8) {
            const int slot = base + (lane >> 2);
            chunk(t, S, slot < n ? (int)leaves[slot] : -1, wlo, whi);
        }
    }

    // phase C without a frontier (it overflowed): every face, split over the replicas
    __device__ __forceinline__ void scan_all(const FaceTree &t) {
        for (int k = lane / PPW; k < t.F; k += REP) test(t, k, __ldg(t.sph_s + k), t.tri_s + 3 * (size_t)k);
    }
};

// Phase B: breadth-first cull of the tree against the warp's box [wlo, whi], every lane's nearest face within ubw (in,
// tightened on the way down: some face lies within the nearest far-corner distance of c, so within that + rw of
// every lane, rw >= every lane's distance to c).  Leaves the surviving leaves in fr[cur][0, n); returns false when the
// frontier overflowed (n > CAP).
template <typename Id, int CAP>
__device__ __forceinline__ bool tree_cull(const FaceTree &t, Id (&fr)[2][CAP], V3 c, float rw, float4 wlo, float4 whi,
                                          float tol, float &ubw, int &cur, int &n) {
    const int lane = threadIdx.x & 31;
    float ub2 = (ubw * 1.00001f + tol) * (ubw * 1.00001f + tol);
    cur = 0; n = 1;
    bool overflow = false;
    if (lane == 0) fr[0][0] = 0;
    __syncwarp();
    for (int lvl = t.nlevels - 1; lvl > 0 && !overflow; --lvl) {
        int nn = 0;
        float far2 = FLT_MAX;
        const int ccnt = t.lvl_cnt[lvl - 1];
        const float4 *nodes = t.nodes + 2 * (size_t)t.lvl_off[lvl - 1];
        for (int base = 0; base < n; base += 8) {
            const int slot = base + (lane >> 2);
            bool pass = false;
            int ch = 0;
            if (slot < n) {
                ch = 4 * (int)fr[cur][slot] + (lane & 3);
                if (ch < ccnt) {
                    const float4 lo = __ldg(nodes + 2 * (size_t)ch), hi = __ldg(nodes + 2 * (size_t)ch + 1);
                    // distance between the node's box and the warp's box bounds every lane's distance to the node
                    const float gx = fmaxf(fmaxf(lo.x - whi.x, wlo.x - hi.x), 0.f);
                    const float gy = fmaxf(fmaxf(lo.y - whi.y, wlo.y - hi.y), 0.f);
                    const float gz = fmaxf(fmaxf(lo.z - whi.z, wlo.z - hi.z), 0.f);
                    pass = fmaf(gz, gz, fmaf(gy, gy, gx * gx)) <= ub2;
                    far2 = fminf(far2, box_far2(c, lo, hi));
                }
            }
            const unsigned mask = __ballot_sync(0xffffffffu, pass);
            const int at = nn + __popc(mask & ((1u << lane) - 1u));
            if (pass && at < CAP) fr[cur ^ 1][at] = (Id)ch;
            nn += __popc(mask);
        }
        overflow = nn > CAP;
        n = nn;
        cur ^= 1;
        const float l2 = sqrtf(warp_min(far2)) + rw;
        if (l2 < ubw) { ubw = l2; ub2 = (ubw * 1.00001f + tol) * (ubw * 1.00001f + tol); }
        __syncwarp();
    }
    return !overflow;
}

// The whole walk for the lanes' points: phases A, B, C and the final merge.  c: the descent centre, rw: a bound on
// every lane's distance to c, [wlo, whi]: the warp's box (both inflated by tol).  Returns the number of leaves that
// survived phase B (> CAP: the frontier overflowed and every face was scanned).
template <int PPW, typename Id, int CAP>
__device__ __forceinline__ int tree_nearest(const FaceTree &t, WalkSmem<Id, CAP> &S, NearestFace<PPW> &q, V3 c,
                                            float rw, float4 wlo, float4 whi) {
    q.descend(t, c);
    float ubw = warp_max(sqrtf(q.best));                       // every lane's nearest is within ubw
    int cur, n;
    const bool ok = tree_cull(t, S.fr, c, rw, wlo, whi, q.tol, ubw, cur, n);
    q.start_scan(ubw, wlo, whi);
    if (ok) q.scan_leaves(t, S, S.fr[cur], n, wlo, whi);
    else q.scan_all(t);
    q.merge();
    return n;
}

}  // namespace icon
