// Remeshing of the demo's reconstruction: replaces lib/dataset/mesh_util.py:109-121 (remesh), pymeshlab's
// laplacian_smooth() followed by remeshing_isotropic_explicit_remeshing(targetlen=Percentage(perc), adaptive=True).
//
// PARITY UNPINNED: pymeshlab's and vcglib's sources are absent.  The rules below restate the two filters at the
// reference's arguments from their documented defaults; what is marked (reading) is this project's choice where the
// documentation fixes nothing.  oracle/remesh.py restates every rule in float64 NumPy, round by round, in the order
// written here (hence -fmad=false): the device's mesh equals the oracle's after every pass, vertices bit for bit and
// faces index for index.  No float atomics; every per-vertex sum runs over the ascending lists of the topology.
//
// Topology, normals and nearest faces are the existing code's: icon_mesh_topology_count / _build (csrc/mesh_priors.cu:
// edges (min, max) ascending, face_to_edge e12 e20 e01, ascending per-vertex edge lists and corners, per-edge
// face-corner entries 3 f + col), icon_area_vertex_normals (csrc/mesh_views.cu) and icon_mesh_prepare /
// icon_mesh_distance (csrc/mesh_dist.cu).  The host loop is icon_b200/remesh.py.
//
// Positions are fp64 throughout; dot(u, w) = (ux wx + uy wy) + uz wz, n(f) = (p1 - p0) x (p2 - p0) written
// (uy wz - uz wy, uz wx - ux wz, ux wy - uy wx), |n|^2 = dot(n, n).
//
// 0. Compaction (icon_remesh_compact): vertices no face references are dropped; survivors keep ascending order.
// 1. Classification (icon_remesh_classify, before every smoothing step and every round).  An edge (a, b) is
//    OK when a != b, it has exactly two face entries, neither face has |n|^2 == 0, and the faces traverse it in
//    opposite directions (entry 3 f + col runs from corner col+1 to corner col+2); BOUNDARY when a != b and it has one
//    entry whose face has |n|^2 > 0; BAD otherwise (self-loop, non-manifold, zero-area face, inconsistent winding).
//    For an OK edge: fa is the face running a -> b and c its opposite corner, fb / d the other's;
//    cos = dot(n_fa, n_fb) / (sqrt|n_fa|^2 sqrt|n_fb|^2); crease when cos < cos 30 deg (0.8660254037844387, the
//    feature angle); kappa = 1 - cos.  A vertex is FROZEN unless every edge of it is OK and its faces form one fan: the
//    walk from its first corner, across the edge to the next corner of each face, first returns to the starting face
//    after exactly as many steps as the vertex has corners (and corners = degree).  Frozen vertices, and every edge
//    that is not OK, are excluded from every topological operation: an operation on edge (a, b) needs the edge OK and
//    none of a, b, c, d frozen.  Boundaries are therefore never flipped, so the valence-4 target of a boundary vertex
//    never applies.  ncrease(v) = crease edges at v; kappa(v) = max kappa over its edges (0 if none).
// 2. Laplacian smooth (icon_remesh_smooth_step), pymeshlab defaults: 3 Jacobi steps, cotangent weights, boundary
//    vertices moved along the boundary only.  Edge weight w = (cot_0 + cot_1) 0.5 over its first two entries in order
//    (one for a boundary edge), cot = dot(u, q) / sqrt|u x q|^2 with u = p_a - p_o, q = p_b - p_o, o the entry's
//    opposite corner, and cot = 0 when |u x q|^2 == 0; w <= 0 (negative, or NaN) gives w = 0 (reading).  A
//    non-frozen vertex moves to sum(w q) / sum(w), or to sum(q) / degree when sum(w) is not > 0.  A vertex with no BAD
//    edge and exactly two BOUNDARY edges moves to the mean of those two neighbours, (sum) / 2.  Any other vertex
//    stays.  Sums start at 0 and run over the vertex's ascending edges.
// 3. Isotropic explicit remeshing, pymeshlab defaults but for the reference's targetlen: 3 iterations, each a split
//    pass, a collapse pass, a flip pass, then tangential relaxation with reprojection.  diag = the smoothed mesh's
//    bounding-box diagonal, L = diag (perc / 100), surface-distance limit 0.01 diag (compared squared, in fp64).
//    adaptive (reading): s(v) = 1 - 0.5 min(1, kappa(v) / (1 - cos 30 deg)), s(e) = min(s(a), s(b)), Le = L s(e), so
//    edges are shortened down to half length where the surface bends by the feature angle or more; not adaptive:
//    Le = L.  hi2 = (Le 4/3)^2, lo2 = (Le 0.8)^2, len2 = |p_b - p_a|^2.
//    Each pass is a sequence of deterministic parallel ROUNDS, each on a fresh topology and classification, until a
//    round has no winner or the pass has run its cap (32 split, 32 collapse, 16 flip rounds).  A candidate's key is
//    (hi32(bits(len2)) << 32 | e), longest first for split and flip (0xffffffff - hi32), shortest first for
//    collapse: its length to 2^-20 relative, then its edge id.  m1(v) = least key over v's edges; m2(v) = least m1
//    over v and its neighbours.  A candidate wins when key <= m(a), m(b), m(c), m(d) with m = m1 for splits (no two
//    winners share a face) and m = m2 for collapses and flips (no winner touches another's one-ring).
//    SPLIT candidate: len2 > hi2.  Winners are numbered in edge order; winner r gets vertex V + r at
//      (p_a + p_b) 0.5.  Faces in order: a face with no winning edge is copied; a face whose column-k edge won, with
//      i0 = f[k], i1 = f[k+1], i2 = f[k+2] and new vertex m, becomes (i0, i1, m), (i0, m, i2).
//    COLLAPSE candidate: len2 < lo2, not a crease, ncrease(a) = ncrease(b) = 0, degree(c), degree(d) > 3, a and b
//      have exactly two common neighbours (link condition), the fp32 midpoint's squared distance to the reference
//      surface (icon_mesh_distance) <= limit^2, and with m = (p_a + p_b) 0.5: every face at a without b (and at b
//      without a) keeps dot(n_old, n_new) > 0 with a (b) moved to m, and every neighbour w != b of a (!= a of b) has
//      |p_w - m|^2 <= hi2.  Winners: b is removed, a moves to m, the two faces of the edge are dropped, b is renamed
//      a in the others; surviving vertices and faces keep ascending old order.
//    FLIP candidate: not a crease, degree(a), degree(b) > 3, c != d, c and d not already neighbours, valence
//      deviation sum |deg - 6| over a, b, c, d strictly lower after (a, b lose one, c, d gain one); with
//      n1 = (p_d - p_a) x (p_c - p_a), n2 = (p_b - p_d) x (p_c - p_d), ns = n_fa + n_fb: dot(n1, n2) >
//      cos30 (sqrt|n1|^2 sqrt|n2|^2), dot(n1, ns) > 0, dot(n2, ns) > 0.  Winners: fa becomes (a, d, c), fb (d, b, c).
//    RELAX (icon_remesh_relax): n = icon_area_vertex_normals of the fp32-rounded vertices.  A non-frozen vertex with
//      no crease edge moves to p + (d - n t), d = sum(q) / degree - p, t = dot(d, n).  One with exactly two crease
//      edges slides along the line of its two crease neighbours q1, q2 (in edge order): e = q2 - q1,
//      p + e (dot((q1 + q2) 0.5 - p, e) / |e|^2) (stays when |e|^2 == 0).  Others (frozen, corners of 1 or >= 3
//      creases) stay.  REPROJECT (icon_remesh_reproject): each moved vertex, rounded to fp32, takes its nearest face
//      of the reference (the smoothed input) from icon_mesh_distance, then the closest point on that face in fp64
//      (Ericson's regions; a zero denominator gives parameter 0, a zero total barycentric weight gives the corner a).
// 4. Output: fp32 vertices [1, V', 3] and int64 faces [1, F', 3]; every vertex is referenced.
//
// Launches and host reads per round: the topology (count and build; one read of E) + classify (3) + select (3-4
// plus a scan, one read of the winner count) + apply (split 3 plus a scan, collapse 3 plus two scans, flip 1);
// a collapse round adds the midpoints and one icon_mesh_distance.  Per iteration the relaxation adds the topology,
// classify, one normals call, relax, one icon_mesh_distance and reproject, with one read (E).
#include "common.cuh"

namespace {

constexpr double COS_FEAT = 0.8660254037844387;
constexpr double KAP0 = 1.0 - COS_FEAT;
constexpr double HI = 4.0 / 3.0;
constexpr double LO = 0.8;
constexpr unsigned long long NONE = 0xFFFFFFFFFFFFFFFFull;
enum { ST_OK = 0, ST_BOUNDARY = 1, ST_BAD = 2 };
enum { OP_SPLIT = 0, OP_COLLAPSE = 1, OP_FLIP = 2 };
constexpr int TPB = 256;

struct D3 { double x, y, z; };
__device__ __forceinline__ D3 ld(const double *p, int64_t i) { return {p[3 * i], p[3 * i + 1], p[3 * i + 2]}; }
__device__ __forceinline__ void st3(double *p, int64_t i, D3 v) { p[3 * i] = v.x; p[3 * i + 1] = v.y; p[3 * i + 2] = v.z; }
__device__ __forceinline__ D3 sub(D3 a, D3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ D3 add(D3 a, D3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ D3 mul(D3 a, double s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ double dot(D3 a, D3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__device__ __forceinline__ D3 cross(D3 u, D3 w) {
    return {u.y * w.z - u.z * w.y, u.z * w.x - u.x * w.z, u.x * w.y - u.y * w.x};
}

// workspace: everything one round needs, sized for (V, F, E)
struct Ws {
    double *fn, *fa2, *kap, *kapv, *cw;
    int32_t *est, *ec, *ed, *efa, *efb, *crease, *ncrease, *frozen, *sbnd;
    unsigned long long *key, *m1, *m2;
    int32_t *win, *rank, *fcnt, *fpos, *keep, *newid, *tgt;
    void *scan;
};

template <typename T> T *carve(char *&p, int64_t n) {
    T *r = reinterpret_cast<T *>(p);
    p += icon::align_up(sizeof(T) * (size_t)(n > 0 ? n : 1), 256);
    return r;
}

size_t ws_layout(int V, int F, int E, void *base, Ws *w) {
    char *p = static_cast<char *>(base);
    Ws t;
    t.fn = carve<double>(p, 3 * (int64_t)F); t.fa2 = carve<double>(p, F);
    t.kap = carve<double>(p, E); t.kapv = carve<double>(p, V); t.cw = carve<double>(p, E);
    t.est = carve<int32_t>(p, E); t.ec = carve<int32_t>(p, E); t.ed = carve<int32_t>(p, E);
    t.efa = carve<int32_t>(p, E); t.efb = carve<int32_t>(p, E); t.crease = carve<int32_t>(p, E);
    t.ncrease = carve<int32_t>(p, V); t.frozen = carve<int32_t>(p, V); t.sbnd = carve<int32_t>(p, V);
    t.key = carve<unsigned long long>(p, E); t.m1 = carve<unsigned long long>(p, V);
    t.m2 = carve<unsigned long long>(p, V);
    t.win = carve<int32_t>(p, E); t.rank = carve<int32_t>(p, E);
    t.fcnt = carve<int32_t>(p, F); t.fpos = carve<int32_t>(p, F);
    t.keep = carve<int32_t>(p, V); t.newid = carve<int32_t>(p, V); t.tgt = carve<int32_t>(p, V);
    int64_t n = V; if (F > n) n = F; if (E > n) n = E;
    t.scan = carve<char>(p, (int64_t)icon::scan_ws_bytes(n));
    if (w) *w = t;
    return (size_t)(p - static_cast<char *>(base)) + 256;
}

Ws ws_view(int V, int F, int E, void *ws) {
    Ws w;
    char *base = reinterpret_cast<char *>(icon::align_up(reinterpret_cast<uintptr_t>(ws), 256));
    ws_layout(V, F, E, base, &w);
    return w;
}

__device__ __forceinline__ int other(const int64_t *edges, int e, int v) {
    const int a = (int)edges[2 * (int64_t)e], b = (int)edges[2 * (int64_t)e + 1];
    return a == v ? b : a;
}

// ------------------------------------------------------------------ classification

__global__ void k_face_normals(const double *__restrict__ P, const int64_t *__restrict__ faces, int F,
                               double *__restrict__ fn, double *__restrict__ fa2) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const D3 p0 = ld(P, faces[3 * (int64_t)f]), p1 = ld(P, faces[3 * (int64_t)f + 1]), p2 = ld(P, faces[3 * (int64_t)f + 2]);
    const D3 n = cross(sub(p1, p0), sub(p2, p0));
    st3(fn, f, n);
    fa2[f] = dot(n, n);
}

__global__ void k_edge_class(icon_mesh_topology t, Ws w) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.E) return;
    const int a = (int)t.edges[2 * (int64_t)e], b = (int)t.edges[2 * (int64_t)e + 1];
    const int o = t.edge_off[e], nent = t.edge_off[e + 1] - o;
    int st = ST_BAD, ec = -1, ed = -1, efa = -1, efb = -1, cr = 0;
    double kap = 0.0;
    const int x0 = t.edge_entries[o], f0 = x0 / 3, c0 = x0 % 3;
    const bool z0 = w.fa2[f0] == 0.0;
    if (nent == 1 && a != b && !z0) st = ST_BOUNDARY;
    if (nent == 2 && a != b && !z0) {
        const int x1 = t.edge_entries[o + 1], f1 = x1 / 3, c1 = x1 % 3;
        const int from0 = (int)t.faces[3 * (int64_t)f0 + (c0 + 1) % 3];
        const int from1 = (int)t.faces[3 * (int64_t)f1 + (c1 + 1) % 3];
        if (w.fa2[f1] != 0.0 && ((from0 == a) != (from1 == a))) {
            st = ST_OK;
            const bool fst = from0 == a;
            efa = fst ? f0 : f1; efb = fst ? f1 : f0;
            ec = (int)t.faces[3 * (int64_t)efa + (fst ? c0 : c1)];
            ed = (int)t.faces[3 * (int64_t)efb + (fst ? c1 : c0)];
            const double cosd = dot(ld(w.fn, efa), ld(w.fn, efb)) / (sqrt(w.fa2[efa]) * sqrt(w.fa2[efb]));
            cr = cosd < COS_FEAT;
            kap = 1.0 - cosd;
        }
    }
    w.est[e] = st; w.ec[e] = ec; w.ed[e] = ed; w.efa[e] = efa; w.efb[e] = efb; w.crease[e] = cr; w.kap[e] = kap;
}

__global__ void k_vert_class(icon_mesh_topology t, Ws w) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= t.V) return;
    const int o = t.vert_off[v], deg = t.vert_off[v + 1] - o;
    int nbad = 0, nbnd = 0, ncr = 0;
    double kv = 0.0;
    for (int i = 0; i < deg; ++i) {
        const int e = t.vert_edges[o + i];
        nbad += w.est[e] == ST_BAD;
        nbnd += w.est[e] == ST_BOUNDARY;
        ncr += w.crease[e];
        if (w.kap[e] > kv) kv = w.kap[e];
    }
    bool fan = false;
    const int ncor = t.corner_off[v + 1] - t.corner_off[v];
    if (nbad == 0 && nbnd == 0 && deg > 0 && ncor == deg) {
        const int k0 = t.vert_corners[t.corner_off[v]], f0 = k0 / 3;
        int fc = f0, cc = k0 % 3, steps = 0;
        while (true) {
            const int e = (int)t.face_to_edge[3 * (int64_t)fc + (cc + 2) % 3];
            const int x = t.edge_entries[t.edge_off[e]], y = t.edge_entries[t.edge_off[e] + 1];
            const int g = (x / 3 == fc) ? y / 3 : x / 3;
            cc = t.faces[3 * (int64_t)g] == v ? 0 : (t.faces[3 * (int64_t)g + 1] == v ? 1 : 2);
            fc = g;
            ++steps;
            if (fc == f0 || steps > ncor) break;
        }
        fan = steps == ncor;
    }
    w.frozen[v] = !fan;
    w.sbnd[v] = nbad == 0 && nbnd == 2;
    w.ncrease[v] = ncr;
    w.kapv[v] = kv;
}

// ------------------------------------------------------------------ Laplacian smoothing

__global__ void k_cot_weights(icon_mesh_topology t, const double *__restrict__ P, Ws w) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.E) return;
    const int o = t.edge_off[e], n = min(t.edge_off[e + 1] - o, 2);
    const D3 pa = ld(P, t.edges[2 * (int64_t)e]), pb = ld(P, t.edges[2 * (int64_t)e + 1]);
    double s = 0.0;
    for (int k = 0; k < n; ++k) {
        const int x = t.edge_entries[o + k];
        const D3 po = ld(P, t.faces[3 * (int64_t)(x / 3) + x % 3]);
        const D3 u = sub(pa, po), q = sub(pb, po);
        const D3 c = cross(u, q);
        const double n2 = dot(c, c);
        s = s + (n2 > 0.0 ? dot(u, q) / sqrt(n2) : 0.0);
    }
    s = s * 0.5;
    w.cw[e] = s > 0.0 ? s : 0.0;
}

__global__ void k_smooth(icon_mesh_topology t, const double *__restrict__ P, Ws w, double *__restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= t.V) return;
    const int o = t.vert_off[v], deg = t.vert_off[v + 1] - o;
    double sw = 0.0;
    D3 s = {0.0, 0.0, 0.0}, su = {0.0, 0.0, 0.0}, sb = {0.0, 0.0, 0.0};
    for (int i = 0; i < deg; ++i) {
        const int e = t.vert_edges[o + i];
        const D3 q = ld(P, other(t.edges, e, v));
        const double we = w.cw[e];
        sw = sw + we;
        s = add(s, mul(q, we));
        su = add(su, q);
        if (w.est[e] == ST_BOUNDARY) sb = add(sb, q);
    }
    D3 r = ld(P, v);
    if (!w.frozen[v]) {
        if (sw > 0.0) r = {s.x / sw, s.y / sw, s.z / sw};
        else { const double d = (double)deg; r = {su.x / d, su.y / d, su.z / d}; }
    }
    if (w.sbnd[v]) r = {sb.x / 2.0, sb.y / 2.0, sb.z / 2.0};
    st3(out, v, r);
}

// ------------------------------------------------------------------ rounds

__global__ void k_midpoints(icon_mesh_topology t, const double *__restrict__ P, float *__restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.E) return;
    const D3 m = mul(add(ld(P, t.edges[2 * (int64_t)e]), ld(P, t.edges[2 * (int64_t)e + 1])), 0.5);
    out[3 * (int64_t)e] = (float)m.x; out[3 * (int64_t)e + 1] = (float)m.y; out[3 * (int64_t)e + 2] = (float)m.z;
}

__device__ __forceinline__ double vscale(const Ws &w, int v) {
    const double x = w.kapv[v] / KAP0;
    return 1.0 - 0.5 * (x > 1.0 ? 1.0 : x);
}

__device__ __forceinline__ bool is_nb(const icon_mesh_topology &t, int v, int u) {
    for (int i = t.vert_off[v]; i < t.vert_off[v + 1]; ++i)
        if (other(t.edges, t.vert_edges[i], v) == u) return true;
    return false;
}

__device__ bool collapse_side(const icon_mesh_topology &t, const double *P, const Ws &w, int x, int y, D3 m,
                              double hi2) {
    for (int i = t.corner_off[x]; i < t.corner_off[x + 1]; ++i) {
        const int k = t.vert_corners[i], f = k / 3, ci = k % 3;
        const int64_t *fv = t.faces + 3 * (int64_t)f;
        if (fv[0] == y || fv[1] == y || fv[2] == y) continue;
        const D3 q0 = ci == 0 ? m : ld(P, fv[0]), q1 = ci == 1 ? m : ld(P, fv[1]), q2 = ci == 2 ? m : ld(P, fv[2]);
        const D3 n1 = cross(sub(q1, q0), sub(q2, q0));
        if (!(dot(ld(w.fn, f), n1) > 0.0)) return false;
    }
    for (int i = t.vert_off[x]; i < t.vert_off[x + 1]; ++i) {
        const int u = other(t.edges, t.vert_edges[i], x);
        if (u == y) continue;
        const D3 d = sub(ld(P, u), m);
        if (dot(d, d) > hi2) return false;
    }
    return true;
}

__global__ void k_candidates(int op, icon_mesh_topology t, const double *__restrict__ P, double L, int adaptive,
                             const float *__restrict__ sqd, double dlim2, Ws w) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.E) return;
    const int a = (int)t.edges[2 * (int64_t)e], b = (int)t.edges[2 * (int64_t)e + 1];
    const int c = w.ec[e], d = w.ed[e];
    unsigned long long key = NONE;
    bool cand = w.est[e] == ST_OK;                               // c, d exist only for an OK edge
    cand = cand && !w.frozen[a] && !w.frozen[b] && !w.frozen[c] && !w.frozen[d];
    const D3 pa = ld(P, a), pb = ld(P, b);
    const D3 dv = sub(pb, pa);
    const double len2 = dot(dv, dv);
    double s = 1.0;
    if (adaptive) { const double sa = vscale(w, a), sb = vscale(w, b); s = sa < sb ? sa : sb; }
    const double Le = L * s;
    const double hi2 = (Le * HI) * (Le * HI), lo2 = (Le * LO) * (Le * LO);
    auto deg = [&](int v) { return t.vert_off[v + 1] - t.vert_off[v]; };
    if (cand) {
        if (op == OP_SPLIT) {
            cand = len2 > hi2;
        } else if (op == OP_FLIP) {
            const int da = deg(a), db = deg(b), dc = deg(c), dd = deg(d);
            cand = !w.crease[e] && da > 3 && db > 3 && c != d;
            const int before = abs(da - 6) + abs(db - 6) + abs(dc - 6) + abs(dd - 6);
            const int after = abs(da - 7) + abs(db - 7) + abs(dc - 5) + abs(dd - 5);
            cand = cand && after < before;
            if (cand) {
                const D3 pc = ld(P, c), pd = ld(P, d);
                const D3 n1 = cross(sub(pd, pa), sub(pc, pa)), n2 = cross(sub(pb, pd), sub(pc, pd));
                const D3 ns = add(ld(w.fn, w.efa[e]), ld(w.fn, w.efb[e]));
                cand = dot(n1, n2) > COS_FEAT * (sqrt(dot(n1, n1)) * sqrt(dot(n2, n2)));
                cand = cand && dot(n1, ns) > 0.0 && dot(n2, ns) > 0.0;
                cand = cand && !is_nb(t, c, d);
            }
        } else {
            cand = !w.crease[e] && w.ncrease[a] == 0 && w.ncrease[b] == 0 && len2 < lo2 && deg(c) > 3 && deg(d) > 3 &&
                   (double)sqd[e] <= dlim2;
            if (cand) {
                int common = 0;
                for (int i = t.vert_off[a]; i < t.vert_off[a + 1]; ++i)
                    common += is_nb(t, b, other(t.edges, t.vert_edges[i], a));
                const D3 m = mul(add(pa, pb), 0.5);
                cand = common == 2 && collapse_side(t, P, w, a, b, m, hi2) && collapse_side(t, P, w, b, a, m, hi2);
            }
        }
    }
    if (cand) {
        unsigned long long q = (unsigned long long)__double_as_longlong(len2) >> 32;
        if (op != OP_COLLAPSE) q = 0xFFFFFFFFull - q;
        key = (q << 32) | (unsigned long long)e;
    }
    w.key[e] = key;
}

__global__ void k_vmin1(icon_mesh_topology t, Ws w) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= t.V) return;
    unsigned long long m = NONE;
    for (int i = t.vert_off[v]; i < t.vert_off[v + 1]; ++i) { const unsigned long long k = w.key[t.vert_edges[i]]; m = k < m ? k : m; }
    w.m1[v] = m;
}

__global__ void k_vmin2(icon_mesh_topology t, Ws w) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= t.V) return;
    unsigned long long m = w.m1[v];
    for (int i = t.vert_off[v]; i < t.vert_off[v + 1]; ++i) {
        const unsigned long long k = w.m1[other(t.edges, t.vert_edges[i], v)];
        m = k < m ? k : m;
    }
    w.m2[v] = m;
}

__global__ void k_winners(icon_mesh_topology t, const unsigned long long *__restrict__ m, Ws w) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= t.E) return;
    const unsigned long long k = w.key[e];
    int win = 0;
    if (k != NONE) {
        const int a = (int)t.edges[2 * (int64_t)e], b = (int)t.edges[2 * (int64_t)e + 1];
        win = k <= m[a] && k <= m[b] && k <= m[w.ec[e]] && k <= m[w.ed[e]];
    }
    w.win[e] = win;
}

// ------------------------------------------------------------------ apply

__device__ __forceinline__ int winning_col(const icon_mesh_topology &t, const Ws &w, int f) {
    for (int k = 0; k < 3; ++k)
        if (w.win[t.face_to_edge[3 * (int64_t)f + k]]) return k;
    return -1;
}

__global__ void k_split_verts(icon_mesh_topology t, const double *__restrict__ P, Ws w, double *__restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < t.V) st3(out, e, ld(P, e));
    if (e < t.E && w.win[e])
        st3(out, (int64_t)t.V + w.rank[e],
            mul(add(ld(P, t.edges[2 * (int64_t)e]), ld(P, t.edges[2 * (int64_t)e + 1])), 0.5));
}

__global__ void k_face_counts(int op, icon_mesh_topology t, Ws w) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= t.F) return;
    const int k = winning_col(t, w, f);
    w.fcnt[f] = op == OP_SPLIT ? (k >= 0 ? 2 : 1) : (k >= 0 ? 0 : 1);
}

__global__ void k_split_faces(icon_mesh_topology t, Ws w, int64_t *__restrict__ out) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= t.F) return;
    const int64_t *fv = t.faces + 3 * (int64_t)f;
    int64_t *o = out + 3 * (int64_t)w.fpos[f];
    const int k = winning_col(t, w, f);
    if (k < 0) { o[0] = fv[0]; o[1] = fv[1]; o[2] = fv[2]; return; }
    const int64_t i0 = fv[k], i1 = fv[(k + 1) % 3], i2 = fv[(k + 2) % 3];
    const int64_t m = (int64_t)t.V + w.rank[t.face_to_edge[3 * (int64_t)f + k]];
    o[0] = i0; o[1] = i1; o[2] = m;
    o[3] = i0; o[4] = m; o[5] = i2;
}

__global__ void k_flip_faces(icon_mesh_topology t, Ws w, int64_t *__restrict__ out) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= t.F) return;
    const int64_t *fv = t.faces + 3 * (int64_t)f;
    int64_t *o = out + 3 * (int64_t)f;
    const int k = winning_col(t, w, f);
    if (k < 0) { o[0] = fv[0]; o[1] = fv[1]; o[2] = fv[2]; return; }
    const int e = (int)t.face_to_edge[3 * (int64_t)f + k];
    const int64_t a = t.edges[2 * (int64_t)e], b = t.edges[2 * (int64_t)e + 1], c = w.ec[e], d = w.ed[e];
    if (w.efa[e] == f) { o[0] = a; o[1] = d; o[2] = c; }
    else { o[0] = d; o[1] = b; o[2] = c; }
}

__global__ void k_collapse_mark(icon_mesh_topology t, Ws w) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= t.V) return;
    int tg = v, keep = 1;
    // v is the b of at most one winner: winners do not share a vertex
    for (int i = t.vert_off[v]; i < t.vert_off[v + 1]; ++i) {
        const int e = t.vert_edges[i];
        if (w.win[e] && t.edges[2 * (int64_t)e + 1] == v) { tg = (int)t.edges[2 * (int64_t)e]; keep = 0; }
    }
    w.tgt[v] = tg;
    w.keep[v] = keep;
}

__global__ void k_collapse_verts(icon_mesh_topology t, const double *__restrict__ P, Ws w, double *__restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= t.V || !w.keep[v]) return;
    D3 p = ld(P, v);
    for (int i = t.vert_off[v]; i < t.vert_off[v + 1]; ++i) {
        const int e = t.vert_edges[i];
        if (w.win[e] && t.edges[2 * (int64_t)e] == v) p = mul(add(ld(P, v), ld(P, t.edges[2 * (int64_t)e + 1])), 0.5);
    }
    st3(out, w.newid[v], p);
}

__global__ void k_collapse_faces(icon_mesh_topology t, Ws w, int64_t *__restrict__ out) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= t.F || !w.fcnt[f]) return;
    const int64_t *fv = t.faces + 3 * (int64_t)f;
    int64_t *o = out + 3 * (int64_t)w.fpos[f];
    for (int k = 0; k < 3; ++k) o[k] = w.newid[w.tgt[fv[k]]];
}

// ------------------------------------------------------------------ relax and reproject

__global__ void k_relax(icon_mesh_topology t, const double *__restrict__ P, const float *__restrict__ nrm, Ws w,
                        double *__restrict__ out, float *__restrict__ out32, int32_t *__restrict__ moved) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= t.V) return;
    const int o = t.vert_off[v], deg = t.vert_off[v + 1] - o;
    D3 s = {0.0, 0.0, 0.0};
    int q1 = -1, q2 = -1;
    for (int i = 0; i < deg; ++i) {
        const int e = t.vert_edges[o + i], u = other(t.edges, e, v);
        s = add(s, ld(P, u));
        if (w.crease[e]) { if (q1 < 0) q1 = u; else q2 = u; }
    }
    const D3 p = ld(P, v);
    D3 r = p;
    int mv = 0;
    if (!w.frozen[v] && w.ncrease[v] == 0) {
        const double dg = (double)deg;
        const D3 dv = sub({s.x / dg, s.y / dg, s.z / dg}, p);
        const D3 n = {(double)nrm[3 * (int64_t)v], (double)nrm[3 * (int64_t)v + 1], (double)nrm[3 * (int64_t)v + 2]};
        const double tt = dot(dv, n);
        r = add(p, sub(dv, mul(n, tt)));
        mv = 1;
    } else if (!w.frozen[v] && w.ncrease[v] == 2) {
        const D3 A = ld(P, q1), B = ld(P, q2);
        const D3 ctr = mul(add(A, B), 0.5), dr = sub(B, A);
        const double dd = dot(dr, dr);
        const double tt = dd > 0.0 ? dot(sub(ctr, p), dr) / dd : 0.0;
        r = add(p, mul(dr, tt));
        mv = 1;
    }
    st3(out, v, r);
    out32[3 * (int64_t)v] = (float)r.x; out32[3 * (int64_t)v + 1] = (float)r.y; out32[3 * (int64_t)v + 2] = (float)r.z;
    moved[v] = mv;
}

__device__ __forceinline__ double safe_div(double x, double y) { return y != 0.0 ? x / y : 0.0; }

__device__ D3 closest_point(D3 p, D3 a, D3 b, D3 c) {
    const D3 ab = sub(b, a), ac = sub(c, a), ap = sub(p, a);
    const double d1 = dot(ab, ap), d2 = dot(ac, ap);
    const D3 bp = sub(p, b);
    const double d3 = dot(ab, bp), d4 = dot(ac, bp);
    const D3 cp = sub(p, c);
    const double d5 = dot(ab, cp), d6 = dot(ac, cp);
    const double vc = d1 * d4 - d3 * d2, vb = d5 * d2 - d1 * d6, va = d3 * d6 - d5 * d4;
    if (d1 <= 0.0 && d2 <= 0.0) return a;
    if (d3 >= 0.0 && d4 <= d3) return b;
    if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) return add(a, mul(ab, safe_div(d1, d1 - d3)));
    if (d6 >= 0.0 && d5 <= d6) return c;
    if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) return add(a, mul(ac, safe_div(d2, d2 - d6)));
    if (va <= 0.0 && (d4 - d3) >= 0.0 && (d5 - d6) >= 0.0)
        return add(b, mul(sub(c, b), safe_div(d4 - d3, (d4 - d3) + (d5 - d6))));
    const double s = (va + vb) + vc;
    if (s == 0.0) return a;
    const double inv = 1.0 / s;
    return add(add(a, mul(ab, vb * inv)), mul(ac, vc * inv));
}

__global__ void k_reproject(const double *__restrict__ P, int V, const int32_t *__restrict__ moved,
                            const int32_t *__restrict__ face, const double *__restrict__ R,
                            const int64_t *__restrict__ rf, double *__restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const D3 p = ld(P, v);
    if (!moved[v]) { st3(out, v, p); return; }
    const int64_t *fv = rf + 3 * (int64_t)face[v];
    st3(out, v, closest_point(p, ld(R, fv[0]), ld(R, fv[1]), ld(R, fv[2])));
}

// ------------------------------------------------------------------ compaction of the input

__global__ void k_ref_mark(const int64_t *__restrict__ faces, int64_t n, int32_t *__restrict__ keep) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) keep[faces[i]] = 1;
}

__global__ void k_ref_gather(const double *__restrict__ P, int V, const int32_t *__restrict__ keep,
                             const int32_t *__restrict__ newid, double *__restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < V && keep[v]) st3(out, newid[v], ld(P, v));
}

__global__ void k_ref_faces(const int64_t *__restrict__ faces, int64_t n, const int32_t *__restrict__ newid,
                            int64_t *__restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = newid[faces[i]];
}

inline unsigned blocks(int64_t n) { return (unsigned)((n + TPB - 1) / TPB); }

bool topo_ok(const icon_mesh_topology *t) {
    return t && t->faces && t->edges && t->face_to_edge && t->vert_off && t->vert_edges && t->edge_off &&
           t->edge_entries && t->corner_off && t->vert_corners && t->V > 0 && t->F > 0 && t->E > 0;
}

}  // namespace

extern "C" size_t icon_remesh_workspace_bytes(int V, int F, int E) {
    if (V < 1) V = 1; if (F < 1) F = 1; if (E < 1) E = 1;
    return ws_layout(V, F, E, nullptr, nullptr);
}

#define REMESH_WS(fn, t)                                                                                         \
    ICON_CHECK_ARG(topo_ok(t), fn ": bad topology");                                                             \
    ICON_CHECK_ARG(ws && ws_bytes >= icon_remesh_workspace_bytes((t)->V, (t)->F, (t)->E), fn ": workspace too small"); \
    const Ws w = ws_view((t)->V, (t)->F, (t)->E, ws)

extern "C" int icon_remesh_compact(const double *verts, int V, const int64_t *faces, int F, double *out_verts,
                                   int64_t *out_faces, int64_t *d_count, void *ws, size_t ws_bytes,
                                   icon_stream_t stream) {
    ICON_CHECK_ARG(verts && faces && out_verts && out_faces && d_count && ws, "icon_remesh_compact: null pointer");
    ICON_CHECK_ARG(V > 0 && F > 0, "icon_remesh_compact: bad sizes V=%d F=%d", V, F);
    ICON_CHECK_ARG(ws_bytes >= icon_remesh_workspace_bytes(V, F, 1), "icon_remesh_compact: workspace too small");
    cudaStream_t s = (cudaStream_t)stream;
    const Ws w = ws_view(V, F, 1, ws);
    const int64_t n = 3 * (int64_t)F;
    ICON_CUDA(cudaMemsetAsync(w.keep, 0, sizeof(int32_t) * V, s));
    k_ref_mark<<<blocks(n), TPB, 0, s>>>(faces, n, w.keep); ICON_LAUNCHED();
    if (int rc = icon::scan_exclusive_i32(w.keep, w.newid, V, d_count, w.scan, s)) return rc;
    k_ref_gather<<<blocks(V), TPB, 0, s>>>(verts, V, w.keep, w.newid, out_verts); ICON_LAUNCHED();
    k_ref_faces<<<blocks(n), TPB, 0, s>>>(faces, n, w.newid, out_faces); ICON_LAUNCHED();
    return 0;
}

extern "C" int icon_remesh_classify(const icon_mesh_topology *t, const double *verts, void *ws, size_t ws_bytes,
                                    icon_stream_t stream) {
    REMESH_WS("icon_remesh_classify", t);
    ICON_CHECK_ARG(verts, "icon_remesh_classify: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    k_face_normals<<<blocks(t->F), TPB, 0, s>>>(verts, t->faces, t->F, w.fn, w.fa2); ICON_LAUNCHED();
    k_edge_class<<<blocks(t->E), TPB, 0, s>>>(*t, w); ICON_LAUNCHED();
    k_vert_class<<<blocks(t->V), TPB, 0, s>>>(*t, w); ICON_LAUNCHED();
    return 0;
}

extern "C" int icon_remesh_smooth_step(const icon_mesh_topology *t, const double *verts, double *out, void *ws,
                                       size_t ws_bytes, icon_stream_t stream) {
    REMESH_WS("icon_remesh_smooth_step", t);
    ICON_CHECK_ARG(verts && out && verts != out, "icon_remesh_smooth_step: null or aliased pointer");
    cudaStream_t s = (cudaStream_t)stream;
    k_cot_weights<<<blocks(t->E), TPB, 0, s>>>(*t, verts, w); ICON_LAUNCHED();
    k_smooth<<<blocks(t->V), TPB, 0, s>>>(*t, verts, w, out); ICON_LAUNCHED();
    return 0;
}

extern "C" int icon_remesh_midpoints(const icon_mesh_topology *t, const double *verts, float *out,
                                     icon_stream_t stream) {
    ICON_CHECK_ARG(topo_ok(t) && verts && out, "icon_remesh_midpoints: null pointer");
    k_midpoints<<<blocks(t->E), TPB, 0, (cudaStream_t)stream>>>(*t, verts, out); ICON_LAUNCHED();
    return 0;
}

extern "C" int icon_remesh_select(int op, const icon_mesh_topology *t, const double *verts, double L, int adaptive,
                                  const float *sqdist, double dlim2, int64_t *d_count, void *ws, size_t ws_bytes,
                                  icon_stream_t stream) {
    REMESH_WS("icon_remesh_select", t);
    ICON_CHECK_ARG(op >= OP_SPLIT && op <= OP_FLIP, "icon_remesh_select: bad op %d", op);
    ICON_CHECK_ARG(verts && d_count && (op != OP_COLLAPSE || sqdist), "icon_remesh_select: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    k_candidates<<<blocks(t->E), TPB, 0, s>>>(op, *t, verts, L, adaptive, sqdist, dlim2, w); ICON_LAUNCHED();
    k_vmin1<<<blocks(t->V), TPB, 0, s>>>(*t, w); ICON_LAUNCHED();
    const unsigned long long *m = w.m1;
    if (op != OP_SPLIT) { k_vmin2<<<blocks(t->V), TPB, 0, s>>>(*t, w); ICON_LAUNCHED(); m = w.m2; }
    k_winners<<<blocks(t->E), TPB, 0, s>>>(*t, m, w); ICON_LAUNCHED();
    return icon::scan_exclusive_i32(w.win, w.rank, t->E, d_count, w.scan, s);
}

extern "C" int icon_remesh_apply(int op, const icon_mesh_topology *t, const double *verts, int W, double *out_verts,
                                 int64_t *out_faces, void *ws, size_t ws_bytes, icon_stream_t stream) {
    REMESH_WS("icon_remesh_apply", t);
    ICON_CHECK_ARG(op >= OP_SPLIT && op <= OP_FLIP, "icon_remesh_apply: bad op %d", op);
    ICON_CHECK_ARG(verts && out_faces && (op == OP_FLIP || out_verts), "icon_remesh_apply: null pointer");
    ICON_CHECK_ARG(W > 0 && W <= t->E, "icon_remesh_apply: bad winner count %d", W);
    cudaStream_t s = (cudaStream_t)stream;
    if (op == OP_FLIP) {
        k_flip_faces<<<blocks(t->F), TPB, 0, s>>>(*t, w, out_faces); ICON_LAUNCHED();
        return 0;
    }
    k_face_counts<<<blocks(t->F), TPB, 0, s>>>(op, *t, w); ICON_LAUNCHED();
    if (int rc = icon::scan_exclusive_i32(w.fcnt, w.fpos, t->F, nullptr, w.scan, s)) return rc;
    if (op == OP_SPLIT) {
        const int n = t->V > t->E ? t->V : t->E;
        k_split_verts<<<blocks(n), TPB, 0, s>>>(*t, verts, w, out_verts); ICON_LAUNCHED();
        k_split_faces<<<blocks(t->F), TPB, 0, s>>>(*t, w, out_faces); ICON_LAUNCHED();
        return 0;
    }
    k_collapse_mark<<<blocks(t->V), TPB, 0, s>>>(*t, w); ICON_LAUNCHED();
    if (int rc = icon::scan_exclusive_i32(w.keep, w.newid, t->V, nullptr, w.scan, s)) return rc;
    k_collapse_verts<<<blocks(t->V), TPB, 0, s>>>(*t, verts, w, out_verts); ICON_LAUNCHED();
    k_collapse_faces<<<blocks(t->F), TPB, 0, s>>>(*t, w, out_faces); ICON_LAUNCHED();
    return 0;
}

extern "C" int icon_remesh_relax(const icon_mesh_topology *t, const double *verts, const float *normals, double *out,
                                 float *out32, int32_t *moved, void *ws, size_t ws_bytes, icon_stream_t stream) {
    REMESH_WS("icon_remesh_relax", t);
    ICON_CHECK_ARG(verts && normals && out && out32 && moved && verts != out, "icon_remesh_relax: null or aliased pointer");
    k_relax<<<blocks(t->V), TPB, 0, (cudaStream_t)stream>>>(*t, verts, normals, w, out, out32, moved); ICON_LAUNCHED();
    return 0;
}

extern "C" int icon_remesh_reproject(const double *verts, int V, const int32_t *moved, const int32_t *face,
                                     const double *ref_verts, const int64_t *ref_faces, double *out,
                                     icon_stream_t stream) {
    ICON_CHECK_ARG(verts && moved && face && ref_verts && ref_faces && out && verts != out,
                   "icon_remesh_reproject: null or aliased pointer");
    ICON_CHECK_ARG(V > 0, "icon_remesh_reproject: bad size V=%d", V);
    k_reproject<<<blocks(V), TPB, 0, (cudaStream_t)stream>>>(verts, V, moved, face, ref_verts, ref_faces, out);
    ICON_LAUNCHED();
    return 0;
}
