// The SMPL-family body model's linear-blend skinning, lbs() of lib/smplx/lbs.py:152-252, forward and backward: the
// body-fit loop of apps/infer.py:168-273 calls it once per iteration through SMPL.forward.  Restated by
// oracle/body_model.py (float64 NumPy, explicit backward); pinned against the reference's own lib/smplx by
// tests/golden/body_model.npz.
//
// Model (icon_lbs_model, fp32 device buffers): v_template [V,3], shapedirs [V,3,NB], posedirs [P,3V] with P = 9(J-1),
// J_regressor [J,V], lbs_weights [V,J], parents (host, checked at prepare: parents[0] = -1, parents[i] < i, J <= 64).
// icon_lbs_prepare builds J_template = J_regressor v_template [J,3] and J_dirs = J_regressor shapedirs [J,3,NB] in
// fp64 (vertex chunks of LBS_PREP_V summed in ascending order, then the chunks in ascending order), so a call's rest
// joints J = J_template + J_dirs beta need no pass over V.
//
// Forward, per batch item b (every value below fp64, from the fp32 inputs; outputs rounded to fp32 once):
//   beta = betas[b] (NB); R_j = pose[b, j] [3,3] as given (pose2rot = 0; never re-orthonormalised), or with
//     pose2rot = 1 Rodrigues of r = pose[b, j] [3] with the reference's quirk: s = r + 1e-8 per component,
//     theta = |s|, d = r / theta, K = [d]x, R = I + sin(theta) K + (1 - cos(theta)) K K.
//   J_j = J_template_j + sum_k J_dirs[j,:,k] beta_k (k ascending).
//   rel_0 = J_0, rel_j = J_j - J_parent(j);  G_0 = [R_0 | rel_0], G_j = G_parent(j) [R_j | rel_j] (3x4, the implied
//     last row 0 0 0 1), computed level by level from the root; joints[b, j] = G_j[:, 3];
//     A_j = [G_j.R | G_j.t - G_j.R J_j].
//   v_shaped = v_template + sum_k shapedirs[v,c,k] beta_k; pf_p = R_{1 + p/9}[p%9] - I[p%9];
//   v_posed = v_shaped + sum_p pf_p posedirs[p, 3v + c] (p ascending);
//   T_v = sum_j lbs_weights[v,j] A_j (j ascending), verts[b, v] = T_v.R v_posed + T_v.t.
// Backward (g_verts and / or g_joints; NULL = zero):
//   gT_v = g_v [v_posed | 1]^T, g_vposed = T_v.R^T g_v;  gA_j = sum_v w[v,j] gT_v;  g_pf = posedirs g_vposed;
//   g_beta = shapedirs^T g_vposed + J_dirs^T g_J.
//   gG_j = [gA_j.R - gA_j.t J_j^T | gA_j.t + g_joints_j], g_J_j = -G_j.R^T gA_j.t; then children before parents:
//   gG_p += [gG_j.R R_j^T + gG_j.t rel_j^T | gG_j.t] (children in ascending order), g_R_j = G_p.R^T gG_j.R,
//   g_rel_j = G_p.R^T gG_j.t (G_p = I for the root); g_J_j += g_rel_j - sum over children g_rel_i;
//   g_R_j += g_pf[9(j-1) ..] for j >= 1; pose2rot: the Rodrigues backward (sin / cos / the 1e-8 shift as above).
// Reductions: the skin backward writes per-tile partials (a tile = LBS_TV vertices; within a tile the sums over
//   vertices are in ascending order, the posedirs / shapedirs dots are a per-lane ascending sum over the tile's
//   columns and a fixed xor-butterfly); the chain backward adds the tiles in ascending order.  No float atomics
//   anywhere: results are bitwise reproducible, and row b of a B-row call equals a one-row call on that row.
// Layout of a call's state (icon_lbs_state_bytes): a header (pose2rot), R [B,J,9], G [B,J,12], A [B,J,12],
//   J [B,J,3], r [B,J,3] (pose2rot only), v_posed [B,V,3], all fp64.
// -fmad=false, as the other geometry units.
//
// Heads: the landmark and joint heads of PIXIE's SMPLX.forward (lib/pixielib/models/SMPLX.py:261-293, lbs.py:38-145,
// 427-434), read from the fp32 `verts` icon_lbs_forward wrote, as the reference reads its own.  Restated by the heads
// part of oracle/body_model.py; pinned against the reference's class by tests/golden/pixie_body_model.npz.
//   Prepared once per model (icon_smplx_heads_prepare, host-checked): corner vertex ids and barycentrics of the
//   static landmarks [Ls,3], the lookup table [79,Ld,3] and the extra joints [E,3] ("slots", in that order), the
//   regressor row written over each joint (source_idxs / target_idxs), the head chain, and per vertex the slots that
//   read it, in (entry, table row, corner) order.
//   Forward, per batch item b (fp64 from the fp32 inputs; each output rounded to fp32 once):
//     row: rel = I, rel <- R[chain[i]] rel for i ascending (the pose as given; the reference detaches it, so the
//       row is not differentiated); a = (-atan2(-rel[2,0], sqrt(rel00^2 + rel10^2)) 180) / pi;
//       y = round_half_even(min(a, 39)); row = y >= 0 ? y : (y < -39 ? 78 : 39 - y).  The reference computes rel in
//       fp32: the row equals the reference's wherever a is at least 1e-3 degrees from a half-integer (fp32 rounding
//       of the six 3x3 products moves a by about 1e-4 degrees for matrices with entries of order 1).
//     landmark / extra entry = (w0 v[i0] + w1 v[i1]) + w2 v[i2] (corner order); the dynamic entries use table row
//       `row`.  reg[r] = sum over v of R[r,v] v[v]: per chunk of HEADS_CV vertices a warp's lanes sum their
//       vertices in ascending order and a fixed xor-butterfly adds the lanes; the chunks are added in ascending
//       order.  joints = cat[J_transformed, landmarks, extra] with joints[source_s] = reg[target_s] (the
//       reference's `detach() * 0 + reg`, equal to reg for a finite J_transformed).
//   Backward (NULL upstreams are zero; fp32 g_verts_heads, one thread per (b, vertex column)): u_e =
//     g_landmarks[e] + g_joints[J + e]; g_v = sum over the slots reading v, in `inc` order, of w_slot u_e (the
//     dynamic slots of other table rows skipped), then + sum over r ascending of R[r,v] g_joints[source of r].
//     g_J_transformed = g_joints[:, :J] with zeros at the sources (the `detach() * 0`).  No float atomics.
//   Launches: two forward (k_heads_reg_partial, k_heads_finish), one backward (k_heads_backward).
//
// Tetra body: PaMIR's TestDataset.compute_voxel_verts (lib/dataset/TestDataset.py:150-192) with TetraSMPLModel.update
// (lib/dataset/body_model.py:344-427) and pymaf's rotation_matrix_to_angle_axis (lib/pymaf/utils/geometry.py).
// Restated by oracle/tetra_body.py; pinned against the reference's own class and conversion, run live, by
// tests/golden/tetra_body.npz.
//   Model (icon_tetra_model, fp64 device buffers, the SMPL vertices then the added ones, N = V + V_added <= 8000):
//   v_template [N,3], shapedirs [10,3N], posedirs [207,3N] (transposed from the files' [N,3,k]), weights [N,24],
//   J_regressor's nonzeros per joint in ascending column order (the order scipy's sparse product sums in; a dense
//   file's zero entries add nothing), parents from kintree_table (checked at prepare: 24 joints, parents[i] < i).
//   T <= 25100 tetrahedra are padded by the host; the kernels never read them.
//   Promotion chain (NumPy >= 2, confirmed on the golden's live run): the pose and betas arrive as fp32 arrays;
//   np.linalg.norm of the fp32 pose stays fp32, np.maximum with np.finfo(np.float64).tiny widens theta, and every
//   later value is fp64 (the fp64 model arrays dotted with the widened betas; r / theta widens r).  NumPy 1.x would
//   keep theta in fp32: this restates NumPy 2.
//   Forward (k_tetra_chain, one CTA):
//     aa_j (fp32): t = R_j^T; d2 = t22 < 1e-6f, d0d1 = t00 > t11, d0nd1 = t00 < -t11; t0 = ((1 + t00) - t11) - t22,
//       t1 = ((1 - t00) + t11) - t22, t2 = ((1 - t00) - t11) + t22, t3 = ((1 + t00) + t11) + t22 and the four
//       candidates q0..q3; with 0/1 masks m0..m3 (d2 d0d1, d2 !d0d1, !d2 d0nd1, !d2 !d0nd1):
//       q = ((((q0 m0 + q1 m1) + q2 m2) + q3 m3) / sqrt(((t0 m0 + t1 m1) + t2 m2) + t3 m3)) 0.5;
//       s2 = (q1^2 + q2^2) + q3^2, two = 2 (q0 < 0 ? atan2(-sqrt s2, -q0) : atan2(sqrt s2, q0)),
//       k = s2 > 0 ? two / sqrt s2 : 2, aa = 0 + q_{1..3} k, NaN -> 0.  Each step one fp32 rounding, as each torch
//       op is; atan2f differs from torch's CPU atan2 by a few ulps.  With rotmats = NULL, aa is read as given.
//     R_j (fp64): theta = max((double)sqrtf((x^2 + y^2) + z^2), DBL_MIN), rh = r / theta,
//       R = (cos I + (1 - cos) rh rh^T) + sin [rh]x (no 1e-8 shift: the model's own rodrigues, not batch_rodrigues).
//     J_j = sum over J_regressor's nonzeros v (ascending) of w v_shaped[v], v_shaped = shapedirs . beta (k
//       ascending) + v_template.  G_0 = [R_0 | J_0], G_j = G_parent [R_j | J_j - J_parent], level by level;
//       A_j = [G_j.R | G_j.t - G_j.R J_j] (the rest-pose removal); lrotmin_p = R_{1 + p/9}[p%9] - I[p%9].
//   Forward (k_tetra_skin, 64 output rows per CTA, one thread per (row, component) of the 8000 x 3 output):
//     v_posed = v_shaped + sum_p lrotmin_p posedirs[p] (p ascending); T = sum_j weights[v,j] A_j (j ascending);
//     v = (((T0 x + T1 y) + T2 z) + T3) + 0 (the model's zero trans); out = fp32(v (double)scale + (double)trans)
//     (the reference's scale.item() and the fp32 trans widened), rows >= N are 0; then x 0.5f, and z x -1.0f (the
//     padding's z is -0.0f, as the reference's array holds).
//   No float atomics, no host sync: scale and trans are read on the device.  Launches: two (k_tetra_chain,
//   k_tetra_skin).
#include <float.h>
#include <math.h>

#include <vector>

#include "common.cuh"

namespace icon {

constexpr int LBS_MAXJ = 64;
constexpr int LBS_MAXP = 9 * (LBS_MAXJ - 1);
constexpr int LBS_MAXNB = 1024;
constexpr int LBS_TV = 64;              // vertices per skin tile
constexpr int LBS_T = 3 * LBS_TV;       // skin threads: one per (vertex, component) column 3 v + c
constexpr int LBS_PREP_V = 1024;        // vertices per prepare chunk
constexpr int LBS_PREP_T = 128;
constexpr int LBS_CB_T = 512;           // chain-backward threads (>= LBS_MAXJ)

struct LbsState {
    int *hdr;
    double *R, *G, *A, *J, *aa, *vp;
};

static size_t lbs_state_carve(void *base, int B, int V, int J, LbsState *s) {
    Carver c(base);
    LbsState t;
    t.hdr = c.take<int>(4);
    t.R = c.take<double>((size_t)B * J * 9);
    t.G = c.take<double>((size_t)B * J * 12);
    t.A = c.take<double>((size_t)B * J * 12);
    t.J = c.take<double>((size_t)B * J * 3);
    t.aa = c.take<double>((size_t)B * J * 3);
    t.vp = c.take<double>((size_t)B * V * 3);
    if (s) *s = t;
    return c.total();
}

static inline int lbs_tiles(int V) { return (V + LBS_TV - 1) / LBS_TV; }
static inline int lbs_outputs(int J, int NB) { return 12 * J + 9 * (J - 1) + NB; }

__device__ __forceinline__ void lbs_rodrigues(const double r[3], double R[9]) {
    const double s0 = r[0] + 1e-8, s1 = r[1] + 1e-8, s2 = r[2] + 1e-8;
    const double th = sqrt(s0 * s0 + s1 * s1 + s2 * s2);
    const double dx = r[0] / th, dy = r[1] / th, dz = r[2] / th;
    const double sn = sin(th), c1 = 1.0 - cos(th);
    const double K[9] = {0.0, -dz, dy, dz, 0.0, -dx, -dy, dx, 0.0};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const double kk = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
            R[3 * i + j] = ((i == j ? 1.0 : 0.0) + sn * K[3 * i + j]) + c1 * kk;
        }
}

// gR [9] -> g_r [3] of lbs_rodrigues
__device__ __forceinline__ void lbs_rodrigues_backward(const double r[3], const double gR[9], double gr[3]) {
    const double s[3] = {r[0] + 1e-8, r[1] + 1e-8, r[2] + 1e-8};
    const double th = sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
    const double dx = r[0] / th, dy = r[1] / th, dz = r[2] / th;
    const double sn = sin(th), cs = cos(th), c1 = 1.0 - cs;
    const double K[9] = {0.0, -dz, dy, dz, 0.0, -dx, -dy, dx, 0.0};
    double gK[9], gsin = 0.0, gc1 = 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            // (gR K^T)_ij = sum_k gR_ik K_jk ; (K^T gR)_ij = sum_k K_ki gR_kj ; (K K)_ij
            const double a = gR[3 * i] * K[3 * j] + gR[3 * i + 1] * K[3 * j + 1] + gR[3 * i + 2] * K[3 * j + 2];
            const double b = K[i] * gR[j] + K[3 + i] * gR[3 + j] + K[6 + i] * gR[6 + j];
            const double kk = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
            gK[3 * i + j] = sn * gR[3 * i + j] + c1 * (a + b);
            gsin = gsin + gR[3 * i + j] * K[3 * i + j];
            gc1 = gc1 + gR[3 * i + j] * kk;
        }
    double gth = cs * gsin + sn * gc1;
    const double gd[3] = {gK[7] - gK[5], gK[2] - gK[6], gK[3] - gK[1]};
    gth = gth - (gd[0] * r[0] + gd[1] * r[1] + gd[2] * r[2]) / (th * th);
#pragma unroll
    for (int c = 0; c < 3; ++c) gr[c] = gd[c] / th + gth * (s[c] / th);
}

// ---------------------------------------------------------------- prepare: J_template, J_dirs

__global__ void __launch_bounds__(LBS_PREP_T) k_lbs_prepare_partial(icon_lbs_model m, double *part) {
    const int j = blockIdx.x, s = blockIdx.y, NB = m.NB, Q = 3 * (NB + 1);
    const int v0 = s * LBS_PREP_V, v1 = min(m.V, v0 + LBS_PREP_V);
    double *out = part + ((size_t)j * gridDim.y + s) * Q;
    for (int q = threadIdx.x; q < Q; q += LBS_PREP_T) {
        double acc = 0.0;
        if (q < 3) {
            for (int v = v0; v < v1; ++v)
                acc = acc + (double)m.J_regressor[(int64_t)j * m.V + v] * (double)m.v_template[3 * (int64_t)v + q];
        } else {
            const int ck = q - 3;          // c * NB + k
            for (int v = v0; v < v1; ++v)
                acc = acc + (double)m.J_regressor[(int64_t)j * m.V + v] *
                                (double)m.shapedirs[(int64_t)v * 3 * NB + ck];
        }
        out[q] = acc;
    }
}

__global__ void __launch_bounds__(LBS_PREP_T) k_lbs_prepare_reduce(icon_lbs_model m, const double *part, int S) {
    const int j = blockIdx.x, NB = m.NB, Q = 3 * (NB + 1);
    for (int q = threadIdx.x; q < Q; q += LBS_PREP_T) {
        double acc = 0.0;
        for (int s = 0; s < S; ++s) acc = acc + part[((size_t)j * S + s) * Q + q];
        if (q < 3) m.J_template[3 * j + q] = acc;
        else m.J_dirs[(size_t)j * 3 * NB + (q - 3)] = acc;
    }
}

// ---------------------------------------------------------------- forward

__device__ __forceinline__ int lbs_depth(const icon_lbs_model &m, int j) {
    int d = 0;
    for (int i = m.parents[j]; i >= 0; i = m.parents[i]) ++d;
    return d;
}

// one CTA per batch item: rest joints, rotations, the chain, A and the posed joints
__global__ void __launch_bounds__(LBS_MAXJ) k_lbs_chain(icon_lbs_model m, const float *__restrict__ betas,
                                                        const float *__restrict__ pose, int pose2rot,
                                                        float *__restrict__ joints, LbsState st) {
    __shared__ double sJ[LBS_MAXJ][3], sR[LBS_MAXJ][9], sG[LBS_MAXJ][12];
    const int b = blockIdx.x, j = threadIdx.x, J = m.J, NB = m.NB;
    const size_t bj = (size_t)b * J + j;
    if (b == 0 && j == 0) st.hdr[0] = pose2rot;
    int depth = 0;
    if (j < J) {
        const float *bt = betas + (size_t)b * NB;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            double acc = m.J_template[3 * j + c];
            const double *jd = m.J_dirs + ((size_t)j * 3 + c) * NB;
            for (int k = 0; k < NB; ++k) acc = acc + jd[k] * (double)bt[k];
            sJ[j][c] = acc;
            st.J[3 * bj + c] = acc;
        }
        double R[9];
        if (pose2rot) {
            double r[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                r[c] = (double)pose[3 * bj + c];
                st.aa[3 * bj + c] = r[c];
            }
            lbs_rodrigues(r, R);
        } else {
#pragma unroll
            for (int e = 0; e < 9; ++e) R[e] = (double)pose[9 * bj + e];
        }
#pragma unroll
        for (int e = 0; e < 9; ++e) {
            sR[j][e] = R[e];
            st.R[9 * bj + e] = R[e];
        }
        depth = lbs_depth(m, j);
    }
    __syncthreads();
    for (int d = 0; __syncthreads_or(j < J && depth >= d); ++d) {
        if (j < J && depth == d) {
            const int p = m.parents[j];
            double rel[3], G[12];
#pragma unroll
            for (int c = 0; c < 3; ++c) rel[c] = p < 0 ? sJ[j][c] : sJ[j][c] - sJ[p][c];
            if (p < 0) {
#pragma unroll
                for (int r = 0; r < 3; ++r) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) G[4 * r + c] = sR[j][3 * r + c];
                    G[4 * r + 3] = rel[r];
                }
            } else {
#pragma unroll
                for (int r = 0; r < 3; ++r) {
#pragma unroll
                    for (int c = 0; c < 3; ++c)
                        G[4 * r + c] = (sG[p][4 * r] * sR[j][c] + sG[p][4 * r + 1] * sR[j][3 + c]) +
                                       sG[p][4 * r + 2] * sR[j][6 + c];
                    G[4 * r + 3] = ((sG[p][4 * r] * rel[0] + sG[p][4 * r + 1] * rel[1]) + sG[p][4 * r + 2] * rel[2]) +
                                   sG[p][4 * r + 3];
                }
            }
#pragma unroll
            for (int e = 0; e < 12; ++e) {
                sG[j][e] = G[e];
                st.G[12 * bj + e] = G[e];
            }
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const double gj = (G[4 * r] * sJ[j][0] + G[4 * r + 1] * sJ[j][1]) + G[4 * r + 2] * sJ[j][2];
#pragma unroll
                for (int c = 0; c < 3; ++c) st.A[12 * bj + 4 * r + c] = G[4 * r + c];
                st.A[12 * bj + 4 * r + 3] = G[4 * r + 3] - gj;
                joints[3 * bj + r] = (float)G[4 * r + 3];
            }
        }
    }
}

// vertex tiles, every batch item per CTA: v_shaped, v_posed (kept in the state) and the skinned vertices
__global__ void __launch_bounds__(LBS_T) k_lbs_skin(icon_lbs_model m, int B, const float *__restrict__ betas,
                                                    LbsState st, float *__restrict__ verts) {
    __shared__ double s_pf[LBS_MAXP], s_A[LBS_MAXJ * 12], s_beta[LBS_MAXNB], s_vp[LBS_T];
    const int t = threadIdx.x, J = m.J, NB = m.NB, P = 9 * (J - 1);
    const int64_t V3 = 3 * (int64_t)m.V, col = (int64_t)blockIdx.x * LBS_T + t, v = col / 3;
    const int c = t % 3, vl = t / 3;
    const bool live = col < V3;
    for (int b = 0; b < B; ++b) {
        __syncthreads();
        for (int p = t; p < P; p += LBS_T) {
            const int e = p % 9;
            s_pf[p] = st.R[((size_t)b * J + 1 + p / 9) * 9 + e] - ((e == 0 || e == 4 || e == 8) ? 1.0 : 0.0);
        }
        for (int i = t; i < 12 * J; i += LBS_T) s_A[i] = st.A[(size_t)b * J * 12 + i];
        for (int k = t; k < NB; k += LBS_T) s_beta[k] = (double)betas[(size_t)b * NB + k];
        __syncthreads();
        double vp = 0.0;
        if (live) {
            double vs = (double)m.v_template[col];
            const float *sd = m.shapedirs + col * NB;
            for (int k = 0; k < NB; ++k) vs = vs + (double)sd[k] * s_beta[k];
            double po = 0.0;
            const float *pd = m.posedirs + col;
#pragma unroll 16
            for (int p = 0; p < P; ++p) po = po + s_pf[p] * (double)__ldg(pd + p * V3);
            vp = vs + po;
            st.vp[(size_t)b * V3 + col] = vp;
        }
        s_vp[t] = vp;
        __syncthreads();
        if (live) {
            double T[4] = {0.0, 0.0, 0.0, 0.0};
            const float *w = m.lbs_weights + v * J;
            for (int jj = 0; jj < J; ++jj) {
                const double wj = (double)w[jj];
#pragma unroll
                for (int q = 0; q < 4; ++q) T[q] = T[q] + wj * s_A[12 * jj + 4 * c + q];
            }
            const double out = ((T[0] * s_vp[3 * vl] + T[1] * s_vp[3 * vl + 1]) + T[2] * s_vp[3 * vl + 2]) + T[3];
            verts[(size_t)b * V3 + col] = (float)out;
        }
    }
}

// ---------------------------------------------------------------- backward

__device__ __forceinline__ double warp_sum_fixed(double x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = x + __shfl_xor_sync(0xffffffffu, x, o);
    return x;       // every lane holds the same value: a + b == b + a
}

// vertex tiles: per-tile partials [B][tiles][12 J + P + NB] of gA, g_pf and g_beta (through shapedirs)
__global__ void __launch_bounds__(LBS_T) k_lbs_skin_backward(icon_lbs_model m, int B, LbsState st,
                                                             const float *__restrict__ gv, double *__restrict__ part) {
    __shared__ double s_A[LBS_MAXJ * 12], s_T[LBS_T * 4], s_gT[LBS_TV * 12], s_g[LBS_T], s_gvp[LBS_T];
    const int t = threadIdx.x, J = m.J, NB = m.NB, P = 9 * (J - 1), NO = 12 * J + P + NB;
    const int lane = t & 31, warp = t >> 5, nwarp = LBS_T / 32;
    const int64_t V3 = 3 * (int64_t)m.V, col0 = (int64_t)blockIdx.x * LBS_T, col = col0 + t, v0 = col0 / 3;
    const int c = t % 3, vl = t / 3;
    const int nv = (int)min((int64_t)LBS_TV, (int64_t)m.V - v0);
    const bool live = col < V3;
    for (int b = 0; b < B; ++b) {
        __syncthreads();
        for (int i = t; i < 12 * J; i += LBS_T) s_A[i] = st.A[(size_t)b * J * 12 + i];
        s_g[t] = live ? (double)gv[(size_t)b * V3 + col] : 0.0;
        __syncthreads();
        if (live) {
            double T[4] = {0.0, 0.0, 0.0, 0.0};
            const float *w = m.lbs_weights + (col / 3) * J;
            for (int jj = 0; jj < J; ++jj) {
                const double wj = (double)w[jj];
#pragma unroll
                for (int q = 0; q < 4; ++q) T[q] = T[q] + wj * s_A[12 * jj + 4 * c + q];
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) s_T[4 * t + q] = T[q];
        }
        __syncthreads();
        double gvp = 0.0;
        if (live) {
            const double *vp = st.vp + (size_t)b * V3 + 3 * (col / 3);
            gvp = (s_T[4 * (3 * vl) + c] * s_g[3 * vl] + s_T[4 * (3 * vl + 1) + c] * s_g[3 * vl + 1]) +
                  s_T[4 * (3 * vl + 2) + c] * s_g[3 * vl + 2];
#pragma unroll
            for (int q = 0; q < 3; ++q) s_gT[12 * vl + 4 * c + q] = s_g[t] * vp[q];
            s_gT[12 * vl + 4 * c + 3] = s_g[t];
        }
        s_gvp[t] = gvp;
        __syncthreads();
        double *out = part + ((size_t)b * gridDim.x + blockIdx.x) * NO;
        for (int o = t; o < 12 * J; o += LBS_T) {
            const int jj = o / 12, e = o % 12;
            double acc = 0.0;
            for (int i = 0; i < nv; ++i) acc = acc + (double)m.lbs_weights[(v0 + i) * J + jj] * s_gT[12 * i + e];
            out[o] = acc;
        }
        for (int p = warp; p < P; p += nwarp) {
            double acc = 0.0;
            const float *pd = m.posedirs + (int64_t)p * V3 + col0;
#pragma unroll
            for (int i = 0; i < LBS_T / 32; ++i) {
                const int cc = lane + 32 * i;
                if (col0 + cc < V3) acc = acc + (double)__ldg(pd + cc) * s_gvp[cc];
            }
            acc = warp_sum_fixed(acc);
            if (lane == 0) out[12 * J + p] = acc;
        }
        for (int k = warp; k < NB; k += nwarp) {
            double acc = 0.0;
#pragma unroll
            for (int i = 0; i < LBS_T / 32; ++i) {
                const int cc = lane + 32 * i;
                if (col0 + cc < V3) acc = acc + (double)m.shapedirs[(col0 + cc) * NB + k] * s_gvp[cc];
            }
            acc = warp_sum_fixed(acc);
            if (lane == 0) out[12 * J + P + k] = acc;
        }
    }
}

// one CTA per batch item: the tile partials in ascending order, the reverse chain, g_pose and g_betas
__global__ void __launch_bounds__(LBS_CB_T) k_lbs_chain_backward(icon_lbs_model m, LbsState st,
                                                                 const double *__restrict__ part, int tiles,
                                                                 const float *__restrict__ gj,
                                                                 float *__restrict__ g_betas,
                                                                 float *__restrict__ g_pose) {
    __shared__ double s_o[12 * LBS_MAXJ + LBS_MAXP + LBS_MAXNB];
    __shared__ double s_gG[LBS_MAXJ][12], s_rel[LBS_MAXJ][3], s_grel[LBS_MAXJ][3], s_gJ[LBS_MAXJ][3];
    __shared__ int s_maxd;
    const int b = blockIdx.x, t = threadIdx.x, J = m.J, NB = m.NB, P = 9 * (J - 1), NO = 12 * J + P + NB;
    const int pose2rot = st.hdr[0];
    if (t == 0) s_maxd = 0;
    for (int o = t; o < NO; o += LBS_CB_T) {
        double acc = 0.0;
        if (part)
            for (int i = 0; i < tiles; ++i) acc = acc + part[((size_t)b * tiles + i) * NO + o];
        s_o[o] = acc;
    }
    __syncthreads();
    const double *gA = s_o, *gpf = s_o + 12 * J, *gb = s_o + 12 * J + P;
    const int j = t;
    const size_t bj = (size_t)b * J + j;
    int depth = 0;
    double gJ[3] = {0.0, 0.0, 0.0};
    if (j < J) {
        const double *Jj = st.J + 3 * bj, *G = st.G + 12 * bj;
        const int p = m.parents[j];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const double gt = gA[12 * j + 4 * r + 3];
#pragma unroll
            for (int c = 0; c < 3; ++c) s_gG[j][4 * r + c] = gA[12 * j + 4 * r + c] - gt * Jj[c];
            s_gG[j][4 * r + 3] = gt + (gj ? (double)gj[3 * bj + r] : 0.0);
            s_rel[j][r] = p < 0 ? Jj[r] : Jj[r] - st.J[3 * ((size_t)b * J + p) + r];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c)
            gJ[c] = -((G[c] * gA[12 * j + 3] + G[4 + c] * gA[12 * j + 7]) + G[8 + c] * gA[12 * j + 11]);
        depth = lbs_depth(m, j);
        atomicMax(&s_maxd, depth);
    }
    __syncthreads();
    // children before parents: a level pulls its children's finished gG in ascending child order
    for (int d = s_maxd; d >= 0; --d) {
        if (j < J && depth == d) {
            for (int i = j + 1; i < J; ++i) {
                if (m.parents[i] != j) continue;
                const double *Ri = st.R + 9 * ((size_t)b * J + i);
#pragma unroll
                for (int r = 0; r < 3; ++r) {
#pragma unroll
                    for (int c = 0; c < 3; ++c)
                        s_gG[j][4 * r + c] = s_gG[j][4 * r + c] +
                                             (((s_gG[i][4 * r] * Ri[3 * c] + s_gG[i][4 * r + 1] * Ri[3 * c + 1]) +
                                               s_gG[i][4 * r + 2] * Ri[3 * c + 2]) +
                                              s_gG[i][4 * r + 3] * s_rel[i][c]);
                    s_gG[j][4 * r + 3] = s_gG[j][4 * r + 3] + s_gG[i][4 * r + 3];
                }
            }
        }
        __syncthreads();
    }
    if (j < J) {
        const int p = m.parents[j];
        double gR[9], grel[3];
        if (p < 0) {
#pragma unroll
            for (int r = 0; r < 3; ++r) {
#pragma unroll
                for (int c = 0; c < 3; ++c) gR[3 * r + c] = s_gG[j][4 * r + c];
                grel[r] = s_gG[j][4 * r + 3];
            }
        } else {
            const double *Gp = st.G + 12 * ((size_t)b * J + p);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    gR[3 * k + c] = (Gp[k] * s_gG[j][c] + Gp[4 + k] * s_gG[j][4 + c]) + Gp[8 + k] * s_gG[j][8 + c];
                grel[k] = (Gp[k] * s_gG[j][3] + Gp[4 + k] * s_gG[j][7]) + Gp[8 + k] * s_gG[j][11];
            }
#pragma unroll
            for (int e = 0; e < 9; ++e) gR[e] = gR[e] + gpf[9 * (j - 1) + e];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) s_grel[j][c] = grel[c];
        if (pose2rot) {
            double gr[3];
            lbs_rodrigues_backward(st.aa + 3 * bj, gR, gr);
#pragma unroll
            for (int c = 0; c < 3; ++c) g_pose[3 * bj + c] = (float)gr[c];
        } else {
#pragma unroll
            for (int e = 0; e < 9; ++e) g_pose[9 * bj + e] = (float)gR[e];
        }
    }
    __syncthreads();
    if (j < J) {
#pragma unroll
        for (int c = 0; c < 3; ++c) gJ[c] = gJ[c] + s_grel[j][c];
        for (int i = j + 1; i < J; ++i)
            if (m.parents[i] == j) {
#pragma unroll
                for (int c = 0; c < 3; ++c) gJ[c] = gJ[c] - s_grel[i][c];
            }
#pragma unroll
        for (int c = 0; c < 3; ++c) s_gJ[j][c] = gJ[c];
    }
    __syncthreads();
    for (int k = t; k < NB; k += LBS_CB_T) {
        double acc = 0.0;
        for (int jj = 0; jj < J; ++jj)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc = acc + m.J_dirs[((size_t)jj * 3 + c) * NB + k] * s_gJ[jj][c];
        g_betas[(size_t)b * NB + k] = (float)(gb[k] + acc);
    }
}

static bool lbs_model_ok(const icon_lbs_model *m) {
    return m && m->V > 0 && m->J >= 2 && m->J <= LBS_MAXJ && m->NB >= 1 && m->NB <= LBS_MAXNB && m->v_template &&
           m->shapedirs && m->posedirs && m->J_regressor && m->lbs_weights && m->J_template && m->J_dirs &&
           (int64_t)m->V * 3 <= INT32_MAX;
}

// ---------------------------------------------------------------- SMPL-X heads (PIXIE)

constexpr int HEADS_LUT = ICON_HEADS_LUT_ROWS;
constexpr int HEADS_MAXR = 64;
constexpr int HEADS_CV = 256;           // vertices per regressor chunk
constexpr int HEADS_T = 256;

static inline int heads_chunks(int V) { return (V + HEADS_CV - 1) / HEADS_CV; }

// the table row of one batch item: rel <- R[chain[i]] rel for i ascending, the reference's Euler angle and rounding
__device__ __forceinline__ int heads_lut_row(const icon_smplx_heads &h, const float *__restrict__ pose_b) {
    double rel[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
#pragma unroll
    for (int i = 0; i < ICON_HEADS_MAX_CHAIN; ++i) {     // static indices: the chain stays in the parameter space
        if (i >= h.nchain) break;
        const float *Rm = pose_b + 9 * h.chain[i];
        double n[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                n[3 * r + c] = ((double)Rm[3 * r] * rel[c] + (double)Rm[3 * r + 1] * rel[3 + c]) +
                               (double)Rm[3 * r + 2] * rel[6 + c];
#pragma unroll
        for (int e = 0; e < 9; ++e) rel[e] = n[e];
    }
    const double sy = sqrt(rel[0] * rel[0] + rel[3] * rel[3]);
    const double a = (-atan2(-rel[6], sy) * 180.0) / 3.141592653589793;
    const double y = rint(fmin(a, 39.0));          // round half to even, as torch.round
    if (y >= 0.0) return (int)y;
    return y < -39.0 ? 78 : 39 - (int)y;
}

// one CTA per (vertex chunk, batch item): a warp per output q = 3 r + c, each lane over its vertices in ascending
// order, then the fixed butterfly
__global__ void __launch_bounds__(HEADS_T) k_heads_reg_partial(icon_smplx_heads h, const float *__restrict__ verts,
                                                               double *__restrict__ part) {
    const int s = blockIdx.x, b = blockIdx.y, S = gridDim.x, Q = 3 * h.R;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int v0 = s * HEADS_CV, nv = min(HEADS_CV, h.V - v0);
    const float *vb = verts + (size_t)b * h.V * 3;
    for (int q = warp; q < Q; q += HEADS_T / 32) {
        const int r = q / 3, c = q % 3;
        const float *Rr = h.regressor + (size_t)r * h.V + v0;
        double acc = 0.0;
        for (int i = lane; i < nv; i += 32) acc = acc + (double)__ldg(Rr + i) * (double)vb[3 * (size_t)(v0 + i) + c];
        acc = warp_sum_fixed(acc);
        if (lane == 0) part[((size_t)b * S + s) * Q + q] = acc;
    }
}

// one CTA per batch item: the table row, the chunk partials in ascending order, the landmarks, the extra joints and
// the joint set
__global__ void __launch_bounds__(HEADS_T) k_heads_finish(icon_smplx_heads h, int S, const double *__restrict__ part,
                                                          const float *__restrict__ verts,
                                                          const float *__restrict__ jl, const float *__restrict__ pose,
                                                          float *__restrict__ landmarks, float *__restrict__ joints,
                                                          int *__restrict__ rows) {
    __shared__ double s_reg[3 * HEADS_MAXR];
    __shared__ int s_row;
    const int b = blockIdx.x, t = threadIdx.x, J = h.J, L = h.Ls + h.Ld, NJ = J + L + h.E, Q = 3 * h.R;
    if (t == 0) {
        s_row = heads_lut_row(h, pose + (size_t)b * J * 9);
        rows[b] = s_row;
    }
    for (int q = t; q < Q; q += HEADS_T) {
        double acc = 0.0;
        for (int s = 0; s < S; ++s) acc = acc + part[((size_t)b * S + s) * Q + q];
        s_reg[q] = acc;
    }
    __syncthreads();
    const float *vb = verts + (size_t)b * h.V * 3;
    for (int o = t; o < 3 * NJ; o += HEADS_T) {
        const int e = o / 3, c = o % 3;
        double val;
        if (e < J) {
            const int r = h.joint_reg[e];
            val = r >= 0 ? s_reg[3 * r + c] : (double)jl[((size_t)b * J + e) * 3 + c];
        } else {
            const int k = e - J;
            const int slot = 3 * (k < h.Ls ? k : k < L ? h.Ls + s_row * h.Ld + (k - h.Ls)
                                                       : h.Ls + HEADS_LUT * h.Ld + (k - L));
            val = ((double)h.bc[slot] * (double)vb[3 * h.vid[slot] + c] +
                   (double)h.bc[slot + 1] * (double)vb[3 * h.vid[slot + 1] + c]) +
                  (double)h.bc[slot + 2] * (double)vb[3 * h.vid[slot + 2] + c];
            if (k < L) landmarks[((size_t)b * L + k) * 3 + c] = (float)val;
        }
        joints[((size_t)b * NJ + e) * 3 + c] = (float)val;
    }
}

// a thread per (batch item, vertex column 3 v + c): the slots that read v in `inc` order, then the regressor rows
// in ascending order; the threads past 3V write the skinned joints' gradient
__global__ void __launch_bounds__(HEADS_T) k_heads_backward(icon_smplx_heads h, const int *__restrict__ rows,
                                                            const float *__restrict__ gl,
                                                            const float *__restrict__ gj, float *__restrict__ gv,
                                                            float *__restrict__ gjl) {
    const int b = blockIdx.y, J = h.J, L = h.Ls + h.Ld, NJ = J + L + h.E;
    const int64_t V3 = 3 * (int64_t)h.V, col = (int64_t)blockIdx.x * HEADS_T + threadIdx.x;
    if (col < V3) {
        const int v = (int)(col / 3), c = (int)(col % 3), row = rows[b];
        const int dyn0 = 3 * h.Ls, dyn1 = 3 * (h.Ls + HEADS_LUT * h.Ld);
        double acc = 0.0;
        for (int i = h.inc_off[v]; i < h.inc_off[v + 1]; ++i) {
            const int slot = h.inc[i];
            int k;
            if (slot < dyn0) {
                k = slot / 3;
            } else if (slot < dyn1) {
                const int d = slot / 3 - h.Ls;
                if (d / h.Ld != row) continue;
                k = h.Ls + d % h.Ld;
            } else {
                k = L + (slot - dyn1) / 3;
            }
            double u = 0.0;
            if (gl && k < L) u = (double)gl[((size_t)b * L + k) * 3 + c];
            if (gj) u = u + (double)gj[((size_t)b * NJ + J + k) * 3 + c];
            acc = acc + (double)h.bc[slot] * u;
        }
        if (gj)
            for (int r = 0; r < h.R; ++r) {
                const int j = h.reg_joint[r];
                if (j >= 0)
                    acc = acc + (double)__ldg(h.regressor + (size_t)r * h.V + v) *
                                    (double)gj[((size_t)b * NJ + j) * 3 + c];
            }
        gv[(size_t)b * V3 + col] = (float)acc;
    } else if (gjl && col < V3 + 3 * J) {
        const int o = (int)(col - V3), j = o / 3;
        gjl[(size_t)b * 3 * J + o] = h.joint_reg[j] >= 0 ? 0.0f : gj[((size_t)b * NJ + j) * 3 + o % 3];
    }
}

static bool heads_ok(const icon_smplx_heads *h) {
    return h && h->V > 0 && (int64_t)h->V * 3 <= INT32_MAX && h->J >= 2 && h->J <= LBS_MAXJ && h->R >= 1 &&
           h->R <= HEADS_MAXR && h->Ls >= 0 && h->Ld >= 0 && h->E >= 0 && h->nchain >= 1 &&
           h->nchain <= ICON_HEADS_MAX_CHAIN && h->regressor && h->vid && h->bc && h->joint_reg && h->reg_joint &&
           h->inc_off && h->inc;
}

// ---------------------------------------------------------------- tetra body (PaMIR's TetraSMPLModel)

constexpr int TETRA_J = ICON_TETRA_JOINTS;
constexpr int TETRA_P = 9 * (TETRA_J - 1);
constexpr int TETRA_NB = ICON_TETRA_BETAS;
constexpr int TETRA_CT = 128;           // chain threads (>= 3 TETRA_J)
constexpr int TETRA_ST = 192;           // skin threads: 64 output rows x 3 components
constexpr int TETRA_STATE = 12 * TETRA_J + TETRA_P;    // A [24,12], then lrotmin [207]

// pymaf's rotation_matrix_to_angle_axis for one [3,3] matrix, op by op in fp32 (every torch op one rounding)
__device__ __forceinline__ void tetra_rotmat_to_aa(const float *__restrict__ R, float aa[3]) {
    float t[3][3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) t[a][b] = R[3 * b + a];          // rmat_t = R^T
    const bool d2 = t[2][2] < 1e-6f, d0d1 = t[0][0] > t[1][1], d0nd1 = t[0][0] < -t[1][1];
    const float t0 = ((1.0f + t[0][0]) - t[1][1]) - t[2][2];
    const float t1 = ((1.0f - t[0][0]) + t[1][1]) - t[2][2];
    const float t2 = ((1.0f - t[0][0]) - t[1][1]) + t[2][2];
    const float t3 = ((1.0f + t[0][0]) + t[1][1]) + t[2][2];
    const float q0[4] = {t[1][2] - t[2][1], t0, t[0][1] + t[1][0], t[2][0] + t[0][2]};
    const float q1[4] = {t[2][0] - t[0][2], t[0][1] + t[1][0], t1, t[1][2] + t[2][1]};
    const float q2[4] = {t[0][1] - t[1][0], t[2][0] + t[0][2], t[1][2] + t[2][1], t2};
    const float q3[4] = {t3, t[1][2] - t[2][1], t[2][0] - t[0][2], t[0][1] - t[1][0]};
    const float m0 = (d2 && d0d1) ? 1.0f : 0.0f, m1 = (d2 && !d0d1) ? 1.0f : 0.0f;
    const float m2 = (!d2 && d0nd1) ? 1.0f : 0.0f, m3 = (!d2 && !d0nd1) ? 1.0f : 0.0f;
    const float den = sqrtf(((t0 * m0 + t1 * m1) + t2 * m2) + t3 * m3);
    float q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) q[i] = ((((q0[i] * m0 + q1[i] * m1) + q2[i] * m2) + q3[i] * m3) / den) * 0.5f;
    const float s2 = (q[1] * q[1] + q[2] * q[2]) + q[3] * q[3];
    const float st = sqrtf(s2), ct = q[0];
    const float two = 2.0f * (ct < 0.0f ? atan2f(-st, -ct) : atan2f(st, ct));
    const float k = s2 > 0.0f ? two / st : 2.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float v = 0.0f + q[1 + c] * k;
        aa[c] = isnan(v) ? 0.0f : v;
    }
}

// TetraSMPLModel.rodrigues: theta = max(fp32 |r|, DBL_MIN) widened, R = (cos I + (1 - cos) rh rh^T) + sin [rh]x
__device__ __forceinline__ void tetra_rodrigues(const float r[3], double R[9]) {
    const float th32 = sqrtf((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]);
    const double th = fmax((double)th32, DBL_MIN);
    const double rh[3] = {(double)r[0] / th, (double)r[1] / th, (double)r[2] / th};
    const double cs = cos(th), sn = sin(th), c1 = 1.0 - cs;
    const double K[9] = {0.0, -rh[2], rh[1], rh[2], 0.0, -rh[0], -rh[1], rh[0], 0.0};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) R[3 * i + j] = (cs * (i == j ? 1.0 : 0.0) + c1 * (rh[i] * rh[j])) + sn * K[3 * i + j];
}

// v_shaped of column col = 3 v + c: shapedirs . beta (k ascending) + v_template
__device__ __forceinline__ double tetra_vshaped(const icon_tetra_model &m, const double *beta, int col) {
    const int N3 = 3 * m.N;
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < TETRA_NB; ++k) acc = acc + m.shapedirs[(size_t)k * N3 + col] * beta[k];
    return acc + m.v_template[col];
}

// one CTA: rotations (from matrices, or the axis-angle as given), rest joints, the chain, A and lrotmin
__global__ void __launch_bounds__(TETRA_CT) k_tetra_chain(icon_tetra_model m, const float *__restrict__ rotmats,
                                                          float *__restrict__ aa, const float *__restrict__ betas,
                                                          double *__restrict__ st) {
    __shared__ double sJ[TETRA_J][3], sR[TETRA_J][9], sG[TETRA_J][12], s_beta[TETRA_NB];
    const int t = threadIdx.x;
    if (t < TETRA_NB) s_beta[t] = (double)betas[t];
    int depth = 0;
    if (t < TETRA_J) {
        float r[3];
        if (rotmats) {
            tetra_rotmat_to_aa(rotmats + 9 * t, r);
#pragma unroll
            for (int c = 0; c < 3; ++c) aa[3 * t + c] = r[c];
        } else {
#pragma unroll
            for (int c = 0; c < 3; ++c) r[c] = aa[3 * t + c];
        }
        tetra_rodrigues(r, sR[t]);
        for (int i = m.parents[t]; i >= 0; i = m.parents[i]) ++depth;
    }
    __syncthreads();
    if (t < 3 * TETRA_J) {
        const int j = t / 3, c = t % 3;
        double acc = 0.0;
        for (int e = m.jr_off[j]; e < m.jr_off[j + 1]; ++e)
            acc = acc + m.jr_val[e] * tetra_vshaped(m, s_beta, 3 * m.jr_col[e] + c);
        sJ[j][c] = acc;
    }
    __syncthreads();
    for (int d = 0; __syncthreads_or(t < TETRA_J && depth >= d); ++d) {
        if (t < TETRA_J && depth == d) {
            const int p = m.parents[t];
            double G[12];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                if (p < 0) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) G[4 * r + c] = sR[t][3 * r + c];
                    G[4 * r + 3] = sJ[t][r];
                } else {
                    const double rel[3] = {sJ[t][0] - sJ[p][0], sJ[t][1] - sJ[p][1], sJ[t][2] - sJ[p][2]};
#pragma unroll
                    for (int c = 0; c < 3; ++c)
                        G[4 * r + c] = (sG[p][4 * r] * sR[t][c] + sG[p][4 * r + 1] * sR[t][3 + c]) +
                                       sG[p][4 * r + 2] * sR[t][6 + c];
                    G[4 * r + 3] = ((sG[p][4 * r] * rel[0] + sG[p][4 * r + 1] * rel[1]) + sG[p][4 * r + 2] * rel[2]) +
                                   sG[p][4 * r + 3];
                }
            }
#pragma unroll
            for (int e = 0; e < 12; ++e) sG[t][e] = G[e];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const double gj = (G[4 * r] * sJ[t][0] + G[4 * r + 1] * sJ[t][1]) + G[4 * r + 2] * sJ[t][2];
#pragma unroll
                for (int c = 0; c < 3; ++c) st[12 * t + 4 * r + c] = G[4 * r + c];
                st[12 * t + 4 * r + 3] = G[4 * r + 3] - gj;
            }
        }
    }
    for (int p = t; p < TETRA_P; p += TETRA_CT) {
        const int e = p % 9;
        st[12 * TETRA_J + p] = sR[1 + p / 9][e] - ((e == 0 || e == 4 || e == 8) ? 1.0 : 0.0);
    }
}

// 64 output rows per CTA, one thread per (row, component): v_posed, the skinning and the epilogue; rows >= N are the
// padding (0 x 0.5, z negated: -0.0f, as the reference's float32 array holds)
__global__ void __launch_bounds__(TETRA_ST) k_tetra_skin(icon_tetra_model m, const float *__restrict__ betas,
                                                         const float *__restrict__ trans,
                                                         const float *__restrict__ scale,
                                                         const double *__restrict__ st, float *__restrict__ out) {
    __shared__ double s_pf[TETRA_P], s_A[12 * TETRA_J], s_beta[TETRA_NB], s_vp[TETRA_ST];
    const int t = threadIdx.x, col = blockIdx.x * TETRA_ST + t, row = col / 3, c = col % 3, N3 = 3 * m.N;
    for (int p = t; p < TETRA_P; p += TETRA_ST) s_pf[p] = st[12 * TETRA_J + p];
    for (int i = t; i < 12 * TETRA_J; i += TETRA_ST) s_A[i] = st[i];
    if (t < TETRA_NB) s_beta[t] = (double)betas[t];
    __syncthreads();
    const bool live = col < N3;
    double vp = 0.0;
    if (live) {
        double po = 0.0;
        const double *pd = m.posedirs + col;
#pragma unroll 9
        for (int p = 0; p < TETRA_P; ++p) po = po + s_pf[p] * __ldg(pd + (size_t)p * N3);
        vp = tetra_vshaped(m, s_beta, col) + po;
    }
    s_vp[t] = vp;
    __syncthreads();
    if (col >= 3 * ICON_TETRA_PAD_V) return;
    float o = 0.0f;
    if (live) {
        double T[4] = {0.0, 0.0, 0.0, 0.0};
        const double *w = m.weights + (size_t)row * TETRA_J;
        for (int j = 0; j < TETRA_J; ++j) {
            const double wj = w[j];
#pragma unroll
            for (int q = 0; q < 4; ++q) T[q] = T[q] + wj * s_A[12 * j + 4 * c + q];
        }
        const int l = 3 * (t / 3);
        const double v = (((T[0] * s_vp[l] + T[1] * s_vp[l + 1]) + T[2] * s_vp[l + 2]) + T[3]) + 0.0;
        o = (float)(v * (double)scale[0] + (double)trans[c]);
    }
    o = o * 0.5f;
    if (c == 2) o = o * -1.0f;
    out[col] = o;
}

static bool tetra_model_ok(const icon_tetra_model *m) {
    return m && m->V >= 1 && m->N >= m->V && m->N <= ICON_TETRA_PAD_V && m->T >= 0 && m->T <= ICON_TETRA_PAD_F &&
           m->v_template && m->shapedirs && m->posedirs && m->weights && m->jr_off && m->jr_col && m->jr_val;
}

}  // namespace icon

// ---------------------------------------------------------------- C ABI

extern "C" size_t icon_lbs_prepare_workspace_bytes(int V, int J, int NB) {
    if (V <= 0 || J <= 0 || NB <= 0) return 0;
    const size_t S = (size_t)(V + icon::LBS_PREP_V - 1) / icon::LBS_PREP_V;
    return icon::align_up((size_t)J * S * 3 * ((size_t)NB + 1) * sizeof(double), 256);
}

extern "C" int icon_lbs_prepare(icon_lbs_model *m, const int64_t *h_parents, int posedirs_rows, void *ws,
                                size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(m && h_parents && ws, "icon_lbs_prepare: null pointer");
    ICON_CHECK_ARG(m->J >= 2 && m->J <= LBS_MAXJ, "icon_lbs_prepare: J=%d joints, the kernels take 2..%d", m->J,
                   LBS_MAXJ);
    ICON_CHECK_ARG(m->NB >= 1 && m->NB <= LBS_MAXNB, "icon_lbs_prepare: NB=%d shape coefficients, the kernels take "
                   "1..%d", m->NB, LBS_MAXNB);
    ICON_CHECK_ARG(posedirs_rows == 9 * (m->J - 1), "icon_lbs_prepare: posedirs has %d rows, 9 (J - 1) = %d",
                   posedirs_rows, 9 * (m->J - 1));
    ICON_CHECK_ARG(h_parents[0] == -1, "icon_lbs_prepare: parents[0] = %lld, the root's must be -1",
                   (long long)h_parents[0]);
    for (int i = 1; i < m->J; ++i)
        ICON_CHECK_ARG(h_parents[i] >= 0 && h_parents[i] < i,
                       "icon_lbs_prepare: parents[%d] = %lld, a joint's parent must come before it", i,
                       (long long)h_parents[i]);
    for (int i = 0; i < m->J; ++i) m->parents[i] = (int)h_parents[i];
    for (int i = m->J; i < LBS_MAXJ; ++i) m->parents[i] = -1;
    ICON_CHECK_ARG(lbs_model_ok(m), "icon_lbs_prepare: null buffer or bad sizes V=%d J=%d NB=%d", m->V, m->J, m->NB);
    ICON_CHECK_ARG(ws_bytes >= icon_lbs_prepare_workspace_bytes(m->V, m->J, m->NB),
                   "icon_lbs_prepare: workspace too small");
    const int S = (m->V + LBS_PREP_V - 1) / LBS_PREP_V;
    k_lbs_prepare_partial<<<dim3((unsigned)m->J, (unsigned)S), LBS_PREP_T, 0, stream>>>(*m, (double *)ws);
    ICON_LAUNCHED();
    k_lbs_prepare_reduce<<<(unsigned)m->J, LBS_PREP_T, 0, stream>>>(*m, (const double *)ws, S);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" size_t icon_lbs_state_bytes(int B, int V, int J, int NB) {
    if (B <= 0 || V <= 0 || J <= 0 || NB <= 0) return 0;
    return icon::lbs_state_carve(nullptr, B, V, J, nullptr);
}

extern "C" size_t icon_lbs_workspace_bytes(int B, int V, int J, int NB, int backward) {
    if (B <= 0 || V <= 0 || J <= 0 || NB <= 0 || !backward) return 0;
    return icon::align_up((size_t)B * icon::lbs_tiles(V) * icon::lbs_outputs(J, NB) * sizeof(double), 256);
}

extern "C" int icon_lbs_forward(const icon_lbs_model *m, int B, const float *betas, const float *pose, int pose2rot,
                                float *verts, float *joints, void *state, size_t state_bytes, void *ws,
                                size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(lbs_model_ok(m), "icon_lbs_forward: model not prepared");
    ICON_CHECK_ARG(B > 0, "icon_lbs_forward: B=%d", B);
    ICON_CHECK_ARG(betas && pose && verts && joints && state, "icon_lbs_forward: null pointer");
    ICON_CHECK_ARG(state_bytes >= icon_lbs_state_bytes(B, m->V, m->J, m->NB), "icon_lbs_forward: state too small");
    ICON_CHECK_ARG(ws_bytes >= icon_lbs_workspace_bytes(B, m->V, m->J, m->NB, 0), "icon_lbs_forward: workspace too small");
    (void)ws;
    LbsState st;
    lbs_state_carve(state, B, m->V, m->J, &st);
    k_lbs_chain<<<(unsigned)B, LBS_MAXJ, 0, stream>>>(*m, betas, pose, pose2rot ? 1 : 0, joints, st);
    ICON_LAUNCHED();
    k_lbs_skin<<<(unsigned)lbs_tiles(m->V), LBS_T, 0, stream>>>(*m, B, betas, st, verts);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_lbs_backward(const icon_lbs_model *m, int B, const void *state, size_t state_bytes,
                                 const float *grad_verts, const float *grad_joints, float *grad_betas,
                                 float *grad_pose, void *ws, size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(lbs_model_ok(m), "icon_lbs_backward: model not prepared");
    ICON_CHECK_ARG(B > 0, "icon_lbs_backward: B=%d", B);
    ICON_CHECK_ARG(state && grad_betas && grad_pose && ws, "icon_lbs_backward: null pointer");
    ICON_CHECK_ARG(state_bytes >= icon_lbs_state_bytes(B, m->V, m->J, m->NB), "icon_lbs_backward: state too small");
    ICON_CHECK_ARG(ws_bytes >= icon_lbs_workspace_bytes(B, m->V, m->J, m->NB, 1),
                   "icon_lbs_backward: workspace too small");
    LbsState st;
    lbs_state_carve((void *)state, B, m->V, m->J, &st);
    const int tiles = lbs_tiles(m->V);
    if (grad_verts) {
        k_lbs_skin_backward<<<(unsigned)tiles, LBS_T, 0, stream>>>(*m, B, st, grad_verts, (double *)ws);
        ICON_LAUNCHED();
    }
    k_lbs_chain_backward<<<(unsigned)B, LBS_CB_T, 0, stream>>>(*m, st, grad_verts ? (const double *)ws : nullptr,
                                                               tiles, grad_joints, grad_betas, grad_pose);
    ICON_LAUNCHED();
    return ICON_OK;
}

// ---------------------------------------------------------------- C ABI: SMPL-X heads

extern "C" int icon_smplx_heads_prepare(icon_smplx_heads *h, const int64_t *h_faces, int F,
                                        const int64_t *h_lmk_faces_idx, const float *h_lmk_bary, int Ls,
                                        const int64_t *h_dyn_faces_idx, const float *h_dyn_bary, int Ld,
                                        const int64_t *h_face_ids, const float *h_bcs, int E,
                                        const int64_t *h_source, const int64_t *h_target, int S,
                                        const int64_t *h_chain, int nchain, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(h && h_faces && h_chain, "icon_smplx_heads_prepare: null pointer");
    ICON_CHECK_ARG(F >= 1 && Ls >= 0 && Ld >= 0 && E >= 0 && S >= 0,
                   "icon_smplx_heads_prepare: bad sizes F=%d Ls=%d Ld=%d E=%d S=%d", F, Ls, Ld, E, S);
    ICON_CHECK_ARG((Ls == 0 || (h_lmk_faces_idx && h_lmk_bary)) && (Ld == 0 || (h_dyn_faces_idx && h_dyn_bary)) &&
                   (E == 0 || (h_face_ids && h_bcs)) && (S == 0 || (h_source && h_target)),
                   "icon_smplx_heads_prepare: null table");
    ICON_CHECK_ARG(nchain >= 1 && nchain <= ICON_HEADS_MAX_CHAIN,
                   "icon_smplx_heads_prepare: head chain of %d joints, the kernels take 1..%d", nchain,
                   ICON_HEADS_MAX_CHAIN);
    h->Ls = Ls;
    h->Ld = Ld;
    h->E = E;
    h->nchain = nchain;
    ICON_CHECK_ARG(heads_ok(h), "icon_smplx_heads_prepare: null buffer or bad sizes V=%d J=%d R=%d", h->V, h->J,
                   h->R);
    const int V = h->V, J = h->J, R = h->R;
    for (int i = 0; i < nchain; ++i) {
        ICON_CHECK_ARG(h_chain[i] >= 0 && h_chain[i] < J,
                       "icon_smplx_heads_prepare: head_kin_chain[%d] = %lld outside [0,%d)", i,
                       (long long)h_chain[i], J);
        h->chain[i] = (int)h_chain[i];
    }
    for (int i = nchain; i < ICON_HEADS_MAX_CHAIN; ++i) h->chain[i] = 0;
    // slots in table order: static [Ls,3], the lookup table [79,Ld,3], extra [E,3]
    const int nf = Ls + HEADS_LUT * Ld + E, N = 3 * nf;
    std::vector<int> vid(N), joint_reg(J, -1), reg_joint(R, -1), off(V + 1, 0), inc(N);
    std::vector<float> bc(N);
    struct Tab { const char *name; const int64_t *f; const float *w; int n; int base; };
    const Tab tabs[3] = {{"lmk_faces_idx", h_lmk_faces_idx, h_lmk_bary, Ls, 0},
                         {"dynamic_lmk_faces_idx", h_dyn_faces_idx, h_dyn_bary, HEADS_LUT * Ld, Ls},
                         {"face_ids", h_face_ids, h_bcs, E, Ls + HEADS_LUT * Ld}};
    for (const Tab &t : tabs)
        for (int i = 0; i < t.n; ++i) {
            const int64_t f = t.f[i];
            ICON_CHECK_ARG(f >= 0 && f < F, "icon_smplx_heads_prepare: %s[%d] = %lld, a face id outside [0,%d)",
                           t.name, i, (long long)f, F);
            for (int k = 0; k < 3; ++k) {
                const int64_t v = h_faces[3 * f + k];
                ICON_CHECK_ARG(v >= 0 && v < V,
                               "icon_smplx_heads_prepare: faces[%lld][%d] = %lld (used by %s[%d]), a vertex id "
                               "outside [0,%d)", (long long)f, k, (long long)v, t.name, i, V);
                vid[3 * (t.base + i) + k] = (int)v;
                bc[3 * (t.base + i) + k] = t.w[3 * i + k];
            }
        }
    for (int s = 0; s < S; ++s) {
        ICON_CHECK_ARG(h_source[s] >= 0 && h_source[s] < J,
                       "icon_smplx_heads_prepare: source_idxs[%d] = %lld outside [0,%d)", s, (long long)h_source[s],
                       J);
        ICON_CHECK_ARG(h_target[s] >= 0 && h_target[s] < R,
                       "icon_smplx_heads_prepare: target_idxs[%d] = %lld outside [0,%d)", s, (long long)h_target[s],
                       R);
        ICON_CHECK_ARG(joint_reg[h_source[s]] < 0 && reg_joint[h_target[s]] < 0,
                       "icon_smplx_heads_prepare: source_idxs / target_idxs[%d] repeats an index", s);
        joint_reg[h_source[s]] = (int)h_target[s];
        reg_joint[h_target[s]] = (int)h_source[s];
    }
    // per-vertex slot lists, stable in (entry, table row, corner) order: a counting sort of that enumeration
    std::vector<int> order;
    order.reserve(N);
    for (int i = 0; i < 3 * Ls; ++i) order.push_back(i);
    for (int l = 0; l < Ld; ++l)
        for (int row = 0; row < HEADS_LUT; ++row)
            for (int k = 0; k < 3; ++k) order.push_back(3 * (Ls + row * Ld + l) + k);
    for (int i = 3 * (Ls + HEADS_LUT * Ld); i < N; ++i) order.push_back(i);
    for (int slot : order) ++off[vid[slot] + 1];
    for (int v = 0; v < V; ++v) off[v + 1] += off[v];
    std::vector<int> fill(off.begin(), off.end() - 1);
    for (int slot : order) inc[fill[vid[slot]]++] = slot;
    if (N > 0) {
        ICON_CUDA(cudaMemcpyAsync(h->vid, vid.data(), N * sizeof(int), cudaMemcpyHostToDevice, stream));
        ICON_CUDA(cudaMemcpyAsync(h->bc, bc.data(), N * sizeof(float), cudaMemcpyHostToDevice, stream));
        ICON_CUDA(cudaMemcpyAsync(h->inc, inc.data(), N * sizeof(int), cudaMemcpyHostToDevice, stream));
    }
    ICON_CUDA(cudaMemcpyAsync(h->joint_reg, joint_reg.data(), J * sizeof(int), cudaMemcpyHostToDevice, stream));
    ICON_CUDA(cudaMemcpyAsync(h->reg_joint, reg_joint.data(), R * sizeof(int), cudaMemcpyHostToDevice, stream));
    ICON_CUDA(cudaMemcpyAsync(h->inc_off, off.data(), (V + 1) * sizeof(int), cudaMemcpyHostToDevice, stream));
    ICON_CUDA(cudaStreamSynchronize(stream));          // the host vectors go out of scope
    return ICON_OK;
}

extern "C" size_t icon_smplx_heads_state_bytes(int B, int V, int R) {
    if (B <= 0 || V <= 0 || R <= 0) return 0;
    return icon::align_up((size_t)B * icon::heads_chunks(V) * 3 * R * sizeof(double), 256);
}

extern "C" int icon_smplx_heads_forward(const icon_smplx_heads *h, int B, const float *verts,
                                        const float *joints_lbs, const float *pose, float *landmarks, float *joints,
                                        int *rows, void *state, size_t state_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(heads_ok(h), "icon_smplx_heads_forward: heads not prepared");
    ICON_CHECK_ARG(B > 0 && B <= 65535, "icon_smplx_heads_forward: B=%d", B);
    ICON_CHECK_ARG(verts && joints_lbs && pose && joints && rows && state && (landmarks || h->Ls + h->Ld == 0),
                   "icon_smplx_heads_forward: null pointer");
    ICON_CHECK_ARG(state_bytes >= icon_smplx_heads_state_bytes(B, h->V, h->R),
                   "icon_smplx_heads_forward: state too small");
    const int S = heads_chunks(h->V);
    k_heads_reg_partial<<<dim3((unsigned)S, (unsigned)B), HEADS_T, 0, stream>>>(*h, verts, (double *)state);
    ICON_LAUNCHED();
    k_heads_finish<<<(unsigned)B, HEADS_T, 0, stream>>>(*h, S, (const double *)state, verts, joints_lbs, pose,
                                                        landmarks, joints, rows);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_smplx_heads_backward(const icon_smplx_heads *h, int B, const int *rows,
                                         const float *grad_landmarks, const float *grad_joints, float *grad_verts,
                                         float *grad_joints_lbs, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(heads_ok(h), "icon_smplx_heads_backward: heads not prepared");
    ICON_CHECK_ARG(B > 0 && B <= 65535, "icon_smplx_heads_backward: B=%d", B);
    ICON_CHECK_ARG(rows && grad_verts && (grad_joints || !grad_joints_lbs),
                   "icon_smplx_heads_backward: null pointer");
    const int64_t cols = 3 * ((int64_t)h->V + h->J);
    k_heads_backward<<<dim3((unsigned)((cols + HEADS_T - 1) / HEADS_T), (unsigned)B), HEADS_T, 0, stream>>>(
        *h, rows, grad_landmarks, grad_joints, grad_verts, grad_joints ? grad_joints_lbs : nullptr);
    ICON_LAUNCHED();
    return ICON_OK;
}

// ---------------------------------------------------------------- C ABI: tetra body

extern "C" int icon_tetra_prepare(icon_tetra_model *m, const int64_t *h_parents, int J, int posedirs_cols,
                                  int nbetas) {
    using namespace icon;
    ICON_CHECK_ARG(m && h_parents, "icon_tetra_prepare: null pointer");
    ICON_CHECK_ARG(J == TETRA_J, "icon_tetra_prepare: kintree_table has %d joints, the kernels take %d", J, TETRA_J);
    ICON_CHECK_ARG(posedirs_cols == TETRA_P, "icon_tetra_prepare: posedirs has %d columns, 9 (J - 1) = %d",
                   posedirs_cols, TETRA_P);
    ICON_CHECK_ARG(nbetas == TETRA_NB, "icon_tetra_prepare: shapedirs has %d columns, the kernels take %d", nbetas,
                   TETRA_NB);
    ICON_CHECK_ARG(h_parents[0] == -1, "icon_tetra_prepare: parents[0] = %lld, the root's must be -1",
                   (long long)h_parents[0]);
    for (int i = 1; i < J; ++i)
        ICON_CHECK_ARG(h_parents[i] >= 0 && h_parents[i] < i,
                       "icon_tetra_prepare: parents[%d] = %lld, a joint's parent must come before it", i,
                       (long long)h_parents[i]);
    ICON_CHECK_ARG(m->N >= m->V && m->N <= ICON_TETRA_PAD_V,
                   "icon_tetra_prepare: V + V_added = %d vertices, the padded voxel_verts hold %d", m->N,
                   ICON_TETRA_PAD_V);
    ICON_CHECK_ARG(m->T >= 0 && m->T <= ICON_TETRA_PAD_F,
                   "icon_tetra_prepare: %d tetrahedra, the padded voxel_faces hold %d", m->T, ICON_TETRA_PAD_F);
    ICON_CHECK_ARG(tetra_model_ok(m), "icon_tetra_prepare: null buffer or bad sizes V=%d N=%d", m->V, m->N);
    for (int i = 0; i < J; ++i) m->parents[i] = (int)h_parents[i];
    return ICON_OK;
}

extern "C" size_t icon_tetra_state_bytes(void) { return icon::align_up(icon::TETRA_STATE * sizeof(double), 256); }

extern "C" int icon_tetra_forward(const icon_tetra_model *m, const float *rotmats, float *aa, const float *betas,
                                  const float *trans, const float *scale, float *voxel_verts, void *state,
                                  size_t state_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(tetra_model_ok(m), "icon_tetra_forward: model not prepared");
    ICON_CHECK_ARG(aa && betas && trans && scale && voxel_verts && state, "icon_tetra_forward: null pointer");
    ICON_CHECK_ARG(state_bytes >= icon_tetra_state_bytes(), "icon_tetra_forward: state too small");
    k_tetra_chain<<<1, TETRA_CT, 0, stream>>>(*m, rotmats, aa, betas, (double *)state);
    ICON_LAUNCHED();
    k_tetra_skin<<<(3 * ICON_TETRA_PAD_V + TETRA_ST - 1) / TETRA_ST, TETRA_ST, 0, stream>>>(
        *m, betas, trans, scale, (const double *)state, voxel_verts);
    ICON_LAUNCHED();
    return ICON_OK;
}
