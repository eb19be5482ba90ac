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
#include <math.h>

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
