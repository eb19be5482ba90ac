// PyMAF's body estimate (lib/pymaf/models/pymaf_net.py, maf_extractor.py, smpl.py, utils/geometry.py): everything
// after the ResNet-50 backbone and the deconvolutions, which run on the NHWC convolution path (icon_b200/hps.py).
//
//   k_maxpool3s2     nn.MaxPool2d(3, 2, 1) of relu(x) (max and relu commute exactly) -> the plain hi / lo operand of
//                    layer1; out-of-image taps are skipped, which is MaxPool2d's -inf padding
//   k_maf_mlp        per sample point: grid_sample(s_feat, align_corners=True) of 256 channels, then the three Conv1d
//                    layers of MAF_Extractor.reduce_dim with their concatenations; writes the regressor's input row
//                    xc = [features channel-major, pose, shape, cam]
//   k_hps_gemv       y = W x + b [+ add], one warp per row (fc1, fc2, and decpose / decshape / deccam as one [157, 1024]
//                    matrix whose `add` is the previous estimate)
//   k_hps_rot6d      rot6d_to_rotmat of the 24 joints; the skinning that follows is icon_lbs_forward (pose2rot = 0)
//   k_hps_regress    J_regressor_extra rows (dense) and Dmap rows (CSR) times the skinned vertices; a Dmap row also
//                    writes its projection, the next iteration's sample point
//   k_hps_tail       joints [24 lbs, 21 vertex joints, 9 extra][joint_map] -> kp_3d, kp_2d = projection, and theta =
//                    [cam, shape, kornia's rotation_matrix_to_angle_axis(rotmat)]
//
// Every dot product accumulates in float64 and rounds once, so a GEMV row's error is its final rounding; the geometry
// runs in float64 too and rounds its outputs to float32.
#include <cuda_fp16.h>

#include "common.cuh"

namespace icon {

constexpr int MAF_C = 256, MAF_H1 = 128, MAF_H2 = 64, MAF_OUT = 5;

__global__ void k_maxpool3s2(const float *__restrict__ x, __half *__restrict__ hi, __half *__restrict__ lo, int N, int H,
                             int W, int C, int Cp, int OH, int OW, int relu) {
    const int64_t total = (int64_t)N * OH * OW * Cp;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % Cp);
    int64_t r = i / Cp;
    const int ox = (int)(r % OW); r /= OW;
    const int oy = (int)(r % OH);
    const int n = (int)(r / OH);
    float m = 0.f;
    if (c < C) {
        m = -INFINITY;
        for (int dy = 0; dy < 3; ++dy) {
            const int y = oy * 2 - 1 + dy;
            if (y < 0 || y >= H) continue;
            for (int dx = 0; dx < 3; ++dx) {
                const int xx = ox * 2 - 1 + dx;
                if (xx < 0 || xx >= W) continue;
                m = fmaxf(m, __ldg(x + (((int64_t)n * H + y) * W + xx) * C + c));
            }
        }
        if (relu) m = fmaxf(m, 0.f);
    }
    const __half h = __float2half_rn(m);
    hi[i] = h;
    lo[i] = __float2half_rn(m - __half2float(h));
}

// grid_sample(bilinear, zeros, align_corners=True) of one channel at source position (ix, iy), in float64
__device__ __forceinline__ double bilinear(const float *__restrict__ f, int H, int W, int C, int c, double ix, double iy) {
    const double x0 = floor(ix), y0 = floor(iy);
    const double tx = ix - x0, ty = iy - y0;
    const int xi = (int)x0, yi = (int)y0;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int xx = xi + (k & 1), yy = yi + (k >> 1);
        if (xx < 0 || xx >= W || yy < 0 || yy >= H) continue;
        const double w = ((k & 1) ? tx : 1.0 - tx) * ((k >> 1) ? ty : 1.0 - ty);
        s += w * (double)__ldg(f + ((int64_t)yy * W + xx) * C + c);
    }
    return s;
}

// one block of MAF_H1 threads per point; pts [2][N] (x row, y row) in [-1, 1] grid coordinates
__global__ void __launch_bounds__(MAF_H1) k_maf_mlp(const float *__restrict__ feat, int H, int W,
                                                    const float *__restrict__ pts, int N,
                                                    const float *__restrict__ w1, const float *__restrict__ b1,
                                                    const float *__restrict__ w2, const float *__restrict__ b2,
                                                    const float *__restrict__ w3, const float *__restrict__ b3,
                                                    const float *__restrict__ prev, int nprev, float *__restrict__ xc) {
    __shared__ float s[MAF_C], y1[MAF_H1], y2[MAF_H2];
    const int n = blockIdx.x, t = threadIdx.x;
    if (n == 0)
        for (int k = t; k < nprev; k += blockDim.x) xc[MAF_OUT * N + k] = prev[k];
    const double ix = ((double)pts[n] + 1.0) * 0.5 * (W - 1), iy = ((double)pts[N + n] + 1.0) * 0.5 * (H - 1);
    for (int c = t; c < MAF_C; c += blockDim.x) s[c] = (float)bilinear(feat, H, W, MAF_C, c, ix, iy);
    __syncthreads();
    {   // conv0: 256 -> 128, leaky 0.01
        const float *w = w1 + (size_t)t * MAF_C;
        double a = 0.0;
        for (int k = 0; k < MAF_C; ++k) a += (double)__ldg(w + k) * s[k];
        const float v = (float)(a + (double)b1[t]);
        y1[t] = v > 0.f ? v : 0.01f * v;
    }
    __syncthreads();
    if (t < MAF_H2) {   // conv1: [y1, s] 384 -> 64, leaky 0.01
        const float *w = w2 + (size_t)t * (MAF_H1 + MAF_C);
        double a = 0.0;
        for (int k = 0; k < MAF_H1; ++k) a += (double)__ldg(w + k) * y1[k];
        for (int k = 0; k < MAF_C; ++k) a += (double)__ldg(w + MAF_H1 + k) * s[k];
        const float v = (float)(a + (double)b2[t]);
        y2[t] = v > 0.f ? v : 0.01f * v;
    }
    __syncthreads();
    if (t < MAF_OUT) {  // conv2: [y2, s] 320 -> 5, relu; flattened channel-major
        const float *w = w3 + (size_t)t * (MAF_H2 + MAF_C);
        double a = 0.0;
        for (int k = 0; k < MAF_H2; ++k) a += (double)__ldg(w + k) * y2[k];
        for (int k = 0; k < MAF_C; ++k) a += (double)__ldg(w + MAF_H2 + k) * s[k];
        const float v = (float)(a + (double)b3[t]);
        xc[(size_t)t * N + n] = fmaxf(v, 0.f);
    }
}

constexpr int GEMV_WARPS = 8;

// y[r] = W[r] . x + b[r] (+ add[r]); x staged in shared memory (K floats)
__global__ void __launch_bounds__(GEMV_WARPS * 32) k_hps_gemv(const float *__restrict__ Wt, const float *__restrict__ x,
                                                              const float *__restrict__ b, const float *__restrict__ add,
                                                              float *__restrict__ y, int R, int K) {
    extern __shared__ float xs[];
    for (int k = threadIdx.x; k < K; k += blockDim.x) xs[k] = x[k];
    __syncthreads();
    const int lane = threadIdx.x & 31, r = blockIdx.x * GEMV_WARPS + (threadIdx.x >> 5);
    if (r >= R) return;
    const float *w = Wt + (size_t)r * K;
    double a = 0.0;
    int k = lane;
    for (; k + 96 < K; k += 128) {
        const float w0 = __ldg(w + k), w1 = __ldg(w + k + 32), w2 = __ldg(w + k + 64), w3 = __ldg(w + k + 96);
        a += (double)w0 * xs[k] + (double)w1 * xs[k + 32] + (double)w2 * xs[k + 64] + (double)w3 * xs[k + 96];
    }
    for (; k < K; k += 32) a += (double)__ldg(w + k) * xs[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) {
        const float v = (float)(a + (double)b[r]);
        y[r] = add ? v + add[r] : v;
    }
}

// rot6d_to_rotmat: x [J][3][2] -> R [J][3][3] with columns b1, b2, b3 (F.normalize's eps 1e-12)
__global__ void k_hps_rot6d(const float *__restrict__ pose, float *__restrict__ rotmat, int J) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= J) return;
    double a1[3], a2[3], b1[3], b2[3], b3[3];
    for (int i = 0; i < 3; ++i) { a1[i] = pose[j * 6 + i * 2]; a2[i] = pose[j * 6 + i * 2 + 1]; }
    const double n1 = fmax(sqrt(a1[0] * a1[0] + a1[1] * a1[1] + a1[2] * a1[2]), 1e-12);
    for (int i = 0; i < 3; ++i) b1[i] = a1[i] / n1;
    const double d = b1[0] * a2[0] + b1[1] * a2[1] + b1[2] * a2[2];
    double u[3];
    for (int i = 0; i < 3; ++i) u[i] = a2[i] - d * b1[i];
    const double n2 = fmax(sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), 1e-12);
    for (int i = 0; i < 3; ++i) b2[i] = u[i] / n2;
    b3[0] = b1[1] * b2[2] - b1[2] * b2[1];
    b3[1] = b1[2] * b2[0] - b1[0] * b2[2];
    b3[2] = b1[0] * b2[1] - b1[1] * b2[0];
    float *R = rotmat + j * 9;
    for (int i = 0; i < 3; ++i) { R[i * 3] = (float)b1[i]; R[i * 3 + 1] = (float)b2[i]; R[i * 3 + 2] = (float)b3[i]; }
}

// projection(p, cam) of lib/pymaf/utils/geometry.py: t = (cam1, cam2, 2 * 5000 / (224 cam0 + 1e-9)), focal 5000,
// principal point 0, then / 112
__device__ __forceinline__ void project(const double p[3], const float *cam, double out[2]) {
    const double tz = 2.0 * 5000.0 / (224.0 * (double)cam[0] + 1e-9);
    const double x = p[0] + (double)cam[1], y = p[1] + (double)cam[2], z = p[2] + tz;
    out[0] = x / z * 5000.0 / 112.0;
    out[1] = y / z * 5000.0 / 112.0;
}

// blocks [0, E): extra-joint row e (dense over V); blocks E..: GEMV_WARPS Dmap rows each (CSR), projected into pts
__global__ void __launch_bounds__(256) k_hps_regress(const float *__restrict__ verts, int V,
                                                     const float *__restrict__ jextra, int E, float *__restrict__ extra,
                                                     const int *__restrict__ row_off, const int *__restrict__ col,
                                                     const float *__restrict__ val, int M, const float *__restrict__ cam,
                                                     float *__restrict__ pts) {
    __shared__ double red[3][8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if ((int)blockIdx.x < E) {
        const float *w = jextra + (size_t)blockIdx.x * V;
        double a[3] = {0.0, 0.0, 0.0};
        for (int v = threadIdx.x; v < V; v += blockDim.x) {
            const double wv = __ldg(w + v);
            if (wv == 0.0) continue;
            for (int c = 0; c < 3; ++c) a[c] += wv * (double)verts[v * 3 + c];
        }
        for (int c = 0; c < 3; ++c) {
            double s = a[c];
#pragma unroll
            for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) red[c][warp] = s;
        }
        __syncthreads();
        if (threadIdx.x < 3) {
            double s = 0.0;
            for (int k = 0; k < 8; ++k) s += red[threadIdx.x][k];
            extra[blockIdx.x * 3 + threadIdx.x] = (float)s;
        }
        return;
    }
    const int m = ((int)blockIdx.x - E) * 8 + warp;
    if (m >= M) return;
    double a[3] = {0.0, 0.0, 0.0};
    for (int k = row_off[m] + lane; k < row_off[m + 1]; k += 32) {
        const double wv = val[k];
        const int v = col[k];
        for (int c = 0; c < 3; ++c) a[c] += wv * (double)verts[v * 3 + c];
    }
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int o = 16; o; o >>= 1) a[c] += __shfl_xor_sync(0xffffffffu, a[c], o);
    if (lane == 0) {
        // the reference projects the float32 product
        const double p[3] = {(double)(float)a[0], (double)(float)a[1], (double)(float)a[2]};
        double q[2];
        project(p, cam, q);
        pts[m] = (float)q[0];
        pts[M + m] = (float)q[1];
    }
}

// kornia's rotation_matrix_to_quaternion (eps 1e-6) + quaternion_to_angle_axis, NaN -> 0, on R [3][3] (row-major)
__device__ void rotmat_to_aa(const float *Rf, double aa[3]) {
    double m[3][3];   // m = R^T (rmat_t)
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) m[i][k] = Rf[k * 3 + i];
    const bool d2 = m[2][2] < 1e-6, d0d1 = m[0][0] > m[1][1], d0nd1 = m[0][0] < -m[1][1];
    double q[4], t;
    if (d2 && d0d1) {
        t = 1 + m[0][0] - m[1][1] - m[2][2];
        q[0] = m[1][2] - m[2][1]; q[1] = t; q[2] = m[0][1] + m[1][0]; q[3] = m[2][0] + m[0][2];
    } else if (d2) {
        t = 1 - m[0][0] + m[1][1] - m[2][2];
        q[0] = m[2][0] - m[0][2]; q[1] = m[0][1] + m[1][0]; q[2] = t; q[3] = m[1][2] + m[2][1];
    } else if (d0nd1) {
        t = 1 - m[0][0] - m[1][1] + m[2][2];
        q[0] = m[0][1] - m[1][0]; q[1] = m[2][0] + m[0][2]; q[2] = m[1][2] + m[2][1]; q[3] = t;
    } else {
        t = 1 + m[0][0] + m[1][1] + m[2][2];
        q[0] = t; q[1] = m[1][2] - m[2][1]; q[2] = m[2][0] - m[0][2]; q[3] = m[0][1] - m[1][0];
    }
    const double st = sqrt(t);   // NaN for t < 0, as the reference's sqrt
    for (int k = 0; k < 4; ++k) q[k] = q[k] / st * 0.5;
    const double ss = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    const double sn = sqrt(ss), cs = q[0];
    const double two_theta = 2.0 * (cs < 0.0 ? atan2(-sn, -cs) : atan2(sn, cs));
    const double k = ss > 0.0 ? two_theta / sn : 2.0;
    for (int c = 0; c < 3; ++c) {
        const double v = q[c + 1] * k;
        aa[c] = isnan(v) ? 0.0 : v;
    }
}

// one block: joints [Jl lbs joints, NV vertex joints, E extra] gathered by joint_map [NJ] -> kp_3d [NJ][3] and kp_2d
// [NJ][2]; theta = [cam 3, shape 10, aa 3 Jl]
__global__ void k_hps_tail(const float *__restrict__ verts, const float *__restrict__ jlbs, int Jl,
                           const int *__restrict__ vid, int NV, const float *__restrict__ extra, int E,
                           const int *__restrict__ jmap, int NJ, const float *__restrict__ rotmat,
                           const float *__restrict__ par, int npose, int nshape, float *__restrict__ kp3d,
                           float *__restrict__ kp2d, float *__restrict__ theta) {
    const float *cam = par + npose + nshape;
    for (int j = threadIdx.x; j < NJ; j += blockDim.x) {
        const int s = jmap[j];
        const float *src = s < Jl ? jlbs + s * 3 : (s < Jl + NV ? verts + (size_t)vid[s - Jl] * 3 : extra + (s - Jl - NV) * 3);
        double p[3], q[2];
        for (int c = 0; c < 3; ++c) { kp3d[j * 3 + c] = src[c]; p[c] = src[c]; }
        project(p, cam, q);
        kp2d[j * 2] = (float)q[0];
        kp2d[j * 2 + 1] = (float)q[1];
    }
    for (int j = threadIdx.x; j < Jl; j += blockDim.x) {
        double aa[3];
        rotmat_to_aa(rotmat + j * 9, aa);
        for (int c = 0; c < 3; ++c) theta[3 + nshape + j * 3 + c] = (float)aa[c];
    }
    for (int k = threadIdx.x; k < 3 + nshape; k += blockDim.x)
        theta[k] = k < 3 ? cam[k] : par[npose + k - 3];
}

}  // namespace icon

using namespace icon;

extern "C" int icon_maxpool3s2_nhwc(const float *x, void *hi, void *lo, int N, int H, int W, int C, int Cp, int relu,
                                    icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(x && hi && lo && N > 0 && H > 0 && W > 0 && C > 0 && Cp >= C && Cp % 64 == 0,
                   "icon_maxpool3s2_nhwc: bad argument");
    const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
    const int64_t total = (int64_t)N * OH * OW * Cp;
    k_maxpool3s2<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, (__half *)hi, (__half *)lo, N, H, W, C, Cp, OH,
                                                                       OW, relu);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_maf_mlp(const float *feat, int H, int W, int C, const float *pts, int N, const float *w1,
                            const float *b1, const float *w2, const float *b2, const float *w3, const float *b3,
                            const float *prev, int nprev, float *xc, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(feat && pts && w1 && b1 && w2 && b2 && w3 && b3 && xc && (prev || nprev == 0),
                   "icon_maf_mlp: null pointer");
    ICON_CHECK_ARG(C == MAF_C && H > 1 && W > 1 && N > 0 && nprev >= 0,
                   "icon_maf_mlp: needs %d channels, H, W > 1 and N > 0 (C=%d, H=%d, W=%d, N=%d)", MAF_C, C, H, W, N);
    k_maf_mlp<<<N, MAF_H1, 0, stream>>>(feat, H, W, pts, N, w1, b1, w2, b2, w3, b3, prev, nprev, xc);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_hps_gemv(const float *w, const float *x, const float *b, const float *add, float *y, int R, int K,
                             icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(w && x && b && y && R > 0 && K > 0, "icon_hps_gemv: bad argument");
    ICON_CHECK_ARG((size_t)K * sizeof(float) <= 48 * 1024, "icon_hps_gemv: K=%d exceeds 12288", K);
    k_hps_gemv<<<(R + GEMV_WARPS - 1) / GEMV_WARPS, GEMV_WARPS * 32, (size_t)K * sizeof(float), stream>>>(w, x, b, add,
                                                                                                         y, R, K);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_hps_rot6d(const float *pose, float *rotmat, int J, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(pose && rotmat && J > 0, "icon_hps_rot6d: bad argument");
    k_hps_rot6d<<<(J + 63) / 64, 64, 0, stream>>>(pose, rotmat, J);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_hps_regress(const float *verts, int V, const float *jextra, int E, float *extra, const int *row_off,
                                const int *col, const float *val, int M, const float *cam, float *pts,
                                icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(verts && V > 0 && E >= 0 && M >= 0 && E + M > 0, "icon_hps_regress: bad argument");
    ICON_CHECK_ARG(E == 0 || (jextra && extra), "icon_hps_regress: extra-joint regressor missing");
    ICON_CHECK_ARG(M == 0 || (row_off && col && val && cam && pts), "icon_hps_regress: Dmap arguments missing");
    k_hps_regress<<<E + (M + 7) / 8, 256, 0, stream>>>(verts, V, jextra, E, extra, row_off, col, val, M, cam, pts);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_hps_tail(const float *verts, const float *jlbs, int Jl, const int *vid, int NV, const float *extra,
                             int E, const int *jmap, int NJ, const float *rotmat, const float *par, int npose,
                             int nshape, float *kp3d, float *kp2d, float *theta, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(verts && jlbs && rotmat && par && kp3d && kp2d && theta && jmap && Jl > 0 && NJ > 0 &&
                       NV >= 0 && E >= 0 && (vid || NV == 0) && (extra || E == 0) && npose == 6 * Jl && nshape >= 0,
                   "icon_hps_tail: bad argument");
    k_hps_tail<<<1, 128, 0, stream>>>(verts, jlbs, Jl, vid, NV, extra, E, jmap, NJ, rotmat, par, npose, nshape, kp3d,
                                      kp2d, theta);
    ICON_LAUNCHED();
    return ICON_OK;
}
