// NHWC companions of conv_nhwc.cu: everything between two convolutions of the encoders in ONE pass each.
//
//   k_norm_finalize   per-(image, channel) sums from the producing kernel's epilogue -> (scale, mean, beta) per channel for
//                     nn.InstanceNorm2d(affine=False) / nn.GroupNorm(32, C)        (FBNet.py:216-261, net_util.py:258-280)
//   k_act_nhwc        y = [relu]( (x - mean) * scale + beta ) [+ residual]  ->  fp16 hi / lo NHWC operand tensors in the layout the
//                     CONSUMING convolution wants (reflection halo, space-to-depth planes for stride 2, channel padding
//                     to 64) and / or an fp32 NHWC tensor
//   k_ew_nhwc         add2 / add3 / 2x2 average pool / bicubic x2 upsample + add (HGFilters.py:49-79), each also
//                     accumulating the statistics of its result for the GroupNorm that reads it next
//   k_nchw_to_nhwc / k_nhwc_to_nchw   layout adaptors at the ends of an encoder (+ statistics)
#include <cuda_fp16.h>

#include "common.cuh"

namespace icon {

// ---------------------------------------------------------------------------------------- statistics -> scale / mean / beta
// stats [N][C][6] doubles (sum, sum of squares over `count` pixels: stats_add in common.cuh) -> ss [N][C][3] (scale, mean,
// beta).  Consumers compute (x - mean) * scale + beta like torch, so a constant channel gives exactly beta (its mean is
// exact), which a folded shift = beta - mean * scale would miss by the rounding of mean * scale.  groups == 0: per
// channel (instance norm).
__global__ void k_norm_finalize(const double *__restrict__ stats, const float *__restrict__ gamma,
                                const float *__restrict__ beta, float *__restrict__ ss, int N, int C, int groups,
                                double count, float eps) {
    pdl_launch_dependents();
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * C) return;
    const int n = i / C, c = i % C;
    double s = 0.0, q = 0.0, cnt = count;
    if (groups <= 0) {
        s = stats_sum(stats + (size_t)i * 6); q = stats_sumsq(stats + (size_t)i * 6);
    } else {
        const int cg = C / groups, g0 = (c / cg) * cg;
        for (int k = 0; k < cg; ++k) {
            s += stats_sum(stats + ((size_t)n * C + g0 + k) * 6);
            q += stats_sumsq(stats + ((size_t)n * C + g0 + k) * 6);
        }
        cnt = count * cg;
    }
    const double mean = s / cnt;
    double var = q / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
    ss[(size_t)i * 3] = rstd * g; ss[(size_t)i * 3 + 1] = (float)mean; ss[(size_t)i * 3 + 2] = b;
}

// ---------------------------------------------------------------------------------------- normalise + split
struct ActParams {
    const float *x;          // fp32 NHWC [N][H][W][Cs_in], channels [ci_off, ci_off + C)
    const float *ss;         // [N][C][3] scale / mean / beta (k_norm_finalize) or null
    const double *stats;     // or: [N][C][6] sums straight from the producer (normalisation folded in here); both null =
    const float *gamma, *beta;   // identity.  gamma / beta: GroupNorm affine or null
    int cg;                  // channels per normalisation group (1 = instance norm), 8 % cg == 0
    double inv_count;        // 1 / (pixels * cg)
    float eps;
    const float *res;        // fp32 NHWC [N][H][W][C] or null: added AFTER the activation
    __half *hi, *lo;         // [N * planes][Hp][Wp][Cp] or null
    float *f32;              // fp32 NHWC [N][H][W][C] or null
    int N, H, W, C, Cs_in, ci_off, Cp;
    int P;                   // halo (reflection) around the image in hi / lo; 0 with s2d
    int s2d;                 // 1: 4 parity planes of (H/2, W/2) -- plane = (y & 1) * 2 + (x & 1)
    int relu;                // 1: ReLU before the residual add; 2: after it (a Bottleneck's relu(bn3(conv3) + residual))
};

// one thread = one (destination pixel, 8-channel group)
__global__ void k_act_nhwc(const __grid_constant__ ActParams p) {
    pdl_launch_dependents();
    pdl_wait();
    const unsigned groups = (unsigned)p.Cp / 8u;                // total < 2^31 is checked by the host: 32-bit index math
    const unsigned Hd = p.s2d ? p.H : p.H + 2 * p.P, Wd = p.s2d ? p.W : p.W + 2 * p.P;
    const unsigned total = (unsigned)p.N * Hd * Wd * groups;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    unsigned r = i / groups;
    const int g = (int)(i - r * groups);
    const int dx = (int)(r % Wd); r /= Wd;
    const int dy = (int)(r % Hd);
    const int n = (int)(r / Hd);
    int sy = dy - p.P, sx = dx - p.P;                          // source pixel (reflection for the halo)
    const bool interior = sy >= 0 && sy < p.H && sx >= 0 && sx < p.W;
    sy = sy < 0 ? -sy : (sy >= p.H ? 2 * p.H - 2 - sy : sy);
    sx = sx < 0 ? -sx : (sx >= p.W ? 2 * p.W - 2 - sx : sx);
    const int c0 = g * 8;
    float v[8];
    const size_t spix = ((size_t)n * p.H + sy) * p.W + sx;
    const float *xs = p.x + spix * p.Cs_in + p.ci_off + c0;
    if (c0 + 8 <= p.C && ((reinterpret_cast<uintptr_t>(xs) & 15) == 0)) {            // 2 x 128-bit loads
        const float4 a = *reinterpret_cast<const float4 *>(xs), b = *reinterpret_cast<const float4 *>(xs + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = (c0 + k < p.C) ? xs[k] : 0.f;
    }
    if (p.ss) {
        const float *ss = p.ss + ((size_t)n * p.C + c0) * 3;
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (c0 + k < p.C) v[k] = fmaf(v[k] - __ldg(ss + 3 * k + 1), __ldg(ss + 3 * k), __ldg(ss + 3 * k + 2));
    } else if (p.stats) {
        // mean / scale from the producer's sums: a thread's 8 channels hold whole groups (cg in {1, 2, 4, 8})
        const double *st = p.stats + ((size_t)n * p.C + c0) * 6;
        for (int g0 = 0; g0 < 8; g0 += p.cg) {
            if (c0 + g0 >= p.C) break;
            double s = 0.0, q = 0.0;
            for (int k = 0; k < p.cg; ++k) { s += stats_sum(st + (g0 + k) * 6); q += stats_sumsq(st + (g0 + k) * 6); }
            const double mean = s * p.inv_count;
            const float var = fmaxf((float)(q * p.inv_count - mean * mean), 0.f);
            const float rstd = rsqrtf(var + p.eps), mf = (float)mean;
            for (int k = 0; k < p.cg; ++k) {
                const int c = c0 + g0 + k;
                const float ga = p.gamma ? __ldg(p.gamma + c) : 1.f, be = p.beta ? __ldg(p.beta + c) : 0.f;
                v[g0 + k] = fmaf(v[g0 + k] - mf, rstd * ga, be);
            }
        }
    }
    if (p.relu == 1) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], 0.f);
    }
    if (p.res) {
        const float *rs = p.res + spix * p.C + c0;
        if (c0 + 8 <= p.C && ((reinterpret_cast<uintptr_t>(rs) & 15) == 0)) {
            const float4 a = *reinterpret_cast<const float4 *>(rs), b = *reinterpret_cast<const float4 *>(rs + 4);
            v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (c0 + k < p.C) v[k] += rs[k];
        }
    }
    if (p.relu == 2) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], 0.f);
    }
    if (p.f32 && interior) {
        float *fd = p.f32 + spix * p.C + c0;
        if (c0 + 8 <= p.C && ((reinterpret_cast<uintptr_t>(fd) & 15) == 0)) {
            *reinterpret_cast<float4 *>(fd) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4 *>(fd + 4) = make_float4(v[4], v[5], v[6], v[7]);
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (c0 + k < p.C) fd[k] = v[k];
        }
    }
    if (p.hi) {
        size_t d;
        if (p.s2d) {
            const int plane = (dy & 1) * 2 + (dx & 1);
            d = ((((size_t)n * 4 + plane) * (p.H / 2) + (dy >> 1)) * (p.W / 2) + (dx >> 1)) * p.Cp + c0;
        } else {
            d = (((size_t)n * Hd + dy) * Wd + dx) * (size_t)p.Cp + c0;
        }
        __align__(16) __half h[8], l[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            h[k] = __float2half_rn(v[k]);
            l[k] = __float2half_rn(v[k] - __half2float(h[k]));
        }
        *reinterpret_cast<uint4 *>(p.hi + d) = *reinterpret_cast<const uint4 *>(h);
        *reinterpret_cast<uint4 *>(p.lo + d) = *reinterpret_cast<const uint4 *>(l);
    }
}

// ---------------------------------------------------------------------------------------- split-K finish + InstanceNorm + act
// The ResnetBlock layers (FBNet.py:268-319: conv -> InstanceNorm2d(affine=False) [-> ReLU] [+ x]) run split-K, and an
// instance norm only needs the statistics of ONE channel over the image: a block that owns 8 channels of all H x W
// pixels can sum the parked split-K partials (fixed order), keep the result in shared memory, compute mean / variance
// locally (two-pass, no atomics: deterministic), normalise, and write the next convolution's hi / lo operand (with its
// reflection halo) + the fp32 copy the residual connection needs -- split-K finish, norm statistics, finalize and the
// act pass in one kernel, the un-normalised tensor never goes to HBM.   grid (C / 8, N), 256 threads, H*W*32 B smem.
struct SkActParams {
    const float *partial;    // [splits][N][H][W][C]
    const float *bias;       // [C] or null
    const float *res;        // fp32 NHWC [N][H][W][C] or null: added after norm (+ ReLU)
    __half *hi, *lo;         // [N][H + 2P][W + 2P][Cp]
    float *f32;              // [N][H][W][C] or null
    int splits, N, H, W, C, Cp, P, relu;
    float eps;
};

__global__ void __launch_bounds__(256) k_splitk_in_act(const __grid_constant__ SkActParams p) {
    extern __shared__ float4 sval[];                           // [H*W][2]: 8 channels per pixel
    __shared__ double sw[8][8];
    __shared__ float s_mean[8], s_rstd[8];
    pdl_launch_dependents();
    pdl_wait();
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int c0 = blockIdx.x * 8, n = blockIdx.y;
    const int HW = p.H * p.W;
    const size_t split_stride = (size_t)p.N * HW * p.C;
    float4 b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
    if (p.bias) { b0 = *reinterpret_cast<const float4 *>(p.bias + c0); b1 = *reinterpret_cast<const float4 *>(p.bias + c0 + 4); }
    double s[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // fp64: the centred pass is only as good as this mean
    for (int pix = tid; pix < HW; pix += 256) {
        const float *src = p.partial + ((size_t)n * HW + pix) * p.C + c0;
        float4 v0 = b0, v1 = b1;
        for (int k = 0; k < p.splits; ++k) {
            const float4 t0 = __ldcg(reinterpret_cast<const float4 *>(src + (size_t)k * split_stride));
            const float4 t1 = __ldcg(reinterpret_cast<const float4 *>(src + (size_t)k * split_stride + 4));
            v0.x += t0.x; v0.y += t0.y; v0.z += t0.z; v0.w += t0.w;
            v1.x += t1.x; v1.y += t1.y; v1.z += t1.z; v1.w += t1.w;
        }
        sval[2 * pix] = v0; sval[2 * pix + 1] = v1;
        s[0] += v0.x; s[1] += v0.y; s[2] += v0.z; s[3] += v0.w; s[4] += v1.x; s[5] += v1.y; s[6] += v1.z; s[7] += v1.w;
    }
    auto block_sum8 = [&](auto (&x)[8], float *out8) {         // deterministic: shuffle tree, then warps in order
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int o = 16; o; o >>= 1) x[k] += __shfl_xor_sync(0xffffffffu, x[k], o);
        __syncthreads();
        if (lane == 0)
#pragma unroll
            for (int k = 0; k < 8; ++k) sw[w][k] = x[k];
        __syncthreads();
        if (tid < 8) {
            double t = 0.0;
            for (int ww = 0; ww < 8; ++ww) t += sw[ww][tid];
            out8[tid] = (float)(t / (double)HW);
        }
        __syncthreads();
    };
    block_sum8(s, s_mean);
    float q[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int pix = tid; pix < HW; pix += 256) {                 // centred second moment from shared memory
        const float4 v0 = sval[2 * pix], v1 = sval[2 * pix + 1];
        float d;
        d = v0.x - s_mean[0]; q[0] = fmaf(d, d, q[0]); d = v0.y - s_mean[1]; q[1] = fmaf(d, d, q[1]);
        d = v0.z - s_mean[2]; q[2] = fmaf(d, d, q[2]); d = v0.w - s_mean[3]; q[3] = fmaf(d, d, q[3]);
        d = v1.x - s_mean[4]; q[4] = fmaf(d, d, q[4]); d = v1.y - s_mean[5]; q[5] = fmaf(d, d, q[5]);
        d = v1.z - s_mean[6]; q[6] = fmaf(d, d, q[6]); d = v1.w - s_mean[7]; q[7] = fmaf(d, d, q[7]);
    }
    block_sum8(q, s_rstd);                                      // holds the (biased) variance for the moment
    if (tid < 8) s_rstd[tid] = rsqrtf(s_rstd[tid] + p.eps);
    __syncthreads();
    const int Hd = p.H + 2 * p.P, Wd = p.W + 2 * p.P;
    for (int d = tid; d < Hd * Wd; d += 256) {
        const int dy = d / Wd, dx = d - dy * Wd;
        int sy = dy - p.P, sx = dx - p.P;
        const bool interior = sy >= 0 && sy < p.H && sx >= 0 && sx < p.W;
        sy = sy < 0 ? -sy : (sy >= p.H ? 2 * p.H - 2 - sy : sy);
        sx = sx < 0 ? -sx : (sx >= p.W ? 2 * p.W - 2 - sx : sx);
        const int pix = sy * p.W + sx;
        const float4 v0 = sval[2 * pix], v1 = sval[2 * pix + 1];
        float y[8] = {(v0.x - s_mean[0]) * s_rstd[0], (v0.y - s_mean[1]) * s_rstd[1], (v0.z - s_mean[2]) * s_rstd[2],
                      (v0.w - s_mean[3]) * s_rstd[3], (v1.x - s_mean[4]) * s_rstd[4], (v1.y - s_mean[5]) * s_rstd[5],
                      (v1.z - s_mean[6]) * s_rstd[6], (v1.w - s_mean[7]) * s_rstd[7]};
        if (p.relu) {
#pragma unroll
            for (int k = 0; k < 8; ++k) y[k] = fmaxf(y[k], 0.f);
        }
        if (p.res) {
            const float *rs = p.res + ((size_t)n * HW + pix) * p.C + c0;
            const float4 r0 = *reinterpret_cast<const float4 *>(rs), r1 = *reinterpret_cast<const float4 *>(rs + 4);
            y[0] += r0.x; y[1] += r0.y; y[2] += r0.z; y[3] += r0.w; y[4] += r1.x; y[5] += r1.y; y[6] += r1.z; y[7] += r1.w;
        }
        if (p.f32 && interior) {
            float *fd = p.f32 + ((size_t)n * HW + pix) * p.C + c0;
            *reinterpret_cast<float4 *>(fd) = make_float4(y[0], y[1], y[2], y[3]);
            *reinterpret_cast<float4 *>(fd + 4) = make_float4(y[4], y[5], y[6], y[7]);
        }
        if (p.hi) {
            __align__(16) __half h[8], l[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                h[k] = __float2half_rn(y[k]);
                l[k] = __float2half_rn(y[k] - __half2float(h[k]));
            }
            const size_t o = (((size_t)n * Hd + dy) * Wd + dx) * (size_t)p.Cp + c0;
            *reinterpret_cast<uint4 *>(p.hi + o) = *reinterpret_cast<const uint4 *>(h);
            *reinterpret_cast<uint4 *>(p.lo + o) = *reinterpret_cast<const uint4 *>(l);
        }
    }
}

// ---------------------------------------------------------------------------------------- elementwise + statistics
struct EwParams {
    const float *a, *b, *c;  // fp32 NHWC
    float *y;
    double *stats;           // [N][C][6] (stats_add in common.cuh) or null
    int N, H, W, C;          // OUTPUT dims
    int mode;                // 0: a + b (+ c)   1: avg_pool2(a) (a is [N][2H][2W][C])   2: b + bicubic_up2(a) (a is [N][H/2][W/2][C])
                             // 3: relu((a - mean) * scale + beta) from ss[n][c][3]   (a norm whose RESULT feeds another norm)
    const float *ss;
};

__device__ __forceinline__ void cubic_w4(float t, float (&w)[4]) {     // torch upsample_bicubic2d, A = -0.75
    const float A = -0.75f;
    float x;
    x = t + 1.f; w[0] = ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A;
    x = t;       w[1] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
    x = 1.f - t; w[2] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
    x = 2.f - t; w[3] = ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A;
}

constexpr int EW_PIX = 64;           // pixels per block (more blocks = more same-address fp64 atomics: 32 measured slower)
// grid (ceil(H*W / EW_PIX), N), 256 threads: thread = (channel quad, pixel row); C % 4 == 0, C / 4 divides 256
__global__ void __launch_bounds__(256) k_ew_nhwc(const __grid_constant__ EwParams p) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ double sred[2][256 * 4];                        // [sum | sum of squares][row][channel]: rows * C = 1024
    const int quads = p.C / 4, rows = 256 / quads;
    const int q = threadIdx.x % quads, r0 = threadIdx.x / quads;
    const int n = blockIdx.y;
    const unsigned hw = (unsigned)p.H * (unsigned)p.W;
    const unsigned pix0 = blockIdx.x * EW_PIX;
    double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
    for (int pr = r0; pr < EW_PIX; pr += rows) {
        const unsigned pix = pix0 + pr;
        if (pix >= hw) break;
        const size_t o = ((size_t)n * hw + pix) * p.C + q * 4;
        float4 v;
        if (p.mode == 0) {
            v = *reinterpret_cast<const float4 *>(p.a + o);
            const float4 b = *reinterpret_cast<const float4 *>(p.b + o);
            v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
            if (p.c) {
                const float4 c = *reinterpret_cast<const float4 *>(p.c + o);
                v.x += c.x; v.y += c.y; v.z += c.z; v.w += c.w;
            }
        } else if (p.mode == 3) {
            v = *reinterpret_cast<const float4 *>(p.a + o);
            const float *ss = p.ss + ((size_t)n * p.C + q * 4) * 3;
            v.x = fmaxf(fmaf(v.x - ss[1], ss[0], ss[2]), 0.f); v.y = fmaxf(fmaf(v.y - ss[4], ss[3], ss[5]), 0.f);
            v.z = fmaxf(fmaf(v.z - ss[7], ss[6], ss[8]), 0.f); v.w = fmaxf(fmaf(v.w - ss[10], ss[9], ss[11]), 0.f);
        } else if (p.mode == 1) {
            const int oy = (int)(pix / p.W), ox = (int)(pix % p.W);
            const int W2 = 2 * p.W;
            const float *s = p.a + (((size_t)n * 2 * p.H + 2 * oy) * W2 + 2 * ox) * p.C + q * 4;
            const float4 a00 = *reinterpret_cast<const float4 *>(s), a01 = *reinterpret_cast<const float4 *>(s + p.C);
            const float4 a10 = *reinterpret_cast<const float4 *>(s + (size_t)W2 * p.C);
            const float4 a11 = *reinterpret_cast<const float4 *>(s + (size_t)W2 * p.C + p.C);
            // F.avg_pool2d: (a00 + a01 + a10 + a11) / 4 in this summation order
            v.x = (a00.x + a01.x + a10.x + a11.x) * 0.25f; v.y = (a00.y + a01.y + a10.y + a11.y) * 0.25f;
            v.z = (a00.z + a01.z + a10.z + a11.z) * 0.25f; v.w = (a00.w + a01.w + a10.w + a11.w) * 0.25f;
        } else {
            const int oy = (int)(pix / p.W), ox = (int)(pix % p.W);
            const int H = p.H / 2, W = p.W / 2;
            const float sy = p.H > 1 ? (float)(H - 1) / (float)(p.H - 1) : 0.f, sx = p.W > 1 ? (float)(W - 1) / (float)(p.W - 1) : 0.f;
            const float fy = sy * oy, fx = sx * ox;
            const int iy = (int)floorf(fy), ix = (int)floorf(fx);
            float wy[4], wx[4];
            cubic_w4(fy - iy, wy);
            cubic_w4(fx - ix, wx);
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int aa = 0; aa < 4; ++aa) {
                const int yy = min(max(iy - 1 + aa, 0), H - 1);
                float4 row = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int bb = 0; bb < 4; ++bb) {
                    const int xx = min(max(ix - 1 + bb, 0), W - 1);
                    const float4 t = *reinterpret_cast<const float4 *>(p.a + (((size_t)n * H + yy) * W + xx) * p.C + q * 4);
                    row.x = fmaf(t.x, wx[bb], row.x); row.y = fmaf(t.y, wx[bb], row.y);
                    row.z = fmaf(t.z, wx[bb], row.z); row.w = fmaf(t.w, wx[bb], row.w);
                }
                acc.x = fmaf(row.x, wy[aa], acc.x); acc.y = fmaf(row.y, wy[aa], acc.y);
                acc.z = fmaf(row.z, wy[aa], acc.z); acc.w = fmaf(row.w, wy[aa], acc.w);
            }
            const float4 b = *reinterpret_cast<const float4 *>(p.b + o);
            v = make_float4(acc.x + b.x, acc.y + b.y, acc.z + b.z, acc.w + b.w);
        }
        *reinterpret_cast<float4 *>(p.y + o) = v;
        if (p.stats) {
            const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) { s1[j] += e[j]; s2[j] = fma((double)e[j], (double)e[j], s2[j]); }
        }
    }
    if (!p.stats) return;
    // per-channel sums of the block in a fixed order (row 0, 1, ...): deterministic, no shared-memory atomics
#pragma unroll
    for (int j = 0; j < 4; ++j) { sred[0][r0 * p.C + q * 4 + j] = s1[j]; sred[1][r0 * p.C + q * 4 + j] = s2[j]; }
    __syncthreads();
    for (int c = threadIdx.x; c < p.C; c += 256) {
        double t1 = 0.0, t2 = 0.0;
        for (int r = 0; r < rows; ++r) { t1 += sred[0][r * p.C + c]; t2 += sred[1][r * p.C + c]; }
        stats_add(p.stats + ((size_t)n * p.C + c) * 6, t1, t2);
    }
}

// ---------------------------------------------------------------------------------------- layout adaptors
// x [N][C][HW] -> y [N][HW][C] (+ stats).  grid (ceil(HW / 32), N, ceil(C / 256)), 256 threads.
__global__ void __launch_bounds__(256) k_nchw_to_nhwc(const float *__restrict__ x, float *__restrict__ y,
                                                      double *__restrict__ stats, int C, int64_t HW) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float tile[];                            // [32][CB + 1]
    const int n = blockIdx.y;
    const int cb0 = blockIdx.z * 256, CB = min(256, C - cb0);
    const int64_t p0 = (int64_t)blockIdx.x * 32;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int cc = w; cc < CB; cc += 8) {
        const int c = cb0 + cc;
        const int64_t pix = p0 + lane;
        const float v = pix < HW ? x[((size_t)n * C + c) * HW + pix] : 0.f;
        tile[lane * (CB + 1) + cc] = v;
        if (stats) {
            double s1 = v, s2 = (double)v * v;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            }
            if (lane == 0) stats_add(stats + ((size_t)n * C + c) * 6, s1, s2);
        }
    }
    __syncthreads();
    const int64_t npx = min((int64_t)32, HW - p0);
    for (int i = threadIdx.x; i < npx * CB; i += 256) {
        const int px = i / CB, cc = i % CB;
        y[((size_t)n * HW + p0 + px) * C + cb0 + cc] = tile[px * (CB + 1) + cc];
    }
}

// x [N][HW][Cs] channels [c_off, c_off + C) -> y [N][C][HW]
__global__ void k_nhwc_to_nchw(const float *__restrict__ x, float *__restrict__ y, int N, int C, int Cs, int c_off, int64_t HW) {
    pdl_launch_dependents();
    pdl_wait();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * C * HW) return;
    const int64_t pix = i % HW;
    const int c = (int)((i / HW) % C), n = (int)(i / (HW * C));
    y[i] = x[((size_t)n * HW + pix) * Cs + c_off + c];
}

// ---------------------------------------------------------------------------------------- 7 x 7 stem operand
// The encoders' first layer has 3..9 input channels: far too few for a 64-channel K-chunk per tap.  Instead the K axis
// of the implicit GEMM runs over (kx, c) inside one filter ROW: with the image stored NHWC with C padded to Cp8 (8 or
// 16), the 8 pixels x Cp8 channels a filter row touches are CONTIGUOUS in memory, so the operand of output pixel x is
// the window starting at input pixel sx * x -- a tensor map whose W dimension has a stride of sx * Cp8 elements
// (overlapping windows) lets the same TMA box load deliver it; the 8th pixel of the window meets zero weights.
// x NCHW fp32 [N][Cin][H][W] -> hi / lo fp16 [N * sy][Hrows][Wp][Cp8] with a halo of 3 (reflection or zeros) and rows
// split into sy parity planes (stride-2 stem: tap row ky reads plane ky % 2 at row offset ky / 2).
__global__ void k_stem_pack(const float *__restrict__ x, __half *__restrict__ hi, __half *__restrict__ lo, int N, int Cin,
                            int H, int W, int Cp8, int Wp, int Hrows, int sy, int reflect) {
    pdl_launch_dependents();
    pdl_wait();
    const int64_t total = (int64_t)N * sy * Hrows * Wp;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int px = (int)(i % Wp);
    int64_t r = i / Wp;
    const int row = (int)(r % Hrows); r /= Hrows;
    const int plane = (int)(r % sy);
    const int n = (int)(r / sy);
    const int py = row * sy + plane;                          // padded row
    int sy_ = py - 3, sx_ = px - 3;
    bool ok = py < H + 6 && px < W + 6;
    if (reflect) {
        sy_ = sy_ < 0 ? -sy_ : (sy_ >= H ? 2 * H - 2 - sy_ : sy_);
        sx_ = sx_ < 0 ? -sx_ : (sx_ >= W ? 2 * W - 2 - sx_ : sx_);
    } else {
        ok = ok && sy_ >= 0 && sy_ < H && sx_ >= 0 && sx_ < W;
    }
    __half *dh = hi + (size_t)i * Cp8, *dl = lo + (size_t)i * Cp8;
    for (int c0 = 0; c0 < Cp8; c0 += 8) {
        __align__(16) __half h[8], l[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int c = c0 + k;
            const float v = (ok && c < Cin) ? x[(((size_t)n * Cin + c) * H + sy_) * W + sx_] : 0.f;
            h[k] = __float2half_rn(v);
            l[k] = __float2half_rn(v - __half2float(h[k]));
        }
        *reinterpret_cast<uint4 *>(dh + c0) = *reinterpret_cast<const uint4 *>(h);
        *reinterpret_cast<uint4 *>(dl + c0) = *reinterpret_cast<const uint4 *>(l);
    }
}

// out[n][co][y][x] = act(bias[co] + sum_{ky,kx} P[n][refl(y + ky - 3)][refl(x + kx - 3)][(ky * 7 + kx) * Cout + co])
// P = the 1 x 1 tensor-core GEMM of the 64-channel activation with the head's weights regrouped per tap
// (49 * Cout columns): the 7 x 7 head (FBNet.py:258-261) as GEMM + col2im instead of an N = 3 implicit GEMM.
__global__ void __launch_bounds__(256) k_col2im7(const float *__restrict__ P, const float *__restrict__ bias,
                                                 float *__restrict__ y, int N, int H, int W, int Cout, int Ps, int act) {
    pdl_launch_dependents();
    pdl_wait();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * H * W) return;
    const int ox = (int)(i % W), oy = (int)((i / W) % H), n = (int)(i / ((int64_t)W * H));
    float acc[3] = {0.f, 0.f, 0.f};
    for (int ky = 0; ky < 7; ++ky) {
        int iy = oy + ky - 3;
        iy = iy < 0 ? -iy : (iy >= H ? 2 * H - 2 - iy : iy);
        const float *row = P + ((size_t)n * H + iy) * W * Ps;
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
            int ix = ox + kx - 3;
            ix = ix < 0 ? -ix : (ix >= W ? 2 * W - 2 - ix : ix);
            const float *s = row + (size_t)ix * Ps + (ky * 7 + kx) * Cout;
            for (int co = 0; co < Cout; ++co) acc[co] += __ldg(s + co);
        }
    }
    for (int co = 0; co < Cout; ++co) {
        float v = acc[co] + (bias ? bias[co] : 0.f);
        if (act == 2) v = tanhf(v);
        else if (act == 1) v = fmaxf(v, 0.f);
        y[(((size_t)n * Cout + co) * H + oy) * W + ox] = v;
    }
}

}  // namespace icon

using namespace icon;

extern "C" int icon_col2im7(const float *P, const float *bias, float *y, int N, int H, int W, int Cout, int Ps, int act,
                            icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(P && y && N > 0 && H > 3 && W > 3 && Cout >= 1 && Cout <= 3 && Ps >= 49 * Cout, "icon_col2im7: bad argument");
    const int64_t total = (int64_t)N * H * W;
    ICON_CUDA(launch_pdl(k_col2im7, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, stream, P, bias, y, N, H, W, Cout, Ps, act));
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_norm_finalize(const double *stats, const float *gamma, const float *beta, float *scale_shift, int N, int C,
                                  int groups, double count, float eps, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(stats && scale_shift && N > 0 && C > 0 && count > 0, "icon_norm_finalize: bad argument");
    ICON_CHECK_ARG(groups <= 0 || C % groups == 0, "icon_norm_finalize: C %% groups != 0");
    ICON_CHECK_ARG((gamma == nullptr) == (beta == nullptr), "icon_norm_finalize: gamma and beta go together");
    ICON_CUDA(launch_pdl(k_norm_finalize, dim3((N * C + 127) / 128), dim3(128), 0, stream, stats, gamma, beta, scale_shift, N,
                         C, groups, count, eps));
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_act_nhwc(const float *x, int Cs_in, int ci_off, const float *scale_shift, const double *stats,
                             const float *gamma, const float *beta, int groups, float eps, const float *res, void *hi,
                             void *lo, float *f32, int N, int H, int W, int C, int Cp, int halo, int s2d, int relu,
                             icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(x && N > 0 && H > 0 && W > 0 && C > 0 && Cp >= C && Cp % 8 == 0, "icon_act_nhwc: bad argument");
    ICON_CHECK_ARG((hi == nullptr) == (lo == nullptr) && (hi || f32), "icon_act_nhwc: hi and lo go together; need an output");
    ICON_CHECK_ARG(!s2d || (halo == 0 && H % 2 == 0 && W % 2 == 0), "icon_act_nhwc: space-to-depth needs even H, W and no halo");
    ICON_CHECK_ARG(halo >= 0 && halo < H && halo < W, "icon_act_nhwc: reflection halo %d needs halo < H, W", halo);
    ICON_CHECK_ARG(ci_off >= 0 && ci_off + C <= Cs_in, "icon_act_nhwc: channel slice outside the input tensor");
    ICON_CHECK_ARG(!(scale_shift && stats), "icon_act_nhwc: scale_shift and stats are exclusive");
    ICON_CHECK_ARG((gamma == nullptr) == (beta == nullptr), "icon_act_nhwc: gamma and beta go together");
    ICON_CHECK_ARG(relu >= 0 && relu <= 2, "icon_act_nhwc: relu %d (0 none, 1 before the residual, 2 after it)", relu);
    ActParams p{};
    p.stats = stats; p.gamma = gamma; p.beta = beta; p.eps = eps; p.cg = 1; p.inv_count = 1.0 / ((double)H * W);
    if (stats && groups > 0) {
        ICON_CHECK_ARG(C % groups == 0, "icon_act_nhwc: C %% groups != 0");
        p.cg = C / groups;
        ICON_CHECK_ARG(p.cg == 1 || p.cg == 2 || p.cg == 4 || p.cg == 8, "icon_act_nhwc: %d channels per group (use icon_norm_finalize)", p.cg);
        p.inv_count = 1.0 / ((double)H * W * p.cg);
    }
    p.x = x; p.ss = scale_shift; p.res = res; p.hi = (__half *)hi; p.lo = (__half *)lo; p.f32 = f32;
    p.N = N; p.H = H; p.W = W; p.C = C; p.Cs_in = Cs_in; p.ci_off = ci_off; p.Cp = Cp; p.P = halo; p.s2d = s2d; p.relu = relu;
    const int64_t total = (int64_t)N * (s2d ? H : H + 2 * halo) * (s2d ? W : W + 2 * halo) * (Cp / 8);
    ICON_CHECK_ARG(total < (int64_t)1 << 31, "icon_act_nhwc: activation too large for 32-bit indexing");
    ICON_CUDA(launch_pdl(k_act_nhwc, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, stream, p));
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_splitk_instnorm_act(const float *partial, int splits, const float *bias, const float *res, void *hi, void *lo,
                                        float *f32, int N, int H, int W, int C, int Cp, int halo, int relu, float eps,
                                        icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(partial && splits >= 1 && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && Cp >= C && Cp % 8 == 0,
                   "icon_splitk_instnorm_act: bad argument (C %% 8 == 0)");
    ICON_CHECK_ARG((hi == nullptr) == (lo == nullptr) && (hi || f32), "icon_splitk_instnorm_act: hi and lo go together; need an output");
    ICON_CHECK_ARG(halo >= 0 && halo < H && halo < W, "icon_splitk_instnorm_act: reflection halo %d needs halo < H, W", halo);
    ICON_CHECK_ARG(Cp == C || !hi, "icon_splitk_instnorm_act: channel padding is not written here (C must be a multiple of 64)");
    const size_t smem = (size_t)H * W * 32;
    ICON_CHECK_ARG(smem <= 200 * 1024, "icon_splitk_instnorm_act: image of %d x %d pixels does not fit shared memory", H, W);
    static bool attr_set[ICON_MAX_DEVICES] = {};
    if (device_needs_setup(attr_set))
        ICON_CUDA(cudaFuncSetAttribute(k_splitk_in_act, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SkActParams p{};
    p.partial = partial; p.bias = bias; p.res = res; p.hi = (__half *)hi; p.lo = (__half *)lo; p.f32 = f32;
    p.splits = splits; p.N = N; p.H = H; p.W = W; p.C = C; p.Cp = Cp; p.P = halo; p.relu = relu; p.eps = eps;
    ICON_CUDA(launch_pdl(k_splitk_in_act, dim3((unsigned)(C / 8), (unsigned)N), dim3(256), smem, stream, p));
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_ew_nhwc(int mode, const float *a, const float *b, const float *c, float *y, double *stats, int N, int H,
                            int W, int C, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(a && y && N > 0 && H > 0 && W > 0 && mode >= 0 && mode <= 3, "icon_ew_nhwc: bad argument");
    ICON_CHECK_ARG(mode == 1 || b, "icon_ew_nhwc: second operand missing");
    ICON_CHECK_ARG(C % 4 == 0 && C <= 1024 && 256 % (C / 4) == 0, "icon_ew_nhwc: C=%d must be a power of two in [4, 1024]", C);
    ICON_CHECK_ARG(mode != 2 || (H % 2 == 0 && W % 2 == 0), "icon_ew_nhwc: upsample output must be even");
    EwParams p{};
    p.a = a; p.b = mode == 3 ? nullptr : b; p.c = c; p.y = y; p.stats = stats; p.N = N; p.H = H; p.W = W; p.C = C; p.mode = mode;
    p.ss = mode == 3 ? b : nullptr;
    dim3 grid((unsigned)(((int64_t)H * W + EW_PIX - 1) / EW_PIX), (unsigned)N);
    ICON_CUDA(launch_pdl(k_ew_nhwc, grid, dim3(256), 0, stream, p));
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_nchw_to_nhwc(const float *x, float *y, double *stats, int N, int C, int64_t HW, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(x && y && N > 0 && C > 0 && HW > 0, "icon_nchw_to_nhwc: bad argument");
    dim3 grid((unsigned)((HW + 31) / 32), (unsigned)N, (unsigned)((C + 255) / 256));
    ICON_CUDA(launch_pdl(k_nchw_to_nhwc, grid, dim3(256), 32 * (min(C, 256) + 1) * sizeof(float), stream, x, y, stats, C, HW));
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_nhwc_to_nchw(const float *x, float *y, int N, int C, int Cs, int c_off, int64_t HW, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(x && y && N > 0 && C > 0 && c_off >= 0 && c_off + C <= Cs && HW > 0, "icon_nhwc_to_nchw: bad argument");
    const int64_t total = (int64_t)N * C * HW;
    ICON_CUDA(launch_pdl(k_nhwc_to_nchw, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, stream, x, y, N, C, Cs, c_off, HW));
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_stem_pack(const float *x, void *hi, void *lo, int N, int Cin, int H, int W, int Cp8, int Wp, int Hrows,
                              int sy, int reflect, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(x && hi && lo && N > 0 && Cin > 0 && H > 3 && W > 3, "icon_stem_pack: bad argument");
    ICON_CHECK_ARG((Cp8 == 8 || Cp8 == 16) && Cin <= Cp8 && (sy == 1 || sy == 2), "icon_stem_pack: Cin <= 16, stride 1 or 2");
    ICON_CHECK_ARG(Wp >= W + 7 && Hrows * sy >= H + 6, "icon_stem_pack: padded extent too small");
    const int64_t total = (int64_t)N * sy * Hrows * Wp;
    ICON_CUDA(launch_pdl(k_stem_pack, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, stream, x, (__half *)hi, (__half *)lo, N, Cin,
                         H, W, Cp8, Wp, Hrows, sy, reflect));
    ICON_LAUNCHED();
    return ICON_OK;
}
