// The encoder kernels that live outside the NHWC path (conv_nhwc.cu, act_nhwc.cu), NCHW fp32:
//   k_normalize_mask   NormalNet.forward's L2 normalisation + background mask   lib/net/NormalNet.py:84-97
//   k_conv3d           PaMIR VolumeEncoder's Conv3d + BatchNorm3d layers        lib/net/VE.py:96-183
#include "common.cuh"

namespace icon {

// NormalNet.py:88-97: y = x / ||x||_2 over the 3 channels (no eps) * (sum_c |image| != 0)
__global__ void k_normalize_mask(const float *__restrict__ x, const float *__restrict__ image, float *__restrict__ y,
                                 int N, int Cimg, int64_t HW) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * HW) return;
    const int n = (int)(i / HW);
    const int64_t r = i % HW;
    const float a = x[((size_t)n * 3 + 0) * HW + r], b = x[((size_t)n * 3 + 1) * HW + r], c = x[((size_t)n * 3 + 2) * HW + r];
    const float nrm = sqrtf(a * a + b * b + c * c);
    float m = 0.f;
    for (int k = 0; k < Cimg; ++k) m += fabsf(image[((size_t)n * Cimg + k) * HW + r]);
    const float mask = m != 0.f ? 1.f : 0.f;
    y[((size_t)n * 3 + 0) * HW + r] = a / nrm * mask;
    y[((size_t)n * 3 + 1) * HW + r] = b / nrm * mask;
    y[((size_t)n * 3 + 2) * HW + r] = c / nrm * mask;
}

}  // namespace icon

using namespace icon;

extern "C" int icon_normalize_mask(const float *x, const float *image, float *y, int N, int Cimg, int64_t HW,
                                   icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(x && image && y && N > 0 && HW > 0, "icon_normalize_mask: bad argument");
    const int64_t n = (int64_t)N * HW;
    k_normalize_mask<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(x, image, y, N, Cimg, HW);
    ICON_LAUNCHED();
    return ICON_OK;
}

// ---------------------------------------------------------------- conv3d (PaMIR VolumeEncoder, lib/net/VE.py:96-183)
// Direct convolution, Cout <= 8, one thread per output voxel computing every output channel; eval-mode
// BatchNorm3d folded into (scale, shift); optional ReLU and residual.  The whole encoder is ~1 GFLOP.
namespace icon {
struct Conv3dParams {
    const float *x, *w, *scale, *shift, *res;
    float *y;
    int Cin, Cout, D, H, W, OD, OH, OW, k, stride, pad, dil, relu;
};
__global__ void __launch_bounds__(128) k_conv3d(Conv3dParams p) {
    extern __shared__ float sw[];                      // [Cout][Cin][k^3]
    const int k3 = p.k * p.k * p.k, nw = p.Cout * p.Cin * k3;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) sw[i] = p.w[i];
    __syncthreads();
    const int64_t n = (int64_t)p.OD * p.OH * p.OW;
    const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= n) return;
    const int ox = (int)(o % p.OW), oy = (int)((o / p.OW) % p.OH), oz = (int)(o / ((int64_t)p.OW * p.OH));
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;
    const size_t plane = (size_t)p.H * p.W, vol = plane * p.D;
    for (int ci = 0; ci < p.Cin; ++ci)
        for (int kz = 0; kz < p.k; ++kz) {
            const int iz = oz * p.stride - p.pad + kz * p.dil;
            if (iz < 0 || iz >= p.D) continue;
            for (int ky = 0; ky < p.k; ++ky) {
                const int iy = oy * p.stride - p.pad + ky * p.dil;
                if (iy < 0 || iy >= p.H) continue;
                for (int kx = 0; kx < p.k; ++kx) {
                    const int ix = ox * p.stride - p.pad + kx * p.dil;
                    if (ix < 0 || ix >= p.W) continue;
                    const float v = __ldg(p.x + ci * vol + (size_t)iz * plane + (size_t)iy * p.W + ix);
                    const int t = (kz * p.k + ky) * p.k + kx;
#pragma unroll
                    for (int c = 0; c < 8; ++c)
                        if (c < p.Cout) acc[c] = fmaf(v, sw[(c * p.Cin + ci) * k3 + t], acc[c]);
                }
            }
        }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        if (c >= p.Cout) break;
        float v = fmaf(acc[c], p.scale[c], p.shift[c]);
        if (p.res) v += p.res[(size_t)c * n + o];
        if (p.relu) v = fmaxf(v, 0.f);
        p.y[(size_t)c * n + o] = v;
    }
}
}  // namespace icon

extern "C" int icon_conv3d(const float *x, const float *w, const float *scale, const float *shift, const float *res,
                           float *y, int Cin, int Cout, int D, int H, int W, int k, int stride, int pad, int dil, int relu,
                           icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(x && w && scale && shift && y && Cin > 0 && Cout > 0 && Cout <= 8 && k > 0 && stride > 0 && dil > 0,
                   "icon_conv3d: bad argument (Cout <= 8)");
    Conv3dParams p{};
    p.x = x; p.w = w; p.scale = scale; p.shift = shift; p.res = res; p.y = y;
    p.Cin = Cin; p.Cout = Cout; p.D = D; p.H = H; p.W = W; p.k = k; p.stride = stride; p.pad = pad; p.dil = dil; p.relu = relu;
    const int ext = dil * (k - 1) + 1;
    p.OD = (D + 2 * pad - ext) / stride + 1; p.OH = (H + 2 * pad - ext) / stride + 1; p.OW = (W + 2 * pad - ext) / stride + 1;
    ICON_CHECK_ARG(p.OD > 0 && p.OH > 0 && p.OW > 0, "icon_conv3d: empty output");
    const size_t smem = (size_t)Cout * Cin * k * k * k * sizeof(float);
    ICON_CHECK_ARG(smem <= 48 * 1024, "icon_conv3d: weights do not fit shared memory");
    const int64_t n = (int64_t)p.OD * p.OH * p.OW;
    icon::k_conv3d<<<(unsigned)((n + 127) / 128), 128, smem, stream>>>(p);
    ICON_LAUNCHED();
    return ICON_OK;
}
