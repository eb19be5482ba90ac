// Implicit-GEMM conv2d / conv-transpose2d on the Hopper tensor cores (wgmma; NCHW fp32 in/out, fp32-class accuracy).
//
// Replaces cuDNN in the encoders' heavy layers (reference: lib/net/FBNet.py:216-319 GlobalGenerator /
// ResnetBlock, lib/net/HGFilters.py + lib/net/net_util.py:258-280 ConvBlock) whenever Cin % 64 == 0.
//
//   D[128 pixels][NT channels] += A[128 x 64] * B[NT x 64]^T   per 64-wide K-chunk, K = taps * Cin,
//   k = tap * Cin + ci, so a chunk is one filter tap x 64 consecutive input channels.
//
// Same numerics as the occupancy MLP (mlp_tc.cu): activations and weights are split x = hi + lo in fp16
// and every k-step issues hi*Whi + hi*Wlo + lo*Whi with fp32 accumulation in registers.
//   warps 0-7   two consumer warpgroups, warpgroup g owns pixels [64 g, 64 g + 64) of the tile: im2col gather of the
//               chunk's input values (two threads per pixel, 32 channels each; zero / reflection padding, stride,
//               transposed-conv index maps), hi/lo split, SWIZZLE_128B store into the warpgroup's rows of the A tile,
//               wgmma (M = 64, N = NT) from shared memory; afterwards the epilogue (+bias/residual/activation -> NCHW)
//               straight from the accumulator fragment.
//   warps 8-11  weight producer (one lane): bulk copies of host-packed K-major SWIZZLE_128B tiles (hi | lo), 2-stage ring.
// Small spatial extents (the 32 x 32 ResnetBlocks) are filled across SMs with split-K: partial sums go to a
// workspace and k_splitk_finish reduces them deterministically.
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace icon {

struct ConvTcParams {
    const float *x;        // [N][Cin][H][W]
    const uint8_t *wt;     // packed tiles: [n_tile][chunk] x (hi NT*128 B | lo NT*128 B)
    const float *bias;     // [Cout] or null   (applied here only when splits == 1)
    const float *res;      // residual or null (splits == 1)
    float *y;              // splits == 1: [N][Cout][OH][OW]; else partial [splits][N][Cout][OH][OW]
    int N, Cin, H, W, Cout, OH, OW, KH, KW, stride, pad, reflect, transposed, act;
    int chunks_total, splits;
};

constexpr int CT_THREADS = 384;

// grid: (pixel tiles, channel tiles, splits).  Shared memory: 2 weight stages (hi NT*128 | lo NT*128), then the A tile
// (hi 16 KB | lo 16 KB, 128 rows x 128 bytes, SWIZZLE_128B).
template <int NT>
__global__ void __launch_bounds__(CT_THREADS, 1) k_conv_tc(ConvTcParams p) {
    using namespace wg;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t bars[4];
    const uint32_t raw = s32(smem_raw), base = (raw + 1023u) & ~1023u;
    uint8_t *sm = smem_raw + (base - raw);
    constexpr uint32_t STAGE = NT * 256;
    constexpr uint32_t A_OFF = 2 * STAGE;
    enum { B_FULL0 = 0, B_FULL1, B_EMPTY0, B_EMPTY1 };
    auto BAR = [&](int i) { return s32(&bars[i]); };
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    const int chunks_per = (p.chunks_total + p.splits - 1) / p.splits;
    const int c_begin = blockIdx.z * chunks_per, c_end = min(p.chunks_total, c_begin + chunks_per);
    const int nchunks = max(0, c_end - c_begin);
    const int n0 = blockIdx.y * NT;

    if (tid == 0) {
        mbar_init(BAR(B_FULL0), 1); mbar_init(BAR(B_FULL1), 1);
        mbar_init(BAR(B_EMPTY0), 8); mbar_init(BAR(B_EMPTY1), 8);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= 8) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && lane == 0) {
            const uint8_t *src = p.wt + ((size_t)blockIdx.y * p.chunks_total + c_begin) * STAGE;
            for (int c = 0; c < nchunks; ++c) {
                const uint32_t s = c & 1, ph = (c >> 1) & 1;
                mbar_wait(BAR(B_EMPTY0 + s), ph ^ 1);
                mbar_expect_tx(BAR(B_FULL0 + s), STAGE);
                bulk_g2s(base + s * STAGE, src + (size_t)c * STAGE, STAGE, BAR(B_FULL0 + s));
            }
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");

    // ---------------------------------------------------- consumers
    const int g = warp >> 2, tw = tid & 127;
    const int r = 64 * g + (tw & 63), half = tw >> 6;            // gather: pixel r of the tile, channels [32 half, +32)
    const int64_t npix = (int64_t)p.N * p.OH * p.OW;
    const int64_t ohw = (int64_t)p.OH * p.OW;
    int pn = 0, oy = 0, ox = 0;
    const int64_t gp = (int64_t)blockIdx.x * 128 + r;
    const bool pv = gp < npix;
    if (pv) {
        pn = (int)(gp / ohw);
        const int rem = (int)(gp % ohw);
        oy = rem / p.OW; ox = rem % p.OW;
    }
    const size_t plane = (size_t)p.H * p.W;
    const float *xn = p.x + (size_t)pn * p.Cin * plane;
    const int cpt = p.Cin / 64;                          // chunks per tap
    const uint32_t a_hi = base + A_OFF, a_lo = a_hi + 16384;
    const uint64_t dah = desc_sw128(a_hi + g * 8192), dal = desc_sw128(a_lo + g * 8192);
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    for (int c = 0; c < nchunks; ++c) {
        const uint32_t s = c & 1, ph = (c >> 1) & 1;
        const int ck = c_begin + c, tap = ck / cpt, ci0 = (ck % cpt) * 64 + 32 * half;
        const int kh = tap / p.KW, kw = tap % p.KW;
        int iy, ix;
        bool ok = pv;
        if (!p.transposed) {
            iy = oy * p.stride - p.pad + kh;
            ix = ox * p.stride - p.pad + kw;
            if (p.reflect) {
                iy = iy < 0 ? -iy : (iy >= p.H ? 2 * p.H - 2 - iy : iy);
                ix = ix < 0 ? -ix : (ix >= p.W ? 2 * p.W - 2 - ix : ix);
            } else ok = ok && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
        } else {
            const int ty2 = oy + p.pad - kh, tx2 = ox + p.pad - kw;
            ok = ok && ty2 >= 0 && tx2 >= 0 && (ty2 % p.stride) == 0 && (tx2 % p.stride) == 0;
            iy = ty2 / p.stride; ix = tx2 / p.stride;
            ok = ok && iy < p.H && ix < p.W;
        }
        uint32_t hi[16], lo[16];
        if (ok) {
            const float *src = xn + (size_t)ci0 * plane + (size_t)iy * p.W + ix;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float a = __ldg(src + (size_t)(2 * j) * plane), b = __ldg(src + (size_t)(2 * j + 1) * plane);
                split2(a, b, hi[j], lo[j]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) { hi[j] = 0u; lo[j] = 0u; }
        }
        if (c) {                                          // chunk c - 1 has finished reading the A tile and its stage
            wait<0>();
            fence_regs(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(BAR(B_EMPTY0 + (s ^ 1)));
        }
        bar_sync(1 + g, 128);
#pragma unroll
        for (int q = 0; q < 4; ++q) {                     // 16-byte chunks 4 half + q of row r, XOR-swizzled by r % 8
            const uint32_t o = (uint32_t)r * 128 + (uint32_t)(((4 * half + q) ^ (r & 7)) * 16);
            *reinterpret_cast<uint4 *>(sm + A_OFF + o) = make_uint4(hi[4 * q], hi[4 * q + 1], hi[4 * q + 2], hi[4 * q + 3]);
            *reinterpret_cast<uint4 *>(sm + A_OFF + 16384 + o) = make_uint4(lo[4 * q], lo[4 * q + 1], lo[4 * q + 2], lo[4 * q + 3]);
        }
        fence_proxy_async();
        bar_sync(1 + g, 128);
        mbar_wait(BAR(B_FULL0 + s), ph);
        const uint64_t bh = desc_sw128(base + s * STAGE), bl = desc_sw128(base + s * STAGE + NT * 128);
        fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {               // 4 x (K = 16): +32 bytes inside the 128-byte row
            mma_ss<NT>(acc, dah + 2 * ks, bh + 2 * ks, 1);
            mma_ss<NT>(acc, dah + 2 * ks, bl + 2 * ks, 1);
            mma_ss<NT>(acc, dal + 2 * ks, bh + 2 * ks, 1);
        }
        commit();
    }
    wait<0>();
    fence_regs(acc);

    // ---- epilogue from the accumulator fragment: rows rf, rf + 8, columns 8 i + cq + (0, 1)
    const int rf = 64 * g + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
    float *yb = p.y + (p.splits > 1 ? (size_t)blockIdx.z * p.N * p.Cout * ohw : 0);
    const bool fin = p.splits == 1;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int64_t gq = (int64_t)blockIdx.x * 128 + rf + 8 * hr;
        if (gq >= npix) continue;
        const int qn = (int)(gq / ohw);
        const int64_t pix = gq % ohw;
#pragma unroll
        for (int i = 0; i < NT / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int co = n0 + 8 * i + cq + e;
                if (co < p.Cout) {
                    const size_t o = ((size_t)qn * p.Cout + co) * ohw + pix;
                    float v = acc[4 * i + 2 * hr + e];
                    if (fin) {
                        if (p.bias) v += __ldg(p.bias + co);
                        if (p.res) v += p.res[o];
                        if (p.act == 1) v = fmaxf(v, 0.f);
                        else if (p.act == 2) v = tanhf(v);
                    }
                    yb[o] = v;
                }
            }
        }
    }
}

// y = act(sum_s partial[s] + bias + res)
__global__ void k_splitk_finish(const float *__restrict__ part, int splits, const float *__restrict__ bias,
                                const float *__restrict__ res, float *__restrict__ y, int64_t total, int Cout,
                                int64_t ohw, int act) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += part[(size_t)s * total + i];
    if (bias) v += __ldg(bias + (int)((i / ohw) % Cout));
    if (res) v += res[i];
    if (act == 1) v = fmaxf(v, 0.f);
    else if (act == 2) v = tanhf(v);
    y[i] = v;
}

template <int NT>
static int launch_conv_tc(const ConvTcParams &p, dim3 grid, cudaStream_t stream) {
    static bool attr_set[ICON_MAX_DEVICES] = {};
    const int smem = 2 * NT * 256 + 32768 + 1024;
    if (device_needs_setup(attr_set))
        ICON_CUDA(cudaFuncSetAttribute(k_conv_tc<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_conv_tc<NT><<<grid, CT_THREADS, smem, stream>>>(p);
    ICON_LAUNCHED();
    return ICON_OK;
}

}  // namespace icon

using namespace icon;

extern "C" size_t icon_conv2d_tc_workspace_bytes(int N, int Cout, int OH, int OW, int splits) {
    return splits > 1 ? (size_t)splits * N * Cout * OH * OW * sizeof(float) : 0;
}

extern "C" int icon_conv2d_tc(const float *x, const void *wt_packed, const float *bias, const float *res, float *y,
                              int N, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad, int out_pad,
                              int reflect, int transposed, int act, int n_tile, int splits, void *ws, size_t ws_bytes,
                              icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(x && wt_packed && y && N > 0 && Cin > 0 && Cout > 0, "icon_conv2d_tc: bad argument");
    ICON_CHECK_ARG(Cin % 64 == 0, "icon_conv2d_tc: Cin=%d must be a multiple of 64 (use icon_conv2d)", Cin);
    ICON_CHECK_ARG(n_tile == 64 || n_tile == 128 || n_tile == 256, "icon_conv2d_tc: n_tile must be 64, 128 or 256");
    ICON_CHECK_ARG(splits >= 1, "icon_conv2d_tc: splits >= 1");
    ICON_CHECK_ARG(((uintptr_t)wt_packed & 15) == 0, "icon_conv2d_tc: packed weights must be 16-byte aligned");
    ConvTcParams p{};
    p.x = x; p.wt = (const uint8_t *)wt_packed; p.bias = bias; p.res = res;
    p.N = N; p.Cin = Cin; p.H = H; p.W = W; p.Cout = Cout; p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad;
    p.reflect = reflect; p.transposed = transposed; p.act = act;
    if (!transposed) { p.OH = (H + 2 * pad - KH) / stride + 1; p.OW = (W + 2 * pad - KW) / stride + 1; }
    else { p.OH = (H - 1) * stride - 2 * pad + KH + out_pad; p.OW = (W - 1) * stride - 2 * pad + KW + out_pad; }
    ICON_CHECK_ARG(p.OH > 0 && p.OW > 0, "icon_conv2d_tc: empty output");
    ICON_CHECK_ARG(!reflect || (pad < H && pad < W && !transposed), "icon_conv2d_tc: bad reflection padding");
    p.chunks_total = KH * KW * (Cin / 64);
    p.splits = splits;
    const size_t need = icon_conv2d_tc_workspace_bytes(N, Cout, p.OH, p.OW, splits);
    if (ws_bytes < need) { set_error("icon_conv2d_tc: workspace %zu < %zu", ws_bytes, need); return ICON_ENOSPC; }
    p.y = splits > 1 ? (float *)ws : y;
    const int64_t npix = (int64_t)N * p.OH * p.OW;
    dim3 grid((unsigned)((npix + 127) / 128), (unsigned)((Cout + n_tile - 1) / n_tile), (unsigned)splits);
    int rc;
    if (n_tile == 256) rc = launch_conv_tc<256>(p, grid, stream);
    else if (n_tile == 128) rc = launch_conv_tc<128>(p, grid, stream);
    else rc = launch_conv_tc<64>(p, grid, stream);
    if (rc) return rc;
    if (splits > 1) {
        const int64_t total = (int64_t)N * Cout * p.OH * p.OW;
        k_splitk_finish<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>((const float *)ws, splits, bias, res, y, total,
                                                                             Cout, (int64_t)p.OH * p.OW, act);
        ICON_LAUNCHED();
    }
    return ICON_OK;
}
