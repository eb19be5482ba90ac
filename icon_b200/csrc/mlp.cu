// Fused feature gather + occupancy MLP (FP32 FMA path).
//
// Replaces, per query point (reference):
//   geometry.index            lib/net/geometry.py:21-43   bilinear / trilinear, align_corners=True
//   feat_select               lib/dataset/mesh_util.py:266-277
//   outlier rule + cat        lib/net/HGPIFuNet.py:298-311, 335-363
//   MLP.forward               lib/net/MLP.py:49-72  (BN folded, skip-concats as extra K rows)
//   preds * in_cube           lib/net/HGPIFuNet.py:362-363
//
// One CTA = 64 points, 256 threads.  Activations never leave the SM: x0 (13->16 rows) and h1
// live in shared memory, h0 is produced 16 channels at a time straight into the K-loop of
// layer 1 and h2 stays in registers for the final dot product.  Weights stream from L2 with
// cp.async double buffering.  Algorithmic HBM traffic: 16 B xyz/in_cube + 32 B SMPL record +
// 4 B rank in, 4 B out per point (DESIGN.md "kernels").
#include "common.cuh"
#include "query_common.cuh"

namespace icon {

constexpr int MP = 64;     // points per CTA
constexpr int MT = 256;    // threads
constexpr int KC = 16;     // K rows per pipeline stage

// packed weight offsets (floats), see icon_b200.h
constexpr int OFF_W0 = 0;                       // [16][512]
constexpr int OFF_B0 = OFF_W0 + 16 * 512;       // [512]
constexpr int OFF_W1 = OFF_B0 + 512;            // [512][256]
constexpr int OFF_B1 = OFF_W1 + 512 * 256;      // [256]
constexpr int OFF_W2 = OFF_B1 + 256;            // [272][128]
constexpr int OFF_B2 = OFF_W2 + 272 * 128;      // [128]
constexpr int OFF_W3 = OFF_B2 + 128;            // [144]
constexpr int OFF_B3 = OFF_W3 + 144;            // [1]
static_assert(OFF_B3 + 1 == ICON_MLP_PACKED_FLOATS, "packed layout");

// MODE: 0 icon, 1 pifu, 2 pamir, 3 raw feature matrix
template <int MODE>
__global__ void __launch_bounds__(MT, 2) k_query_mlp(QueryParams q) {
    extern __shared__ __align__(16) float sm[];
    float *x0s = sm;                    // [16][MP]
    float *stage = sm + 16 * MP;        // 10240 floats: L1: w1c[2][KC][256] + h0c[2][KC][MP]; L2: w2c[2][KC][128]
    float *h1s = stage + 10240;         // [256][MP]
    float *w1c = stage;                 // [2][KC*256]
    float *h0c = stage + 2 * KC * 256;  // [2][KC*MP]
    float *w2c = stage;                 // [2][KC*128]
    float *red = stage + 2 * KC * 128;  // [8][MP] layer-3 partials (inside stage, free in L2/L3 phase)

    const int tid = threadIdx.x;
    const int64_t p0 = (int64_t)blockIdx.x * MP;
    const float *__restrict__ W = q.mlp;
    const int c0 = q.c0;

    // prefetch first W1 stage while features are gathered
    {
        const float4 *src = (const float4 *)(W + OFF_W1);
        for (int i = tid; i < KC * 256 / 4; i += MT) cp_async16(w1c + 4 * i, src + i);
        cp_async_commit();
    }

    // ------------------------------------------------------------ gather x0 [16][MP]
    {
        const int pl = tid & (MP - 1), grp = tid >> 6;   // 4 groups of 64 threads
        const int64_t pi = p0 + pl;
        const bool live = pi < q.N;
        if (MODE == 3) {
            for (int r = grp; r < 16; r += 4) x0s[r * MP + pl] = (live && r < c0) ? q.raw[(size_t)r * q.N + pi] : 0.f;
        } else {
            float4 xyz = live ? q.xyz4[pi] : make_float4(0.f, 0.f, 0.f, 0.f);
            if (MODE == 0) {
                // columns: L image channels, sdf, [cmap xyz], [norm xyz] (include/icon_b200.h icon_query_feats)
                const bool has_vis = q.feats & ICON_FEAT_VIS;
                const int d = has_vis ? q.C / 2 : q.C;
                float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0;
                if (live) {
                    const float4 *r = (const float4 *)(q.rec + 8 * pi);
                    r0 = r[0]; r1 = r[1];
                }
                const float vis = r1.w;
                if (grp == 0) {
                    float sdf = r0.x, cx = r0.y, cy = r0.z, cz = r0.w;
                    const bool outlier = live && fabsf(sdf) >= q.clip;
                    if (outlier) sdf = sdf > 0.f ? 1.f : -1.f;   // HGPIFuNet.py:299-302
                    int col = d;
                    x0s[col++ * MP + pl] = sdf;
                    if (q.feats & ICON_FEAT_CMAP) {
                        if (outlier) {
                            // HGPIFuNet.py:303-304: cmap[k][c] <- s[(3k+c) mod K]
                            long long K = *q.d_K;
                            long long k3 = 3ll * (long long)q.krank[pi];
                            cx = (float)q.signs[(k3) % K];
                            cy = (float)q.signs[(k3 + 1) % K];
                            cz = (float)q.signs[(k3 + 2) % K];
                        }
                        x0s[col++ * MP + pl] = cx;
                        x0s[col++ * MP + pl] = cy;
                        x0s[col++ * MP + pl] = cz;
                    }
                    if (q.feats & ICON_FEAT_NORM) {
                        x0s[col++ * MP + pl] = r1.x;
                        x0s[col++ * MP + pl] = r1.y;
                        x0s[col++ * MP + pl] = r1.z;
                    }
                    for (int r = col; r < 16; ++r) x0s[r * MP + pl] = 0.f;
                } else {
                    // feat_select: vis=1 -> channels [0,d), vis=0 -> [d,2d); without vis all C channels
                    const int base = !has_vis || vis != 0.f ? 0 : d;
                    for (int ch = grp - 1; ch < d; ch += 3) {
                        float v = live ? bilinear(q.feat + (size_t)(base + ch) * q.H * q.W, q.H, q.W, xyz.x, xyz.y) : 0.f;
                        x0s[ch * MP + pl] = v;
                    }
                }
            } else if (MODE == 1) {
                for (int ch = grp; ch < q.C; ch += 4) {
                    float v = live ? bilinear(q.feat + (size_t)ch * q.H * q.W, q.H, q.W, xyz.x, xyz.y) : 0.f;
                    x0s[ch * MP + pl] = v;
                }
                if (grp == 0) {
                    x0s[q.C * MP + pl] = live ? xyz.z : 0.f;
                    for (int r = q.C + 1; r < 16; ++r) x0s[r * MP + pl] = 0.f;
                }
            } else {
                if (grp < 3) {
                    for (int ch = grp; ch < q.C; ch += 3) {
                        float v = live ? bilinear(q.feat + (size_t)ch * q.H * q.W, q.H, q.W, xyz.x, xyz.y) : 0.f;
                        x0s[ch * MP + pl] = v;
                    }
                } else {
                    const size_t vs = (size_t)q.VD * q.VD * q.VD;
                    for (int ch = 0; ch < 7; ++ch) {
                        float v = live ? trilinear(q.vol + ch * vs, q.VD, xyz.x, xyz.y, xyz.z) : 0.f;
                        x0s[(q.C + ch) * MP + pl] = v;
                    }
                    for (int r = q.C + 7; r < 16; ++r) x0s[r * MP + pl] = 0.f;
                }
            }
        }
    }
    __syncthreads();

    // ------------------------------------------------------------ layers 0+1
    // thread tile: 8 channels (ty*8..) x 8 points ({tx*4..+3} and {32+tx*4..+3})
    const int ty = tid >> 3, tx = tid & 7;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    // h0 producer mapping: channel hc = tid>>4 (0..15) within the stage, points hp*4..+3, hp = tid&15
    const int hc = tid >> 4, hp = tid & 15;

    constexpr int NST1 = 512 / KC;
    for (int st = 0; st < NST1; ++st) {
        const int buf = st & 1;
        // produce h0 rows [st*KC, st*KC+KC) into h0c[buf]
        {
            const int ch = st * KC + hc;
            float a0 = __ldg(W + OFF_B0 + ch), a1 = a0, a2 = a0, a3 = a0;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                float w = __ldg(W + OFF_W0 + j * 512 + ch);
                float4 xv = *(const float4 *)(x0s + j * MP + hp * 4);
                a0 = fmaf(w, xv.x, a0); a1 = fmaf(w, xv.y, a1); a2 = fmaf(w, xv.z, a2); a3 = fmaf(w, xv.w, a3);
            }
            *(float4 *)(h0c + buf * KC * MP + hc * MP + hp * 4) = make_float4(lrelu(a0), lrelu(a1), lrelu(a2), lrelu(a3));
        }
        // prefetch next W1 stage
        if (st + 1 < NST1) {
            const float4 *src = (const float4 *)(W + OFF_W1 + (size_t)(st + 1) * KC * 256);
            float *dst = w1c + (buf ^ 1) * KC * 256;
            for (int i = tid; i < KC * 256 / 4; i += MT) cp_async16(dst + 4 * i, src + i);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float *wb = w1c + buf * KC * 256 + ty * 8;
        const float *hb = h0c + buf * KC * MP + tx * 4;
#pragma unroll
        for (int k = 0; k < KC; ++k) {
            float4 a0 = *(const float4 *)(wb + k * 256), a1 = *(const float4 *)(wb + k * 256 + 4);
            float4 b0 = *(const float4 *)(hb + k * MP), b1 = *(const float4 *)(hb + k * MP + 32);
            float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    // epilogue layer 1 -> h1s
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int ch = ty * 8 + i;
        const float bia = __ldg(W + OFF_B1 + ch);
        *(float4 *)(h1s + ch * MP + tx * 4) = make_float4(lrelu(acc[i][0] + bia), lrelu(acc[i][1] + bia),
                                                         lrelu(acc[i][2] + bia), lrelu(acc[i][3] + bia));
        *(float4 *)(h1s + ch * MP + 32 + tx * 4) = make_float4(lrelu(acc[i][4] + bia), lrelu(acc[i][5] + bia),
                                                              lrelu(acc[i][6] + bia), lrelu(acc[i][7] + bia));
    }
    // first W2 stage (stage buffers are free: all threads passed the last barrier of the loop)
    {
        const float4 *src = (const float4 *)(W + OFF_W2);
        for (int i = tid; i < KC * 128 / 4; i += MT) cp_async16(w2c + 4 * i, src + i);
        cp_async_commit();
    }
    __syncthreads();

    // ------------------------------------------------------------ layer 2: K = 256 (h1) + 16 (x0)
    // thread tile: 4 channels (ty*4..) x 8 points
    float acc2[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc2[i][j] = 0.f;
    constexpr int NST2 = 272 / KC;   // 17
    for (int st = 0; st < NST2; ++st) {
        const int buf = st & 1;
        if (st + 1 < NST2) {
            const float4 *src = (const float4 *)(W + OFF_W2 + (size_t)(st + 1) * KC * 128);
            float *dst = w2c + (buf ^ 1) * KC * 128;
            for (int i = tid; i < KC * 128 / 4; i += MT) cp_async16(dst + 4 * i, src + i);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float *wb = w2c + buf * KC * 128 + ty * 4;
        const float *hb = (st < 16 ? h1s + (size_t)st * KC * MP : x0s) + tx * 4;
#pragma unroll
        for (int k = 0; k < KC; ++k) {
            float4 a0 = *(const float4 *)(wb + k * 128);
            float4 b0 = *(const float4 *)(hb + k * MP), b1 = *(const float4 *)(hb + k * MP + 32);
            float a[4] = {a0.x, a0.y, a0.z, a0.w};
            float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc2[i][j] = fmaf(a[i], b[j], acc2[i][j]);
        }
        __syncthreads();
    }

    // ------------------------------------------------------------ layer 3 (128 + 16 -> 1) and output
    float part[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) part[j] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int ch = ty * 4 + i;
        const float bia = __ldg(W + OFF_B2 + ch), w3 = __ldg(W + OFF_W3 + ch);
#pragma unroll
        for (int j = 0; j < 8; ++j) part[j] = fmaf(w3, lrelu(acc2[i][j] + bia), part[j]);
    }
    // reduce over the 4 ty values inside the warp (lanes differ in bits 3,4), then over 8 warps
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        part[j] += __shfl_xor_sync(0xffffffffu, part[j], 8);
        part[j] += __shfl_xor_sync(0xffffffffu, part[j], 16);
    }
    const int lane = tid & 31, wid = tid >> 5;
    if (lane < 8) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            red[wid * MP + lane * 4 + j] = part[j];
            red[wid * MP + 32 + lane * 4 + j] = part[4 + j];
        }
    }
    __syncthreads();
    if (tid < MP) {
        const int64_t pi = p0 + tid;
        if (pi < q.N) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) s += red[w * MP + tid];
            for (int j = 0; j < 16; ++j) s = fmaf(__ldg(W + OFF_W3 + 128 + j), x0s[j * MP + tid], s);
            s += __ldg(W + OFF_B3);
            float in_cube = (MODE == 3) ? 1.f : q.xyz4[pi].w;
            q.out[pi] = in_cube * s;
        }
    }
}

// ---------------------------------------------------------------- outlier rank (icon prior)
__global__ void k_outlier_flag(const float *__restrict__ rec, int64_t N, float clip, int32_t *__restrict__ flag) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) flag[i] = fabsf(rec[8 * i]) >= clip ? 1 : 0;
}
__global__ void k_outlier_signs(const float *__restrict__ rec, int64_t N, float clip,
                                const int32_t *__restrict__ krank, int8_t *__restrict__ signs) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) {
        float s = rec[8 * i];
        if (fabsf(s) >= clip) signs[krank[i]] = s > 0.f ? 1 : -1;
    }
}

constexpr size_t MLP_SMEM = (16 * MP + 10240 + 256 * MP) * sizeof(float);

template <int MODE>
static int launch_mlp(const QueryParams &q, cudaStream_t stream) {
    static bool attr_set[ICON_MAX_DEVICES] = {};
    if (device_needs_setup(attr_set))
        ICON_CUDA(cudaFuncSetAttribute(k_query_mlp<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MLP_SMEM));
    unsigned nblk = (unsigned)((q.N + MP - 1) / MP);
    k_query_mlp<MODE><<<nblk, MT, MLP_SMEM, stream>>>(q);
    ICON_LAUNCHED();
    return ICON_OK;
}

// defined in mlp_tc.cu
int launch_mlp_tc(int mode, const QueryParams &q, const void *blob, cudaStream_t stream);
static int g_mlp_impl = 1;

template <int MODE>
static int launch_any(const QueryParams &q, const void *tc, cudaStream_t stream) {
    if (g_mlp_impl == 1) {
        if (!tc) {          // never degrade silently to the 10x slower FP32 kernel: the caller asked for the tensor cores
            set_error("icon_query / icon_mlp_only: the tensor-core MLP needs the packed tensor-core weight blob (mlp_tc == NULL); "
                      "pass it or select the FP32 kernel with icon_set_mlp_impl(0)");
            return ICON_EINVAL;
        }
        if (q.c0 > 15) {    // x0 column 15 is the constant 1 that carries the folded biases
            set_error("icon_query / icon_mlp_only: the tensor-core MLP takes c0 <= 15 input channels (got %d)", q.c0);
            return ICON_EINVAL;
        }
        return launch_mlp_tc(MODE, q, tc, stream);
    }
    return launch_mlp<MODE>(q, stream);
}

// defined in sdf.cu
size_t sdf_ws_bytes(int64_t N);
int run_sdf(const float *points, int64_t sc, int64_t sn, int64_t N, const float *h_calib, const MeshView &m,
            float *rec, int32_t *face, void *ws, float4 **xyz4_out, cudaStream_t stream);
int run_points_only(const float *points, int64_t sc, int64_t sn, int64_t N, const float *h_calib,
                    float4 *xyz4, cudaStream_t stream);

struct QueryWs {
    void *sdf_ws;
    float *rec;
    int32_t *krank;
    int8_t *signs;
    int64_t *d_K;
    void *scan_ws;
    float4 *xyz4;   // non-icon priors
};

static QueryWs carve_query(Carver &c, int64_t N, int prior) {
    QueryWs w{};
    if (prior == ICON_PRIOR_ICON) {
        w.sdf_ws = c.take<char>(sdf_ws_bytes(N));
        w.rec = c.take<float>((size_t)N * 8);
        w.krank = c.take<int32_t>((size_t)N);
        w.signs = c.take<int8_t>((size_t)N);
        w.d_K = c.take<int64_t>(1);
        w.scan_ws = c.take<char>(scan_ws_bytes(N));
    } else {
        w.xyz4 = c.take<float4>((size_t)N);
    }
    return w;
}

}  // namespace icon

using namespace icon;

extern "C" size_t icon_query_workspace_bytes(int64_t N, int F, int prior) {
    (void)F;
    Carver c(nullptr);
    carve_query(c, N, prior);
    return c.total();
}

extern "C" int icon_query(int prior, const float *points, int64_t stride_c, int64_t stride_n, int64_t N,
                          const float *h_calib, const float *feat, int C, int H, int W,
                          const float *vol_feat, int VD, const void *mesh_ws, int V, int F,
                          const float *mlp_packed, const void *mlp_tc, int c0, float sdf_clip, float *out,
                          void *ws, size_t ws_bytes, icon_stream_t stream) {
    return icon_query_feats(prior, points, stride_c, stride_n, N, h_calib, feat, C, H, W, vol_feat, VD, mesh_ws, V, F,
                            mlp_packed, mlp_tc, c0, sdf_clip, ICON_FEAT_ALL, out, ws, ws_bytes, stream);
}

extern "C" int icon_query_feats(int prior, const float *points, int64_t stride_c, int64_t stride_n, int64_t N,
                                const float *h_calib, const float *feat, int C, int H, int W,
                                const float *vol_feat, int VD, const void *mesh_ws, int V, int F,
                                const float *mlp_packed, const void *mlp_tc, int c0, float sdf_clip, int smpl_feats,
                                float *out, void *ws, size_t ws_bytes, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(N >= 0 && N < (int64_t)INT32_MAX, "icon_query: N=%lld out of range", (long long)N);
    if (N == 0) return ICON_OK;
    ICON_CHECK_ARG(points && h_calib && feat && mlp_packed && out && ws, "icon_query: null pointer");
    ICON_CHECK_ARG(((uintptr_t)mlp_tc & 15) == 0, "icon_query: mlp_tc must be 16-byte aligned");
    ICON_CHECK_ARG(c0 >= 1 && c0 <= 16, "icon_query: c0=%d unsupported (1..16)", c0);
    ICON_CHECK_ARG(H >= 2 && W >= 2, "icon_query: feature map %dx%d too small", H, W);
    {
        Carver c(nullptr);
        carve_query(c, N, prior);
        if (ws_bytes < c.total()) {
            set_error("icon_query: workspace %zu < %zu", ws_bytes, c.total());
            return ICON_ENOSPC;
        }
    }
    Carver c(ws);
    QueryWs w = carve_query(c, N, prior);
    QueryParams q{};
    q.feat = feat; q.C = C; q.H = H; q.W = W; q.vol = vol_feat; q.VD = VD;
    q.mlp = mlp_packed; q.c0 = c0; q.clip = sdf_clip; q.out = out; q.N = N;
    if (prior == ICON_PRIOR_ICON) {
        ICON_CHECK_ARG(mesh_ws && V > 0 && F > 0, "icon_query: icon prior needs a prepared body mesh");
        ICON_CHECK_ARG((smpl_feats & ~ICON_FEAT_ALL) == 0, "icon_query: smpl_feats mask %d has bits outside ICON_FEAT_ALL",
                       smpl_feats);
        const int cm = smpl_feats & ICON_FEAT_CMAP ? 1 : 0, nm = smpl_feats & ICON_FEAT_NORM ? 1 : 0;
        const bool vs = smpl_feats & ICON_FEAT_VIS;   // with vis, feat_select keeps half of the C image channels
        const int tail = 1 + 3 * cm + 3 * nm;          // sdf [, cmap xyz] [, norm xyz]
        ICON_CHECK_ARG((!vs || C % 2 == 0) && c0 == (vs ? C / 2 : C) + tail,
                       "icon_query: icon prior with smpl_feats mask %d expects c0 = %s + %d (C=%d c0=%d)", smpl_feats,
                       vs ? "C/2" : "C", tail, C, c0);
        q.feats = smpl_feats;
        MeshView m = mesh_view(mesh_ws, V, F);
        float4 *xyz4 = nullptr;
        int rc = run_sdf(points, stride_c, stride_n, N, h_calib, m, w.rec, nullptr, w.sdf_ws, &xyz4, stream);
        if (rc) return rc;
        if (cm) {
            // the cmap overwrite needs each outlier's rank over the whole call; without cmap the query is point-local
            unsigned nb = (unsigned)((N + 255) / 256);
            k_outlier_flag<<<nb, 256, 0, stream>>>(w.rec, N, sdf_clip, w.krank);
            ICON_LAUNCHED();
            rc = scan_exclusive_i32(w.krank, w.krank, N, w.d_K, w.scan_ws, stream);
            if (rc) return rc;
            k_outlier_signs<<<nb, 256, 0, stream>>>(w.rec, N, sdf_clip, w.krank, w.signs);
            ICON_LAUNCHED();
            q.krank = w.krank; q.signs = w.signs; q.d_K = w.d_K;
        }
        q.xyz4 = xyz4; q.rec = w.rec;
        profile_mark(3, stream);
        rc = launch_any<0>(q, mlp_tc, stream);
        profile_mark(4, stream);
        return rc;
    }
    profile_mark(0, stream);                         // stage timers: [0,1) point transform, [1,3) empty, [3,4) gather + MLP
    int rc = run_points_only(points, stride_c, stride_n, N, h_calib, w.xyz4, stream);
    if (rc) return rc;
    profile_mark(1, stream); profile_mark(2, stream); profile_mark(3, stream);
    q.xyz4 = w.xyz4;
    if (prior == ICON_PRIOR_PIFU) {
        ICON_CHECK_ARG(C + 1 == c0, "icon_query: pifu prior expects c0 = C + 1 (C=%d c0=%d)", C, c0);
        rc = launch_any<1>(q, mlp_tc, stream);
        profile_mark(4, stream);
        return rc;
    }
    if (prior == ICON_PRIOR_PAMIR) {
        ICON_CHECK_ARG(vol_feat && VD >= 2 && C + 7 == c0, "icon_query: pamir prior expects vol_feat and c0 = C + 7");
        rc = launch_any<2>(q, mlp_tc, stream);
        profile_mark(4, stream);
        return rc;
    }
    set_error("icon_query: unknown prior %d", prior);
    return ICON_EINVAL;
}

extern "C" int icon_set_mlp_impl(int impl) {
    ICON_CHECK_ARG(impl == 0 || impl == 1, "icon_set_mlp_impl: 0 (fp32) or 1 (tensor cores)");
    g_mlp_impl = impl;
    return ICON_OK;
}
extern "C" int icon_get_mlp_impl(void) { return g_mlp_impl; }

extern "C" int icon_mlp_only(const float *feature, int c0, int64_t N, const float *mlp_packed, const void *mlp_tc,
                             float *out, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (N == 0) return ICON_OK;
    ICON_CHECK_ARG(feature && mlp_packed && out && c0 >= 1 && c0 <= 16, "icon_mlp_only: bad argument");
    QueryParams q{};
    q.raw = feature; q.mlp = mlp_packed; q.c0 = c0; q.out = out; q.N = N;
    return launch_any<3>(q, mlp_tc, stream);
}
