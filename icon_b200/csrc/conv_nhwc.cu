// Encoder convolutions: implicit GEMM on the Hopper tensor cores (wgmma) with BOTH operands staged by the TMA engine.
//
// Replaces cuDNN in the encoders (reference: lib/net/FBNet.py:216-319 GlobalGenerator / ResnetBlock,
// lib/net/HGFilters.py:49-197 + lib/net/net_util.py:258-280 HGFilter / HourGlass / ConvBlock).
//
// Activations live in HBM as NHWC, already split x = hi + lo into two fp16 tensors by the kernel that produced them
// (k_act_nhwc: normalisation + ReLU + split in one pass).  A K-chunk of the implicit GEMM is one filter tap x 64
// input channels, i.e. for a tile of BH x BW output pixels a [BH][BW][64] box of the input shifted by the tap:
// exactly one 4-D tiled TMA load (cp.async.bulk.tensor, SWIZZLE_128B) per operand half -- zero padding is the TMA's
// out-of-bounds fill, reflection padding is a halo the producer wrote, stride 2 is a space-to-depth layout the
// producer wrote (4 parity planes), a transposed convolution is 4 output phases with 1/2/2/4 taps each.  The box
// lands in shared memory as 128 rows (pixels) x 128 bytes (64 fp16), 16-byte chunks XOR-swizzled by row % 8 --
// the K-major SWIZZLE_128B operand layout of wgmma, so the MMA reads it through a descriptor with no thread
// ever touching the data.  Weights: host-packed tiles in the same layout (1-D bulk copies).
//
//   D[128 pixels][NT channels] += A_hi*B_hi + A_hi*B_lo + A_lo*B_hi      (3 f16 wgmmas per k-step, fp32 in registers)
//
//   warps 0-7   two consumer warpgroups (warpgroup g: pixels [64 g, 64 g + 64) of the tile, M = 64, N = NT), then the
//               epilogue: accumulators -> shared memory -> one column (channel) per thread walking the pixels:
//               coalesced fp32 NHWC stores (optionally into a channel slice of a wider tensor = torch.cat for free),
//               +bias, and per-(image, channel) sum / sum-of-squares for the Instance/GroupNorm that follows (fp64,
//               added with exact atomics: stats_add), so the norm needs no statistics pass.
//   warp 8      producer: 2 tensor-map loads (A hi, A lo) + 1 bulk copy (B hi|lo) per chunk, STAGES-deep ring
// Small spatial extents (the 32 x 32 ResnetBlocks) fill the machine through split-K (partials + k_splitk_nhwc).
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace icon {

struct TapDesc { int8_t dy, dx; uint8_t plane, wtap; };
constexpr int MAX_TAPS = 49;

struct ConvNhwcParams {
    const uint8_t *wt;       // [n tiles][wt_chunks] x (hi NT*128 B | lo NT*128 B)
    const float *bias;       // [Cout] or null
    float *out;              // fp32 NHWC [N][OHf][OWf][Cs], this conv writes channels [co_off, co_off + Cout)
    float *partial;          // splits > 1: [splits][N][Ht][Wt][Cout]
    double *stats;           // [N][Cout][6] (sum, sum of squares: stats_add in common.cuh) or null
    int N, Ht, Wt;           // logical output grid of this launch (per image)
    int BW, BH, tiles_x, tiles_y;
    int OHf, OWf, osy, osx, ooy, oox;     // out (y, x) = (a * osy + ooy, b * osx + oox)
    int Cs, co_off, Cout;
    int cpt;                 // 64-channel chunks per tap
    int ntaps, nplanes, wt_chunks, splits;
    TapDesc taps[MAX_TAPS];
};

constexpr int CN_THREADS = 288;

template <int NT, int STAGES>
__global__ void __launch_bounds__(CN_THREADS, NT == 64 ? 2 : 1)
k_conv_nhwc(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
            const __grid_constant__ ConvNhwcParams p) {
    using namespace wg;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t bar_full[STAGES], bar_empty[STAGES];
    constexpr uint32_t A_BYTES = 128 * 128;                   // one half (hi or lo) of the A tile
    constexpr uint32_t B_BYTES = NT * 256;                    // hi | lo
    constexpr uint32_t STAGE = 2 * A_BYTES + B_BYTES;
    constexpr int LD = NT + 8;                                // epilogue tile [128][LD] fp32 over the drained stages
    static_assert(128 * LD * 4 <= STAGES * STAGE, "epilogue tile");
    const uint32_t base = (s32(smem_raw) + 1023u) & ~1023u;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    pdl_launch_dependents();

    const int nchunks_all = p.ntaps * p.cpt;
    const int per = (nchunks_all + p.splits - 1) / p.splits;
    const int c_begin = blockIdx.z * per, c_end = min(nchunks_all, c_begin + per);
    const int nchunks = max(0, c_end - c_begin);

    int t = blockIdx.x;
    const int tx = t % p.tiles_x; t /= p.tiles_x;
    const int ty = t % p.tiles_y;
    const int n = t / p.tiles_y;
    const int x0 = tx * p.BW, y0 = ty * p.BH;

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(s32(&bar_full[s]), 1); mbar_init(s32(&bar_empty[s]), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        tma_prefetch_desc(&map_hi);
        tma_prefetch_desc(&map_lo);
    }
    __syncthreads();
    pdl_wait();                       // everything above is local set-up; the predecessor's outputs are read from here on

    if (warp == 8) {
        if (lane == 0) {
            const uint8_t *wsrc = p.wt + (size_t)blockIdx.y * p.wt_chunks * B_BYTES;
            for (int i = 0; i < nchunks; ++i) {
                const int c = c_begin + i, tap = c / p.cpt, cb = c - tap * p.cpt;
                const TapDesc td = p.taps[tap];
                const uint32_t s = i % STAGES, ph = (i / STAGES) & 1;
                mbar_wait(s32(&bar_empty[s]), ph ^ 1);
                const uint32_t full = s32(&bar_full[s]), dst = base + s * STAGE;
                mbar_expect_tx(full, STAGE);
                const int cx = x0 + td.dx, cy = y0 + td.dy, cn = n * p.nplanes + td.plane;
                tma_load_4d(dst, &map_hi, cb * 64, cx, cy, cn, full);
                tma_load_4d(dst + A_BYTES, &map_lo, cb * 64, cx, cy, cn, full);
                bulk_g2s(dst + 2 * A_BYTES, wsrc + (size_t)(td.wtap * p.cpt + cb) * B_BYTES, B_BYTES, full);
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers: mainloop
    const int g = warp >> 2;
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    for (int i = 0; i < nchunks; ++i) {
        const uint32_t s = i % STAGES, ph = (i / STAGES) & 1;
        mbar_wait(s32(&bar_full[s]), ph);
        const uint32_t sb = base + s * STAGE;
        const uint64_t ah = desc_sw128(sb + g * 8192), al = desc_sw128(sb + A_BYTES + g * 8192);
        const uint64_t bh = desc_sw128(sb + 2 * A_BYTES), bl = desc_sw128(sb + 2 * A_BYTES + NT * 128);
        fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {               // 4 x (K = 16): +32 bytes inside the 128-byte row
            mma_ss<NT>(acc, ah + 2 * ks, bh + 2 * ks, 1);
            mma_ss<NT>(acc, ah + 2 * ks, bl + 2 * ks, 1);
            mma_ss<NT>(acc, al + 2 * ks, bh + 2 * ks, 1);
        }
        commit();
        wait<1>();                                       // chunk i - 1 is complete: hand its stage back
        fence_regs(acc);
        if (i) {
            __syncwarp();
            if (lane == 0) mbar_arrive(s32(&bar_empty[(i - 1) % STAGES]));
        }
    }
    wait<0>();
    fence_regs(acc);

    // ---------------------------------------------------------------- epilogue
    // The accumulator fragment gives a thread 2 pixels x NT / 4 channels; global memory wants a warp on one pixel's
    // CHANNELS.  Both warpgroups park their fragments in shared memory (the drained stages), then every thread walks the
    // pixels of one channel: lane = channel, one coalesced 128-byte store per pixel and warp, and the per-channel sums
    // for the following norm fall out of the same walk.
    float *tile = reinterpret_cast<float *>(smem_raw + (base - s32(smem_raw)));
    bar_sync(1, 256);                                    // both warpgroups' wgmmas have drained every stage
    {
        const int rf = 64 * g + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < NT / 8; ++i) {
            *reinterpret_cast<float2 *>(tile + rf * LD + 8 * i + cq) = make_float2(acc[4 * i], acc[4 * i + 1]);
            *reinterpret_cast<float2 *>(tile + (rf + 8) * LD + 8 * i + cq) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
        }
    }
    bar_sync(1, 256);
    const int col = tid % NT, row0 = tid / NT;
    constexpr int RSTEP = 256 / NT;
    const int co = blockIdx.y * NT + col;
    if (co >= p.Cout) return;
    const bool fin = p.splits == 1;
    const int bw_shift = 31 - __clz(p.BW), bw_mask = p.BW - 1;
    const size_t split_stride = (size_t)p.N * p.Ht * p.Wt * p.Cout;
    const float bias = (fin && p.bias) ? __ldg(p.bias + co) : 0.f;
    double s1 = 0.0, s2 = 0.0;
    for (int row = row0; row < 128; row += RSTEP) {
        const int a = y0 + (row >> bw_shift), b = x0 + (row & bw_mask);
        if (a >= p.Ht || b >= p.Wt) continue;
        const float val = tile[row * LD + col] + bias;
        if (fin) {
            p.out[(((size_t)n * p.OHf + (size_t)(a * p.osy + p.ooy)) * p.OWf + (size_t)(b * p.osx + p.oox)) * p.Cs + p.co_off + co] = val;
            s1 += val; s2 = fma((double)val, (double)val, s2);
        } else {
            p.partial[(size_t)blockIdx.z * split_stride + (((size_t)n * p.Ht + a) * p.Wt + b) * p.Cout + co] = val;
        }
    }
    if (fin && p.stats) stats_add(p.stats + ((size_t)n * p.Cout + co) * 6, s1, s2);
}

// split-K finish: out = bias + sum_s partial[s] in split order (deterministic) + per-(image, channel) statistics.
// Block = 32 pixels x 128 channels, 256 threads: lane = channel quad (128-bit loads, coalesced), warp = pixel slot,
// 4 pixels per thread, every load of a thread independent.  grid (ceil(HW / 32), ceil(Cout / 128), N).
__global__ void __launch_bounds__(256) k_splitk_nhwc(const __grid_constant__ ConvNhwcParams p) {
    __shared__ double sred[2][8][128];
    pdl_launch_dependents();
    pdl_wait();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.y * 128 + lane * 4;
    const int n = blockIdx.z;
    const int64_t hw = (int64_t)p.Ht * p.Wt;
    const size_t split_stride = (size_t)p.N * hw * p.Cout;
    const bool cv = c < p.Cout;                                 // Cout % 4 == 0 is checked by the host for this kernel
    float4 bias = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cv && p.bias) bias = *reinterpret_cast<const float4 *>(p.bias + c);
    double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int64_t pix = (int64_t)blockIdx.x * 32 + k * 8 + w;
        if (!cv || pix >= hw) continue;
        const float *src = p.partial + ((size_t)n * hw + pix) * p.Cout + c;
        float4 v = bias;
        for (int s = 0; s < p.splits; ++s) {
            const float4 t = __ldcg(reinterpret_cast<const float4 *>(src + (size_t)s * split_stride));
            v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
        }
        const int a = (int)(pix / p.Wt), b = (int)(pix % p.Wt);
        *reinterpret_cast<float4 *>(p.out + (((size_t)n * p.OHf + (size_t)(a * p.osy + p.ooy)) * p.OWf + (size_t)(b * p.osx + p.oox)) * p.Cs +
                                    p.co_off + c) = v;
        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) { s1[j] += e[j]; s2[j] = fma((double)e[j], (double)e[j], s2[j]); }
    }
    if (!p.stats) return;
#pragma unroll
    for (int j = 0; j < 4; ++j) { sred[0][w][lane * 4 + j] = s1[j]; sred[1][w][lane * 4 + j] = s2[j]; }
    __syncthreads();
    const int cc = threadIdx.x, co = blockIdx.y * 128 + cc;
    if (cc < 128 && co < p.Cout) {                              // the block's 8 pixel slots in a fixed order
        double t1 = 0.0, t2 = 0.0;
        for (int k = 0; k < 8; ++k) { t1 += sred[0][k][cc]; t2 += sred[1][k][cc]; }
        stats_add(p.stats + ((size_t)n * p.Cout + co) * 6, t1, t2);
    }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// fp16 tensor, dims innermost first (elements), strides of dims 1..3 in elements; box [64][bw][bh][1], SWIZZLE_128B
static int make_map(CUtensorMap *m, const void *ptr, const int64_t dims[4], const int64_t strides[3], int bw, int bh) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return ICON_ECUDA; }
    cuuint64_t gd[4] = {(cuuint64_t)dims[0], (cuuint64_t)dims[1], (cuuint64_t)dims[2], (cuuint64_t)dims[3]};
    cuuint64_t gs[3] = {(cuuint64_t)strides[0] * 2, (cuuint64_t)strides[1] * 2, (cuuint64_t)strides[2] * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)bh, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(ptr), gd, gs, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): dims %lld %lld %lld %lld strides %lld %lld %lld box %d %d", (int)r,
                  (long long)dims[0], (long long)dims[1], (long long)dims[2], (long long)dims[3], (long long)strides[0],
                  (long long)strides[1], (long long)strides[2], bw, bh);
        return ICON_ECUDA;
    }
    return ICON_OK;
}

template <int NT, int STAGES>
static int launch_conv_nhwc(const CUtensorMap &mh, const CUtensorMap &ml, const ConvNhwcParams &p, dim3 grid,
                            cudaStream_t stream) {
    constexpr int smem = STAGES * (2 * 128 * 128 + NT * 256) + 1024;
    static bool attr_set[ICON_MAX_DEVICES] = {};
    if (device_needs_setup(attr_set))
        ICON_CUDA(cudaFuncSetAttribute(k_conv_nhwc<NT, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    ICON_CUDA(launch_pdl(k_conv_nhwc<NT, STAGES>, grid, dim3(CN_THREADS), (size_t)smem, stream, mh, ml, p));
    ICON_LAUNCHED();
    return ICON_OK;
}

}  // namespace icon

using namespace icon;

extern "C" size_t icon_conv_nhwc_workspace_bytes(int N, int Ht, int Wt, int Cout, int splits) {
    return splits > 1 ? (size_t)splits * N * Ht * Wt * Cout * sizeof(float) : 0;
}

extern "C" int icon_conv_nhwc(const void *a_hi, const void *a_lo, const int64_t *dims, const int64_t *strides,
                              const void *wt_packed, int wt_chunks, const float *bias, float *out, int OHf, int OWf, int Cs,
                              int co_off, int Cout, int N, int Ht, int Wt, int osy, int osx, int ooy, int oox, int nplanes,
                              int ntaps, const int *taps /* ntaps x (dy, dx, plane, wtap) */, int cpt, int n_tile, int splits,
                              double *stats, void *ws, size_t ws_bytes, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(a_hi && a_lo && dims && strides && wt_packed && taps, "icon_conv_nhwc: null pointer");
    ICON_CHECK_ARG(out || splits > 1, "icon_conv_nhwc: out == NULL (park the split-K partials only) needs splits > 1");
    ICON_CHECK_ARG(N > 0 && Ht > 0 && Wt > 0 && Cout > 0 && cpt > 0 && nplanes > 0, "icon_conv_nhwc: bad size");
    ICON_CHECK_ARG(ntaps >= 1 && ntaps <= MAX_TAPS, "icon_conv_nhwc: 1..%d taps", MAX_TAPS);
    ICON_CHECK_ARG(n_tile == 64 || n_tile == 128 || n_tile == 256, "icon_conv_nhwc: n_tile must be 64, 128 or 256");
    ICON_CHECK_ARG(splits >= 1 && splits <= ntaps * cpt, "icon_conv_nhwc: 1 <= splits <= chunks");
    ICON_CHECK_ARG((((uintptr_t)a_hi | (uintptr_t)a_lo | (uintptr_t)wt_packed) & 15) == 0, "icon_conv_nhwc: 16-byte alignment");
    ICON_CHECK_ARG(dims[0] % 8 == 0 && strides[0] % 8 == 0 && strides[1] % 8 == 0 && strides[2] % 8 == 0,
                   "icon_conv_nhwc: tensor-map strides must be multiples of 16 bytes");
    ICON_CHECK_ARG(co_off >= 0 && co_off + Cout <= Cs, "icon_conv_nhwc: channel slice outside the output tensor");
    ConvNhwcParams p{};
    p.wt = (const uint8_t *)wt_packed; p.bias = bias; p.out = out; p.stats = splits == 1 ? stats : nullptr;
    p.N = N; p.Ht = Ht; p.Wt = Wt;
    int bw = 1;
    while (bw < Wt && bw < 16) bw <<= 1;                       // 8 x 16 pixel tiles (taps of neighbouring tiles overlap
                                                               // in L2); narrower boxes for images under 16 wide
    p.BW = bw; p.BH = 128 / bw;
    p.tiles_x = (Wt + p.BW - 1) / p.BW; p.tiles_y = (Ht + p.BH - 1) / p.BH;
    p.OHf = OHf; p.OWf = OWf; p.osy = osy; p.osx = osx; p.ooy = ooy; p.oox = oox;
    p.Cs = Cs; p.co_off = co_off; p.Cout = Cout; p.cpt = cpt; p.ntaps = ntaps; p.nplanes = nplanes;
    p.wt_chunks = wt_chunks; p.splits = splits;
    for (int i = 0; i < ntaps; ++i) {
        p.taps[i].dy = (int8_t)taps[4 * i]; p.taps[i].dx = (int8_t)taps[4 * i + 1];
        p.taps[i].plane = (uint8_t)taps[4 * i + 2]; p.taps[i].wtap = (uint8_t)taps[4 * i + 3];
        ICON_CHECK_ARG(taps[4 * i + 2] >= 0 && taps[4 * i + 2] < nplanes && (taps[4 * i + 3] + 1) * cpt <= wt_chunks,
                       "icon_conv_nhwc: tap %d out of range", i);
    }
    ICON_CHECK_ARG(!out || ((Ht - 1) * osy + ooy < OHf && (Wt - 1) * osx + oox < OWf), "icon_conv_nhwc: output mapping outside the tensor");
    const size_t need = icon_conv_nhwc_workspace_bytes(N, Ht, Wt, Cout, splits);
    if (ws_bytes < need || (need && !ws)) { set_error("icon_conv_nhwc: workspace %zu < %zu", ws_bytes, need); return ICON_ENOSPC; }
    p.partial = splits > 1 ? (float *)ws : nullptr;
    ICON_CHECK_ARG(splits == 1 || !out || (Cout % 4 == 0 && Cs % 4 == 0 && co_off % 4 == 0 && ((uintptr_t)out & 15) == 0 &&
                                           (!bias || ((uintptr_t)bias & 15) == 0)),
                   "icon_conv_nhwc: split-K needs channel counts / offsets that are multiples of 4");
    CUtensorMap mh, ml;
    int rc = make_map(&mh, a_hi, dims, strides, p.BW, p.BH);
    if (rc) return rc;
    rc = make_map(&ml, a_lo, dims, strides, p.BW, p.BH);
    if (rc) return rc;
    dim3 grid((unsigned)(p.tiles_x * p.tiles_y * N), (unsigned)((Cout + n_tile - 1) / n_tile), (unsigned)splits);
    if (n_tile == 256) rc = launch_conv_nhwc<256, 2>(mh, ml, p, grid, stream);
    else if (n_tile == 128) rc = launch_conv_nhwc<128, 3>(mh, ml, p, grid, stream);
    else rc = launch_conv_nhwc<64, 2>(mh, ml, p, grid, stream);     // 97 KB: two CTAs per SM overlap prologue / epilogue
    if (rc) return rc;
    if (splits > 1 && out) {
        p.stats = stats;
        dim3 g2((unsigned)(((int64_t)Ht * Wt + 31) / 32), (unsigned)((Cout + 127) / 128), (unsigned)N);
        ICON_CUDA(launch_pdl(k_splitk_nhwc, g2, dim3(256), 0, stream, p));
        ICON_LAUNCHED();
    }
    return ICON_OK;
}
