// Fused feature gather + occupancy MLP on the Hopper tensor cores (wgmma, sm_90a).
//
// Same contract as mlp.cu (reference: lib/net/MLP.py:49-72, lib/net/geometry.py:21-43,
// lib/dataset/mesh_util.py:266-277, lib/net/HGPIFuNet.py:298-311, 335-363).
//
// Precision: every layer input x is split x = hi + lo with hi = fp16(x), lo = fp16(x - hi) (22
// significant bits), the BN-folded weights likewise on the host, and each layer is evaluated as
// hi*Whi + hi*Wlo + lo*Whi with fp32 accumulation -- three f16 wgmmas per k-step, fp32-class accuracy
// (parity bar 1e-4 on the logit).
//
// One persistent CTA per SM, 128 query points per tile, 384 threads (3 warpgroups):
//   warps 0-7   two consumer warpgroups, warpgroup g owns rows [64 g, 64 g + 64) of the tile.  Per tile, with the
//               tile's x0 operand (fp16 hi / lo, column 15 is the constant 1 that carries b0 and b2) taken from one of
//               two shared-memory slots: for each of layer 1's 8 K-chunks j, layer 0's outputs [64 j, 64 j + 64)
//               (wgmma from shared memory) -> LeakyReLU -> hi / lo register A fragments -> layer-1 K-chunk, N = 256,
//               A from registers.  Two fragment buffers alternate: layer 0 of chunk j + 1 is issued and converted
//               while layer 1 of chunk j runs.  Then LeakyReLU(+ b1) of the 256-wide accumulator, 64 columns at a
//               time, feeds layer 2's four K-chunks (N = 128), each slice converted while the previous chunk runs ->
//               x0 tail of layer 2 -> layer 3 (144 -> 1) as an fp32 dot over the accumulator fragment, reduced
//               across the 4 lanes that share a row.
//   warps 8-11  producer warpgroup (hands its registers to the consumers with setmaxnreg).
//               warp 8, one lane: 1-D bulk copies (cp.async.bulk, TMA engine) of host-pre-swizzled K-major SWIZZLE_128B
//               weight tiles from L2 into a 4 x 32 KB ring, mbarrier complete_tx (per tile 8 layer-1 chunks as hi / lo
//               stage pairs and 4 layer-2 chunks; layer 0, the x0 tail of layer 2 and the fp32 tail stay resident).
//               warps 9-11: the feature gather of the next tile (bilinear / trilinear samples, SMPL record, outlier
//               rule) into the free x0 slot, so it runs while the consumers compute the current one.
#include <cuda_fp16.h>

#include "common.cuh"
#include "query_common.cuh"
#include "wgmma.cuh"

namespace icon {

constexpr int TC_THREADS = 384;      // 2 consumer warpgroups + 1 producer warpgroup
constexpr int TC_M = 128;
constexpr int NSTAGE = 4;            // weight ring depth: two layer-1 chunks
constexpr int STAGE_BYTES = 32768;   // one SW128 operand: 256 rows x 64 k (layer 1, hi or lo) or 128 rows, hi | lo (layer 2)
constexpr int STAGES_PER_TILE = 20;  // 8 x 2 layer-1 + 4 layer-2; a multiple of NSTAGE, so every tile starts at stage 0
static_assert(STAGES_PER_TILE % NSTAGE == 0 && NSTAGE % 2 == 0, "layer-1 hi / lo pairs must stay on stages (2i, 2i + 1)");
constexpr int GATHER_THREADS = 96;   // warps 9-11

// byte offsets inside the packed tensor-core weight blob (host: icon_b200/ops.py pack_mlp)
constexpr int TCB_W0 = 0;                         // hi 16384 | lo 16384, no swizzle, LBO 8192, SBO 128
constexpr int TCB_W1 = 32768;                     // 8 x (hi 32768 | lo 32768), SW128, 256 rows x 64 k
constexpr int TCB_W2 = TCB_W1 + 8 * 65536;        // 4 x (hi 16384 | lo 16384), SW128, 128 rows x 64 k
constexpr int TCB_W2T = TCB_W2 + 4 * 32768;       // hi 4096 | lo 4096, no swizzle, 128 rows x 16 k
constexpr int TCB_F32 = TCB_W2T + 8192;           // b0[512] b1[256] b2[128] w3[144] b3[1] pad
constexpr int TCB_F32_FLOATS = 512 + 256 + 128 + 144 + 4;
constexpr int TCB_BYTES = TCB_F32 + TCB_F32_FLOATS * 4;
static_assert(TCB_BYTES == ICON_MLP_TC_BYTES, "blob layout");

// shared memory map (bytes from a 1024-aligned base)
constexpr int SM_STAGE = 0;                       // NSTAGE x 32768
constexpr int SM_W0 = NSTAGE * STAGE_BYTES;       // 32768
constexpr int SM_X0 = SM_W0 + 32768;              // 2 x0 slots of X0_SLOT bytes:
constexpr int X0_H = 0;                           //   4096  A tile of x0 (hi), no swizzle, LBO 2048, SBO 128
constexpr int X0_L = 4096;                        //   4096
constexpr int X0_F = 8192;                        //   [16][128] fp32 (layer 3 skip connection, row 15 = in_cube)
constexpr int X0_SLOT = 16384;
constexpr int SM_F32 = SM_X0 + 2 * X0_SLOT;       // biases etc.
constexpr int SM_W2T = (SM_F32 + TCB_F32_FLOATS * 4 + 127) / 128 * 128;   // x0 tail of layer 2 (hi 4096 | lo 4096)
constexpr int SM_BAR = SM_W2T + 8192;
constexpr int NBAR = 2 * NSTAGE + 5;
constexpr int SM_TOTAL = SM_BAR + NBAR * 8;
constexpr int TC_SMEM_BYTES = SM_TOTAL + 1024;    // slack for manual 1024-B alignment
static_assert(TC_SMEM_BYTES <= 227 * 1024, "shared memory");

enum { B_FULL0 = 0, B_EMPTY0 = NSTAGE, B_W0RDY = 2 * NSTAGE, B_XFULL0 = 2 * NSTAGE + 1, B_XEMPTY0 = 2 * NSTAGE + 3 };

// Register split of setmaxnreg.  At launch the CTA holds 168 registers x 384 threads (the __launch_bounds__ cap), and
// setmaxnreg.inc only hands out what setmaxnreg.dec returned, so 2 x 128 x CONSUMER + 128 x PRODUCER <= 168 x 384.
constexpr int REG_CONSUMER = 224, REG_PRODUCER = 56;
static_assert(2 * 128 * REG_CONSUMER + 128 * REG_PRODUCER <= 168 * TC_THREADS, "register split");

// LeakyReLU(d + bias) of 4 k-steps (64 columns) of an accumulator fragment -> hi / lo register A fragments.
// d points at the fragment of the chunk's first 8-column block; bias (or null) at the chunk's column 2 (lane % 4).
__device__ __forceinline__ void act_frag64(const float *d, const float *bias, uint32_t (&ah)[4][4], uint32_t (&al)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {            // q: (row, row + 8) x (cols 0..7, 8..15) in fragment order
            const int nb = 2 * kk + (q >> 1), e = 4 * nb + 2 * (q & 1);
            float v0 = d[e], v1 = d[e + 1];
            if (bias) { v0 += bias[8 * nb]; v1 += bias[8 * nb + 1]; }
            v0 = fmaxf(v0, 0.01f * v0); v1 = fmaxf(v1, 0.01f * v1);
            wg::split2(v0, v1, ah[kk][q], al[kk][q]);
        }
    }
}

// Gather of one point into its x0 slot: xf = the point's column of the slot's [16][128] fp32 matrix (stride TC_M).
// Columns are placed as mlp.cu and the reference do (image channels first, then the prior's own columns); columns
// c0..14 stay zero, since layer 0, the x0 tail of layer 2 and layer 3's skip connection read all of rows 0..14.  Each
// value goes to shared memory as soon as it is computed, which keeps the gather inside the producer's register budget.
template <int MODE>
__device__ __forceinline__ void gather_point(const QueryParams &q, int64_t pi, float *xf) {
#pragma unroll
    for (int j = 0; j < 15; ++j) xf[j * TC_M] = 0.f;
    float in_cube = 1.f;
    if (pi < q.N) {
        if (MODE == 3) {
            const int c0 = q.c0;
#pragma unroll
            for (int j = 0; j < 15; ++j)
                if (j < c0) xf[j * TC_M] = q.raw[(size_t)j * q.N + pi];
        } else {
            const float4 xyz = q.xyz4[pi];
            in_cube = xyz.w;
            if (MODE == 0) {
                // d image channels, then sdf [, cmap xyz] [, norm xyz] (include/icon_b200.h icon_query_feats); the host
                // checked c0 = d + 1 + 3 cmap + 3 norm <= 15, so every column written here is below 15
                const bool has_vis = q.feats & ICON_FEAT_VIS;
                const int d = has_vis ? q.C / 2 : q.C;
                const float4 *rp = (const float4 *)(q.rec + 8 * pi);
                const float4 r0 = rp[0], r1 = rp[1];
                const int fb = has_vis && r1.w == 0.f ? d : 0;   // feat_select: vis=1 front, vis=0 back; no vis: all C
                float sdf = r0.x;
                const bool outlier = fabsf(sdf) >= q.clip;
                if (outlier) sdf = sdf > 0.f ? 1.f : -1.f;       // HGPIFuNet.py:299-302
                float *col = xf + d * TC_M;                      // next SMPL column
                col[0] = sdf;
                col += TC_M;
                if (q.feats & ICON_FEAT_CMAP) {
                    float cx = r0.y, cy = r0.z, cz = r0.w;
                    if (outlier) {                               // HGPIFuNet.py:303-304
                        const long long K = *q.d_K, k3 = 3ll * (long long)q.krank[pi];
                        cx = (float)q.signs[k3 % K];
                        cy = (float)q.signs[(k3 + 1) % K];
                        cz = (float)q.signs[(k3 + 2) % K];
                    }
                    col[0] = cx; col[TC_M] = cy; col[2 * TC_M] = cz;
                    col += 3 * TC_M;
                }
                if (q.feats & ICON_FEAT_NORM) { col[0] = r1.x; col[TC_M] = r1.y; col[2 * TC_M] = r1.z; }
                if (d == 6) {                                    // icon-filter (C = 12, vis) and icon-mvp (C = 6)
#pragma unroll
                    for (int ch = 0; ch < 6; ++ch)
                        xf[ch * TC_M] = bilinear(q.feat + (size_t)(fb + ch) * q.H * q.W, q.H, q.W, xyz.x, xyz.y);
                } else {                                     // any d in 1..14 (c0 >= d + 1)
#pragma unroll
                    for (int ch = 0; ch < 14; ++ch)
                        if (ch < d) xf[ch * TC_M] = bilinear(q.feat + (size_t)(fb + ch) * q.H * q.W, q.H, q.W, xyz.x, xyz.y);
                }
            } else if (MODE == 1) {
                if (q.C == 12) {
#pragma unroll
                    for (int ch = 0; ch < 12; ++ch)
                        xf[ch * TC_M] = bilinear(q.feat + (size_t)ch * q.H * q.W, q.H, q.W, xyz.x, xyz.y);
                } else {                                     // any C in 1..14 (c0 = C + 1 <= 15)
#pragma unroll
                    for (int ch = 0; ch < 14; ++ch)
                        if (ch < q.C) xf[ch * TC_M] = bilinear(q.feat + (size_t)ch * q.H * q.W, q.H, q.W, xyz.x, xyz.y);
                }
                if (q.C < 15) xf[q.C * TC_M] = xyz.z;
            } else {
                const size_t vs = (size_t)q.VD * q.VD * q.VD;
                if (q.C == 6) {
#pragma unroll
                    for (int ch = 0; ch < 6; ++ch)
                        xf[ch * TC_M] = bilinear(q.feat + (size_t)ch * q.H * q.W, q.H, q.W, xyz.x, xyz.y);
                } else {                                     // any C in 1..8 (c0 = C + 7 <= 15)
#pragma unroll
                    for (int ch = 0; ch < 8; ++ch)
                        if (ch < q.C) xf[ch * TC_M] = bilinear(q.feat + (size_t)ch * q.H * q.W, q.H, q.W, xyz.x, xyz.y);
                }
#pragma unroll
                for (int ch = 0; ch < 7; ++ch)
                    if (q.C + ch < 15) xf[(q.C + ch) * TC_M] = trilinear(q.vol + ch * vs, q.VD, xyz.x, xyz.y, xyz.z);
            }
        }
    }
    xf[15 * TC_M] = in_cube;                             // c0 <= 15: row 15 is spare
}

template <int MODE>
__global__ void __launch_bounds__(TC_THREADS, 1) k_query_mlp_tc(QueryParams q, const uint8_t *__restrict__ blob) {
    using namespace wg;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = s32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t *sm = smem_raw + (base - raw);
    const float *sf32 = reinterpret_cast<const float *>(sm + SM_F32);
    const float *sb1 = sf32 + 512, *sw3 = sf32 + 896, *sb3 = sf32 + 1040;     // b0 [0,512) and b2 [768,896) ride in the weight tiles
    const uint32_t bar0 = base + SM_BAR;
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t ntiles = (q.N + TC_M - 1) / TC_M;

    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(BAR(B_FULL0 + s), 1); mbar_init(BAR(B_EMPTY0 + s), 8); }
        mbar_init(BAR(B_W0RDY), 1);
        for (int b = 0; b < 2; ++b) { mbar_init(BAR(B_XFULL0 + b), GATHER_THREADS); mbar_init(BAR(B_XEMPTY0 + b), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= 8) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REG_PRODUCER));
        if (warp == 8) {
            // ==================================================== weight producer
            if (lane == 0) {
                mbar_expect_tx(BAR(B_W0RDY), 32768 + TCB_F32_FLOATS * 4 + 8192);
                bulk_g2s(base + SM_W0, blob + TCB_W0, 32768, BAR(B_W0RDY));
                bulk_g2s(base + SM_F32, blob + TCB_F32, TCB_F32_FLOATS * 4, BAR(B_W0RDY));
                bulk_g2s(base + SM_W2T, blob + TCB_W2T, 8192, BAR(B_W0RDY));
                uint32_t cnt = 0;
                for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
                    // consumption order: layer-1 chunks 0..7 as (hi, lo) stage pairs, then layer-2 chunks 0..3
                    for (int i = 0; i < STAGES_PER_TILE; ++i, ++cnt) {
                        const uint32_t s = cnt % NSTAGE, ph = (cnt / NSTAGE) & 1;
                        mbar_wait(BAR(B_EMPTY0 + s), ph ^ 1);
                        const uint32_t dst = base + SM_STAGE + s * STAGE_BYTES, full = BAR(B_FULL0 + s);
                        mbar_expect_tx(full, STAGE_BYTES);
                        const uint8_t *src = i < 16 ? blob + TCB_W1 + (size_t)i * 32768 : blob + TCB_W2 + (size_t)(i - 16) * 32768;
                        bulk_g2s(dst, src, STAGE_BYTES, full);
                    }
                }
            }
        } else {
            // ==================================================== feature gather, one tile ahead of the consumers
            const int gt = tid - 9 * 32;
            for (uint32_t it = 0; blockIdx.x + (int64_t)it * gridDim.x < ntiles; ++it) {
                const int b = it & 1;
                mbar_wait(BAR(B_XEMPTY0 + b), ((it >> 1) & 1) ^ 1);
                uint8_t *xs = sm + SM_X0 + b * X0_SLOT;
                for (int r = gt; r < TC_M; r += GATHER_THREADS) {
                    float *xf = reinterpret_cast<float *>(xs + X0_F) + r;
                    gather_point<MODE>(q, (blockIdx.x + (int64_t)it * gridDim.x) * TC_M + r, xf);
                    uint32_t hi[8], lo[8];
#pragma unroll
                    for (int i = 0; i < 7; ++i) split2(xf[2 * i * TC_M], xf[(2 * i + 1) * TC_M], hi[i], lo[i]);
                    split2(xf[14 * TC_M], 1.f, hi[7], lo[7]);          // column 15 = 1: carries b0 (layer 0) and b2 (x0 tail of layer 2)
                    const int off = (r >> 3) * 128 + (r & 7) * 16;
                    *reinterpret_cast<uint4 *>(xs + X0_H + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                    *reinterpret_cast<uint4 *>(xs + X0_H + off + 2048) = make_uint4(hi[4], hi[5], hi[6], hi[7]);
                    *reinterpret_cast<uint4 *>(xs + X0_L + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                    *reinterpret_cast<uint4 *>(xs + X0_L + off + 2048) = make_uint4(lo[4], lo[5], lo[6], lo[7]);
                }
                fence_proxy_async();                 // the x0 tiles are read by wgmma (async proxy)
                mbar_arrive(BAR(B_XFULL0 + b));
            }
        }
        return;
    }

    // ============================================================ consumer warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REG_CONSUMER));
    const int g = warp >> 2;
    const int rf = 64 * g + 16 * (warp & 3) + (lane >> 2);       // fragment rows rf, rf + 8 of the tile
    const int cq = 2 * (lane & 3);                               // fragment column offset inside an 8-column block
    uint32_t cnt = 0;
    auto stage_wait = [&](uint32_t c) {
        const uint32_t s = c % NSTAGE;
        mbar_wait(BAR(B_FULL0 + s), (c / NSTAGE) & 1);
        return s;
    };
    auto warp_arrive = [&](int bar) {          // after the wgmmas / loads that read the buffer are complete
        __syncwarp();
        if (lane == 0) mbar_arrive(BAR(bar));
    };
    const uint64_t dw2th = desc_nosw(base + SM_W2T, 2048, 128), dw2tl = desc_nosw(base + SM_W2T + 4096, 2048, 128);
    mbar_wait(BAR(B_W0RDY), 0);

    uint32_t it = 0;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const int b = it & 1;
        const uint32_t xs = base + SM_X0 + b * X0_SLOT;
        const uint64_t dx0h = desc_nosw(xs + X0_H + g * 1024, 2048, 128), dx0l = desc_nosw(xs + X0_L + g * 1024, 2048, 128);
        mbar_wait(BAR(B_XFULL0 + b), (it >> 1) & 1);

        // layer 0, outputs [64 j, 64 j + 64): K = 16, one k-step; b0 rides on x0 column 15 = 1
        auto layer0 = [&](int j, float (&a0)[32]) {
            const uint64_t w0h = desc_nosw(base + SM_W0 + j * 1024, 8192, 128), w0l = w0h + (16384 >> 4);
            fence();
            mma_ss<64>(a0, dx0h, w0h, 0);
            mma_ss<64>(a0, dx0h, w0l, 1);
            mma_ss<64>(a0, dx0l, w0h, 1);
            commit();
        };
        float acc1[128];
        // layer-1 K-chunk j from fragments (ch, cl), with layer 0 of chunk j + 1 converted into (nh, nl) meanwhile.
        // On entry layer 1 of chunk j - 1, which read (nh, nl), may still run.
        auto layer1 = [&](int j, uint32_t (&ch)[4][4], uint32_t (&cl)[4][4], uint32_t (&nh)[4][4], uint32_t (&nl)[4][4]) {
            wait<0>();
            if (j) { warp_arrive(B_EMPTY0 + (cnt - 2) % NSTAGE); warp_arrive(B_EMPTY0 + (cnt - 1) % NSTAGE); }
            float a0[32];
            if (j < 7) layer0(j + 1, a0);
            const uint32_t s = stage_wait(cnt);
            stage_wait(cnt + 1);
            const uint64_t bh = desc_sw128(base + SM_STAGE + s * STAGE_BYTES), bl = bh + (STAGE_BYTES >> 4);
            fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                mma_rs<256>(acc1, ch[kk], bh + 2 * kk, (j | kk) != 0);
                mma_rs<256>(acc1, ch[kk], bl + 2 * kk, 1);
                mma_rs<256>(acc1, cl[kk], bh + 2 * kk, 1);
            }
            commit();
            cnt += 2;
            if (j < 7) {
                wait<1>();                           // layer 0 of chunk j + 1 is complete; layer 1 of chunk j runs on
                fence_regs(a0);
                act_frag64(a0, nullptr, nh, nl);
            }
        };
        uint32_t xh[4][4], xl[4][4], yh[4][4], yl[4][4];
        {
            float a0[32];
            layer0(0, a0);
            wait<0>();
            fence_regs(a0);
            act_frag64(a0, nullptr, xh, xl);
        }
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            layer1(j, xh, xl, yh, yl);
            layer1(j + 1, yh, yl, xh, xl);
        }
        wait<0>();
        fence_regs(acc1);
        warp_arrive(B_EMPTY0 + (cnt - 2) % NSTAGE);
        warp_arrive(B_EMPTY0 + (cnt - 1) % NSTAGE);

        // layer 2: K-chunk c reads LeakyReLU(acc1 + b1) of layer-1 outputs [64 c, 64 c + 64); slice c + 1 is converted
        // while chunk c runs
        float acc2[64];
        auto layer2 = [&](int c, uint32_t (&ch)[4][4], uint32_t (&cl)[4][4]) {
            const uint32_t s = stage_wait(cnt);
            const uint64_t bh = desc_sw128(base + SM_STAGE + s * STAGE_BYTES), bl = bh + (16384 >> 4);
            fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                mma_rs<128>(acc2, ch[kk], bh + 2 * kk, (c | kk) != 0);
                mma_rs<128>(acc2, ch[kk], bl + 2 * kk, 1);
                mma_rs<128>(acc2, cl[kk], bh + 2 * kk, 1);
            }
            commit();
            ++cnt;
            if (c) {                                 // chunk c - 1 is complete: its stage and fragments are free
                wait<1>();
                warp_arrive(B_EMPTY0 + (cnt - 2) % NSTAGE);
            }
        };
        act_frag64(acc1, sb1 + cq, xh, xl);
        layer2(0, xh, xl);
        act_frag64(acc1 + 32, sb1 + 64 + cq, yh, yl);
        layer2(1, yh, yl);
        act_frag64(acc1 + 64, sb1 + 128 + cq, xh, xl);
        layer2(2, xh, xl);
        act_frag64(acc1 + 96, sb1 + 192 + cq, yh, yl);
        layer2(3, yh, yl);
        // x0 tail of layer 2 (b2 through the constant-1 column)
        fence();
        mma_ss<128>(acc2, dx0h, dw2th, 1);
        mma_ss<128>(acc2, dx0h, dw2tl, 1);
        mma_ss<128>(acc2, dx0l, dw2th, 1);
        commit();
        wait<0>();
        fence_regs(acc2);
        warp_arrive(B_EMPTY0 + (cnt - 1) % NSTAGE);

        // layer 3: LeakyReLU(acc2) . w3 over this thread's 32 columns of rows rf and rf + 8, then across the quad
        const float *x0f = reinterpret_cast<const float *>(sm + (xs - base) + X0_F);
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float w0 = sw3[8 * i + cq], w1 = sw3[8 * i + cq + 1];
            float v0 = acc2[4 * i], v1 = acc2[4 * i + 1], v2 = acc2[4 * i + 2], v3 = acc2[4 * i + 3];
            v0 = fmaxf(v0, 0.01f * v0); v1 = fmaxf(v1, 0.01f * v1);
            v2 = fmaxf(v2, 0.01f * v2); v3 = fmaxf(v3, 0.01f * v3);
            s0 = fmaf(w0, v0, s0); s0 = fmaf(w1, v1, s0);
            s1 = fmaf(w0, v2, s1); s1 = fmaf(w1, v3, s1);
        }
        s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
        s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
        if ((lane & 3) < 2) {
            const int r = rf + 8 * (lane & 1);
            float s = (lane & 1) ? s1 : s0;
            const int64_t pi = tile * TC_M + r;
            if (pi < q.N) {
#pragma unroll
                for (int j = 0; j < 15; ++j) s = fmaf(sw3[128 + j], x0f[j * TC_M + r], s);    // skip connection; rows >= c0 are zero
                s += sb3[0];
                // in_cube * s as the reference computes it, signed zero included; but outside the cube the features
                // are unbounded (pifu's z, icon's normals far from the body) and can overflow the fp16 operands,
                // so a non-finite s must not turn the product into NaN there
                q.out[pi] = x0f[15 * TC_M + r] != 0.f ? s : copysignf(0.f, s);
            }
        }
        warp_arrive(B_XEMPTY0 + b);                  // layer 0, the x0 tail and layer 3 are done with this slot
    }
}

template <int MODE>
int launch_mlp_tc_t(const QueryParams &q, const void *blob, cudaStream_t stream) {
    static bool attr_set[ICON_MAX_DEVICES] = {};
    if (device_needs_setup(attr_set)) {
        ICON_CUDA(cudaFuncSetAttribute(k_query_mlp_tc<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES));
    }

    const int sms = device_sm_count();
    const int64_t ntiles = (q.N + TC_M - 1) / TC_M;
    const unsigned grid = (unsigned)(ntiles < sms ? ntiles : sms);
    k_query_mlp_tc<MODE><<<grid, TC_THREADS, TC_SMEM_BYTES, stream>>>(q, (const uint8_t *)blob);
    ICON_LAUNCHED();
    return ICON_OK;
}

int launch_mlp_tc(int mode, const QueryParams &q, const void *blob, cudaStream_t stream) {
    switch (mode) {
        case 0: return launch_mlp_tc_t<0>(q, blob, stream);
        case 1: return launch_mlp_tc_t<1>(q, blob, stream);
        case 2: return launch_mlp_tc_t<2>(q, blob, stream);
        default: return launch_mlp_tc_t<3>(q, blob, stream);
    }
}

}  // namespace icon
