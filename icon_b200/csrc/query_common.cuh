// Shared by the two implementations of the fused gather + MLP kernel (mlp.cu: FP32 FMA,
// mlp_tc.cu: wgmma fp16x3): kernel parameters and the grid_sample restatements.
#pragma once
#include "common.cuh"

namespace icon {

struct QueryParams {
    const float4 *xyz4;      // [N] transformed xyz + in_cube
    const float *rec;        // [N][8] icon prior
    const int32_t *krank;    // [N] exclusive outlier rank (icon)
    const int8_t *signs;     // [K] sign of the k-th outlier (icon, with cmap)
    const int64_t *d_K;      // number of outliers (icon, with cmap)
    int feats;               // icon: ICON_FEAT_* mask of the smpl_feats subset (include/icon_b200.h icon_query_feats)
    const float *feat;       // [C][H][W]
    int C, H, W;
    const float *vol;        // [7][VD][VD][VD] (pamir)
    int VD;
    const float *raw;        // [c0][N] (mlp_only)
    const float *mlp;
    int c0;
    float clip;
    float *out;
    int64_t N;
};

__device__ __forceinline__ float lrelu(float x) { return x > 0.f ? x : 0.01f * x; }

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// grid_sample, bilinear, zero padding, align_corners=True; one channel plane [H][W]
__device__ __forceinline__ float bilinear(const float *__restrict__ plane, int H, int W, float x, float y) {
    float ix = ((x + 1.f) / 2.f) * (float)(W - 1);
    float iy = ((y + 1.f) / 2.f) * (float)(H - 1);
    float fx = floorf(ix), fy = floorf(iy);
    int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    float wx1 = ix - fx, wy1 = iy - fy, wx0 = (fx + 1.f) - ix, wy0 = (fy + 1.f) - iy;
    float o = 0.f;
    bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
    if (vx0 && vy0) o += __ldg(plane + (size_t)y0 * W + x0) * (wx0 * wy0);
    if (vx1 && vy0) o += __ldg(plane + (size_t)y0 * W + x1) * (wx1 * wy0);
    if (vx0 && vy1) o += __ldg(plane + (size_t)y1 * W + x0) * (wx0 * wy1);
    if (vx1 && vy1) o += __ldg(plane + (size_t)y1 * W + x1) * (wx1 * wy1);
    return o;
}

// grid_sample 5-D, trilinear, zero padding, align_corners=True; one channel volume [D][D][D]
__device__ __forceinline__ float trilinear(const float *__restrict__ v, int D, float x, float y, float z) {
    float ix = ((x + 1.f) / 2.f) * (float)(D - 1);
    float iy = ((y + 1.f) / 2.f) * (float)(D - 1);
    float iz = ((z + 1.f) / 2.f) * (float)(D - 1);
    float fx = floorf(ix), fy = floorf(iy), fz = floorf(iz);
    int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
    float tx = ix - fx, ty = iy - fy, tz = iz - fz;
    float o = 0.f;
#pragma unroll
    for (int dz = 0; dz < 2; ++dz)
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                int xx = x0 + dx, yy = y0 + dy, zz = z0 + dz;
                if (xx >= 0 && xx < D && yy >= 0 && yy < D && zz >= 0 && zz < D) {
                    float w = (dx ? tx : 1.f - tx) * (dy ? ty : 1.f - ty) * (dz ? tz : 1.f - tz);
                    o += __ldg(v + ((size_t)zz * D + yy) * D + xx) * w;
                }
            }
    return o;
}

}  // namespace icon
