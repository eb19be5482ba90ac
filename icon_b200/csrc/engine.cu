// Per-level kernels of the coarse-to-fine reconstruction engine.
//
// Replace the body of Seg3dLossless._forward_faster (lib/common/seg3d_lossless.py:152-265):
// two F.interpolate(trilinear) calls, the boundary test, the SmoothConv3D dilation
// (lib/common/seg3d_utils.py:169-181), the nonzero / unique / scatter_ bookkeeping and
// batch_eval's coordinate normalisation (:125-138).  All grids are [R,R,R], [z][y][x].
// These are HBM-bound byte movers: one thread per voxel, coalesced along x.
#include "common.cuh"

namespace icon {

// ---------------------------------------------------------------- upsample + boundary + carry
// torch upsample_trilinear3d with align_corners=True and R_out = 2 R_in - 1 has weights 0, 1/2, 1 only; the
// nesting is w innermost, then h, then d, and a tap with weight 0 contributes exactly 0, so skipping it keeps the
// result bit-identical:  lerp(a, b) = 0.5 a + 0.5 b on odd coordinates, a on even ones.
__device__ __forceinline__ float half_sum(float a, float b) { return __fadd_rn(__fmul_rn(0.5f, a), __fmul_rn(0.5f, b)); }

// one thread = output voxels (2i, 2i+1) of row (y, z); rows are flattened into the x grid dimension
__global__ void __launch_bounds__(256) k_grid_upsample(const float *__restrict__ in, const uint8_t *__restrict__ done_in,
                                                       int Ri, float bal, float *__restrict__ out,
                                                       uint8_t *__restrict__ boundary, uint8_t *__restrict__ done_out) {
    const int Ro = 2 * Ri - 1;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = t % Ri, y = t / Ri, z = blockIdx.y;
    if (y >= Ro) return;
    const int y0 = y >> 1, z0 = z >> 1;
    const bool oy = y & 1, oz = z & 1;
    const int i1 = min(i + 1, Ri - 1);
    const size_t RR = (size_t)Ri * Ri;
    const float *r00 = in + z0 * RR + (size_t)y0 * Ri;
    const float *r01 = r00 + (oy ? Ri : 0), *r10 = r00 + (oz ? RR : 0), *r11 = r10 + (oy ? Ri : 0);
    // taps at x index i and i+1 for the (up to) four contributing input rows
    const float a00 = r00[i], b00 = r00[i1];
    float e, o;                      // outputs at x = 2i (even) and x = 2i+1 (odd)
    bool any1, any0, any1o, any0o;   // boundary = some contributing tap above `bal` and some not
    {
        const bool pa = a00 > bal, pb = b00 > bal;
        e = a00; o = half_sum(a00, b00);
        any1 = pa; any0 = !pa; any1o = pa | pb; any0o = !pa | !pb;
    }
    if (oy) {
        const float a = r01[i], b = r01[i1];
        const bool pa = a > bal, pb = b > bal;
        e = half_sum(e, a); o = half_sum(o, half_sum(a, b));
        any1 |= pa; any0 |= !pa; any1o |= pa | pb; any0o |= !pa | !pb;
    }
    if (oz) {
        const float a = r10[i], b = r10[i1];
        bool pa = a > bal, pb = b > bal;
        float e2 = a, o2 = half_sum(a, b);
        any1 |= pa; any0 |= !pa; any1o |= pa | pb; any0o |= !pa | !pb;
        if (oy) {
            const float c = r11[i], d = r11[i1];
            pa = c > bal; pb = d > bal;
            e2 = half_sum(e2, c); o2 = half_sum(o2, half_sum(c, d));
            any1 |= pa; any0 |= !pa; any1o |= pa | pb; any0o |= !pa | !pb;
        }
        e = half_sum(e, e2); o = half_sum(o, o2);
    }
    const size_t ob = ((size_t)z * Ro + y) * Ro + 2 * i;
    const bool has_odd = 2 * i + 1 < Ro;
    out[ob] = e;
    if (has_odd) out[ob + 1] = o;
    if (boundary) {
        boundary[ob] = (any1 && any0) ? 1 : 0;
        if (has_odd) boundary[ob + 1] = (any1o && any0o) ? 1 : 0;
    }
    if (done_out) {
        uint8_t d = 0;
        if (!oy && !oz) d = done_in ? done_in[z0 * RR + (size_t)y0 * Ri + i] : 1;
        done_out[ob] = d;
        if (has_odd) done_out[ob + 1] = 0;
    }
}

// ---------------------------------------------------------------- separable box dilation
// axis 0: along x ([z][y][x] -> [z][y][x]); axis 1: along y; axis 2: along z, written as [x][y][z]
template <int AXIS>
__global__ void k_dilate(const uint8_t *__restrict__ in, int R, int rad, uint8_t *__restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y, z = blockIdx.z;
    if (x >= R) return;
    const size_t RR = (size_t)R * R;
    uint8_t any = 0;
    if (AXIS == 0) {
        const uint8_t *row = in + z * RR + (size_t)y * R;
        for (int k = max(0, x - rad); k <= min(R - 1, x + rad); ++k) any |= row[k];
        out[z * RR + (size_t)y * R + x] = any;
    } else if (AXIS == 1) {
        for (int k = max(0, y - rad); k <= min(R - 1, y + rad); ++k) any |= in[z * RR + (size_t)k * R + x];
        out[z * RR + (size_t)y * R + x] = any;
    } else {
        for (int k = max(0, z - rad); k <= min(R - 1, z + rad); ++k) any |= in[k * RR + (size_t)y * R + x];
        out[(size_t)x * RR + (size_t)y * R + z] = any;
    }
}

// ---------------------------------------------------------------- ordered compaction
__global__ void k_compact_flag(const uint8_t *__restrict__ mask_xyz, const uint8_t *__restrict__ done, int R,
                               int32_t *__restrict__ flag) {
    const int64_t n = (int64_t)R * R * R;
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // j = (x*R + y)*R + z
    if (j >= n) return;
    const int z = (int)(j % R), y = (int)((j / R) % R), x = (int)(j / ((int64_t)R * R));
    const size_t zyx = ((size_t)z * R + y) * R + x;
    flag[j] = (mask_xyz[j] && !done[zyx]) ? 1 : 0;
}

struct Box {
    float bmin[3], bmax[3];
};

// batch_eval (seg3d_lossless.py:131-138): coords.float() / (R_last-1) * (b_max-b_min) + b_min,
// elementwise torch ops -> separate roundings (no contraction)
__device__ __forceinline__ float norm_coord(float c, float denom, float lo, float hi) {
    return __fadd_rn(__fmul_rn(__fdiv_rn(c, denom), __fsub_rn(hi, lo)), lo);
}

__global__ void k_compact_write(const uint8_t *__restrict__ mask_xyz, uint8_t *__restrict__ done, int R,
                                int R_last, Box box, const int32_t *__restrict__ pos,
                                float *__restrict__ points, int64_t *__restrict__ indices, int64_t capacity) {
    const int64_t n = (int64_t)R * R * R;
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int z = (int)(j % R), y = (int)((j / R) % R), x = (int)(j / ((int64_t)R * R));
    const size_t zyx = ((size_t)z * R + y) * R + x;
    if (!(mask_xyz[j] && !done[zyx])) return;
    const int64_t p = pos[j];
    if (p >= capacity) return;
    const float stride = (float)(R_last - 1) / (float)(R - 1);
    const float den = (float)(R_last - 1);
    points[3 * p + 0] = norm_coord((float)x * stride, den, box.bmin[0], box.bmax[0]);
    points[3 * p + 1] = norm_coord((float)y * stride, den, box.bmin[1], box.bmax[1]);
    points[3 * p + 2] = norm_coord((float)z * stride, den, box.bmin[2], box.bmax[2]);
    indices[p] = (int64_t)zyx;
    done[zyx] = 1;
}

__global__ void k_scatter(float *__restrict__ occ, const int64_t *__restrict__ idx,
                          const float *__restrict__ val, int64_t n) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) occ[idx[j]] = val[j];
}

__global__ void k_init_points(int R0, int R_last, Box box, float *__restrict__ points) {
    const int64_t n = (int64_t)R0 * R0 * R0;
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // z slowest, x fastest
    if (j >= n) return;
    const int x = (int)(j % R0), y = (int)((j / R0) % R0), z = (int)(j / ((int64_t)R0 * R0));
    // create_grid3D: linspace(0, R_last-1, R0).long() -- exact multiples of the stride
    const int stride = (R_last - 1) / (R0 - 1);
    const float den = (float)(R_last - 1);
    points[3 * j + 0] = norm_coord((float)(x * stride), den, box.bmin[0], box.bmax[0]);
    points[3 * j + 1] = norm_coord((float)(y * stride), den, box.bmin[1], box.bmax[1]);
    points[3 * j + 2] = norm_coord((float)(z * stride), den, box.bmin[2], box.bmax[2]);
}

__global__ void k_count_above(const float *__restrict__ occ, int64_t n, float bal,
                              unsigned long long *__restrict__ cnt) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int c = 0;
    for (; j < n; j += (int64_t)gridDim.x * blockDim.x) c += occ[j] > bal;
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(cnt, (unsigned long long)c);
}

static Box make_box(const float *bmin, const float *bmax) {
    Box b;
    for (int i = 0; i < 3; ++i) { b.bmin[i] = bmin[i]; b.bmax[i] = bmax[i]; }
    return b;
}

}  // namespace icon

using namespace icon;

// ---------------------------------------------------------------- 4-view normal preview (Seg3dLossless.display)
// seg3d_lossless.py:497-581 (find_vertices / render_normal / display), what ICON.render_func shows during training:
// for each of the views front / left / right / back and each image column (a, b): the FIRST voxel along the view axis
// whose occupancy exceeds 0.5; its colour is the normalised backward finite difference (step 2, clamped at the border)
// of the occupancy along (a, b, c), mapped to [0, 1]; columns that hit nothing stay white.  out: uint8 [R][4 R][3].
// View v reads the volume [z][y][x] as s(a, b, c) = occ[R-1-c][b][a] (front), occ[a][b][R-1-c] (left),
// occ[a][b][c] (right), occ[c][b][a] (back) -- the reference's permute / flip chains written out.
__global__ void k_display(const float *__restrict__ occ, int R, uint8_t *__restrict__ out) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y, view = blockIdx.z;
    if (a >= R) return;
    const size_t RR = (size_t)R * R;
    auto S = [&](int aa, int bb, int cc) -> float {
        switch (view) {
            case 0: return occ[(size_t)(R - 1 - cc) * RR + (size_t)bb * R + aa];      // front
            case 1: return occ[(size_t)aa * RR + (size_t)bb * R + (R - 1 - cc)];      // left
            case 2: return occ[(size_t)aa * RR + (size_t)bb * R + cc];                // right
            default: return occ[(size_t)cc * RR + (size_t)bb * R + aa];               // back
        }
    };
    float r = 1.f, g = 1.f, bl = 1.f;
    for (int c = 0; c < R; ++c) {
        const float v1 = S(a, b, c);
        if (!(v1 > 0.5f)) continue;
        const float nx = S(max(a - 2, 0), b, c) - v1, ny = S(a, max(b - 2, 0), c) - v1, nz = S(a, b, max(c - 2, 0)) - v1;
        const float nrm = sqrtf(nx * nx + ny * ny + nz * nz);
        r = fminf(fmaxf((nx / nrm + 1.f) / 2.f, 0.f), 1.f);
        g = fminf(fmaxf((ny / nrm + 1.f) / 2.f, 0.f), 1.f);
        bl = fminf(fmaxf((nz / nrm + 1.f) / 2.f, 0.f), 1.f);
        break;
    }
    uint8_t *px = out + ((size_t)b * 4 * R + (size_t)view * R + a) * 3;
    px[0] = (uint8_t)(r * 255.0f); px[1] = (uint8_t)(g * 255.0f); px[2] = (uint8_t)(bl * 255.0f);
}

extern "C" int icon_display(const float *occ, int R, uint8_t *out, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(occ && out && R >= 3 && R <= 4096, "icon_display: bad argument (R=%d)", R);
    dim3 grid((unsigned)((R + 127) / 128), (unsigned)R, 4);
    k_display<<<grid, 128, 0, stream>>>(occ, R, out);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_grid_upsample(const float *occ_in, const uint8_t *done_in, int R_in, float balance,
                                  float *occ_out, uint8_t *boundary, uint8_t *done_out, icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(occ_in && occ_out && R_in >= 2 && R_in <= 32768, "icon_grid_upsample: bad argument (R_in=%d)", R_in);
    const int Ro = 2 * R_in - 1;
    dim3 grid((unsigned)(((int64_t)Ro * R_in + 255) / 256), Ro);
    k_grid_upsample<<<grid, 256, 0, stream>>>(occ_in, done_in, R_in, balance, occ_out, boundary, done_out);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_grid_dilate(const uint8_t *mask, int R, int k, uint8_t *tmp, uint8_t *out_xyz,
                                icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(mask && tmp && out_xyz && R >= 1 && k >= 1 && (k & 1), "icon_grid_dilate: bad argument (R=%d k=%d)", R, k);
    const int rad = (k - 1) / 2;
    dim3 grid((R + 127) / 128, R, R);
    // x pass: mask -> out_xyz (used as scratch), y pass: -> tmp, z pass: -> out_xyz transposed
    k_dilate<0><<<grid, 128, 0, stream>>>(mask, R, rad, out_xyz);
    ICON_LAUNCHED();
    k_dilate<1><<<grid, 128, 0, stream>>>(out_xyz, R, rad, tmp);
    ICON_LAUNCHED();
    k_dilate<2><<<grid, 128, 0, stream>>>(tmp, R, rad, out_xyz);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" size_t icon_compact_workspace_bytes(int R) {
    const int64_t n = (int64_t)R * R * R;
    return align_up((size_t)n * sizeof(int32_t), 256) + scan_ws_bytes(n);
}

extern "C" int icon_grid_compact(const uint8_t *mask_xyz, uint8_t *done, int R, int R_last,
                                 const float *h_bmin, const float *h_bmax, float *points, int64_t *indices,
                                 int64_t capacity, int64_t *d_count, void *ws, size_t ws_bytes,
                                 icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(mask_xyz && done && points && indices && d_count && ws && R >= 2, "icon_grid_compact: bad argument");
    if (ws_bytes < icon_compact_workspace_bytes(R)) {
        set_error("icon_grid_compact: workspace %zu < %zu", ws_bytes, icon_compact_workspace_bytes(R));
        return ICON_ENOSPC;
    }
    const int64_t n = (int64_t)R * R * R;
    int32_t *flag = (int32_t *)ws;
    void *sws = (char *)ws + align_up((size_t)n * sizeof(int32_t), 256);
    unsigned nb = (unsigned)((n + 255) / 256);
    k_compact_flag<<<nb, 256, 0, stream>>>(mask_xyz, done, R, flag);
    ICON_LAUNCHED();
    int rc = scan_exclusive_i32(flag, flag, n, d_count, sws, stream);
    if (rc) return rc;
    k_compact_write<<<nb, 256, 0, stream>>>(mask_xyz, done, R, R_last, make_box(h_bmin, h_bmax), flag, points,
                                            indices, capacity);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_grid_scatter(float *occ, const int64_t *indices, const float *values, int64_t n,
                                 icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (n == 0) return ICON_OK;
    ICON_CHECK_ARG(occ && indices && values && n > 0, "icon_grid_scatter: bad argument");
    k_scatter<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(occ, indices, values, n);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_grid_init_points(int R0, int R_last, const float *h_bmin, const float *h_bmax, float *points,
                                     icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(points && R0 >= 2 && R_last >= R0 && (R_last - 1) % (R0 - 1) == 0,
                   "icon_grid_init_points: resolutions %d / %d not nested", R0, R_last);
    const int64_t n = (int64_t)R0 * R0 * R0;
    k_init_points<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(R0, R_last, make_box(h_bmin, h_bmax), points);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" int icon_grid_count_above(const float *occ, int64_t n, float balance, int64_t *d_count,
                                     icon_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(occ && d_count && n >= 0, "icon_grid_count_above: bad argument");
    ICON_CUDA(cudaMemsetAsync(d_count, 0, sizeof(int64_t), stream));
    if (n == 0) return ICON_OK;
    unsigned nb = (unsigned)min((int64_t)device_sm_count() * 8, (n + 255) / 256);
    k_count_above<<<nb, 256, 0, stream>>>(occ, n, balance, (unsigned long long *)d_count);
    ICON_LAUNCHED();
    return ICON_OK;
}
