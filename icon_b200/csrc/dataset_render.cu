// Views of the dataset renderer: replaces lib.renderer.gl.prt_render.PRTRender (shaders prt.vs / prt.fs, 16x MSAA)
// and lib.renderer.gl.color_render.ColorRender (color.vs / color.fs, no MSAA) as scripts/render_single.py drives
// them.  The reference needs an OpenGL context; this does not.
//
// PARITY UNPINNED: the GL implementation is not a dependency of this project, and what GL leaves to the
// implementation (MSAA sample positions, the resolve, glGenerateMipmap's filter, the LOD approximation, texture-filter
// precision, depth-buffer width) is fixed here as this file's rules.  They are restated operation for operation by
// oracle/dataset_render.py and the images are compared bit for bit (hence -fmad=false).  All arithmetic is fp32 in the
// order written, except the two transcendental steps marked fp64 below.
//
// Inputs as GL receives them.  Attributes are float64 on the host (GL_DOUBLE) and rounded to fp32 once; so are the
// uniforms NormMat, RotMat, ModelMat, PerspMat and SHCoeffs.  Every attribute is indexed per face corner c = 3 f + k
// by its own index array, as set_mesh does: position by faces, normal by faces_nml, uv by faces_uvs, PRT by faces_prt
// (PRTRender); position, colour and normal by faces (ColorRender).  A face with an index outside its array, a
// non-finite vertex or one outside the exact range is not drawn.
//
// Vertex stage (prt.vs / color.vs), per corner.  A 4x4 product row is ((m0 x + m1 y) + m2 z) + m3 w, a 3x3 row
// (m0 x + m1 y) + m2 z; the host forms the uniform products MP = PerspMat ModelMat and R = mat3(ModelMat) RotMat
// entry by entry with those sums (GLSL evaluates PerspMat * ModelMat * v left to right):
//   pos = NormMat (p, 1); q = RotMat pos; g = MP (q, 1); orthographic only: g.w = 1 (the host checks PerspMat's last
//   row is (0, 0, 0, 1)), so z_ndc = g.z.  Normal R n.  PRT: p0 kept, band 1 = OptRotateBand1(p1..p3, R), band 2 =
//   OptRotateBand2(p4..p8, R), restated with GLSL's column-major indexing (R[i][j] = column i, row j) and copy-in /
//   copy-out parameters (the output does not alias the input).
// Viewport, snapping, coverage, depth (raster.cuh; normal_render.cu's rules, generalised to S samples per pixel):
//   x_w = g.x (W/2) + W/2, y_w likewise, snapped to 1/256 pixel; z_w = (z_ndc + 1) 0.5.  S = 1 (ColorRender) samples
//   the pixel centre; S = 16 (PRTRender(ms_rate=16)) samples 256 p + 128 + 16 d for the 16 offsets d of DR_PATTERN
//   (the D3D11 standard 16-sample pattern, in 1/16 pixel: all distinct, all inside the pixel).  Per sample: exact int64
//   edge functions with the top-left rule, depth from that sample's barycentrics, 24-bit GL_LESS on
//   rint(z_w (2^24 - 1)), then the lowest face index: a 64-bit atomicMin of (q << 32 | face) per sample.  Front and
//   back views differ only by Camera's near / far.
// Shading, once per (pixel, face), at the pixel centre (GL 3.3 MSAA without sample shading, no `centroid`): the
//   barycentrics l_k = float(E_k) / float(2 area) of the centre, extrapolated when it lies outside the face; every
//   sample of the face takes that one result.  An attribute interpolates as (l0 a0 + l1 a1) + l2 a2.
//   Attachment 1: n = interpolated normal, r = sqrt((n.x n.x + n.y n.y) + n.z n.z), (n / r + 1) 0.5, alpha 1; r == 0
//   gives rgb 0.5 (normal_render.cu's rule).  Attachment 2: (z, z, z, 1), z = interpolated z_ndc.
//   Attachment 0, ColorRender: (interpolated colour, 1), unclamped.
//   Attachment 0, PRTRender (analytic off, no normal map): s_c = sum over k = 0..8 of p_k SH[k][c], accumulated from 0
//   in k order; gamma g_c = fp32(pow(fp64 s_c, fp64(1.0f / 2.2f))) for s_c >= 0 and 0 for s_c < 0 (GLSL's pow is
//   undefined there; 0 is what clamp gives a NaN with IEEE fmax); rgb = min(max(albedo_c g_c, 0), 1), alpha 1.
// Albedo (set_albedo): level 0 = the image flipped vertically, texel u8 / 255.f, alpha 1.  Levels 1-3: size
//   max(1, floor(w / 2)) x max(1, floor(h / 2)); texel (i, j) = (a + b + c + d + 2) >> 2 of sources (2i + di, 2j + dj),
//   di, dj in {0, 1}, each clamped to the previous level's last column / row (an odd size drops its last column / row).
//   Level of detail, constant per face (orthographic): g_k = d l_k / d x_w = float(-dy_k 256) / float(2 area) (and
//   dx_k for y), du/dx = ((u0 gx0 + u1 gx1) + u2 gx2) w0, dv/dx likewise with h0, rho = max(sqrt(du/dx^2 + dv/dx^2),
//   sqrt(du/dy^2 + dv/dy^2)) in level-0 texels, lambda = fp32(log2(fp64 rho)).  lambda > 0 (minification,
//   LINEAR_MIPMAP_LINEAR): lc = min(lambda, 3), d = floor(lc); d == 3 samples level 3, else lerp(T_d, T_d+1, lc - d);
//   otherwise (magnification, also NaN) LINEAR on level 0.  Bilinear T_L at uv: x = u w_L - 0.5 clamped to
//   [-1, w_L] (IEEE fmin / fmax), i = floor(x), a = x - i, columns i and i + 1 clamped to [0, w_L - 1] (CLAMP_TO_EDGE),
//   rows likewise; lerp(lerp(t00, t10, a), lerp(t01, t11, a), b) with lerp(p, q, a) = p + a (q - p).  Without an
//   albedo map the albedo is 1.
// Resolve: each attachment is the mean of its S samples, summed in sample order from +0 and then times 1 / S;
//   background samples add the clear colour (0, 0, 0, 0).  No clamp (GL_CLAMP_* off) but where the shader clamps.
// Output [3][H][W][4] f32, attachments 0-2 in get_color's layout (row 0 at the top).
#include "raster.cuh"

namespace icon {

constexpr int DR_SMALL = 256;                // faces with at most this many (pixel, sample) pairs: one thread each
constexpr int DR_BIG_BLOCKS = 1024;

// D3D11 standard 16-sample pattern, in 1/16 pixel from the pixel centre
__constant__ signed char DR_PATTERN[16][2] = {{1, 1},   {-1, -3}, {-3, 2},  {4, -1},  {-5, -2}, {2, 5},
                                              {5, 3},   {3, -5},  {-2, 6},  {0, -7},  {-4, -6}, {-6, 4},
                                              {-8, 0},  {7, -4},  {6, 7},   {-7, -8}};
constexpr int DR_LO16 = 128 - 8 * 16, DR_HI16 = 128 + 7 * 16;   // sample span in a pixel, 1/256 units

struct DrView {
    float norm[12], rot[9], mp[12], r[9], sh[27];
};

__device__ __forceinline__ float dr_row3(const float *m, float x, float y, float z) { return (m[0] * x + m[1] * y) + m[2] * z; }
__device__ __forceinline__ bool dr_in(int64_t i, int n) { return i >= 0 && i < n; }

// OptRotateBand1 / OptRotateBand2 of prt.vs; G(i, j) = GLSL R[i][j] = column i, row j of the row-major r
#define G(i, j) r[3 * (j) + (i)]
__device__ __forceinline__ void dr_band1(const float *r, const float x[3], float d[3]) {
    d[0] = (G(1, 1) * x[0] + (-G(1, 2)) * x[1]) + G(1, 0) * x[2];
    d[1] = ((-G(2, 1)) * x[0] + G(2, 2) * x[1]) + (-G(2, 0)) * x[2];
    d[2] = (G(0, 1) * x[0] + (-G(0, 2)) * x[1]) + G(0, 0) * x[2];
}

__device__ __forceinline__ void dr_band2(const float *r, const float x[5], float dst[5]) {
    const float s_c3 = 0.94617469575f, s_c4 = -0.31539156525f, s_c5 = 0.54627421529f;
    const float s_c_scale = 1.0f / 0.91529123286551084f, s_c_scale_inv = 0.91529123286551084f;
    const float s_rc2 = 1.5853309190550713f * s_c_scale;
    const float s_c4_div_c3 = s_c4 / s_c3, s_c4_div_c3_x2 = (s_c4 / s_c3) * 2.0f;
    const float s_scale_dst2 = s_c3 * s_c_scale_inv, s_scale_dst4 = s_c5 * s_c_scale_inv;
    const float sh0 = ((x[3] + x[4]) + x[4]) - x[1];
    const float sh1 = ((x[0] + s_rc2 * x[2]) + x[3]) + x[4];
    const float sh2 = x[0], sh3 = -x[3], sh4 = -x[1];
    const float r2x = G(0, 0) + G(0, 1), r2y = G(1, 0) + G(1, 1), r2z = G(2, 0) + G(2, 1);
    const float r3x = G(0, 0) + G(0, 2), r3y = G(1, 0) + G(1, 2), r3z = G(2, 0) + G(2, 2);
    const float r4x = G(0, 1) + G(0, 2), r4y = G(1, 1) + G(1, 2), r4z = G(2, 1) + G(2, 2);
    const float sh0_x = sh0 * G(0, 0), sh0_y = sh0 * G(1, 0);
    float d0 = sh0_x * G(1, 0);
    float d1 = sh0_y * G(2, 0);
    float d2 = sh0 * (G(2, 0) * G(2, 0) + s_c4_div_c3);
    float d3 = sh0_x * G(2, 0);
    float d4 = sh0_x * G(0, 0) - sh0_y * G(1, 0);
    const float sh1_x = sh1 * G(0, 2), sh1_y = sh1 * G(1, 2);
    d0 += sh1_x * G(1, 2);
    d1 += sh1_y * G(2, 2);
    d2 += sh1 * (G(2, 2) * G(2, 2) + s_c4_div_c3);
    d3 += sh1_x * G(2, 2);
    d4 += sh1_x * G(0, 2) - sh1_y * G(1, 2);
    const float sh2_x = sh2 * r2x, sh2_y = sh2 * r2y;
    d0 += sh2_x * r2y;
    d1 += sh2_y * r2z;
    d2 += sh2 * (r2z * r2z + s_c4_div_c3_x2);
    d3 += sh2_x * r2z;
    d4 += sh2_x * r2x - sh2_y * r2y;
    const float sh3_x = sh3 * r3x, sh3_y = sh3 * r3y;
    d0 += sh3_x * r3y;
    d1 += sh3_y * r3z;
    d2 += sh3 * (r3z * r3z + s_c4_div_c3_x2);
    d3 += sh3_x * r3z;
    d4 += sh3_x * r3x - sh3_y * r3y;
    const float sh4_x = sh4 * r4x, sh4_y = sh4 * r4y;
    d0 += sh4_x * r4y;
    d1 += sh4_y * r4z;
    d2 += sh4 * (r4z * r4z + s_c4_div_c3_x2);
    d3 += sh4_x * r4z;
    d4 += sh4_x * r4x - sh4_y * r4y;
    dst[0] = d0;
    dst[1] = -d1;
    dst[2] = d2 * s_scale_dst2;
    dst[3] = -d3;
    dst[4] = d4 * s_scale_dst4;
}
#undef G

// per corner: the raster record and the attributes (z_ndc, n.xyz) (u, v, a0, a1) (a2..a5) (a6, a7, a8, -), a = the
// rotated PRT (PRTRender) or the colour in a0..a2 (ColorRender)
__global__ void k_dr_vertex(icon_dr_mesh m, DrView vw, int W, int H, int4 *__restrict__ vrec,
                            float4 *__restrict__ cattr) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= 3 * (int64_t)m.F) return;
    const int64_t ip = m.f_pos[c], in = m.f_nrm[c], ia = m.f_attr[c];
    const bool textured = m.tex != nullptr;
    const int64_t iu = textured ? m.f_uv[c] : 0;
    if (!dr_in(ip, m.V) || !dr_in(in, m.Vn) || !dr_in(ia, m.Va) || (textured && !dr_in(iu, m.Vt))) {
        vrec[c] = make_int4(0, 0, 0, 0);
        return;
    }
    const float *p = m.pos + 3 * ip;
    const float px = dr_row3(vw.norm, p[0], p[1], p[2]) + vw.norm[3];
    const float py = dr_row3(vw.norm + 4, p[0], p[1], p[2]) + vw.norm[7];
    const float pz = dr_row3(vw.norm + 8, p[0], p[1], p[2]) + vw.norm[11];
    const float qx = dr_row3(vw.rot, px, py, pz), qy = dr_row3(vw.rot + 3, px, py, pz), qz = dr_row3(vw.rot + 6, px, py, pz);
    const float gx = dr_row3(vw.mp, qx, qy, qz) + vw.mp[3], gy = dr_row3(vw.mp + 4, qx, qy, qz) + vw.mp[7];
    const float gz = dr_row3(vw.mp + 8, qx, qy, qz) + vw.mp[11];
    const float hw = (float)W * 0.5f, hh = (float)H * 0.5f;
    const float xw = gx * hw + hw, yw = gy * hh + hh;
    const float zw = (gz + 1.f) * 0.5f;
    const int ok = fabsf(xw) <= RS_RANGE && fabsf(yw) <= RS_RANGE && isfinite(zw);
    vrec[c] = make_int4(ok ? (int)rintf(xw * 256.f) : 0, ok ? (int)rintf(yw * 256.f) : 0, __float_as_int(zw), ok);
    const float *n = m.nrm + 3 * in;
    float4 *o = cattr + 4 * c;
    o[0] = make_float4(gz, dr_row3(vw.r, n[0], n[1], n[2]), dr_row3(vw.r + 3, n[0], n[1], n[2]),
                       dr_row3(vw.r + 6, n[0], n[1], n[2]));
    const float u = textured ? m.uv[2 * iu] : 0.f, v = textured ? m.uv[2 * iu + 1] : 0.f;
    if (m.mode == ICON_DR_PRT) {
        const float *a = m.attr + 9 * ia;
        const float x1[3] = {a[1], a[2], a[3]}, x2[5] = {a[4], a[5], a[6], a[7], a[8]};
        float b1[3], b2[5];
        dr_band1(vw.r, x1, b1);
        dr_band2(vw.r, x2, b2);
        o[1] = make_float4(u, v, a[0], b1[0]);
        o[2] = make_float4(b1[1], b1[2], b2[0], b2[1]);
        o[3] = make_float4(b2[2], b2[3], b2[4], 0.f);
    } else {
        const float *a = m.attr + 3 * ia;
        o[1] = make_float4(u, v, a[0], a[1]);
        o[2] = make_float4(a[2], 0.f, 0.f, 0.f);
        o[3] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

__device__ __forceinline__ void dr_span(int S, int &lo, int &hi) {
    lo = S == 1 ? 128 : DR_LO16;
    hi = S == 1 ? 128 : DR_HI16;
}

__device__ __forceinline__ bool dr_tri(const int4 *__restrict__ vrec, int f, int W, int H, int S, RsTri &t,
                                       float zw[3]) {
    int4 r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        r[k] = vrec[3 * (int64_t)f + k];
        zw[k] = __int_as_float(r[k].z);
    }
    int lo, hi;
    dr_span(S, lo, hi);
    return rs_setup(r, W, H, lo, hi, t);
}

// sample s of pixel (px, py)
__device__ __forceinline__ void dr_fragment(const RsTri &t, const float zw[3], int f, int px, int py, int s, int W, int S,
                                            unsigned long long *__restrict__ zbuf) {
    const int Px = px * 256 + 128 + (S == 1 ? 0 : 16 * DR_PATTERN[s][0]);
    const int Py = py * 256 + 128 + (S == 1 ? 0 : 16 * DR_PATTERN[s][1]);
    long long e[3];
    if (!rs_cover(t, Px, Py, e)) return;
    float l[3];
    rs_weights(t, e, l);
    const float z = (l[0] * zw[0] + l[1] * zw[1]) + l[2] * zw[2];
    unsigned long long key;
    if (rs_depth_key(z, f, key)) atomicMin(&zbuf[((size_t)py * W + px) * S + s], key);
}

__global__ void k_dr_small(int F, const int4 *__restrict__ vrec, int W, int H, int S,
                           unsigned long long *__restrict__ zbuf, int32_t *__restrict__ big, int32_t *__restrict__ nbig) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    RsTri t;
    float zw[3];
    if (!dr_tri(vrec, f, W, H, S, t, zw)) return;
    const int nx = t.bx1 - t.bx0 + 1, ny = t.by1 - t.by0 + 1;
    if ((long long)nx * ny * S > DR_SMALL) {
        big[atomicAdd(nbig, 1)] = f;
        return;
    }
    for (int py = t.by0; py <= t.by1; ++py)
        for (int px = t.bx0; px <= t.bx1; ++px)
            for (int s = 0; s < S; ++s) dr_fragment(t, zw, f, px, py, s, W, S, zbuf);
}

__global__ void __launch_bounds__(256) k_dr_big(const int4 *__restrict__ vrec, int W, int H, int S,
                                                unsigned long long *__restrict__ zbuf, const int32_t *__restrict__ big,
                                                const int32_t *__restrict__ nbig) {
    const int n = *nbig;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const int f = big[i];
        RsTri t;
        float zw[3];
        if (!dr_tri(vrec, f, W, H, S, t, zw)) continue;
        const int nx = t.bx1 - t.bx0 + 1;
        const long long np = (long long)nx * (t.by1 - t.by0 + 1) * S;
        for (long long q = threadIdx.x; q < np; q += blockDim.x) {
            const long long p = q / S;
            dr_fragment(t, zw, f, t.bx0 + (int)(p % nx), t.by0 + (int)(p / nx), (int)(q % S), W, S, zbuf);
        }
    }
}

// ---------------------------------------------------------------- albedo texture

struct DrTex {
    const uchar4 *t;
    int w, h;
};

__host__ __device__ __forceinline__ void dr_level(int w0, int h0, int L, int &w, int &h, int64_t &off) {
    w = w0; h = h0; off = 0;
    for (int i = 0; i < L; ++i) {
        off += (int64_t)w * h;
        w = w > 1 ? w >> 1 : 1;
        h = h > 1 ? h >> 1 : 1;
    }
}

__device__ __forceinline__ float dr_lerp(float p, float q, float a) { return p + a * (q - p); }

__device__ __forceinline__ float3 dr_texel(const uchar4 *t, int w, int i, int j) {
    const uchar4 c = t[(int64_t)j * w + i];
    return make_float3((float)c.x / 255.f, (float)c.y / 255.f, (float)c.z / 255.f);
}

__device__ float3 dr_bilinear(const DrTex &tx, int L, float u, float v) {
    int w, h;
    int64_t off;
    dr_level(tx.w, tx.h, L, w, h, off);
    const uchar4 *t = tx.t + off;
    const float x = fminf(fmaxf(u * (float)w - 0.5f, -1.f), (float)w), y = fminf(fmaxf(v * (float)h - 0.5f, -1.f), (float)h);
    const float xf = floorf(x), yf = floorf(y);
    const float a = x - xf, b = y - yf;
    const int i0 = min(max((int)xf, 0), w - 1), i1 = min(max((int)xf + 1, 0), w - 1);
    const int j0 = min(max((int)yf, 0), h - 1), j1 = min(max((int)yf + 1, 0), h - 1);
    const float3 t00 = dr_texel(t, w, i0, j0), t10 = dr_texel(t, w, i1, j0);
    const float3 t01 = dr_texel(t, w, i0, j1), t11 = dr_texel(t, w, i1, j1);
    return make_float3(dr_lerp(dr_lerp(t00.x, t10.x, a), dr_lerp(t01.x, t11.x, a), b),
                       dr_lerp(dr_lerp(t00.y, t10.y, a), dr_lerp(t01.y, t11.y, a), b),
                       dr_lerp(dr_lerp(t00.z, t10.z, a), dr_lerp(t01.z, t11.z, a), b));
}

__device__ float3 dr_trilinear(const DrTex &tx, float lambda, float u, float v) {
    if (!(lambda > 0.f)) return dr_bilinear(tx, 0, u, v);
    const float lc = fminf(lambda, 3.f), d = floorf(lc);
    if (d >= 3.f) return dr_bilinear(tx, 3, u, v);
    const float fr = lc - d;
    const float3 c1 = dr_bilinear(tx, (int)d, u, v), c2 = dr_bilinear(tx, (int)d + 1, u, v);
    return make_float3(dr_lerp(c1.x, c2.x, fr), dr_lerp(c1.y, c2.y, fr), dr_lerp(c1.z, c2.z, fr));
}

// level 0: the image flipped vertically, RGBA with alpha 255
__global__ void k_dr_tex0(const uint8_t *__restrict__ rgb, int w, int h, uchar4 *__restrict__ t) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)w * h) return;
    const int i = (int)(p % w), j = (int)(p / w);
    const uint8_t *s = rgb + 3 * ((int64_t)(h - 1 - j) * w + i);
    t[p] = make_uchar4(s[0], s[1], s[2], 255);
}

// level L + 1 from level L: 2x2 box, sources clamped to the last column / row, rounded half up
__global__ void k_dr_mip(const uchar4 *__restrict__ src, int ws, int hs, uchar4 *__restrict__ dst, int wd, int hd) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)wd * hd) return;
    const int i = (int)(p % wd), j = (int)(p / wd);
    const int x0 = min(2 * i, ws - 1), x1 = min(2 * i + 1, ws - 1), y0 = min(2 * j, hs - 1), y1 = min(2 * j + 1, hs - 1);
    const uchar4 a = src[(int64_t)y0 * ws + x0], b = src[(int64_t)y0 * ws + x1];
    const uchar4 c = src[(int64_t)y1 * ws + x0], d = src[(int64_t)y1 * ws + x1];
    dst[p] = make_uchar4((a.x + b.x + c.x + d.x + 2) >> 2, (a.y + b.y + c.y + d.y + 2) >> 2,
                         (a.z + b.z + c.z + d.z + 2) >> 2, 255);
}

// ---------------------------------------------------------------- shading and resolve

struct DrShade {
    float4 a0, a1, a2;
};

__device__ __forceinline__ float dr_interp(const float l[3], float a, float b, float c) { return (l[0] * a + l[1] * b) + l[2] * c; }

__device__ DrShade dr_shade(const icon_dr_mesh &m, const DrView &vw, const int4 *__restrict__ vrec,
                            const float4 *__restrict__ cattr, int f, int px, int py, int W, int H, int S) {
    RsTri t;
    float zw[3];
    dr_tri(vrec, f, W, H, S, t, zw);                       // succeeded in the raster pass
    long long ei[3], e[3];
    rs_edges(t, px * 256 + 128, py * 256 + 128, ei);       // the centre, covered or not
    rs_orig(t, ei, e);
    float l[3];
    rs_weights(t, e, l);
    const float4 *c0 = cattr + 12 * (int64_t)f, *c1 = c0 + 4, *c2 = c0 + 8;
    DrShade o;
    const float z = dr_interp(l, c0[0].x, c1[0].x, c2[0].x);
    o.a2 = make_float4(z, z, z, 1.f);
    const float nx = dr_interp(l, c0[0].y, c1[0].y, c2[0].y), ny = dr_interp(l, c0[0].z, c1[0].z, c2[0].z);
    const float nz = dr_interp(l, c0[0].w, c1[0].w, c2[0].w);
    const float r = sqrtf((nx * nx + ny * ny) + nz * nz);
    o.a1 = r == 0.f ? make_float4(0.5f, 0.5f, 0.5f, 1.f)
                    : make_float4((nx / r + 1.f) * 0.5f, (ny / r + 1.f) * 0.5f, (nz / r + 1.f) * 0.5f, 1.f);
    if (m.mode != ICON_DR_PRT) {
        o.a0 = make_float4(dr_interp(l, c0[1].z, c1[1].z, c2[1].z), dr_interp(l, c0[1].w, c1[1].w, c2[1].w),
                           dr_interp(l, c0[2].x, c1[2].x, c2[2].x), 1.f);
        return o;
    }
    float p[9];
    p[0] = dr_interp(l, c0[1].z, c1[1].z, c2[1].z);
    p[1] = dr_interp(l, c0[1].w, c1[1].w, c2[1].w);
    p[2] = dr_interp(l, c0[2].x, c1[2].x, c2[2].x);
    p[3] = dr_interp(l, c0[2].y, c1[2].y, c2[2].y);
    p[4] = dr_interp(l, c0[2].z, c1[2].z, c2[2].z);
    p[5] = dr_interp(l, c0[2].w, c1[2].w, c2[2].w);
    p[6] = dr_interp(l, c0[3].x, c1[3].x, c2[3].x);
    p[7] = dr_interp(l, c0[3].y, c1[3].y, c2[3].y);
    p[8] = dr_interp(l, c0[3].z, c1[3].z, c2[3].z);
    float g[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 9; ++k) s = s + p[k] * vw.sh[3 * k + ch];
        g[ch] = s >= 0.f ? (float)pow((double)s, (double)(1.0f / 2.2f)) : 0.f;
    }
    float3 alb = make_float3(1.f, 1.f, 1.f);
    if (m.tex) {
        // level of detail from the face's screen-space uv derivatives (constant per face)
        long long exi[3], eyi[3], ex[3], ey[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int a = (k + 1) % 3, b = (k + 2) % 3;
            exi[k] = -(long long)(t.Y[b] - t.Y[a]) * 256;
            eyi[k] = (long long)(t.X[b] - t.X[a]) * 256;
        }
        rs_orig(t, exi, ex);
        rs_orig(t, eyi, ey);
        float gx[3], gy[3];
        rs_weights(t, ex, gx);
        rs_weights(t, ey, gy);
        const float fw = (float)m.tex_w, fh = (float)m.tex_h;
        const float us[3] = {c0[1].x, c1[1].x, c2[1].x}, vs[3] = {c0[1].y, c1[1].y, c2[1].y};
        const float dudx = dr_interp(gx, us[0], us[1], us[2]) * fw, dvdx = dr_interp(gx, vs[0], vs[1], vs[2]) * fh;
        const float dudy = dr_interp(gy, us[0], us[1], us[2]) * fw, dvdy = dr_interp(gy, vs[0], vs[1], vs[2]) * fh;
        const float rho = fmaxf(sqrtf(dudx * dudx + dvdx * dvdx), sqrtf(dudy * dudy + dvdy * dvdy));
        const float lambda = (float)log2((double)rho);
        const float u = dr_interp(l, us[0], us[1], us[2]), v = dr_interp(l, vs[0], vs[1], vs[2]);
        DrTex tx{(const uchar4 *)m.tex, m.tex_w, m.tex_h};
        alb = dr_trilinear(tx, lambda, u, v);
    }
    o.a0 = make_float4(fminf(fmaxf(alb.x * g[0], 0.f), 1.f), fminf(fmaxf(alb.y * g[1], 0.f), 1.f),
                       fminf(fmaxf(alb.z * g[2], 0.f), 1.f), 1.f);
    return o;
}

__device__ __forceinline__ void dr_add(float4 &a, const float4 &b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ float4 dr_scale(const float4 &a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }

// one thread per pixel: the distinct faces of its samples are shaded once each (a two-entry cache; shading is
// deterministic, so the cache only saves work) and the samples are averaged in sample order
__global__ void k_dr_resolve(icon_dr_mesh m, DrView vw, const unsigned long long *__restrict__ zbuf,
                             const int4 *__restrict__ vrec, const float4 *__restrict__ cattr, int W, int H, int S,
                             float4 *__restrict__ out) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)W * H) return;
    const int px = (int)(p % W), py = (int)(p / W);
    float4 acc[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) acc[a] = make_float4(0.f, 0.f, 0.f, 0.f);
    int cf0 = -1, cf1 = -1, next = 0;
    DrShade cs0, cs1;
    for (int s = 0; s < S; ++s) {
        const unsigned long long key = zbuf[p * S + s];
        if (key == RS_EMPTY) continue;
        const int f = (int)(key & 0xffffffffull);
        if (f != cf0 && f != cf1) {
            const DrShade o = dr_shade(m, vw, vrec, cattr, f, px, py, W, H, S);
            if (next) { cf1 = f; cs1 = o; } else { cf0 = f; cs0 = o; }
            next ^= 1;
        }
        const DrShade &o = f == cf0 ? cs0 : cs1;
        dr_add(acc[0], o.a0);
        dr_add(acc[1], o.a1);
        dr_add(acc[2], o.a2);
    }
    const float inv = 1.f / (float)S;
    const int64_t o = (int64_t)(H - 1 - py) * W + px;          // get_color flips the rows
    const int64_t plane = (int64_t)W * H;
#pragma unroll
    for (int a = 0; a < 3; ++a) out[a * plane + o] = dr_scale(acc[a], inv);
}

struct DrWs {
    unsigned long long *zbuf;
    int4 *vrec;
    float4 *cattr;
    int32_t *big, *nbig;
};

static size_t dr_carve(void *ws, int F, int W, int H, int S, DrWs *o) {
    Carver c(ws);
    DrWs w;
    w.zbuf = c.take<unsigned long long>((size_t)W * H * S);
    w.vrec = c.take<int4>((size_t)3 * F);
    w.cattr = c.take<float4>((size_t)12 * F);
    w.big = c.take<int32_t>((size_t)F);
    w.nbig = c.take<int32_t>(1);
    if (o) *o = w;
    return c.total();
}

static bool dr_sizes_ok(int F, int W, int H, int S) {
    return F > 0 && F <= (1 << 29) && W > 0 && H > 0 && W <= 16384 && H <= 16384 && (S == 1 || S == 16);
}

}  // namespace icon

extern "C" size_t icon_dataset_render_workspace_bytes(int F, int width, int height, int samples) {
    if (!icon::dr_sizes_ok(F, width, height, samples)) return 0;
    return icon::dr_carve(nullptr, F, width, height, samples, nullptr);
}

extern "C" int icon_dataset_render(const icon_dr_mesh *mesh, const float *h_view, int width, int height, int samples,
                                   float *out, void *ws, size_t ws_bytes, icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(mesh && h_view && out && ws, "icon_dataset_render: null pointer");
    const icon_dr_mesh &m = *mesh;
    ICON_CHECK_ARG(dr_sizes_ok(m.F, width, height, samples),
                   "icon_dataset_render: bad sizes F=%d %dx%d samples=%d (samples must be 1 or 16)", m.F, width, height,
                   samples);
    ICON_CHECK_ARG(m.mode == ICON_DR_PRT || m.mode == ICON_DR_COLOR, "icon_dataset_render: bad mode %d", m.mode);
    ICON_CHECK_ARG(m.pos && m.nrm && m.attr && m.f_pos && m.f_nrm && m.f_attr && m.V > 0 && m.Vn > 0 && m.Va > 0,
                   "icon_dataset_render: missing mesh arrays");
    ICON_CHECK_ARG(!m.tex || (m.mode == ICON_DR_PRT && m.uv && m.f_uv && m.Vt > 0 && m.tex_w > 0 && m.tex_h > 0 &&
                              m.tex_w <= 65536 && m.tex_h <= 65536),
                   "icon_dataset_render: a texture needs PRT mode, uvs and a size in [1, 65536]");
    ICON_CHECK_ARG(ws_bytes >= icon_dataset_render_workspace_bytes(m.F, width, height, samples),
                   "icon_dataset_render: workspace too small");
    DrWs w;
    dr_carve(ws, m.F, width, height, samples, &w);
    DrView vw;
    float *dst = (float *)&vw;
    for (int k = 0; k < (int)(sizeof(DrView) / sizeof(float)); ++k) dst[k] = h_view[k];
    const int64_t npix = (int64_t)width * height;
    const int64_t nc = 3 * (int64_t)m.F;
    ICON_CUDA(cudaMemsetAsync(w.zbuf, 0xff, (size_t)npix * samples * sizeof(unsigned long long), stream));
    ICON_CUDA(cudaMemsetAsync(w.nbig, 0, sizeof(int32_t), stream));
    k_dr_vertex<<<(unsigned)((nc + 255) / 256), 256, 0, stream>>>(m, vw, width, height, w.vrec, w.cattr);
    ICON_LAUNCHED();
    k_dr_small<<<(unsigned)((m.F + 255) / 256), 256, 0, stream>>>(m.F, w.vrec, width, height, samples, w.zbuf, w.big,
                                                                    w.nbig);
    ICON_LAUNCHED();
    k_dr_big<<<DR_BIG_BLOCKS, 256, 0, stream>>>(w.vrec, width, height, samples, w.zbuf, w.big, w.nbig);
    ICON_LAUNCHED();
    k_dr_resolve<<<(unsigned)((npix + 127) / 128), 128, 0, stream>>>(m, vw, w.zbuf, w.vrec, w.cattr, width, height,
                                                                       samples, (float4 *)out);
    ICON_LAUNCHED();
    return ICON_OK;
}

extern "C" size_t icon_dataset_texture_bytes(int w, int h) {
    if (w <= 0 || h <= 0 || w > 65536 || h > 65536) return 0;
    int wl, hl;
    int64_t off;
    icon::dr_level(w, h, 4, wl, hl, off);
    return (size_t)off * 4;
}

extern "C" int icon_dataset_texture(const uint8_t *rgb, int w, int h, uint8_t *tex, size_t tex_bytes,
                                    icon_stream_t stream_) {
    using namespace icon;
    cudaStream_t stream = (cudaStream_t)stream_;
    ICON_CHECK_ARG(rgb && tex, "icon_dataset_texture: null pointer");
    ICON_CHECK_ARG(w > 0 && h > 0 && w <= 65536 && h <= 65536, "icon_dataset_texture: bad size %dx%d", w, h);
    ICON_CHECK_ARG(tex_bytes >= icon_dataset_texture_bytes(w, h), "icon_dataset_texture: buffer too small");
    uchar4 *t = (uchar4 *)tex;
    const int64_t n0 = (int64_t)w * h;
    k_dr_tex0<<<(unsigned)((n0 + 255) / 256), 256, 0, stream>>>(rgb, w, h, t);
    ICON_LAUNCHED();
    for (int L = 0; L < 3; ++L) {
        int ws, hs, wd, hd;
        int64_t os, od;
        dr_level(w, h, L, ws, hs, os);
        dr_level(w, h, L + 1, wd, hd, od);
        const int64_t n = (int64_t)wd * hd;
        k_dr_mip<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(t + os, ws, hs, t + od, wd, hd);
        ICON_LAUNCHED();
    }
    return ICON_OK;
}
