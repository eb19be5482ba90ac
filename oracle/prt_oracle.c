/*
 * oracle/prt_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Brute-force any-hit ray cast of the PRT transfer (lib/renderer/prt_util.py:115-182, computePRT): every ray
 * against every face in index order until the first hit.  PARITY UNPINNED against trimesh's own ray intersector
 * (absent here); this is the checker of icon_prt's hit bits.
 *
 * any_hit_block is geom.cuh's ray_hit_tri performed with the same fp32 operations in the same order (gcc
 * -ffp-contract=off, fmaf only where written), which is what makes icon_prt's verdicts bit-exact against it.
 * The vector helpers are sdf_oracle.c's, included as mesh_oracle.c includes them.  Built into its own library by
 * oracle/prt.py.
 */
#include "sdf_oracle.c"

/* geom.cuh's ray_hit_tri over a block of faces held as structure of arrays, without early exits so that the
 * compiler can vectorise it: the same operations on the same values, so the same verdict face by face (each of
 * ray_hit_tri's early misses is a false factor here, NaN included). */
#define PRT_BLK 64
static int any_hit_block(v3 o, v3 d, const float *const t[9], int f0, int n) {
    int any = 0;
    for (int k = 0; k < n; ++k) {
        const int f = f0 + k;
        v3 a = {t[0][f], t[1][f], t[2][f]}, e1 = {t[3][f], t[4][f], t[5][f]}, e2 = {t[6][f], t[7][f], t[8][f]};
        v3 p = v3cross(d, e2);
        float det = v3dot(e1, p);
        float sg = det > 0.f ? 1.f : -1.f, ad = fabsf(det);
        v3 s = v3sub(o, a);
        float u = v3dot(s, p) * sg;
        v3 q = v3cross(s, e1);
        float v = v3dot(d, q) * sg;
        float w = v3dot(e2, q) * sg;
        any |= (det != 0.f) & (u >= 0.f) & (u <= ad) & (v >= 0.f) & (u + v <= ad) & (w > 0.f);
    }
    return any;
}

/* origins [N,3] f32 (o + delta n, already rounded), dirs [D,3] f32; verts [V,3] f32, faces [F,3] int64.
 * bits [N, ceil(D/32)]: bit d % 32 of word d / 32 = ray (origin i, direction d) meets a face. */
void oracle_prt_hits(const float *origins, int64_t N, const float *dirs, int D, const float *verts, int V,
                     const int64_t *faces, int F, uint32_t *bits) {
    (void)V;
    const int W = (D + 31) / 32;
    float *soa = (float *)malloc(sizeof(float) * 9 * (size_t)F);
    const float *t[9];
    for (int c = 0; c < 9; ++c) t[c] = soa + (size_t)c * F;
    for (int f = 0; f < F; ++f) {
        v3 a = ld3(verts + 3 * faces[3 * f]), b = ld3(verts + 3 * faces[3 * f + 1]),
           c = ld3(verts + 3 * faces[3 * f + 2]);
        v3 ab = v3sub(b, a), ac = v3sub(c, a);
        const float r[9] = {a.x, a.y, a.z, ab.x, ab.y, ab.z, ac.x, ac.y, ac.z};
        for (int k = 0; k < 9; ++k) soa[(size_t)k * F + f] = r[k];
    }
#pragma omp parallel for schedule(dynamic, 4)
    for (int64_t i = 0; i < N; ++i) {
        v3 o = ld3(origins + 3 * i);
        uint32_t *row = bits + (size_t)i * W;
        memset(row, 0, sizeof(uint32_t) * (size_t)W);
        for (int j = 0; j < D; ++j) {
            v3 d = ld3(dirs + 3 * j);
            for (int f0 = 0; f0 < F; f0 += PRT_BLK) {
                if (any_hit_block(o, d, t, f0, F - f0 < PRT_BLK ? F - f0 : PRT_BLK)) {
                    row[j >> 5] |= 1u << (j & 31);
                    break;
                }
            }
        }
    }
    free(soa);
}
