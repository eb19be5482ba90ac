// Point/triangle primitives of the SMPL-body SDF block.
//
// Arithmetic contract (DESIGN.md "bit-exact geometry"): IEEE fp32, round-to-nearest, NO implicit
// contraction -- every translation unit that includes this header is compiled with
// `-fmad=false`; fused multiply-adds appear only where fmaf() is written.  The CPU oracle
// (oracle/sdf_oracle.c, gcc -ffp-contract=off) performs the same operations in the same order,
// which is what makes nearest face / sign / visibility bit-exact between the two.
//
// Replaces (reference call sites): kaolin point_to_mesh_distance (lib/dataset/mesh_util.py:374),
// kaolin check_sign (mesh_util.py:393).
#pragma once
#include <cuda_runtime.h>

namespace icon {

struct V3 {
    float x, y, z;
};
__device__ __forceinline__ V3 mk3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)); }
__device__ __forceinline__ V3 cross3(V3 a, V3 b) {
    return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

struct Tri {
    V3 a, ab, ac;
};

// per-face record: 3 x float4 = (a.xyz, ab.x) (ab.yz, ac.xy) (ac.z, 0, 0, 0)
__device__ __forceinline__ Tri load_tri(const float4 *__restrict__ rec) {
    float4 r0 = __ldg(rec), r1 = __ldg(rec + 1), r2 = __ldg(rec + 2);
    Tri t;
    t.a = mk3(r0.x, r0.y, r0.z);
    t.ab = mk3(r0.w, r1.x, r1.y);
    t.ac = mk3(r1.z, r1.w, r2.x);
    return t;
}

// Exact squared distance from p to triangle (a, a+ab, a+ac): region walk vertex A, vertex B,
// edge AB, vertex C, edge AC, edge BC, face.  Mirrors tri_sqdist() of oracle/sdf_oracle.c.
__device__ __forceinline__ float tri_sqdist(V3 p, V3 a, V3 ab, V3 ac) {
    V3 ap = sub3(p, a);
    float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
    V3 q;
    if (d1 <= 0.f && d2 <= 0.f) {
        q = ap;
    } else {
        V3 b = mk3(a.x + ab.x, a.y + ab.y, a.z + ab.z);
        V3 bp = sub3(p, b);
        float d3 = dot3(ab, bp), d4 = dot3(ac, bp);
        if (d3 >= 0.f && d4 <= d3) {
            q = bp;
        } else {
            float vc = d1 * d4 - d3 * d2;
            if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {
                float v = d1 / (d1 - d3);
                q = mk3(ap.x - v * ab.x, ap.y - v * ab.y, ap.z - v * ab.z);
            } else {
                V3 c = mk3(a.x + ac.x, a.y + ac.y, a.z + ac.z);
                V3 cp = sub3(p, c);
                float d5 = dot3(ab, cp), d6 = dot3(ac, cp);
                if (d6 >= 0.f && d5 <= d6) {
                    q = cp;
                } else {
                    float vb = d5 * d2 - d1 * d6;
                    if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {
                        float w = d2 / (d2 - d6);
                        q = mk3(ap.x - w * ac.x, ap.y - w * ac.y, ap.z - w * ac.z);
                    } else {
                        float va = d3 * d6 - d5 * d4;
                        float d43 = d4 - d3, d56 = d5 - d6;
                        if (va <= 0.f && d43 >= 0.f && d56 >= 0.f) {
                            float w = d43 / (d43 + d56);
                            q = mk3(bp.x - w * (ac.x - ab.x), bp.y - w * (ac.y - ab.y),
                                    bp.z - w * (ac.z - ab.z));
                        } else {
                            float denom = 1.0f / (va + vb + vc);
                            float v = vb * denom, w = vc * denom;
                            q = mk3(ap.x - (ab.x * v + ac.x * w), ap.y - (ab.y * v + ac.y * w),
                                    ap.z - (ab.z * v + ac.z * w));
                        }
                    }
                }
            }
        }
    }
    return dot3(q, q);
}

// +x ray from p against triangle (a, e1, e2): Moller-Trumbore with dir = (1,0,0).
// Mirrors ray_hit_px() of oracle/sdf_oracle.c.
__device__ __forceinline__ int ray_hit_px(V3 p, V3 a, V3 e1, V3 e2) {
    float det = e1.z * e2.y - e1.y * e2.z;
    if (det == 0.f) return 0;
    float inv = 1.0f / det;
    float ty = p.y - a.y, tz = p.z - a.z, tx = p.x - a.x;
    float u = (tz * e2.y - ty * e2.z) * inv;
    if (u < 0.f || u > 1.f) return 0;
    float qx = ty * e1.z - tz * e1.y;
    float v = qx * inv;
    if (v < 0.f || u + v > 1.f) return 0;
    float qy = tz * e1.x - tx * e1.z;
    float qz = tx * e1.y - ty * e1.x;
    float t = fmaf(e2.z, qz, fmaf(e2.y, qy, e2.x * qx)) * inv;
    return t > 0.f ? 1 : 0;
}

// Ray o + t d (t > 0) against triangle (a, a + e1, a + e2): Moller-Trumbore without the division, the any-hit test of
// the PRT transfer (prt.cu).  With det = e1.(d x e2), u' = s.(d x e2), v' = d.(s x e1), t' = e2.(s x e1), s = o - a,
// each taken times sign(det) (exact), the convention is:
//   * edges and vertices count as hits: u' >= 0, v' >= 0, u' + v' <= |det|  (u = u' / det, v = v' / det);
//   * the hit must lie strictly ahead of the origin: t' > 0;
//   * det == 0 (the ray parallel to the face's plane, or a zero-area face) is a miss, and so is a NaN anywhere
//     (every comparison is written so that NaN fails it).
// Mirrored face by face by any_hit_block() of oracle/prt_oracle.c.
__device__ __forceinline__ bool ray_hit_tri(V3 o, V3 d, V3 a, V3 e1, V3 e2) {
    const V3 p = cross3(d, e2);
    const float det = dot3(e1, p);
    if (det == 0.f) return false;
    const float sg = det > 0.f ? 1.f : -1.f, ad = fabsf(det);
    const V3 s = sub3(o, a);
    const float u = dot3(s, p) * sg;
    if (!(u >= 0.f && u <= ad)) return false;
    const V3 q = cross3(s, e1);
    const float v = dot3(d, q) * sg;
    if (!(v >= 0.f && u + v <= ad)) return false;
    return dot3(e2, q) * sg > 0.f;
}

}  // namespace icon
