/*
 * oracle/mesh_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Distance-only brute force for any triangle mesh: trimesh.proximity.closest_point as the
 * benchmark's Chamfer / P2S metric uses it (lib/dataset/Evaluator.py:219-222; no attributes, no
 * sign).  PARITY UNPINNED against trimesh itself (absent here).
 *
 * The point-triangle distance is sdf_oracle.c's tri_sqdist, included rather than restated so that
 * the SMPL oracle and this one cannot drift apart; the same arithmetic contract holds (gcc
 * -ffp-contract=off, fmaf only where written), which is what makes icon_mesh_distance bit-exact
 * against it.  Built into its own library by oracle/mesh_distance.py.
 */
#include "sdf_oracle.c"

/* points [N,3]; verts [V,3]; faces [F,3] int64.  Outputs: sqdist[N] exact squared distance,
 * face[N] first strict minimum in face order (lowest index on ties). */
void oracle_mesh_distance(const float *points, int64_t N, const float *verts, int V,
                          const int64_t *faces, int F, float *sqdist, int32_t *face_out) {
    (void)V;
    float *tri = (float *)malloc(sizeof(float) * 9 * (size_t)F);
    for (int f = 0; f < F; ++f) {
        v3 a = ld3(verts + 3 * faces[3 * f]), b = ld3(verts + 3 * faces[3 * f + 1]),
           c = ld3(verts + 3 * faces[3 * f + 2]);
        v3 ab = v3sub(b, a), ac = v3sub(c, a);
        float *t = tri + 9 * (size_t)f;
        t[0] = a.x; t[1] = a.y; t[2] = a.z; t[3] = ab.x; t[4] = ab.y; t[5] = ab.z;
        t[6] = ac.x; t[7] = ac.y; t[8] = ac.z;
    }
#pragma omp parallel for schedule(dynamic, 16)
    for (int64_t i = 0; i < N; ++i) {
        v3 p = ld3(points + 3 * i);
        float best = INFINITY; int bi = 0;
        for (int f = 0; f < F; ++f) {
            const float *t = tri + 9 * (size_t)f;
            float d = tri_sqdist(p, ld3(t), ld3(t + 3), ld3(t + 6));
            if (d < best) { best = d; bi = f; }
        }
        sqdist[i] = best;
        face_out[i] = bi;
    }
    free(tri);
}
