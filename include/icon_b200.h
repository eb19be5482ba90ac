/*
 * icon_b200.h -- C ABI of libicon_b200.so (sm_90a kernels for ICON's occupancy-query +
 * mesh-extraction hot path).
 *
 * The reference (YuliangXiu/ICON) has no FFI: its "plugin API" for this path is Python
 * nn.Module duck typing (SURVEY.md 8b).  The Python mirror in icon_b200/ (re-exported under
 * the reference's import paths in lib/) keeps those signatures and calls the entry points
 * below through ctypes with raw device pointers.  Each entry point cites the reference
 * code it replaces.  Conventions:
 *
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless named h_*;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing
 *     synchronises unless stated;
 *   - no hidden allocation: the caller (torch's caching allocator) provides outputs and
 *     workspaces; *_workspace_bytes() tell how much;
 *   - return 0 on success, a negative ICON_E* code otherwise; icon_last_error() gives the
 *     message (thread local).  There is no CPU fallback anywhere.
 */
#ifndef ICON_B200_H
#define ICON_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ICON_OK 0
#define ICON_EINVAL (-1)   /* bad argument / unsupported size */
#define ICON_ECUDA (-2)    /* CUDA runtime error (message has the cudaError string) */
#define ICON_ENOSPC (-3)   /* workspace or output buffer too small */

#define ICON_PRIOR_ICON 0
#define ICON_PRIOR_PIFU 1
#define ICON_PRIOR_PAMIR 2

typedef void *icon_stream_t;

int icon_version(void);
const char *icon_last_error(void);
/* Number of kernel launches issued by this library since load (bench.py's gpu_launches). */
int64_t icon_launch_count(void);

/* Measurement hook (bench.py roofline): when enabled, icon_query records CUDA events on its
 * stream around its stages; icon_profile_last_query synchronises on the last one and returns
 * the stage durations of the most recent icon_query in milliseconds:
 * h_ms[0] binning+sort, [1] SDF brick kernel, [2] outlier rank (empty without cmap), [3] gather+MLP kernel. */
int icon_profile_enable(int on);
int icon_profile_last_query(float *h_ms);

/* ------------------------------------------------------------------ SMPL body preparation
 * Replaces the per-call preamble of cal_sdf_batch, lib/dataset/mesh_util.py:367-372:
 * pytorch3d Meshes.verts_normals_padded (area-weighted vertex normals, deterministic
 * sequential-index_add order) and the four face_vertices gathers
 * (lib/common/render_utils.py:149-163).  Builds, into `mesh_ws`, the face tree (Morton-sorted
 * records and bounding spheres, AABB levels), per-face records (a, ab, ac), per-face attribute
 * records (normals, cmap, vis at the three corners) and the +x-ray culling boxes.  Done once per
 * body, not once per query.
 * verts [V,3] f32, faces [F,3] i64, cmap [V,3] f32, vis [V] f32 (0/1). */
size_t icon_smpl_workspace_bytes(int V, int F);
int icon_smpl_prepare(const float *verts, const int64_t *faces, const float *cmap,
                      const float *vis, int V, int F, void *mesh_ws, size_t mesh_ws_bytes,
                      icon_stream_t stream);

/* ------------------------------------------------------------------ occupancy MLP weights
 * Replaces MLP.__init__/forward's per-layer Conv1d + BatchNorm1d(eval) (lib/net/MLP.py:26-72):
 * the host folds BN into the 1x1 convs and packs the layers; this copies nothing, it only
 * describes the packed device buffer so the kernels can check it.
 * Packed layout (floats): W0t [16][512] | b0 [512] | W1t [512][256] | b1 [256] |
 *                         W2t [272][128] | b2 [128] | W3 [144] | b3 [1]
 * with k-major ("t") storage, the c0 input channels zero-padded to 16, and skip-concat
 * columns ordered [y | x0]. */
#define ICON_MLP_PACKED_FLOATS (16 * 512 + 512 + 512 * 256 + 256 + 272 * 128 + 128 + 144 + 1)
/* Tensor-core form of the same folded weights (host: icon_b200/ops.py pack_mlp): every matrix
 * split W = hi + lo in fp16 and stored as ready-to-use K-major wgmma tiles (bytes):
 *   W0  hi 16384 | lo 16384    512 rows x 16 k, no swizzle (LBO 8192, SBO 128); k = 15 holds b0: the kernel feeds
 *                              x0 column 15 = 1, so the tensor-core path takes c0 <= 15
 *   W1  8 x (hi 32768 | lo 32768)   256 rows x 64 k per chunk, SWIZZLE_128B
 *   W2  4 x (hi 16384 | lo 16384)   128 rows x 64 k per chunk, SWIZZLE_128B
 *   W2t hi 4096 | lo 4096      128 rows x 16 k (the skip-concat x0 columns), no swizzle; k = 15 holds b2
 *   f32 b0[512] b1[256] b2[128] w3[144] b3[1] pad[3] */
#define ICON_MLP_TC_BYTES (32768 + 8 * 65536 + 4 * 32768 + 8192 + (512 + 256 + 128 + 144 + 4) * 4)
/* 0 = FP32 FMA kernel (mlp.cu), 1 = wgmma fp16x3 kernel (mlp_tc.cu, default when mlp_tc != NULL) */
int icon_set_mlp_impl(int impl);
int icon_get_mlp_impl(void);

/* ------------------------------------------------------------------ fused occupancy query
 * Replaces HGPIFuNet.query (lib/net/HGPIFuNet.py:268-367) + cal_sdf_batch
 * (lib/dataset/mesh_util.py:357-396; kaolin point_to_mesh_distance / check_sign) +
 * geometry.index / orthogonal (lib/net/geometry.py:21-61) + feat_select
 * (mesh_util.py:266-277) + MLP.forward (lib/net/MLP.py:49-72) for one feature stack, B=1.
 *
 *   points      : xyz of point i at points[c*stride_c + i*stride_n], c in 0..2
 *   calib       : HOST pointer to 12 floats, rows of [R|t] (calibs[0,:3,:4])
 *   feat        : image feature map [C,H,W] f32 (C = 12 or 6 for icon, 12 pifu, 6 pamir)
 *   vol_feat    : pamir only: [7,D,D,D] f32; else NULL
 *   mesh_ws     : icon only: workspace filled by icon_smpl_prepare (same V,F); else NULL
 *   mlp_packed  : ICON_MLP_PACKED_FLOATS floats
 *   mlp_tc      : ICON_MLP_TC_BYTES bytes (16-byte aligned) or NULL (-> FP32 kernel)
 *   c0          : MLP input channels (13 or 10 for the icon prior's full smpl_feats; see icon_query_feats)
 *   sdf_clip    : cfg.sdf_clip/100 (icon)
 *   out         : [N] f32 occupancy (preds[0,0,:])
 *   ws          : scratch, icon_query_workspace_bytes(N, F) bytes
 */
size_t icon_query_workspace_bytes(int64_t N, int F, int prior);
int icon_query(int prior, const float *points, int64_t stride_c, int64_t stride_n, int64_t N,
               const float *h_calib, const float *feat, int C, int H, int W,
               const float *vol_feat, int VD, const void *mesh_ws, int V, int F,
               const float *mlp_packed, const void *mlp_tc, int c0, float sdf_clip, float *out,
               void *ws, size_t ws_bytes, icon_stream_t stream);

/* icon_query for any `smpl_feats` subset of the icon prior (HGPIFuNet.py:97-104, 298-346).  smpl_feats is a bitmask
 * of the ICON_FEAT_* bits below; `sdf` is always a column.  The MLP input columns are, in order:
 *   image features   with VIS: the C/2 channels feat_select picks (vis = 1: [0, C/2), vis = 0: [C/2, C));
 *                    without:  all C channels in order
 *   sdf              |sdf| >= sdf_clip becomes sign(sdf)
 *   cmap xyz         if CMAP, with the call-level outlier overwrite (HGPIFuNet.py:303-304)
 *   norm xyz         if NORM
 * so c0 = C/2 + 1 + 3 cmap + 3 norm with VIS (C even) and C + 1 + 3 cmap + 3 norm without.  Without CMAP the query
 * is point-local (no outlier rank: a call split into pieces gives the same values).  The mask is ignored for pifu /
 * pamir.  icon_query is this function with all three bits set. */
#define ICON_FEAT_CMAP 1
#define ICON_FEAT_NORM 2
#define ICON_FEAT_VIS 4
#define ICON_FEAT_ALL (ICON_FEAT_CMAP | ICON_FEAT_NORM | ICON_FEAT_VIS)
int icon_query_feats(int prior, const float *points, int64_t stride_c, int64_t stride_n, int64_t N,
                     const float *h_calib, const float *feat, int C, int H, int W,
                     const float *vol_feat, int VD, const void *mesh_ws, int V, int F,
                     const float *mlp_packed, const void *mlp_tc, int c0, float sdf_clip, int smpl_feats,
                     float *out, void *ws, size_t ws_bytes, icon_stream_t stream);

/* Points-per-warp policy of the SDF kernel: force_ppw in {1, 8, 32} pins it (0 = automatic: 1 below ppw8_from
 * points per call, 8 below ppw32_from, else 32; negative thresholds keep the current value).  Results are
 * identical for every setting. */
int icon_set_sdf_policy(int force_ppw, int64_t ppw8_from, int64_t ppw32_from);
/* Brick face lists of the PPW = 32 path (default on): a body's first dense call builds, into its mesh workspace, a
 * sorted list of candidate faces for each of 32^3 bricks over [-1,1]^3; warps inside one brick then skip the tree
 * walk.  enable = 0 turns the path off (A/B runs).  max_entries > 0 caps the face-list entries later builds may use
 * (a build past the cap marks the lists overflowed and dense calls walk the tree); 0 = the workspace's capacity.
 * Results are identical either way. */
int icon_set_sdf_bricks(int enable, int64_t max_entries);
/* Brick list state of a prepared body (synchronises the device): out[0] built, [1] overflowed, [2] face-list
 * entries, [3] face-list entry capacity of the workspace, [4] builds enqueued by this process so far (all bodies). */
int icon_sdf_brick_info(const void *mesh_ws, int V, int F, int64_t *out);
/* Read-back of a prepared body's built brick lists (diagnostics; synchronises the device).  dims[0] = bricks per axis
 * A, dims[1] = face-list entries E; with every array null only dims is written.  Host arrays, B = A^3 bricks, brick
 * b = (bz * A + by) * A + bx: foff [B + 1] list offsets, flist [E] original face ids, fkey [E] their keys, bub [B] the
 * bound on every point's nearest distance, bface [B] the face nearest each brick centre, sph [F][4] the bounding
 * sphere (centre, radius) of each original face that the keys were computed from.  ICON_EINVAL when the lists are not
 * built or overflowed. */
int icon_sdf_brick_lists(const void *mesh_ws, int V, int F, int64_t *dims, int32_t *foff, int32_t *flist,
                         float *fkey, float *bub, int32_t *bface, float *sph);

/* Debug / parity tap: the SMPL block alone (cal_sdf_batch outputs before the outlier rule).
 * rec [N,8] f32 = sdf, cmap xyz, norm xyz, vis(0/1); face [N] i32 nearest face id. */
int icon_sdf_only(const float *points, int64_t stride_c, int64_t stride_n, int64_t N,
                  const float *h_calib, const void *mesh_ws, int V, int F, float *rec,
                  int32_t *face, void *ws, size_t ws_bytes, icon_stream_t stream);
/* Same outputs by brute force over all faces (no bricks); slow, for cross-checks. */
int icon_sdf_bruteforce(const float *points, int64_t stride_c, int64_t stride_n, int64_t N,
                        const float *h_calib, const void *mesh_ws, int V, int F, float *rec,
                        int32_t *face, icon_stream_t stream);
/* Read-back of the face tree at the start of a workspace icon_smpl_prepare or icon_mesh_prepare filled (diagnostics;
 * synchronises the device).  Host arrays: order [F] original face id at each sorted position, tri_s [F][12] records
 * (a.xyz, ab.xyz, ac.xyz, then 3 zeros) and sph_s [F][4] bounding spheres (centre, radius) in sorted order, nodes
 * [N][2][4] boxes (min.xyz, 0) (max.xyz, 0), leaves first, N = sum over levels of the node counts ceil(F / 4),
 * ceil(F / 16), ... down to 1. */
int icon_face_tree_read(const void *mesh_ws, int V, int F, int32_t *order, float *tri_s, float *sph_s, float *nodes);
/* ------------------------------------------------------------------ any triangle mesh: distance and sampling
 * The two trimesh calls of the benchmark's Chamfer / P2S metric (lib/dataset/Evaluator.py:200-230,
 * calculate_chamfer_p2s): trimesh.proximity.closest_point and trimesh.sample.sample_surface_even.
 *
 * icon_mesh_prepare: distance-only workspace for verts [V,3] f32, faces [F,3] i64 (no cmap, vis or normals; F is
 * bounded by memory only): per-face records, Morton-sorted 4-ary AABB tree with 32-bit ids, and the cumulative
 * area weights the sampler draws from.  The workspace stays valid while verts / faces are unchanged. */
size_t icon_mesh_workspace_bytes(int V, int F);
int icon_mesh_prepare(const float *verts, const int64_t *faces, int V, int F, void *mesh_ws, size_t mesh_ws_bytes,
                      icon_stream_t stream);
/* Unsigned nearest face of points [N,3] f32 (contiguous): out_sqdist [N] f32 exact squared distance, out_face [N] i32
 * (may be NULL) the nearest face, lowest index on ties.  Bit-identical to brute force over all faces
 * (oracle_mesh_distance).  Needs no scratch. */
int icon_mesh_distance(const float *points, int64_t N, const void *mesh_ws, int V, int F, float *out_sqdist,
                       int32_t *out_face, icon_stream_t stream);
/* sample_surface_even(mesh, count) (trimesh 3.9.35 semantics, seeded): 3 count area-weighted uniform candidates, then
 * greedy removal in candidate order of every candidate within radius sqrt(area / (3 count)) of a kept one, keeping at
 * most count (<= 8192).  out_points [count,3] f32, out_face [count] i32, *out_count (device i32) = samples kept.
 * verts / faces are the arrays the workspace was prepared from; ws: icon_mesh_sample_workspace_bytes(count). */
size_t icon_mesh_sample_workspace_bytes(int count);
int icon_mesh_sample(const float *verts, const int64_t *faces, int V, int F, const void *mesh_ws, int count,
                     uint64_t seed, float *out_points, int32_t *out_face, int32_t *out_count, void *ws,
                     size_t ws_bytes, icon_stream_t stream);
/* Precomputed radiance transfer (lib/renderer/prt_util.py:115-182, computePRT) over a workspace icon_mesh_prepare
 * filled for the mesh (Vm vertices, F faces).  For the V ray origins origins [V,3] f64 with unit normals normals [V,3]
 * f64 and the D directions dirs [D,3] f64 with their K real SH values sh [D,K] f64:
 *   prt_out[v,k] = w * sum_d (d.n_v > 0) (1 - hit) (d.n_v) sh[d,k]        [V,K] f64,
 * hit = any face met by the ray fp32(o_v + delta n_v) + t fp32(d), t > 0 (Moller-Trumbore, convention in geom.cuh).
 * The sum runs over blocks of n directions when D = n^2 (one block otherwise), in order.  hit_bits [V, ceil(D/32)]
 * u32 (may be NULL): bit d % 32 of word d / 32 is ray d's verdict; when given, every ray is cast, else only the
 * front-facing ones.  ws: at least ceil(D/32) * 4 bytes; vertices go in chunks of as many rows as it holds
 * (icon_prt_workspace_bytes: up to 65536).  The results do not depend on the chunking. */
size_t icon_prt_workspace_bytes(int V, int D, int K);
int icon_prt(const void *mesh_ws, int Vm, int F, const double *origins, const double *normals, int V, double delta,
             const double *dirs, const double *sh, int D, int K, double w, double *prt_out, uint32_t *hit_bits,
             void *ws, size_t ws_bytes, icon_stream_t stream);

/* MLP alone on a ready [c0,N] feature matrix (parity tap for lib/net/MLP.py:49-72). */
int icon_mlp_only(const float *feature, int c0, int64_t N, const float *mlp_packed,
                  const void *mlp_tc, float *out, icon_stream_t stream);

/* ------------------------------------------------------------------ reconstruction engine
 * Replace the per-level body of Seg3dLossless._forward_faster
 * (lib/common/seg3d_lossless.py:186-263).  Grids are [R,R,R] indexed [z][y][x]. */

/* seg3d_lossless.py:190-223: both F.interpolate(trilinear, align_corners=True) calls
 * (occupancy and (occ>balance) mask) fused with is_boundary = 0<valid<1 and with the
 * carry-over of the already-evaluated set (coords_accum*2).  R_out = 2*R_in-1.
 * boundary/done_out may be NULL (last level: upsample only, :186-203). */
int icon_display(const float *occ, int R, uint8_t *out /* [R][4R][3] */, icon_stream_t stream);   /* Seg3dLossless.display:
   first-hit + finite-difference normal preview, views front | left | right | back (seg3d_lossless.py:497-581) */
int icon_grid_upsample(const float *occ_in, const uint8_t *done_in, int R_in, float balance,
                       float *occ_out, uint8_t *boundary, uint8_t *done_out,
                       icon_stream_t stream);
/* seg3d_lossless.py:226-234 + seg3d_utils.py:169-181: (SmoothConv3D(k)(mask) > 0) == binary
 * dilation by a k^3 box; separable.  tmp: R^3 bytes.  The result is written TRANSPOSED,
 * out_xyz[x][y][z], which is the order `is_boundary.permute(2,1,0).nonzero()` walks. */
int icon_grid_dilate(const uint8_t *mask, int R, int k, uint8_t *tmp, uint8_t *out_xyz,
                     icon_stream_t stream);
/* seg3d_lossless.py:236-249 + batch_eval :125-138: clear already-evaluated voxels, stable
 * compaction in (x,y,z)-lexicographic order, emit query points
 * p = c*stride/(R_last-1)*(b_max-b_min)+b_min and linear indices z*R*R+y*R+x; marks the
 * selected voxels in `done`.  *d_count (device int64) receives n.  ws: icon_compact_workspace_bytes(R). */
size_t icon_compact_workspace_bytes(int R);
int icon_grid_compact(const uint8_t *mask_xyz, uint8_t *done, int R, int R_last,
                      const float *h_bmin, const float *h_bmax, float *points, int64_t *indices,
                      int64_t capacity, int64_t *d_count, void *ws, size_t ws_bytes,
                      icon_stream_t stream);
/* seg3d_lossless.py:255-258: occupancys.scatter_(2, point_indices, occupancys_topk). */
int icon_grid_scatter(float *occ, const int64_t *indices, const float *values, int64_t n,
                      icon_stream_t stream);
/* seg3d_lossless.py:168-177: level-0 lattice points (create_grid3D + batch_eval) and the
 * "(occupancys > 0.5).sum() == 0" test (d_count receives the number above balance). */
int icon_grid_init_points(int R0, int R_last, const float *h_bmin, const float *h_bmax,
                          float *points, icon_stream_t stream);
int icon_grid_count_above(const float *occ, int64_t n, float balance, int64_t *d_count,
                          icon_stream_t stream);

/* ------------------------------------------------------------------ marching cubes
 * Replaces Seg3dLossless.export_mesh (lib/common/seg3d_lossless.py:583-604): kaolin
 * voxelgrids_to_trianglemeshes (<=256^3) / PyMCubes (>256^3) at iso `balance`, including the
 * occupancys[1:,1:,1:] crop and the [:, [2,1,0]] / [:, [0,2,1]] permutations.  Indexing
 * contract: DESIGN.md "marching cubes" (oracle/mcubes.py restates it).
 *   occ [R,R,R]; padded=1 -> kaolin branch (zero pad, padded-frame coords, f32 verts),
 *   padded=0 -> PyMCubes branch (f64 verts).  Each branch classifies and interpolates in its vertex precision:
 *   f < (float)iso and fp32 t padded, (double)f < iso and fp64 t plain (PyMCubes takes the iso value as a double).
 * icon_mc_count fills ws and writes {n_verts, n_tris} to d_counts (device int64[2]);
 * icon_mc_emit writes verts [n_verts,3] (f32 or f64) and faces [n_tris,3] i64. */
size_t icon_mc_workspace_bytes(int R, int padded);
int icon_mc_count(const float *occ, int R, double iso, int padded, void *ws, size_t ws_bytes,
                  int64_t *d_counts, icon_stream_t stream);
int icon_mc_emit(const float *occ, int R, double iso, int padded, const void *ws, void *verts,
                 int64_t *faces, int64_t n_verts, int64_t n_tris, icon_stream_t stream);

/* ------------------------------------------------------------------ PaMIR semantic voxelisation
 * Replaces voxelize_cuda.forward_semantic_voxelization as called by VoxelizationFunction.forward
 * (lib/net/voxelize.py:57-59) plus the bzyxc -> bcdhw permute of Voxelization.forward (:137).
 * verts [NV,3] f32 (surface vertices first, then the tetra-SMPL interior ones, in [-0.5,0.5]^3),
 * codes [NVsurf,3] f32, tets [NT,4] i32 (indices into verts), out [3,res,res,res] f32 (c,z,y,x).
 * Source of voxelize_cuda is absent: the algorithm is restated (csrc/voxelize.cu header), parity unpinned. */
size_t icon_voxelize_workspace_bytes(int res);
int icon_voxelize(const float *verts, int NV, int NVsurf, const float *codes, const int32_t *tets, int NT,
                  int res, float sigma, float *out, void *ws, size_t ws_bytes, icon_stream_t stream);

/* ------------------------------------------------------------------ vertex visibility (producer of smpl_vis)
 * Replaces get_visibility (lib/dataset/mesh_util.py:280-316): z-buffer rasterisation of the body at
 * image_size^2 (4096 in the reference) with pytorch3d's conventions (csrc/visibility.cu header; parity unpinned),
 * vis[v] = 1 for the vertices of every face that owns a pixel (plus the last face's, as faces[-1] does upstream).
 * xyz [V,3] f32 = (cat(xy, -z) + 1) / 2 as the reference builds it, faces [F,3] i64, vis [V] f32. */
size_t icon_visibility_workspace_bytes(int image_size);
int icon_visibility(const float *xyz, int V, const int64_t *faces, int F, int image_size, float *vis,
                    void *ws, size_t ws_bytes, icon_stream_t stream);

/* ------------------------------------------------------------------ normal images of the evaluation
 * Replace the OpenGL NormalRender behind Evaluator._render_normal (lib/dataset/Evaluator.py:58-73) and trimesh's
 * vertex_normals it draws by default.  Rules (parity unpinned): csrc/normal_render.cu header (the vertex normals:
 * csrc/normals.cu header).
 *
 * icon_vertex_normals: trimesh's angle-weighted vertex normals of verts [V,3] f64, faces [F,3] i64, computed in fp64
 * and written as out [V,3] f32; bitwise reproducible (no float atomics).  Unreferenced vertices get zero. */
size_t icon_vertex_normals_workspace_bytes(int V, int F);
int icon_vertex_normals(const double *verts, int V, const int64_t *faces, int F, float *out, void *ws,
                        size_t ws_bytes, icon_stream_t stream);
/* icon_normal_render: one orthographic normal image at width x height (each <= 16384).
 * verts [V,3] f32 (already scale_factor * vertices), norms [V,3] f32, faces [F,3] i64, h_model: HOST pointer to the
 * 12 floats of the model matrix's first three rows.  out_rgba [height,width,4] f32 (16-byte aligned) in get_color's
 * row order, background (1,1,1,0); out_face [height,width] i32 the drawn face (-1 background) or NULL. */
size_t icon_normal_render_workspace_bytes(int V, int F, int width, int height);
int icon_normal_render(const float *verts, const float *norms, int V, const int64_t *faces, int F,
                       const float *h_model, int width, int height, float *out_rgba, int32_t *out_face,
                       void *ws, size_t ws_bytes, icon_stream_t stream);

/* ------------------------------------------------------------------ views of the dataset renderer
 * Replace the OpenGL PRTRender (lib/renderer/gl/prt_render.py, shaders prt.vs / prt.fs, 16x MSAA) and ColorRender
 * (color_render.py, color.vs / color.fs) that scripts/render_single.py draws with.  Rules (parity unpinned):
 * csrc/dataset_render.cu header.
 *
 * icon_dr_mesh: device arrays of one mesh, every attribute indexed per face corner by its own [F,3] i64 index array.
 * mode ICON_DR_PRT: pos [V,3], nrm [Vn,3], uv [Vt,2], attr = PRT [Va,9] (f32); tex = icon_dataset_texture's levels or
 * NULL (albedo 1; uv / f_uv are then not read).  ICON_DR_COLOR: attr = colour [Va,3]; tex must be NULL. */
#define ICON_DR_PRT 0
#define ICON_DR_COLOR 1
typedef struct {
    int mode, F, V, Vn, Vt, Va;
    const float *pos, *nrm, *uv, *attr;
    const int64_t *f_pos, *f_nrm, *f_uv, *f_attr;
    const uint8_t *tex;
    int tex_w, tex_h;
} icon_dr_mesh;
/* icon_dataset_render: one view at width x height (each <= 16384) with samples in {1, 16} per pixel.  h_view: HOST
 * pointer to 69 floats: NormMat rows 0-2 (12), RotMat (9, row-major), PerspMat ModelMat rows 0-2 (12; its row 3 must
 * be (0, 0, 0, 1)), mat3(ModelMat) RotMat (9), SHCoeffs [9][3] (27).  out [3][height][width][4] f32 (16-byte
 * aligned): attachments 0-2 in get_color's layout.  ws: icon_dataset_render_workspace_bytes (0 for bad sizes). */
size_t icon_dataset_render_workspace_bytes(int F, int width, int height, int samples);
int icon_dataset_render(const icon_dr_mesh *mesh, const float *h_view, int width, int height, int samples, float *out,
                        void *ws, size_t ws_bytes, icon_stream_t stream);
/* icon_dataset_texture: the albedo's mip levels 0-3 (RGBA8, level 0 = rgb [h,w,3] u8 flipped vertically, then 2x2
 * boxes) into tex (icon_dataset_texture_bytes(w, h) bytes, 4-byte aligned), once per texture. */
size_t icon_dataset_texture_bytes(int w, int h);
int icon_dataset_texture(const uint8_t *rgb, int w, int h, uint8_t *tex, size_t tex_bytes, icon_stream_t stream);

/* ------------------------------------------------------------------ self-rotation video of the demo
 * Replace the pytorch3d renders of Render.get_rendered_video (lib/common/render.py:327-374; MeshRasterizer +
 * cleanShader at get_camera / init_renderer(camera, "clean_mesh", "gray")) and the colours VF2Mesh gives a mesh.
 * Rules (parity unpinned): csrc/mesh_views.cu header (the vertex normals: csrc/normals.cu header).
 *
 * icon_area_vertex_normals: pytorch3d's verts_normals_packed of verts [V,3] f32, faces [F,3] i64 -> out [V,3] f32;
 * bitwise reproducible (no float atomics). */
size_t icon_area_vertex_normals_workspace_bytes(int V, int F);
int icon_area_vertex_normals(const float *verts, int V, const int64_t *faces, int F, float *out, void *ws,
                             size_t ws_bytes, icon_stream_t stream);
/* icon_area_vertex_normals_backward: grad_normals [V,3] f32 (the upstream gradient of out) -> grad_verts [V,3] f32,
 * overwritten; fp64 sums in the forward's (pass, face) order, bitwise reproducible.  ws:
 * icon_area_vertex_normals_backward_workspace_bytes(V, F) bytes. */
size_t icon_area_vertex_normals_backward_workspace_bytes(int V, int F);
int icon_area_vertex_normals_backward(const float *verts, int V, const int64_t *faces, int F,
                                      const float *grad_normals, float *grad_verts, void *ws, size_t ws_bytes,
                                      icon_stream_t stream);
/* icon_mesh_views: A orthographic views at S x S (S <= 4096, A F < 2^31) in one call.  verts [V,3] f32, colors
 * [V,3] f32 (per-vertex RGB), faces [F,3] i64, h_view_mats: HOST pointer to A x 12 floats (each view's 3 x 4 matrix,
 * rows; icon_b200/mesh_views.py view_matrices).  out [A,S,S,3] u8 RGB, row 0 at the top; face_out [A,S,S] i32 the
 * nearest fragment's face (-1 background) or NULL; rgb_out [A,S,S,3] f32 the blended colour before the uint8
 * conversion, or NULL.  ws: icon_mesh_views_workspace_bytes(V, F, S, A) bytes (about 250 A S^2 + 16 A V + 8 A F). */
size_t icon_mesh_views_workspace_bytes(int V, int F, int S, int A);
int icon_mesh_views(const float *verts, const float *colors, int V, const int64_t *faces, int F,
                    const float *h_view_mats, int A, int S, uint8_t *out, int32_t *face_out, float *rgb_out,
                    void *ws, size_t ws_bytes, icon_stream_t stream);
/* Differentiable renders of the fitting loops: Render.get_rgb_image (mode ICON_RENDER_NORMAL, the rules of
 * icon_mesh_views) and Render.get_silhouette_image (ICON_RENDER_SILHOUETTE), forward and backward; rules and
 * gradient formulas (parity unpinned) in the csrc/mesh_views.cu header.  Arguments as icon_mesh_views (h_view_mats on
 * the host; colors may be NULL for the silhouette).
 * icon_mesh_render_forward: out [A,S,S,3] f32 rgb (NORMAL) or [A,S,S] f32 alpha (SILHOUETTE).  state: the K slot keys
 *   of every pixel, [A][S][S][K] u64 (z bits << 32 | face, ascending, all ones when empty; K = 30 / 50), which the
 *   backward reads: icon_mesh_render_state_bytes(mode, S, A) bytes.
 * icon_mesh_render_backward: grad_out shaped as out -> grad_verts [V,3] f32 and (NORMAL, or NULL) grad_colors [V,3]
 *   f32, overwritten; bitwise reproducible (no float atomics).
 * ws: icon_mesh_render_workspace_bytes(mode, backward, V, F, S, A) bytes (backward = 0 forward, 1 backward). */
#define ICON_RENDER_NORMAL 0
#define ICON_RENDER_SILHOUETTE 1
size_t icon_mesh_render_state_bytes(int mode, int S, int A);
size_t icon_mesh_render_workspace_bytes(int mode, int backward, int V, int F, int S, int A);
int icon_mesh_render_forward(int mode, const float *verts, const float *colors, int V, const int64_t *faces, int F,
                             const float *h_view_mats, int A, int S, float *out, void *state, size_t state_bytes,
                             void *ws, size_t ws_bytes, icon_stream_t stream);
int icon_mesh_render_backward(int mode, const float *verts, const float *colors, int V, const int64_t *faces, int F,
                              const float *h_view_mats, int A, int S, const float *grad_out, const void *state,
                              size_t state_bytes, float *grad_verts, float *grad_colors, void *ws, size_t ws_bytes,
                              icon_stream_t stream);

/* ------------------------------------------------------------------ cloth-refinement geometry
 * The mesh topology, the three shape priors of update_mesh_shape_prior_losses (lib/dataset/mesh_util.py:168-176) and
 * LocalAffine (lib/net/local_affine.py), forward and backward; rules and gradient formulas (parity unpinned) in the
 * csrc/mesh_priors.cu header.  No float atomics: bitwise reproducible.  One mesh (B = 1).
 *
 * Topology: icon_mesh_topology_count(faces [F,3] i64) rejects an index outside [0, V) and returns the edge count E
 *   to the host (it synchronises the stream); icon_mesh_topology_build, with the same unchanged ws, fills the arrays
 *   of the struct (all device memory, caller-allocated to the sizes given). */
typedef struct {
    int V, F, E;
    const int64_t *faces;      /* [F,3] */
    int64_t *edges;            /* [E,2] (min, max), ascending */
    int64_t *face_to_edge;     /* [F,3] columns e12, e20, e01 */
    int32_t *vert_off;         /* [V+1] */
    int32_t *vert_edges;       /* [2E] per vertex its edge ids, ascending (a self-loop twice); degree = row length */
    int32_t *edge_off;         /* [E+1] */
    int32_t *edge_entries;     /* [3F] per edge its face-corner entries 3 f + col, ascending */
    int32_t *corner_off;       /* [V+1] */
    int32_t *vert_corners;     /* [3F] per vertex its corners 3 f + c, ascending */
} icon_mesh_topology;
size_t icon_mesh_topology_workspace_bytes(int V, int F);
int icon_mesh_topology_count(const int64_t *faces, int V, int F, int64_t *h_E, void *ws, size_t ws_bytes,
                             icon_stream_t stream);
int icon_mesh_topology_build(const icon_mesh_topology *t, void *ws, size_t ws_bytes, icon_stream_t stream);
/* icon_vertex_edges: the vert_edges lists of caller edges [E,2] i64 (indices in [0, V), checked by the caller),
 * built by the same code as the topology's. */
size_t icon_vertex_edges_workspace_bytes(int V, int E);
int icon_vertex_edges(const int64_t *edges, int E, int V, int32_t *vert_off, int32_t *vert_edges, void *ws,
                      size_t ws_bytes, icon_stream_t stream);
/* Priors of verts [V,3] f32: forward -> three f32 device scalars (edge, normal consistency, uniform laplacian);
 * backward: the three upstream gradients as device scalars, NULL = absent (that term is skipped) -> grad_verts [V,3]
 * f32, overwritten.  ws: icon_mesh_priors_workspace_bytes(V, F, E, backward) bytes. */
size_t icon_mesh_priors_workspace_bytes(int V, int F, int E, int backward);
int icon_mesh_priors_forward(const icon_mesh_topology *t, const float *verts, float *out_edge, float *out_nc,
                             float *out_lap, void *ws, size_t ws_bytes, icon_stream_t stream);
int icon_mesh_priors_backward(const icon_mesh_topology *t, const float *verts, const float *g_edge, const float *g_nc,
                              const float *g_lap, float *grad_verts, void *ws, size_t ws_bytes, icon_stream_t stream);
/* ------------------------------------------------------------------ remeshing of the reconstruction
 * lib/dataset/mesh_util.py:109-121 (remesh: pymeshlab laplacian_smooth + isotropic explicit remeshing); rules
 * (parity unpinned) in the csrc/remesh.cu header; the host loop is icon_b200/remesh.py.  Vertices are f64 [V,3].
 * ws: icon_remesh_workspace_bytes(V, F, E) bytes for the topology t the call is given; classify fills it and the
 * other calls of the same round read it.
 * compact: drop unreferenced vertices (out_verts [V,3], out_faces [F,3], *d_count (device i64) = vertices kept;
 *   ws sized for (V, F, 1)).  smooth_step: one Jacobi step (after classify).  midpoints: fp32 edge midpoints [E,3].
 * select: op 0 split, 1 collapse (sqdist [E] f32: squared distance of each midpoint to the reference surface), 2
 *   flip; marks the round's winners, *d_count (device i64) = their number W.  apply: split -> out_verts [V+W,3],
 *   out_faces [F+2W,3]; collapse -> [V-W,3], [F-2W,3]; flip -> out_faces [F,3] (out_verts unused).
 * relax: normals [V,3] f32 (icon_area_vertex_normals) -> out [V,3] f64, out32 [V,3] f32, moved [V] i32.
 * reproject: each moved vertex onto its nearest reference face face[v] (icon_mesh_distance of out32). */
size_t icon_remesh_workspace_bytes(int V, int F, int E);
int icon_remesh_compact(const double *verts, int V, const int64_t *faces, int F, double *out_verts,
                        int64_t *out_faces, int64_t *d_count, void *ws, size_t ws_bytes, icon_stream_t stream);
int icon_remesh_classify(const icon_mesh_topology *t, const double *verts, void *ws, size_t ws_bytes,
                         icon_stream_t stream);
int icon_remesh_smooth_step(const icon_mesh_topology *t, const double *verts, double *out, void *ws,
                            size_t ws_bytes, icon_stream_t stream);
int icon_remesh_midpoints(const icon_mesh_topology *t, const double *verts, float *out, icon_stream_t stream);
int icon_remesh_select(int op, const icon_mesh_topology *t, const double *verts, double L, int adaptive,
                       const float *sqdist, double dlim2, int64_t *d_count, void *ws, size_t ws_bytes,
                       icon_stream_t stream);
int icon_remesh_apply(int op, const icon_mesh_topology *t, const double *verts, int W, double *out_verts,
                      int64_t *out_faces, void *ws, size_t ws_bytes, icon_stream_t stream);
int icon_remesh_relax(const icon_mesh_topology *t, const double *verts, const float *normals, double *out,
                      float *out32, int32_t *moved, void *ws, size_t ws_bytes, icon_stream_t stream);
int icon_remesh_reproject(const double *verts, int V, const int32_t *moved, const int32_t *face,
                          const double *ref_verts, const int64_t *ref_faces, double *out, icon_stream_t stream);
/* LocalAffine, B = 1: A [N,3,3], b [N,3], x [N,3], edges [E,2] i64 -> out [N,3], w_diff [E,3,4], w_rigid [N] (all
 * f32).  Backward: g_out / g_diff / g_rigid shaped as those (NULL = absent), vert_off / vert_edges from
 * icon_vertex_edges of the same edges -> grad_A, grad_b and (when not NULL) grad_x, overwritten. */
int icon_local_affine_forward(const float *A, const float *b, const float *x, int N, const int64_t *edges, int E,
                              float *out, float *w_diff, float *w_rigid, icon_stream_t stream);
int icon_local_affine_backward(const float *A, const float *b, const float *x, int N, const int64_t *edges, int E,
                               const int32_t *vert_off, const int32_t *vert_edges, const float *g_out,
                               const float *g_diff, const float *g_rigid, float *grad_A, float *grad_b, float *grad_x,
                               icon_stream_t stream);

/* ------------------------------------------------------------------ body model (linear-blend skinning)
 * lbs() of lib/smplx/lbs.py for an SMPL-family model, forward and backward; rules, layouts and reduction order in the
 * csrc/body_model.cu header.  fp32 inputs and outputs, fp64 inside.  No float atomics: bitwise reproducible, and row b
 * of a B-row call equals a one-row call on that row.
 *
 * icon_lbs_model: the caller fills V, J (2..64), NB (1..1024) and the buffer pointers (device, fp32, contiguous);
 *   icon_lbs_prepare checks h_parents (host [J] i64: parents[0] = -1, parents[i] < i) and posedirs_rows = 9 (J - 1),
 *   copies the parents into the struct and writes J_template / J_dirs (caller-allocated device fp64). */
typedef struct {
    int V, J, NB;
    int parents[64];
    const float *v_template;   /* [V,3] */
    const float *shapedirs;    /* [V,3,NB] */
    const float *posedirs;     /* [9(J-1), 3V] */
    const float *J_regressor;  /* [J,V] */
    const float *lbs_weights;  /* [V,J] */
    double *J_template;        /* [J,3]    = J_regressor v_template */
    double *J_dirs;            /* [J,3,NB] = J_regressor shapedirs */
} icon_lbs_model;
size_t icon_lbs_prepare_workspace_bytes(int V, int J, int NB);
int icon_lbs_prepare(icon_lbs_model *m, const int64_t *h_parents, int posedirs_rows, void *ws, size_t ws_bytes,
                     icon_stream_t stream);
/* Forward: betas [B,NB], pose [B,J,3] (pose2rot = 1, axis-angle) or [B,J,3,3] (pose2rot = 0, used as given) ->
 * verts [B,V,3], joints [B,J,3]; `state` (icon_lbs_state_bytes) keeps what the backward needs.  Backward:
 * grad_verts [B,V,3] and / or grad_joints [B,J,3] (NULL = zero) -> grad_betas [B,NB] and grad_pose (the pose's
 * shape), overwritten.  ws: icon_lbs_workspace_bytes(..., backward) bytes (the forward needs none). */
size_t icon_lbs_state_bytes(int B, int V, int J, int NB);
size_t icon_lbs_workspace_bytes(int B, int V, int J, int NB, int backward);
int icon_lbs_forward(const icon_lbs_model *m, int B, const float *betas, const float *pose, int pose2rot, float *verts,
                     float *joints, void *state, size_t state_bytes, void *ws, size_t ws_bytes, icon_stream_t stream);
int icon_lbs_backward(const icon_lbs_model *m, int B, const void *state, size_t state_bytes, const float *grad_verts,
                      const float *grad_joints, float *grad_betas, float *grad_pose, void *ws, size_t ws_bytes,
                      icon_stream_t stream);

/* ------------------------------------------------------------------ SMPL-X heads (PIXIE's landmarks and joints)
 * The landmark and joint heads PIXIE's SMPLX.forward (lib/pixielib/models/SMPLX.py) runs on the skinned vertices:
 * the head-yaw lookup-table row, the static and dynamic face landmarks, the extra joints picked from faces and the
 * dense joint regressor written over `source` joints.  Rules, tolerances and the backward's order in the "heads"
 * section of the csrc/body_model.cu header.  No float atomics.
 *
 * icon_smplx_heads: the caller fills V, J (2..64), R (regressor rows, 1..64), `regressor` (device fp32 [R,V]) and
 *   allocates the device arrays below with N = 3 (Ls + 79 Ld + E) slots; icon_smplx_heads_prepare checks the host
 *   tables (every face id in [0,F), every vertex id of a used face in [0,V), chain and source in [0,J), target in
 *   [0,R), sources and targets each distinct), fills Ls, Ld, E, nchain, chain and writes the arrays.  It copies to
 *   the device and synchronises `stream` (a one-time fill, not a per-call cost). */
#define ICON_HEADS_LUT_ROWS 79
#define ICON_HEADS_MAX_CHAIN 8
typedef struct {
    int V, J, R;
    int Ls, Ld, E, nchain;
    int chain[ICON_HEADS_MAX_CHAIN];
    const float *regressor;  /* [R,V] */
    int *vid;                /* [N]   corner vertex ids: static [Ls,3], then the table [79,Ld,3], then extra [E,3] */
    float *bc;               /* [N]   their barycentric weights, same layout */
    int *joint_reg;          /* [J]   the regressor row written over joint j, or -1 */
    int *reg_joint;          /* [R]   the joint regressor row r is written over, or -1 */
    int *inc_off;            /* [V+1] per vertex, its range of `inc` */
    int *inc;                /* [N]   the slots that read each vertex, in (entry, table row, corner) order */
} icon_smplx_heads;
int icon_smplx_heads_prepare(icon_smplx_heads *h, const int64_t *h_faces, int F, const int64_t *h_lmk_faces_idx,
                             const float *h_lmk_bary, int Ls, const int64_t *h_dyn_faces_idx, const float *h_dyn_bary,
                             int Ld, const int64_t *h_face_ids, const float *h_bcs, int E, const int64_t *h_source,
                             const int64_t *h_target, int S, const int64_t *h_chain, int nchain,
                             icon_stream_t stream);
/* Forward: verts [B,V,3] and joints_lbs [B,J,3] (icon_lbs_forward's outputs), pose [B,J,3,3] -> landmarks
 * [B,Ls+Ld,3], joints [B,J+Ls+Ld+E,3] and rows [B] (int32 lookup-table rows); `state` (icon_smplx_heads_state_bytes)
 * is scratch for the regressor's partial sums.  Two launches.  Backward: grad_landmarks and / or grad_joints
 * (NULL = zero) -> grad_verts [B,V,3] (overwritten) and, when grad_joints is given, grad_joints_lbs [B,J,3] (zero
 * at the regressed joints).  One launch. */
size_t icon_smplx_heads_state_bytes(int B, int V, int R);
int icon_smplx_heads_forward(const icon_smplx_heads *h, int B, const float *verts, const float *joints_lbs,
                             const float *pose, float *landmarks, float *joints, int *rows, void *state,
                             size_t state_bytes, icon_stream_t stream);
int icon_smplx_heads_backward(const icon_smplx_heads *h, int B, const int *rows, const float *grad_landmarks,
                              const float *grad_joints, float *grad_verts, float *grad_joints_lbs,
                              icon_stream_t stream);

/* ------------------------------------------------------------------ tetra body (PaMIR's TetraSMPLModel)
 * TestDataset.compute_voxel_verts of the pamir demo: rotation matrices -> pymaf's axis-angle (fp32) ->
 * TetraSMPLModel.update (fp64) of the SMPL vertices and the added interior vertices -> the padded, halved, z-flipped
 * voxel_verts [8000,3].  Rules and promotion chain in the "tetra body" section of the csrc/body_model.cu header.
 *
 * icon_tetra_model: the caller fills V (SMPL vertices), N = V + V_added, T (tetrahedra), nnz and the device buffers
 *   (fp64 / int32, contiguous; both vertex sets stacked, SMPL's first); icon_tetra_prepare checks J = 24,
 *   posedirs_cols = 207, nbetas = 10, h_parents (host [24] i64: parents[0] = -1, parents[i] < i), N <= 8000 and
 *   T <= 25100, and copies the parents into the struct.  It launches nothing. */
#define ICON_TETRA_JOINTS 24
#define ICON_TETRA_BETAS 10
#define ICON_TETRA_PAD_V 8000
#define ICON_TETRA_PAD_F 25100
typedef struct {
    int V, N, T, nnz;
    int parents[ICON_TETRA_JOINTS];
    const double *v_template;  /* [N,3] */
    const double *shapedirs;   /* [10,3N]  column k of shapedirs / shapedirs_added */
    const double *posedirs;    /* [207,3N] column p of posedirs / posedirs_added */
    const double *weights;     /* [N,24] */
    const int *jr_off;         /* [25]    per joint, its range of jr_col / jr_val */
    const int *jr_col;         /* [nnz]   J_regressor's nonzero columns (SMPL vertex ids), ascending per joint */
    const double *jr_val;      /* [nnz]   their values */
} icon_tetra_model;
int icon_tetra_prepare(icon_tetra_model *m, const int64_t *h_parents, int J, int posedirs_cols, int nbetas);
/* Forward: rotmats [24,3,3] fp32 (cat of global_orient[0], body_pose[0]) -> aa [24,3] (written), or rotmats = NULL
 * and aa read as given; betas [10], trans [3], scale [1] fp32 (read on the device) -> voxel_verts [8000,3].  `state`:
 * icon_tetra_state_bytes() bytes of scratch.  Two launches, no host sync. */
size_t icon_tetra_state_bytes(void);
int icon_tetra_forward(const icon_tetra_model *m, const float *rotmats, float *aa, const float *betas,
                       const float *trans, const float *scale, float *voxel_verts, void *state, size_t state_bytes,
                       icon_stream_t stream);

/* ------------------------------------------------------------------ encoder operators
 * Replace the cuDNN / torch calls of the encoders (lib/net/HGFilters.py, FBNet.py, NormalNet.py, VE.py).  The first
 * two take NCHW fp32 tensors; every 2-D convolution and normalisation runs on the NHWC path after them. */
/* y = x / ||x||_2 (over 3 channels, no eps) * (sum_c |image| != 0): NormalNet.forward (NormalNet.py:84-97) */
int icon_normalize_mask(const float *x, const float *image, float *y, int N, int Cimg, int64_t HW,
                        icon_stream_t stream);
/* nn.Conv3d (B = 1, Cout <= 8, cubic kernel / stride / padding / dilation) followed by eval-mode BatchNorm3d
 * folded into per-channel (scale, shift), optional residual add and ReLU: the layers of PaMIR's VolumeEncoder
 * (lib/net/VE.py:96-183).  x [Cin,D,H,W], w [Cout,Cin,k,k,k], y [Cout,OD,OH,OW]. */
int icon_conv3d(const float *x, const float *w, const float *scale, const float *shift, const float *res, float *y,
                int Cin, int Cout, int D, int H, int W, int k, int stride, int pad, int dil, int relu,
                icon_stream_t stream);
/* ---- NHWC encoder path (csrc/conv_nhwc.cu, csrc/act_nhwc.cu): activations between layers are NHWC, pre-split
 * x = hi + lo into two fp16 tensors [N * nplanes][Hp][Wp][Cp] (Cp % 64 == 0) by icon_act_nhwc.
 *
 * icon_conv_nhwc: implicit-GEMM convolution on wgmma, A operand staged by 4-D tiled TMA loads straight from the
 *   hi / lo tensors (`dims` = tensor-map extents innermost first, `strides` = element strides of dims 1..3), weights
 *   from `wt_packed` (per n_tile output channels and per chunk a K-major SWIZZLE_128B fp16 hi tile followed by the lo
 *   tile; `wt_chunks` chunks per tile, chunk index = wtap * cpt + channel block).  `wt_scale` (optional, NULL = 1):
 *   per output channel factor 2^-e applied to the products before the bias, for rows packed as w * 2^e so that the
 *   fp16 lo half stays a normal number (icon_b200/nhwc.py pack_tiles).  The launch covers a logical
 *   Ht x Wt grid per image; output pixel (a, b) is written to out[n][a * osy + ooy][b * osx + oox][co_off + co] of an
 *   fp32 NHWC tensor with Cs channels (channel slices = concatenation for free; osy = 2 = one phase of a transposed
 *   convolution).  `taps`: ntaps x (dy, dx, plane, wtap) -- the A box of tap t is read at (y0 + dy, x0 + dx) of image
 *   n * nplanes + plane (out-of-range coordinates read zeros = zero padding).  stats (optional, zeroed by the
 *   caller): [N][Cout][6] doubles receive per-channel sum / sum of squares of the result (bias included), each as
 *   three words (sum = stats[0] + stats[1] + stats[2], sum of squares = stats[3] + stats[4] + stats[5]) so that the
 *   atomic adds are exact and the result does not depend on block order.  icon_ew_nhwc and icon_nchw_to_nhwc write the
 *   same.
 * icon_norm_finalize: stats -> [N][C][3] (scale, mean, beta) for InstanceNorm2d (groups = 0) / GroupNorm(groups) with
 *   affine; a consumer computes y = (x - mean) * scale + beta, so a constant channel gives exactly beta.
 * icon_act_nhwc: y = [relu]((x - mean) * scale + beta) [+ res] (relu = 1), or relu(... + res) (relu = 2: the ReLU
 *   after the residual add that ends a ResNet Bottleneck), from the `scale_shift` table or folded in from the
 *   producer's `stats` (+ GroupNorm gamma / beta, groups = 0: instance norm; 1, 2, 4 or 8 channels per group)
 *   -> hi / lo operand tensors (halo > 0: reflection halo;
 *   s2d = 1: four parity planes for a stride-2 consumer; channels padded to Cp with zeros) and / or fp32 NHWC.
 * icon_ew_nhwc: mode 0 a + b (+ c), 1 avg_pool2(a), 2 b + bicubic_up2(a, align_corners), 3 relu((a - mean) * scale + beta)
 *   with b = the [N][C][3] table of icon_norm_finalize; optional stats of the result.
 * icon_nchw_to_nhwc / icon_nhwc_to_nchw: layout adaptors (the former with optional stats). */
size_t icon_conv_nhwc_workspace_bytes(int N, int Ht, int Wt, int Cout, int splits);
int icon_conv_nhwc(const void *a_hi, const void *a_lo, const int64_t *dims, const int64_t *strides, const void *wt_packed,
                   int wt_chunks, const float *wt_scale, const float *bias, float *out, int OHf, int OWf, int Cs, int co_off,
                   int Cout, int N,
                   int Ht, int Wt, int osy, int osx, int ooy, int oox, int nplanes, int ntaps, const int *taps, int cpt,
                   int n_tile, int splits, double *stats, void *ws, size_t ws_bytes, icon_stream_t stream);
int icon_norm_finalize(const double *stats, const float *gamma, const float *beta, float *scale_shift, int N, int C,
                       int groups, double count, float eps, icon_stream_t stream);
int icon_act_nhwc(const float *x, int Cs_in, int ci_off, const float *scale_shift, const double *stats, const float *gamma,
                  const float *beta, int groups, float eps, const float *res, void *hi, void *lo, float *f32, int N, int H,
                  int W, int C, int Cp, int halo, int s2d, int relu, icon_stream_t stream);
/* icon_splitk_instnorm_act: for a split-K convolution followed by InstanceNorm2d(affine=False) [+ ReLU] [+ residual]
 * (the ResnetBlocks): call icon_conv_nhwc with out == NULL (the split partials stay parked in its workspace
 * [splits][N][H][W][C]), then this -- one kernel sums the partials in split order, computes each channel's mean /
 * variance over the image inside a block (no atomics), normalises and writes the next operand (hi / lo with a
 * reflection halo) and / or the fp32 tensor. */
int icon_splitk_instnorm_act(const float *partial, int splits, const float *bias, const float *res, void *hi, void *lo,
                             float *f32, int N, int H, int W, int C, int Cp, int halo, int relu, float eps,
                             icon_stream_t stream);
/* icon_col2im7: second half of the 7 x 7 output head computed as GEMM + col2im: P [N][H][W][Ps] holds, per INPUT pixel,
 * the products with every tap's weights (column (ky * 7 + kx) * Cout + co; the first half is icon_conv_nhwc with the
 * regrouped 1 x 1 weights); out[n][co][y][x] = act(bias + sum over the 49 reflected neighbours). */
int icon_col2im7(const float *P, const float *bias, float *y, int N, int H, int W, int Cout, int Ps, int act,
                 icon_stream_t stream);
int icon_ew_nhwc(int mode, const float *a, const float *b, const float *c, float *y, double *stats, int N, int H, int W,
                 int C, icon_stream_t stream);
int icon_nchw_to_nhwc(const float *x, float *y, double *stats, int N, int C, int64_t HW, icon_stream_t stream);
int icon_nhwc_to_nchw(const float *x, float *y, int N, int C, int Cs, int c_off, int64_t HW, icon_stream_t stream);
/* icon_stem_pack: NCHW fp32 image -> hi / lo fp16 [N * sy][Hrows][Wp][Cp8] (Cp8 = 8 | 16 >= Cin) with a 3-pixel halo
 * (reflect = 1: ReflectionPad2d(3); 0: zeros) and rows split into sy parity planes: the operand layout of the 7 x 7
 * first layers (K runs over the 8 x Cp8 contiguous values of a filter row; icon_conv_nhwc reads it through a tensor
 * map whose W stride is sx * Cp8 elements). */
int icon_stem_pack(const float *x, void *hi, void *lo, int N, int Cin, int H, int W, int Cp8, int Wp, int Hrows, int sy,
                   int reflect, icon_stream_t stream);
/* ---- clean_mesh (csrc/clean.cu; reference lib/dataset/mesh_util.py:778-791: trimesh split + largest component).
 * faces int64 [nf][3] indexing nv vertices (nf < 2^28).  _count: trimesh's components (faces joined across edges used
 * by exactly two faces), picks the one with the most distinct vertices (ties: the one with the smallest face index),
 * leaves the kept counts in d_counts[0..1] and the re-index tables in `ws`; _emit writes the compacted float32
 * vertices / int32 faces (ascending original order).  Deterministic: the result does not depend on block order. */
size_t icon_clean_mesh_workspace_bytes(int64_t nv, int64_t nf);
int icon_clean_mesh_count(const int64_t *faces, int64_t nv, int64_t nf, void *ws, size_t ws_bytes, int64_t *d_counts,
                          icon_stream_t stream);
int icon_clean_mesh_emit(const void *verts, int verts_f64, const int64_t *faces, int64_t nv, int64_t nf, const void *ws,
                         float *out_verts, int32_t *out_faces, icon_stream_t stream);

/* ---- garment extraction (csrc/garments.cu; reference lib/common/cloth_extraction.py:extract_cloth, called from
 * apps/infer.py:566-605 with -seg_dir).  DESIGN.md 4.16.
 * icon_garment_labels: labels[v] = h_smpl_parts[j*], j* the SMPL vertex nearest to reconstruction vertex v in the
 *   float64 rdist ((x0-y0)^2 + (x1-y1)^2) + (x2-y2)^2, exact ties to the lowest j.  recon_verts [V,3] f64,
 *   smpl_verts [S,3] f64, labels [V] u8 on the device; h_smpl_parts [S] u8 on the host (copied into `ws`),
 *   ICON_EINVAL when one is 32 or more.  Brute force.
 * icon_garment_face_mask: keep[v] = inside(v) && !(remove_parts >> labels[v] & 1), inside(v) = (x, y) of verts[v]
 *   inside any polygon under matplotlib's crossings rule (a non-finite point is never inside; a polygon of fewer than
 *   three vertices encloses nothing); face_mask[f] = keep of any corner of faces[f]; *kept_count = sum of face_mask.
 *   Polygon p is poly_xy[h_poly_off[p] .. h_poly_off[p+1]) ([NP,2] f64 on the device; offsets [npoly+1] i32 on the
 *   host, ICON_EINVAL when one decreases or leaves [0, NP]).  verts [V,3] f64, faces [F,3] i64, labels [V] u8,
 *   face_mask [F] u8, kept_count one i32 on the device.  Synchronises `stream` before it returns: the kernels check
 *   the labels and faces on the device and the verdict is read back; ICON_EINVAL when a label is 32 or more or a
 *   face index is outside [0, V). */
size_t icon_garment_labels_workspace_bytes(int S);
int icon_garment_labels(const double *recon_verts, int V, const double *smpl_verts, int S, const uint8_t *h_smpl_parts,
                        uint8_t *labels, void *ws, size_t ws_bytes, icon_stream_t stream);
size_t icon_garment_face_mask_workspace_bytes(int V, int npoly);
int icon_garment_face_mask(const double *verts, int V, const int64_t *faces, int F, const uint8_t *labels,
                           uint32_t remove_parts, const double *poly_xy, int NP, const int32_t *h_poly_off, int npoly,
                           uint8_t *face_mask, int32_t *kept_count, void *ws, size_t ws_bytes, icon_stream_t stream);

/* ---- PyMAF's body estimate (csrc/hps.cu; reference lib/pymaf/models/pymaf_net.py, maf_extractor.py, smpl.py,
 * utils/geometry.py).  DESIGN.md 4.17.  All buffers fp32 on the device; dot products accumulate in float64.
 * icon_maxpool3s2_nhwc: MaxPool2d(3, 2, 1) of x [N,H,W,C] (of relu(x) when relu != 0) -> the plain hi / lo operand
 *   [N,OH,OW,Cp] (Cp % 64 == 0, channels >= C written 0), OH = (H - 1) / 2 + 1.
 * icon_maf_mlp: per point n of pts [2,N] (x row, y row): bilinear grid_sample (align_corners, zero padding) of the
 *   256 channels of feat [H,W,256], then Conv1d 256->128 + leaky 0.01, [., feature] 384->64 + leaky,
 *   [., feature] 320->5 + ReLU (w1 [128,256], w2 [64,384], w3 [5,320]) -> xc[c * N + n]; xc[5N .. 5N + nprev) = prev.
 * icon_hps_gemv: y [R] = w [R,K] x [K] + b [+ add], K <= 12288.
 * icon_hps_rot6d: rot6d_to_rotmat of pose [J,6] -> rotmat [J,3,3].
 * icon_hps_regress: extra [E,3] = jextra [E,V] verts [V,3]; for Dmap in CSR (row_off [M+1], col, val), the
 *   projection of Dmap verts with cam [3] -> pts [2,M].
 * icon_hps_tail: kp_3d [NJ,3] = [jlbs [Jl,3], verts[vid] [NV,3], extra [E,3]][jmap], kp_2d [NJ,2] its projection with
 *   the cam at par[npose + nshape], theta = [cam, par[npose .. npose + nshape), angle-axis of rotmat [Jl,3,3]]
 *   (kornia's quaternion route, NaN -> 0).  vid and jmap are checked by the caller. */
int icon_maxpool3s2_nhwc(const float *x, void *hi, void *lo, int N, int H, int W, int C, int Cp, int relu,
                         icon_stream_t stream);
int icon_maf_mlp(const float *feat, int H, int W, int C, const float *pts, int N, const float *w1, const float *b1,
                 const float *w2, const float *b2, const float *w3, const float *b3, const float *prev, int nprev,
                 float *xc, icon_stream_t stream);
int icon_hps_gemv(const float *w, const float *x, const float *b, const float *add, float *y, int R, int K,
                  icon_stream_t stream);
int icon_hps_rot6d(const float *pose, float *rotmat, int J, icon_stream_t stream);
int icon_hps_regress(const float *verts, int V, const float *jextra, int E, float *extra, const int *row_off,
                     const int *col, const float *val, int M, const float *cam, float *pts, icon_stream_t stream);
int icon_hps_tail(const float *verts, const float *jlbs, int Jl, const int *vid, int NV, const float *extra, int E,
                  const int *jmap, int NJ, const float *rotmat, const float *par, int npose, int nshape, float *kp3d,
                  float *kp2d, float *theta, icon_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif
