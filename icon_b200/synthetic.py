"""Synthetic, seeded inputs shaped like the reference's (SURVEY.md section 8d).

No checkpoints, SMPL model files or datasets exist offline, so the parity tests, smoke()
and bench.py all run on inputs built here:

* a closed genus-0 "body" mesh with SMPL's exact counts (V=6890, F=13776; the counts
  `lib/dataset/TestDataset.py:280-285` of the reference works with),
* per-vertex cmap / vis attributes (what `TestDataset.compute_vis_cmap` produces),
* image-feature maps and MLP weights with the reference's state_dict shapes.
"""
import math

import numpy as np
import torch


def body_mesh(rings=82, segs=84, seed=0, extent=(0.5, 0.9, 0.25)):
    """Star-shaped closed mesh: rings*segs+2 vertices, 2*rings*segs faces.

    Default 82 x 84 gives V=6890, F=13776 (SMPL's counts).  The radial function is a smooth
    low-order perturbation of an ellipsoid, so the surface is watertight, consistently
    outward-oriented and free of self-intersections.
    Returns (verts float32 [V,3], faces int64 [F,3]).
    """
    rng = np.random.RandomState(seed)
    th = (np.arange(rings) + 1.0) / (rings + 1.0) * math.pi  # polar, poles excluded
    ph = np.arange(segs) / segs * 2.0 * math.pi
    T, P = np.meshgrid(th, ph, indexing="ij")

    coef = rng.uniform(-1.0, 1.0, size=6)

    def radius(t, p):
        r = 1.0
        r = r + 0.18 * coef[0] * np.sin(2 * t) * np.cos(p)
        r = r + 0.15 * coef[1] * np.sin(t) ** 2 * np.cos(2 * p + coef[2])
        r = r + 0.12 * coef[3] * np.sin(3 * t) * np.sin(p)
        r = r + 0.10 * coef[4] * np.sin(t) ** 3 * np.cos(3 * p + coef[5])
        return r

    def point(t, p):
        r = radius(t, p)
        # y is the long (polar) axis, like a standing body
        return np.stack([r * np.sin(t) * np.cos(p), r * np.cos(t), r * np.sin(t) * np.sin(p)], -1)

    body = point(T, P).reshape(-1, 3)
    north = point(np.array(0.0), np.array(0.0))[None]
    south = point(np.array(math.pi), np.array(0.0))[None]
    verts = np.concatenate([body, north, south], 0)
    verts = verts / np.abs(verts).max(0, keepdims=True) * np.asarray(extent)[None]

    def vid(i, j):
        return i * segs + (j % segs)

    n_id, s_id = rings * segs, rings * segs + 1
    faces = []
    for j in range(segs):
        faces.append((n_id, vid(0, j + 1), vid(0, j)))
        faces.append((s_id, vid(rings - 1, j), vid(rings - 1, j + 1)))
    for i in range(rings - 1):
        for j in range(segs):
            a, b, c, d = vid(i, j), vid(i, j + 1), vid(i + 1, j), vid(i + 1, j + 1)
            faces.append((a, b, c))
            faces.append((b, d, c))
    faces = np.asarray(faces, dtype=np.int64)
    # orient outward: signed volume must be positive
    v0, v1, v2 = verts[faces[:, 0]], verts[faces[:, 1]], verts[faces[:, 2]]
    if np.einsum("ij,ij->i", v0, np.cross(v1, v2)).sum() < 0:
        faces = faces[:, [0, 2, 1]]
    # shuffle face order so that "lowest face index wins" is not correlated with position
    faces = faces[rng.permutation(len(faces))]
    return verts.astype(np.float32), faces


def body_attributes(verts, seed=0):
    """cmap in [-1,1]^3 per vertex and a 0/1 visibility flag (front-facing half)."""
    rng = np.random.RandomState(seed + 1)
    cmap = rng.uniform(-1.0, 1.0, size=verts.shape).astype(np.float32)
    vis = (verts[:, 2:3] + 0.05 * rng.standard_normal((len(verts), 1)) > 0).astype(np.float32)
    return cmap, vis


def collapse_faces(faces, n=16, seed=0):
    """A copy of `faces` with faces 0..3 and n - 4 random others collapsed to a segment (corner 1 moved onto corner 0).
    The exact point-triangle distance to such a face is NaN (0/0) wherever (c - a).(p - a) > 0, which a nearest-face
    search must never take; faces 0..3 have the lowest ids, so they would win the tie rule if it did."""
    rng = np.random.RandomState(seed)
    k = np.concatenate([np.arange(4), 4 + rng.choice(len(faces) - 4, n - 4, replace=False)])
    out = faces.copy()
    out[k, 1] = out[k, 0]
    return out


def lattice_points(res, device="cpu"):
    """Cell-centre lattice p = -1 + 2 (i + 0.5) / res per axis, x fastest; [1, res^3, 3]."""
    a = (-1.0 + 2.0 * (torch.arange(res, dtype=torch.float64) + 0.5) / res).float()
    z, y, x = torch.meshgrid(a, a, a, indexing="ij")
    return torch.stack([x, y, z], -1).reshape(1, -1, 3).to(device)


def mlp_state_dict(c0=13, dims=(512, 256, 128, 1), res_layers=(2, 3, 4), seed=0, trained_bn=False):
    """Random weights with the reference MLP's state_dict keys (lib/net/MLP.py:26-47).

    By default the BatchNorm statistics are mild (running_var in [0.5, 1.5], gamma near 1).  trained_bn=True gives
    BatchNorm layers like a trained network's instead: running_var log-uniform in [1e-4, 10], |gamma| log-uniform in
    [0.1, 10] with random signs, running_mean up to about +-30.  As in training, the statistics agree with the conv
    they follow: a channel's weight row is scaled by sqrt(running_var) and its bias sits near running_mean, so the
    normalised pre-activations stay O(1) while the folded weights and biases (gamma / sqrt(var + eps) up to ~1e3)
    exercise the fold."""
    g = torch.Generator().manual_seed(seed)
    chans = [c0] + list(dims)
    sd = {}
    for l in range(len(chans) - 1):
        cin = chans[l] + (c0 if l in res_layers else 0)
        cout = chans[l + 1]
        sd[f"filters.{l}.weight"] = torch.randn(cout, cin, 1, generator=g) / math.sqrt(cin)
        sd[f"filters.{l}.bias"] = 0.1 * torch.randn(cout, generator=g)
        if l != len(chans) - 2:
            sd[f"norms.{l}.weight"] = 1.0 + 0.1 * torch.randn(cout, generator=g)
            sd[f"norms.{l}.bias"] = 0.1 * torch.randn(cout, generator=g)
            sd[f"norms.{l}.running_mean"] = 0.1 * torch.randn(cout, generator=g)
            sd[f"norms.{l}.running_var"] = 0.5 + torch.rand(cout, generator=g)
            sd[f"norms.{l}.num_batches_tracked"] = torch.tensor(100)
    if trained_bn:
        t = torch.Generator().manual_seed(seed + 1000)
        for l in range(len(chans) - 2):
            cout = chans[l + 1]
            var = 10.0 ** (torch.rand(cout, generator=t) * 5 - 4)
            mean = 10.0 * torch.randn(cout, generator=t)
            sign = torch.where(torch.rand(cout, generator=t) < 0.5, -1.0, 1.0)
            sd[f"norms.{l}.running_var"] = var
            sd[f"norms.{l}.running_mean"] = mean
            sd[f"norms.{l}.weight"] = sign * 10.0 ** (torch.rand(cout, generator=t) * 2 - 1)
            sd[f"filters.{l}.weight"] = sd[f"filters.{l}.weight"] * var.sqrt()[:, None, None]
            sd[f"filters.{l}.bias"] = mean + var.sqrt() * sd[f"filters.{l}.bias"]
    return sd


def wide_range_features(c0, n, seed=0):
    """[1, c0, n] MLP inputs over a wide dynamic range: magnitudes log-uniform in [1e-6, 1e4] with random signs and
    about 10 % exact zeros.  In the last quarter of the points column 0 is in [-1e4, -1e3] and the other columns are
    N(0, 1): with a layer-0 weight column of one sign (positive after the BatchNorm fold) those points drive nearly
    every layer-0 unit onto the LeakyReLU negative branch."""
    g = torch.Generator().manual_seed(seed)
    mag = 10.0 ** (torch.rand(1, c0, n, generator=g, dtype=torch.float64) * 10 - 6)
    sign = torch.where(torch.rand(1, c0, n, generator=g) < 0.5, -1.0, 1.0).double()
    x = (mag * sign).float()
    x[torch.rand(1, c0, n, generator=g) < 0.1] = 0.0
    q = n - n // 4
    x[:, :, q:] = torch.randn(1, c0, n - q, generator=g)
    x[:, 0, q:] = -(10.0 ** (3 + torch.rand(n - q, generator=g)))
    return x


def feature_map(channels=12, size=128, seed=0):
    g = torch.Generator().manual_seed(seed + 7)
    return torch.randn(1, channels, size, size, generator=g)


def seeded_like(state_dict, seed):
    """Deterministic, well-scaled values for every entry of a state_dict (sorted key order):
    conv weights N(0, 1/fan_in), 1-D affine weights 1 + 0.1 N, biases / means 0.1 N,
    running_var U(0.5, 1.5)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(state_dict.keys()):
        ref = state_dict[k]
        shape = tuple(ref.shape)
        if k.endswith("num_batches_tracked"):
            out[k] = torch.tensor(100)
        elif k.endswith("running_var"):
            out[k] = 0.5 + torch.rand(shape, generator=g)
        elif len(shape) >= 2:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            out[k] = torch.randn(shape, generator=g) / math.sqrt(fan_in)
        elif k.endswith("weight"):
            out[k] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            out[k] = 0.1 * torch.randn(shape, generator=g)
    return out


def tet_body(rings=82, segs=84, seed=0, extent=(0.22, 0.42, 0.12)):
    """Tetra-SMPL stand-in (what TestDataset.compute_voxel_verts hands to the pamir prior): the star-shaped
    body_mesh inside [-0.5,0.5]^3 plus one interior vertex at the origin, every face joined to it.
    Returns (verts [V+1,3] f32, n_surface V, tets [F,4] int32, vertex_code [V,3] f32 in [0,1])."""
    verts, faces = body_mesh(rings, segs, seed, extent)
    V = len(verts)
    allv = np.concatenate([verts, np.zeros((1, 3), np.float32)], 0)
    tets = np.concatenate([faces.astype(np.int32), np.full((len(faces), 1), V, np.int32)], 1)
    lo, hi = verts.min(0, keepdims=True), verts.max(0, keepdims=True)
    code = ((verts - lo) / (hi - lo)).astype(np.float32)
    return allv.astype(np.float32), V, tets, code


def encoder_inputs_512(seed=5, size=512):
    """image / T_normal_F / T_normal_B [1,3,size,size] in [-1,1] with a centred elliptical foreground; everything
    outside the ellipse is exactly 0 in all three maps (the background NormalNet masks, lib/net/NormalNet.py:93-97)."""
    g = torch.Generator().manual_seed(seed)
    a = (torch.arange(size, dtype=torch.float32) + 0.5) / size * 2 - 1
    yy, xx = torch.meshgrid(a, a, indexing="ij")
    fg = ((xx / 0.55) ** 2 + (yy / 0.9) ** 2 < 1.0).float()[None, None]
    out = {}
    for k in ("image", "T_normal_F", "T_normal_B"):
        lo = torch.rand(1, 3, size // 8, size // 8, generator=g) * 2 - 1          # smooth part
        hi = torch.rand(1, 3, size, size, generator=g) * 2 - 1                      # pixel noise
        smooth = torch.nn.functional.interpolate(lo, size=(size, size), mode="bilinear", align_corners=False)
        out[k] = ((0.7 * smooth + 0.3 * hi).clamp(-1, 1) * fg).contiguous()
    return out


def adversarial_points(verts, faces, n_each=600, seed=0):
    """Query points that sit on the decision boundaries of cal_sdf_batch for a given mesh: exactly on vertices, on
    fp32 edge midpoints and face centroids (distance 0, many equidistant faces), points whose +x ray passes exactly
    through a vertex or an edge midpoint (same y, z; the parity ray of check_sign), and random points near the
    surface.  Returns [1, n, 3] float32."""
    rng = np.random.RandomState(seed)
    v = verts.astype(np.float32)
    f = faces.astype(np.int64)
    vi = rng.randint(len(v), size=n_each)
    fi = rng.randint(len(f), size=n_each)
    on_vert = v[vi]
    mid = ((v[f[fi, 0]] + v[f[fi, 1]]) * np.float32(0.5)).astype(np.float32)
    cen = ((v[f[fi, 0]] + v[f[fi, 1]] + v[f[fi, 2]]) / np.float32(3.0)).astype(np.float32)
    ray_v = v[vi].copy(); ray_v[:, 0] -= rng.uniform(0.01, 0.6, n_each).astype(np.float32)
    ray_e = mid.copy(); ray_e[:, 0] -= rng.uniform(0.01, 0.6, n_each).astype(np.float32)
    near = (cen + 0.02 * rng.standard_normal(cen.shape)).astype(np.float32)
    pts = np.concatenate([on_vert, mid, cen, ray_v, ray_e, near], 0).astype(np.float32)
    return torch.from_numpy(pts)[None]


SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]


def smplx_parents():
    """A 55-joint tree shaped like SMPL-X's: SMPL's first 22 body joints, jaw and two eyes under the head (15), and
    three-joint fingers under each wrist (20, 21), five per hand; the fingertips are at depth 10."""
    par = SMPL_PARENTS[:22] + [15, 15, 15]
    for wrist in (20, 21):
        for _ in range(5):
            n = len(par)
            par += [wrist, n, n + 1]
    return par


def body_model(kind="smpl", seed=0, V=None):
    """Seeded SMPL-family model arrays (float32; parents int64), for lbs (lib/smplx/lbs.py):
    "smpl": v_template = body_mesh() (V 6890, its faces under "faces"), SMPL's 24-joint tree, NB 10;
    "smplx": V 10475 points of an ellipsoidal cloud, smplx_parents() (55 joints, depth 10), NB 20;
    "tiny": V points (default 31), J 2, NB 3.
    J_regressor rows are 4 nearby vertices with positive weights summing to 1; lbs_weights rows are the at most 4
    nearest joints (inverse-distance weights summing to 1); shapedirs [V,3,NB] and posedirs [9(J-1),3V] are small
    Gaussians."""
    rng = np.random.RandomState(seed)
    out = {}
    if kind == "smpl":
        v, f = body_mesh(seed=seed)
        out["faces"] = f
        parents, NB = list(SMPL_PARENTS), 10
    elif kind == "smplx":
        v = (rng.standard_normal((10475, 3)) * np.array([0.25, 0.45, 0.12])).astype(np.float32)
        parents, NB = smplx_parents(), 20
    elif kind == "tiny":
        v = (rng.standard_normal((31 if V is None else V, 3)) * 0.3).astype(np.float32)
        parents, NB = [-1, 0], 3
    else:
        raise ValueError(f"body_model: unknown kind {kind!r}")
    out.update(model_arrays(v, parents, NB, rng))
    return out


def model_arrays(v, parents, NB, rng):
    """body_model()'s regressor, weights and blend shapes for points v [V,3] and a kinematic tree (see there)."""
    nv, J = len(v), len(parents)
    centres = rng.choice(nv, J, replace=nv < J)
    jr = np.zeros((J, nv), np.float64)
    for j, c in enumerate(centres):
        near = np.argsort(((v - v[c]) ** 2).sum(1), kind="stable")[:min(4, nv)]
        w = rng.uniform(0.5, 1.5, len(near))
        jr[j, near] = w / w.sum()
    joints = jr @ v.astype(np.float64)
    d = np.sqrt(((v[:, None, :].astype(np.float64) - joints[None]) ** 2).sum(-1))
    lw = np.zeros((nv, J), np.float64)
    near = np.argsort(d, 1, kind="stable")[:, :min(4, J)]
    w = 1.0 / (np.take_along_axis(d, near, 1) + 0.05)
    np.put_along_axis(lw, near, w / w.sum(1, keepdims=True), 1)
    return dict(v_template=v.astype(np.float32), J_regressor=jr.astype(np.float32), lbs_weights=lw.astype(np.float32),
               shapedirs=(0.01 * rng.standard_normal((nv, 3, NB))).astype(np.float32),
               posedirs=(0.01 * rng.standard_normal((9 * (J - 1), 3 * nv))).astype(np.float32),
               parents=np.asarray(parents, np.int64))


PIXIE_SIZES = {"tiny": dict(rings=8, segs=12, V=98, F=192, n_shape=10, n_exp=10),
               "real": dict(rings=100, segs=104, V=10475, F=20908, n_shape=200, n_exp=50)}
# PIXIE's J14 regressor rows written over SMPL-X joints: SMPLX.__init__'s (source, target) pairs for its
# keypoint_names and J14_NAMES (lib/pixielib/models/SMPLX.py:186-198)
PIXIE_J14_SOURCE = [1, 2, 4, 5, 7, 8, 12, 15, 16, 17, 18, 19, 20, 21]
PIXIE_J14_TARGET = [3, 2, 4, 1, 5, 0, 12, 13, 9, 8, 10, 7, 11, 6]
PIXIE_HEAD_CHAIN = [15, 12, 9, 6, 3, 0]


def pixie_model(kind="tiny", seed=0, grid=None):
    """Seeded arrays shaped like PIXIE's SMPL-X model file and side files (lib/pixielib/models/SMPLX.py:114-202):
    v_template [V,3], f [F,3], shapedirs [V,3,300 + n_exp] (the class keeps [:n_shape] and [300:300 + n_exp]; the
    columns between are zero), posedirs [V,3,9(J-1)] (the file's layout), J_regressor [J,V], kintree_table [2,J],
    weights [V,J], lmk_faces_idx [51], lmk_bary_coords [51,3], dynamic_lmk_faces_idx [79,17],
    dynamic_lmk_bary_coords [79,17,3], the extra joints' face_ids [22] / bcs [22,3] and the J14 regressor [14,V];
    n_shape, n_exp.  "tiny": body_mesh(8, 12) (V 98, F 192), n_shape = n_exp = 10; "real": V 10 475, F 20 908,
    n_shape 200, n_exp 50 (a closed body_mesh plus loose vertices and faces to SMPL-X's counts).  J = 55 (the
    smplx_parents() tree).  `grid`: round blend shapes to multiples of 2^-grid.  Barycentrics are positive and sum
    to about 1."""
    z = PIXIE_SIZES[kind]
    rng = np.random.RandomState(seed)
    v, f = body_mesh(rings=z["rings"], segs=z["segs"], seed=seed)
    extra_v = z["V"] - len(v)
    if extra_v:
        v = np.concatenate([v, (0.05 * rng.standard_normal((extra_v, 3)) + [0.0, 0.85, 0.1]).astype(np.float32)], 0)
        lo = z["V"] - extra_v
        tri = np.stack([rng.choice(extra_v, 3, replace=False) + lo for _ in range(z["F"] - len(f))])
        f = np.concatenate([f, tri.astype(np.int64)], 0)
    parents = smplx_parents()
    J, ns, ne = len(parents), z["n_shape"], z["n_exp"]
    m = model_arrays(v, parents, ns + ne, rng)
    sd = np.zeros((z["V"], 3, 300 + ne), np.float32)
    sd[:, :, :ns], sd[:, :, 300:] = m["shapedirs"][:, :, :ns], m["shapedirs"][:, :, ns:]
    pd = m["posedirs"]
    if grid is not None:
        sd = (np.round(sd.astype(np.float64) * 2.0 ** grid) / 2.0 ** grid).astype(np.float32)
        pd = (np.round(pd.astype(np.float64) * 2.0 ** grid) / 2.0 ** grid).astype(np.float32)
    F = len(f)

    def bary(*shape):
        w = rng.uniform(0.05, 1.0, shape + (3,))
        return (w / w.sum(-1, keepdims=True)).astype(np.float32)
    j14 = np.zeros((14, z["V"]), np.float64)
    for r in range(14):
        near = rng.choice(z["V"], 6, replace=False)
        w = rng.uniform(0.2, 1.0, 6)
        j14[r, near] = w / w.sum()
    kin = np.stack([np.asarray(parents, np.int64), np.arange(J, dtype=np.int64)])
    kin[0, 0] = 4294967295                     # the file's root entry; the class sets parents[0] = -1
    return dict(v_template=v.astype(np.float32), f=f.astype(np.int64), shapedirs=sd,
                posedirs=pd.T.reshape(z["V"], 3, 9 * (J - 1)).copy(), J_regressor=m["J_regressor"],
                kintree_table=kin, weights=m["lbs_weights"], lmk_faces_idx=rng.randint(0, F, 51).astype(np.int64),
                lmk_bary_coords=bary(51), dynamic_lmk_faces_idx=rng.randint(0, F, (79, 17)).astype(np.int64),
                dynamic_lmk_bary_coords=bary(79, 17), face_ids=rng.randint(0, F, 22).astype(np.int64), bcs=bary(22),
                j14_regressor=j14.astype(np.float32), n_shape=ns, n_exp=ne)


def pixie_buffers(arr):
    """The buffers PIXIE's SMPLX.__init__ registers from pixie_model() arrays (float32 / int64 numpy), by the same
    slicing and reshapes: v_template, shapedirs [V,3,n_shape + n_exp], posedirs [9(J-1),3V], J_regressor, parents,
    lbs_weights, faces_tensor, the landmark tables, head_kin_chain, face_ids, bcs, extra_joint_regressor,
    source_idxs, target_idxs."""
    ns, ne = arr["n_shape"], arr["n_exp"]
    P = arr["posedirs"].shape[-1]
    parents = arr["kintree_table"][0].astype(np.int64).copy()
    parents[0] = -1
    return dict(v_template=arr["v_template"], shapedirs=np.concatenate([arr["shapedirs"][:, :, :ns],
                                                                         arr["shapedirs"][:, :, 300:300 + ne]], 2),
                posedirs=np.ascontiguousarray(arr["posedirs"].reshape(-1, P).T), J_regressor=arr["J_regressor"],
                parents=parents, lbs_weights=arr["weights"], faces_tensor=arr["f"],
                lmk_faces_idx=arr["lmk_faces_idx"], lmk_bary_coords=arr["lmk_bary_coords"],
                dynamic_lmk_faces_idx=arr["dynamic_lmk_faces_idx"],
                dynamic_lmk_bary_coords=arr["dynamic_lmk_bary_coords"],
                head_kin_chain=np.asarray(PIXIE_HEAD_CHAIN, np.int64), face_ids=arr["face_ids"], bcs=arr["bcs"],
                extra_joint_regressor=arr["j14_regressor"], source_idxs=np.asarray(PIXIE_J14_SOURCE, np.int64),
                target_idxs=np.asarray(PIXIE_J14_TARGET, np.int64))


def pixie_smplx_standin():
    """A fresh class standing in for PIXIE's SMPLX (lib/pixielib/models/SMPLX.py) where no checkout exists, for
    body_model.make_pixie_SMPLX to patch: `__init__(buffers, n_shape)` registers what the reference's `__init__` registers,
    from pixie_buffers() arrays (the extra joints under `extra_joint_selector`, the default poses and parameters as
    identities and zeros) and calls `super(SMPLX, self).__init__()` as the reference does; `forward(*args)` records
    its arguments in the class's `calls` list and returns "reference"."""
    import torch.nn as nn

    class SMPLX(nn.Module):
        calls = []

        def __init__(self, buffers, n_shape=10):
            super(SMPLX, self).__init__()
            for k, v in buffers.items():
                if k not in ("face_ids", "bcs"):
                    self.register_buffer(k, torch.as_tensor(np.asarray(v)).clone())
            self.extra_joint_selector = nn.Module()
            for k in ("face_ids", "bcs"):
                self.extra_joint_selector.register_buffer(k, torch.as_tensor(np.asarray(buffers[k])).clone())
            ne = int(np.asarray(buffers["shapedirs"]).shape[2]) - n_shape
            self.register_buffer("shape_params", torch.zeros(1, n_shape))
            self.register_buffer("expression_params", torch.zeros(1, ne))
            for k, n in (("global_pose", 1), ("body_pose", 21), ("jaw_pose", 1), ("eye_pose", 2),
                         ("left_hand_pose", 15), ("right_hand_pose", 15)):
                self.register_buffer(k, torch.eye(3)[None].repeat(n, 1, 1))
            self.use_joint_regressor = True

        def forward(self, *args):
            SMPLX.calls.append(args)
            return "reference"

    return SMPLX


TETRA_SIZES = {"tiny": dict(rings=4, segs=6, V_added=7, T=60),
               "smpl": dict(rings=82, segs=84, V_added=1110, T=25100)}
TETRA_FILES = ("smpl/SMPL_NEUTRAL.pkl", "tetra_neutral_adult_smpl.npz", "tetrahedrons_neutral_adult.txt")


def tetra_model(kind="tiny", seed=0, folder=None):
    """Seeded arrays of PaMIR's tetrahedral SMPL (lib/dataset/body_model.py:234-306), float64 on a 2^-20 grid (so
    they do not depend on the machine's libm): the SMPL pkl's v_template [V,3], f, J_regressor (scipy csc [24,V], 4
    to 8 nearby vertices per joint, as SMPL's file stores it), weights [V,24], posedirs [V,3,207], shapedirs
    [V,3,10], kintree_table [2,24] (SMPL's tree, root entry 4294967295); the tetra npz's v_template_added [Va,3],
    weights_added, shapedirs_added, posedirs_added, tetrahedrons; and `tets` [T,4], the 1-based text file's rows.
    Built on tet_body: "tiny" is tet_body(4, 6) (V 26) with 7 added vertices and 60 tetrahedra; "smpl" is
    tet_body() (V 6890) with V + V_added = 8000 and T = 25100, the padded sizes TestDataset.compute_voxel_verts
    allots, exactly.  The added vertices are the interior one at the origin and shrunken surface vertices; the extra
    tetrahedra join surface faces to them.  With `folder`, writes the three files under TETRA_FILES' names and
    returns their paths as well."""
    import pickle

    import scipy.sparse as sp
    z = TETRA_SIZES[kind]
    rng = np.random.RandomState(seed)
    allv, V, tets, _ = tet_body(rings=z["rings"], segs=z["segs"], seed=seed)
    surf = allv[:V].astype(np.float64)
    Va, F = z["V_added"], len(tets)
    shrink = 0.5 * surf[rng.choice(V, Va - 1, replace=False)]
    va = np.concatenate([np.zeros((1, 3)), shrink], 0)
    extra = tets[rng.choice(F, z["T"] - F, replace=F < z["T"] - F)].copy()
    extra[:, 3] = V + 1 + rng.randint(0, Va - 1, len(extra))
    tets = np.concatenate([tets, extra], 0).astype(np.int64)
    q = lambda x: np.round(np.asarray(x, np.float64) * 2.0 ** 20) / 2.0 ** 20   # noqa: E731
    both = np.concatenate([surf, va], 0)
    m = model_arrays(both.astype(np.float32), SMPL_PARENTS, 10, rng)
    jr = np.zeros((24, V))
    for j in range(24):
        near = np.argsort(((surf - surf[rng.randint(V)]) ** 2).sum(1), kind="stable")[:rng.randint(4, 9)]
        w = rng.uniform(0.5, 1.5, len(near))
        jr[j, near] = w / w.sum()
    pd = m["posedirs"].T.reshape(V + Va, 3, 207)
    kin = np.stack([np.asarray(SMPL_PARENTS, np.int64), np.arange(24, dtype=np.int64)])
    kin[0, 0] = 4294967295
    out = dict(v_template=q(surf), f=tets[:F, :3].copy(), J_regressor=sp.csc_matrix(q(jr)),
               weights=q(m["lbs_weights"][:V]), posedirs=q(pd[:V]), shapedirs=q(m["shapedirs"][:V]),
               kintree_table=kin, v_template_added=q(va), weights_added=q(m["lbs_weights"][V:]),
               shapedirs_added=q(m["shapedirs"][V:]), posedirs_added=q(pd[V:]), tetrahedrons=tets,
               tets=tets + 1)
    if folder is None:
        return out
    import os
    paths = tuple(os.path.join(folder, n) for n in TETRA_FILES)
    os.makedirs(os.path.dirname(paths[0]), exist_ok=True)
    with open(paths[0], "wb") as fh:
        pickle.dump({k: out[k] for k in ("v_template", "f", "J_regressor", "weights", "posedirs", "shapedirs",
                                         "kintree_table")}, fh, protocol=2)
    np.savez(paths[1], **{k: out[k] for k in ("v_template_added", "weights_added", "shapedirs_added",
                                              "posedirs_added", "tetrahedrons")})
    np.savetxt(paths[2], out["tets"], fmt="%d")
    return out, paths


# ---------------------------------------------------------------- PyMAF (lib/pymaf/models/pymaf_net.py)

PYMAF_DMAP_SIZES = (6890, 1723, 431)


def pymaf_tables(seed=0):
    """Seeded SMPL tables PyMAF reads besides the body model (float32 unless stated): J_regressor_extra [9,6890]
    (rows of 4 nearby vertices, positive weights summing to 1), the two sparse downsampling matrices D0 [1723,6890]
    and D1 [431,1723] (rows of 1..3 positive weights summing to 1) and their product Dmap [431,6890], 21 vertex-joint
    ids (int64, distinct), a joint_map of 49 entries into the 54 [24 lbs, 21 vertex, 9 extra] joints (int64), and the
    mean parameters pose [144] (6-D rotations near the identity), shape [10] and cam [3] (scale near 0.9)."""
    rng = np.random.RandomState(seed + 7001)
    bm = body_model("smpl", seed=seed)
    v = bm["v_template"].astype(np.float64)
    nv = len(v)
    jx = np.zeros((9, nv), np.float64)
    for r, c in enumerate(rng.choice(nv, 9, replace=False)):
        near = np.argsort(((v - v[c]) ** 2).sum(1), kind="stable")[:4]
        w = rng.uniform(0.5, 1.5, 4)
        jx[r, near] = w / w.sum()
    D = []
    for rows, cols in ((PYMAF_DMAP_SIZES[1], PYMAF_DMAP_SIZES[0]), (PYMAF_DMAP_SIZES[2], PYMAF_DMAP_SIZES[1])):
        d = np.zeros((rows, cols), np.float32)
        for r in range(rows):
            k = rng.randint(1, 4)
            w = rng.uniform(0.5, 1.5, k)
            d[r, rng.choice(cols, k, replace=False)] = w / w.sum()
        D.append(d)
    eye6 = np.tile(np.array([1, 0, 0, 1, 0, 0], np.float32), 24)
    return dict(body=bm, J_regressor_extra=jx.astype(np.float32), D=D,
                Dmap=(D[1].astype(np.float64) @ D[0].astype(np.float64)).astype(np.float32),
                vertex_ids=np.sort(rng.choice(nv, 21, replace=False)).astype(np.int64),
                joint_map=rng.choice(54, 49, replace=False).astype(np.int64),
                pose=(eye6 + 0.1 * rng.standard_normal(144)).astype(np.float32),
                shape=(0.5 * rng.standard_normal(10)).astype(np.float32),
                cam=np.array([0.9, 0.05, 0.2], np.float32) + (0.02 * rng.standard_normal(3)).astype(np.float32))


def pymaf_state_dict(seed=0, tables=None):
    """Every key and shape of PyMAF's state_dict (res50 backbone, three k4 deconvolutions of 256 channels, three MAF
    extractors with MLP_DIM [256, 128, 64, 5], three regressors with their SMPL, dp_head), seeded with NumPy's
    RandomState: He-scaled convolutions; trained-like BatchNorms (running mean ~ N(0, 0.1), variance U(0.5, 1.5),
    gamma U(0.5, 1.5) and U(0.2, 1) for the last BN of each block, beta ~ N(0, 0.1)); MAF and fc layers uniform in
    +-1 / sqrt(fan_in) (torch's defaults); decpose / decshape / deccam xavier-uniform with gain 0.01.  The SMPL
    buffers and mean parameters come from pymaf_tables(seed)."""
    rng = np.random.RandomState(seed)
    T = pymaf_tables(seed) if tables is None else tables
    sd = {}

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a))

    def conv(name, cout, cin, k):
        sd[name] = t((rng.standard_normal((cout, cin, k, k)) * math.sqrt(2.0 / (cin * k * k))).astype(np.float32))

    def bn(name, c, last=False):
        sd[name + ".weight"] = t(rng.uniform(0.2, 1.0, c) if last else rng.uniform(0.5, 1.5, c)).float()
        sd[name + ".bias"] = t(0.1 * rng.standard_normal(c)).float()
        sd[name + ".running_mean"] = t(0.1 * rng.standard_normal(c)).float()
        sd[name + ".running_var"] = t(rng.uniform(0.5, 1.5, c)).float()
        sd[name + ".num_batches_tracked"] = torch.tensor(0, dtype=torch.int64)

    def uni(shape, fan_in, gain=None, fan_out=None):
        b = 1.0 / math.sqrt(fan_in) if gain is None else gain * math.sqrt(6.0 / (fan_in + fan_out))
        return t(rng.uniform(-b, b, shape).astype(np.float32))

    fe = "feature_extractor."
    conv(fe + "conv1.weight", 64, 3, 7)
    bn(fe + "bn1", 64)
    inplanes = 64
    for li, (planes, n) in enumerate(zip((64, 128, 256, 512), (3, 4, 6, 3))):
        for b in range(n):
            pre = f"{fe}layer{li + 1}.{b}."
            conv(pre + "conv1.weight", planes, inplanes, 1)
            bn(pre + "bn1", planes)
            conv(pre + "conv2.weight", planes, planes, 3)
            bn(pre + "bn2", planes)
            conv(pre + "conv3.weight", planes * 4, planes, 1)
            bn(pre + "bn3", planes * 4, last=True)
            if b == 0:
                conv(pre + "downsample.0.weight", planes * 4, inplanes, 1)
                bn(pre + "downsample.1", planes * 4, last=True)
            inplanes = planes * 4
    for i in range(3):
        cin = inplanes if i == 0 else 256
        sd[f"deconv_layers.{3 * i}.weight"] = t((rng.standard_normal((cin, 256, 4, 4))
                                                  * math.sqrt(2.0 / (cin * 4))).astype(np.float32))
        bn(f"deconv_layers.{3 * i + 1}", 256)
    bm = T["body"]
    for i in range(3):
        m = f"maf_extractor.{i}."
        for k, (cout, cin) in enumerate(((128, 256), (64, 384), (5, 320))):
            sd[m + f"conv{k}.weight"] = uni((cout, cin, 1), cin)
            sd[m + f"conv{k}.bias"] = uni((cout,), cin)
        sd[m + "Dmap"] = t(T["Dmap"])
    lin = torch.linspace(-1, 1, 21)
    xv, yv = torch.meshgrid([lin, lin], indexing="ij")
    sd["points_grid"] = torch.stack([xv.reshape(-1), yv.reshape(-1)]).unsqueeze(0)
    for i in range(3):
        r = f"regressor.{i}."
        feat = 441 * 5 if i == 0 else 431 * 5
        for name, (cout, cin) in (("fc1", (1024, feat + 157)), ("fc2", (1024, 1024))):
            sd[r + name + ".weight"] = uni((cout, cin), cin)
            sd[r + name + ".bias"] = uni((cout,), cin)
        for name, cout in (("decpose", 144), ("decshape", 10), ("deccam", 3)):
            sd[r + name + ".weight"] = uni((cout, 1024), 1024, gain=0.01, fan_out=cout)
            sd[r + name + ".bias"] = uni((cout,), 1024)
        s = r + "smpl."
        sd[s + "betas"] = torch.zeros(64, 10)
        sd[s + "global_orient"] = torch.zeros(64, 3)
        sd[s + "body_pose"] = torch.zeros(64, 69)
        sd[s + "faces_tensor"] = t(bm["faces"].astype(np.int64))
        sd[s + "v_template"] = t(bm["v_template"])
        sd[s + "shapedirs"] = t(bm["shapedirs"])
        sd[s + "J_regressor"] = t(bm["J_regressor"])
        sd[s + "posedirs"] = t(bm["posedirs"])
        sd[s + "parents"] = t(bm["parents"])
        sd[s + "lbs_weights"] = t(bm["lbs_weights"])
        sd[s + "vertex_joint_selector.extra_joints_idxs"] = t(T["vertex_ids"])
        sd[s + "J_regressor_extra"] = t(T["J_regressor_extra"])
        sd[r + "init_pose"] = t(T["pose"][None])
        sd[r + "init_shape"] = t(T["shape"][None])
        sd[r + "init_cam"] = t(T["cam"][None])
    for name, cout in (("predict_u", 25), ("predict_v", 25), ("predict_ann_index", 15), ("predict_uv_index", 25)):
        sd[f"dp_head.{name}.weight"] = uni((cout, 256, 3, 3), 256 * 9)
        sd[f"dp_head.{name}.bias"] = uni((cout,), 256 * 9)
    return sd


def pymaf_image(seed=0):
    """An ImageNet-normalised-looking [1,3,224,224] float32 image: a smooth seeded field plus noise."""
    rng = np.random.RandomState(seed + 9100)
    yy, xx = np.meshgrid(np.linspace(-1, 1, 224), np.linspace(-1, 1, 224), indexing="ij")
    img = np.stack([np.sin(3 * xx + c) * np.cos(2 * yy - c) for c in range(3)])
    img = img + 0.3 * rng.standard_normal((3, 224, 224))
    return torch.from_numpy(img[None].astype(np.float32))


PYMAF_PARAMETERS = ("weight", "bias", "betas", "global_orient", "body_pose")


def pymaf_standin(state_dict, joint_map, cfg):
    """A fresh class standing in for the reference's PyMAF where no checkout exists: a module tree whose state_dict
    has exactly `state_dict`'s keys (`weight` / `bias` and SMPL's betas / pose are parameters that require grad, as
    in the reference's module, every other tensor a buffer; numeric children as ModuleLists so that
    `regressor[i].smpl.joint_map` resolves), a `forward(x, J_regressor=None)` that records its calls and returns
    "reference", and `cfg` bound in a module of its own, as lib.pymaf.models.pymaf_net binds it."""
    import sys
    import types
    from torch import nn

    mod = types.ModuleType(f"icon_b200_pymaf_standin_{len([m for m in sys.modules if 'pymaf_standin' in m])}")
    mod.cfg = cfg
    sys.modules[mod.__name__] = mod

    def tree(names):
        kids = {}
        for k in names:
            head, _, rest = k.partition(".")
            kids.setdefault(head, []).append(rest)
        return kids

    def build(m, prefix, names):
        for head, rests in tree(names).items():
            if rests == [""]:
                t = state_dict[prefix + head].clone()
                if head in PYMAF_PARAMETERS and t.is_floating_point() and "running" not in head:
                    m.register_parameter(head, nn.Parameter(t))
                else:
                    m.register_buffer(head, t)
                continue
            sub = tree(rests)
            if all(h.isdigit() for h in sub):
                child = nn.ModuleList([nn.Module() for _ in range(max(int(h) for h in sub) + 1)])
                for h, rs in sub.items():
                    build(child[int(h)], f"{prefix}{head}.{h}.", rs)
            else:
                child = nn.Module()
                build(child, f"{prefix}{head}.", rests)
            m.add_module(head, child)

    class PyMAF(nn.Module):
        calls = []

        def __init__(self):
            super().__init__()
            build(self, "", list(state_dict))
            for r in self.regressor:
                r.smpl.joint_map = torch.as_tensor(joint_map).long()

        def forward(self, x, J_regressor=None):
            PyMAF.calls.append((x, J_regressor))
            return "reference"

    PyMAF.__module__ = mod.__name__
    mod.PyMAF = PyMAF
    return PyMAF


def pymaf_cfg():
    """The shipped lib/pymaf/configs/pymaf_config.yaml values PyMAF reads, as attribute namespaces."""
    from types import SimpleNamespace as NS
    return NS(MODEL=NS(PyMAF=NS(BACKBONE="res50", MLP_DIM=[256, 128, 64, 5], N_ITER=3, AUX_SUPV_ON=True)),
              RES_MODEL=NS(DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[256, 256, 256],
                           NUM_DECONV_KERNELS=[4, 4, 4]),
              LOSS=NS(POINT_REGRESSION_WEIGHTS=0.5))


PYMAF_FILES = ("smpl_related/models/smpl/SMPL_NEUTRAL.pkl", "pymaf_data/J_regressor_extra.npy",
               "pymaf_data/mesh_downsampling.npz", "pymaf_data/smpl_mean_params.npz")


def pymaf_files(folder, seed=0):
    """Write, under `folder`, the model files PyMAF loads (PYMAF_FILES), at the real sizes, from pymaf_tables(seed):
    SMPL_NEUTRAL.pkl (plain NumPy arrays: v_template, f, J_regressor, weights, posedirs [V,3,207], shapedirs [V,3,10],
    kintree_table with the root entry 4294967295), J_regressor_extra.npy [9,6890], mesh_downsampling.npz (D: the two
    sparse downsampling matrices; U: their transposes; A: the adjacency of the three levels as sparse identities) and
    smpl_mean_params.npz (pose [144], shape [10], cam [3], float32).  Returns (tables, paths)."""
    import os
    import pickle

    import scipy.sparse as sp
    T = pymaf_tables(seed)
    bm = T["body"]
    V = len(bm["v_template"])
    paths = tuple(os.path.join(folder, n) for n in PYMAF_FILES)
    for p in paths:
        os.makedirs(os.path.dirname(p), exist_ok=True)
    kin = np.stack([np.asarray(SMPL_PARENTS, np.int64), np.arange(24, dtype=np.int64)])
    kin[0, 0] = 4294967295
    with open(paths[0], "wb") as fh:
        pickle.dump(dict(v_template=bm["v_template"].astype(np.float64), f=bm["faces"].astype(np.int64),
                         J_regressor=sp.csc_matrix(bm["J_regressor"].astype(np.float64)),
                         weights=bm["lbs_weights"].astype(np.float64),
                         posedirs=bm["posedirs"].T.reshape(V, 3, -1).astype(np.float64),
                         shapedirs=bm["shapedirs"].astype(np.float64), kintree_table=kin), fh, protocol=2)
    np.save(paths[1], T["J_regressor_extra"])

    def objs(xs):
        a = np.empty(len(xs), dtype=object)
        for i, x in enumerate(xs):
            a[i] = x
        return a
    D = [sp.csr_matrix(d) for d in T["D"]]
    np.savez(paths[2], D=objs(D), U=objs([d.T.tocsr() for d in D]),
             A=objs([sp.identity(n, format="csr", dtype=np.float32) for n in PYMAF_DMAP_SIZES]))
    np.savez(paths[3], pose=T["pose"], shape=T["shape"], cam=T["cam"])
    return T, paths


def pymaf_sha256(state_dict):
    """SHA-256 over the state dict's keys, dtypes, shapes and bytes in key order: seed drift fails loudly."""
    import hashlib
    h = hashlib.sha256()
    for k in sorted(state_dict):
        t = state_dict[k].detach().cpu().contiguous()
        h.update(k.encode())
        h.update(str(t.dtype).encode())
        h.update(str(tuple(t.shape)).encode())
        h.update(t.numpy().tobytes())
    return h.hexdigest()
