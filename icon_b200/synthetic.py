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
