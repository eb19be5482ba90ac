"""Marching cubes (csrc/mc.cu) and clean_mesh (csrc/clean.cu) at their edges, index-exact against the oracle.

Marching cubes: fields that reach the volume border (the cropped occ[0] shell and the zero shells of the padded branch,
an open surface in the plain branch), nodes exactly on the iso value, NaN / +-inf nodes, every cube case, the densest
field (a 3-D checkerboard: every cell ambiguous, the most vertices and triangles a 1024-voxel block can carry), grid
sizes giving every G mod 4 on both sides of the 256^3 branch switch, and iso values fp32 cannot represent.  Faces
compare with array_equal, vertices bit for bit through an integer view (NaN positions compare as NaN).

clean_mesh: hand-built non-manifold meshes (tests/test_mesh_cpu.py), order="lex" meshes, the fields above, fp64
vertices, thousands of tied components and a 513^3 surface, against oracle/mesh.py (trimesh's split restated).
"""
import numpy as np
import pytest
import torch

from oracle import mcubes as OM
from oracle.mc_table import NUM_VERTS
from oracle import mesh as OMesh
from test_mesh_cpu import HAND_MESHES

pytestmark = pytest.mark.gpu

LEVELS = np.array([0.0, 0.25, 0.5, 0.75, 1.0], np.float32)


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _grid(R):
    a = np.linspace(-1.0, 1.0, R)
    return np.meshgrid(a, a, a, indexing="ij")             # z, y, x


def _same_bits(a, b):
    """Equal dtype, shape and bits; NaN matches NaN whatever its payload (the GPU writes one canonical NaN)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    it = np.int64 if a.dtype == np.float64 else np.int32
    return np.array_equal(na, nb) and np.array_equal(np.where(na, 0, a.view(it)), np.where(nb, 0, b.view(it)))


def _oracle(occ, iso=0.5, order="edge"):
    """export_mesh restated with `iso` in both branches (the kaolin branch at any iso, in fp32)."""
    final = np.ascontiguousarray(occ[1:, 1:, 1:])
    pad = final.shape[0] <= 256
    with np.errstate(invalid="ignore", divide="ignore"):
        v, f = OM.marching_cubes(final, iso, pad=pad, dtype=np.float32 if pad else np.float64)
    if order == "lex":
        v, f = OM.lexicographic_merge(v, f)
    return v[:, [2, 1, 0]], f[:, [0, 2, 1]]


def _check(occ, iso=0.5, order="edge"):
    """ops.marching_cubes(occ, iso, order) == the oracle, index-exact; returns the oracle's (verts, faces)."""
    from icon_b200 import ops
    occ = np.ascontiguousarray(occ, np.float32)
    v, f = ops.marching_cubes(torch.from_numpy(occ).to(_cuda()), iso, order=order)
    rv, rf = _oracle(occ, iso, order)
    plain = occ.shape[0] - 1 > 256
    assert v.dtype == (torch.float64 if plain else torch.float32) and f.dtype == torch.int64
    assert np.array_equal(f.cpu().numpy(), rf)
    assert _same_bits(v.cpu().numpy(), rv)
    if iso == 0.5 and order == "edge":
        ev, ef = OM.export_mesh(occ, 0.5) if np.isfinite(occ).all() else (rv, rf)
        assert np.array_equal(ef, rf) and _same_bits(ev, rv)
    return rv, rf


def _edge_use(f):
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    k, c = np.unique(e[:, 0] * (int(f.max()) + 1) + e[:, 1], return_counts=True)
    return np.stack(np.divmod(k, int(f.max()) + 1), 1), c


def _assert_closed(f):
    _, c = _edge_use(f)
    assert (c == 2).all()


def _assert_open_only_on_the_border(v, f, R):
    """Plain branch: edges used once lie on the grid's outer faces (coordinate 0 or G - 1 = R - 2 on one axis)."""
    e, c = _edge_use(f)
    b = e[c == 1]
    assert len(b) > 0 and (c <= 2).all()
    pa, pb = v[b[:, 0]], v[b[:, 1]]
    on = ((pa == 0) & (pb == 0)) | ((pa == R - 2) & (pb == R - 2))
    assert on.any(axis=1).all()


# --------------------------------------------------------------------------- fields
def _ramp(R, axis, sign):
    c = _grid(R)[2 - axis]                                  # axis 0 = x
    return (0.5 + sign * 0.9 * (c - 0.137)).astype(np.float32)


def _slab(R):
    z, y, x = _grid(R)
    return (0.5 + 0.8 * (0.6 - np.abs(x + y + z - 0.1))).astype(np.float32)


def _all_inside(R):
    rng = np.random.default_rng(R)
    return (0.8 + 0.2 * rng.random((R, R, R))).astype(np.float32)


def _only_cropped_planes(R):
    occ = np.zeros((R, R, R), np.float32)
    occ[0], occ[:, 0], occ[:, :, 0] = 1.0, 0.9, 0.8
    return occ


def _corner_blob(R, s):
    z, y, x = _grid(R)
    return (0.5 + 1.5 * (0.9 - np.sqrt((x - s) ** 2 + (y - s) ** 2 + (z - s) ** 2))).astype(np.float32)


def _offset_blob(R, seed=0, noise=0.05):
    """a sphere that crosses the volume border on three faces, plus noise (ambiguous cases)"""
    z, y, x = _grid(R)
    occ = 0.5 + 1.5 * (0.85 - np.sqrt((x - 0.35) ** 2 + (y + 0.2) ** 2 + (z - 0.4) ** 2))
    return (occ + noise * np.random.default_rng(seed).standard_normal(occ.shape)).astype(np.float32)


def _quantised(R, density, seed, box=None):
    """values in {0, 0.25, 0.5, 0.75, 1}: nodes on iso (t = 0 / t = 1, coincident vertices); `box` = the corner
    sub-box holding them (the rest 0) for plain-branch sizes"""
    rng = np.random.default_rng(seed)
    n = box or R
    q = rng.choice(LEVELS, size=(n, n, n), p=[1 - density, density / 4, density / 4, density / 4, density / 4])
    occ = np.zeros((R, R, R), np.float32)
    occ[R - n:, :n, R - n:] = q                             # touches three outer faces
    return occ


BORDER = {
    **{f"ramp_{'xyz'[a]}{'+' if s > 0 else '-'}": (lambda R, a=a, s=s: _ramp(R, a, s)) for a in range(3) for s in (1, -1)},
    "slab": _slab,
    "all_inside": _all_inside,
    "only_cropped_planes": _only_cropped_planes,
    "corner_blob_lo": lambda R: _corner_blob(R, -1.0),
    "corner_blob_hi": lambda R: _corner_blob(R, 1.0),
}


# --------------------------------------------------------------------------- marching cubes
@pytest.mark.parametrize("R", [33, 259])
@pytest.mark.parametrize("name", sorted(BORDER))
def test_mc_surface_at_the_volume_border(name, R):
    occ = BORDER[name](R)
    rv, rf = _check(occ)
    if name == "only_cropped_planes" or (name == "all_inside" and R > 257):
        assert len(rf) == 0                                 # cropped away / no level crossing without the zero pad
        return
    assert len(rf) > 0
    if R - 1 <= 256:
        _assert_closed(rf)                                  # the zero shells close every surface
    else:
        _assert_open_only_on_the_border(rv, rf, R)


@pytest.mark.parametrize("order", ["edge", "lex"])
@pytest.mark.parametrize("density", [0.1, 0.3, 0.5])
@pytest.mark.parametrize("R", [12, 33, 259])
def test_mc_iso_valued_nodes(R, density, order):
    occ = _quantised(R, density, seed=R + int(100 * density), box=24 if R > 257 else None)
    rv, rf = _check(occ, order=order)
    assert len(rf) > 0
    if order == "edge" and R <= 257:
        _assert_closed(rf)


def test_mc_iso_valued_nodes_existing_lex_field():
    """the field of test_marching_cubes_lexicographic_order_contract with many more nodes on the level set"""
    z, y, x = _grid(41)
    occ = (0.5 + (0.6 - np.sqrt(x * x + y * y + z * z))).astype(np.float32)
    occ[::4, ::3, ::2] = np.where(np.abs(occ[::4, ::3, ::2] - 0.5) < 0.1, 0.5, occ[::4, ::3, ::2])
    for order in ("edge", "lex"):
        _check(occ, order=order)


def _nearest_to_iso(occ, box):
    sub = np.abs(occ[box] - 0.5)
    idx = np.unravel_index(np.argmin(sub), sub.shape)
    return tuple(s.start + i for s, i in zip(box, idx))


@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf], ids=["nan", "+inf", "-inf"])
@pytest.mark.parametrize("R", [33, 259])
def test_mc_non_finite_nodes(R, value):
    """NaN is not below iso, +-inf compare as themselves, t follows IEEE (inf / inf = NaN): one node at a time on the
    first and last kept layer and in the interior, then all of them at once."""
    occ = _offset_blob(R, seed=R, noise=0.0)
    full = slice(1, R)
    nodes = [_nearest_to_iso(occ, (slice(R - 1, R), full, full)), _nearest_to_iso(occ, (full, slice(1, 2), full)),
             _nearest_to_iso(occ, (slice(R // 4, 3 * R // 4),) * 3)]
    for n in nodes:
        o = occ.copy()
        o[n] = value
        _check(o)
    o = occ.copy()
    for n in nodes:
        o[n] = value
    rv, _ = _check(o)
    if np.isnan(value):
        assert np.isnan(rv).any()


def test_mc_every_cube_case():
    rng = np.random.default_rng(7)
    for R, p in ((33, 0.5), (33, 0.3), (259, 0.5)):
        occ = np.zeros((R, R, R), np.float32)
        n = min(R, 40)
        occ[:n, :n, :n] = (rng.random((n, n, n)) < p).astype(np.float32)
        final = occ[1:, 1:, 1:]
        hist = np.bincount(OM.cube_cases(final, 0.5, pad=R - 1 <= 256, dtype=np.float64).ravel(), minlength=256)
        assert (hist > 0).all(), np.flatnonzero(hist == 0)
        _check(occ)


@pytest.mark.parametrize("R,box", [(129, None), (259, 64)])
def test_mc_checkerboard_densest_blocks(R, box):
    """every cell ambiguous: 3 vertices per voxel and 4 triangles per cell, i.e. 3072 vertices and 4096 triangles
    per interior 1024-voxel block, which k_mc_count packs into 16-bit halves"""
    n = box or R
    i, j, k = np.indices((n, n, n))
    occ = np.zeros((R, R, R), np.float32)
    occ[:n, :n, :n] = ((i + j + k) % 2).astype(np.float32)
    rv, rf = _check(occ)
    cases = np.unique(OM.cube_cases(occ[1:n, 1:n, 1:n], 0.5, pad=False))
    assert len(cases) == 2 and cases.sum() == 255 and (np.asarray(NUM_VERTS)[cases] == 12).all()
    assert len(rf) >= 4 * (n - 2) ** 3


@pytest.mark.parametrize("R", [3, 4, 5, 6, 7, 8, 31, 32, 33, 34, 129, 255, 256, 257, 258, 259, 260, 261])
def test_mc_grid_sizes(R):
    """G = R + 1 (padded, R <= 257) or R - 1 (plain): every G mod 4, quad rows across 1024-voxel blocks, both sides
    of the branch switch"""
    occ = _offset_blob(R, seed=R, noise=0.05 if R > 8 else 0.0)
    if R <= 8:
        occ[1:, 1:, 1:] = np.random.default_rng(R).choice(LEVELS, size=(R - 1,) * 3)
    rv, rf = _check(occ)
    assert len(rf) > 0
    if R - 1 <= 256:
        _assert_closed(rf)


@pytest.mark.parametrize("iso", [0.3, 0.1 + 2.0 ** -24, 0.7])
def test_mc_plain_branch_iso_not_representable_in_fp32(iso):
    """PyMCubes takes the iso value as a double: the cube test is float64(f) < iso and t uses the double, so nodes
    equal to fl32(iso) sit on the side the double puts them (below when fl32(iso) < iso)."""
    R = 259
    iso32 = float(np.float32(iso))
    assert iso32 != iso
    z, y, x = _grid(R)
    occ = (iso + 1.5 * (0.7 - np.sqrt((x / 0.9) ** 2 + (y / 0.7) ** 2 + (z / 0.8) ** 2))).astype(np.float32)
    near = np.abs(occ - iso32) < 0.01
    occ[near & (np.random.default_rng(0).random(occ.shape) < 0.3)] = iso32
    assert (occ[1:, 1:, 1:] == iso32).sum() > 100
    _check(occ, iso)
    _check(occ, iso, order="lex")
    # levels {0, .25, .5, .75, 1} moved so that .5 lands exactly on fl32(iso)
    q = (_quantised(R, 0.4, seed=3, box=30) - np.float32(0.5) + np.float32(iso32)).astype(np.float32)
    assert (q[1:, 1:, 1:] == iso32).sum() > 100
    _check(q, iso)


def test_mc_padded_branch_any_iso_in_fp32():
    occ = _offset_blob(33, seed=1)
    for iso in (0.3, 0.7, 0.1 + 2.0 ** -24):
        _check(occ, iso)


def test_mc_bench_call_unchanged_at_iso_half():
    """ops.marching_cubes(occ, 0.5): the call the benchmark times, both branches"""
    for R in (257, 513):
        z, y, x = _grid(R)
        occ = (0.5 + 2.0 * (0.8 - np.sqrt((x / 0.45) ** 2 + (y / 0.8) ** 2 + (z / 0.3) ** 2))).astype(np.float32)
        _check(occ, 0.5)


# --------------------------------------------------------------------------- clean_mesh
def _clean_check(v, f):
    """clean_mesh_device and the drop-in clean_mesh on (v, f) == OMesh.clean_mesh, index-exact; returns the result."""
    from icon_b200 import mesh
    dev = _cuda()
    vt = torch.as_tensor(v).to(dev)
    ft = torch.as_tensor(np.asarray(f, np.int64)).to(dev)
    rv, rf = OMesh.clean_mesh(np.asarray(v), np.asarray(f, np.int64))
    cv, cf = mesh.clean_mesh_device(vt, ft)
    assert cv.dtype == torch.float32 and cf.dtype == torch.int32
    assert np.array_equal(cf.cpu().numpy(), rf) and _same_bits(cv.cpu().numpy(), rv)
    dv, df = mesh.clean_mesh(vt.cpu(), ft.cpu())                     # CPU tensors in, CPU tensors out
    assert dv.device.type == "cpu" and torch.equal(df, cf.cpu()) and _same_bits(dv.numpy(), rv)
    return rv, rf


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", sorted(HAND_MESHES))
def test_clean_mesh_hand_built_meshes(name, dtype):
    nv, faces, keep_v, keep_f = HAND_MESHES[name]
    v = (np.arange(3 * nv, dtype=np.float64).reshape(nv, 3) * 0.1 + 1.0 / 3.0).astype(dtype)
    rv, rf = _clean_check(v, faces)
    assert _same_bits(rv, v[keep_v].astype(np.float32)) and np.array_equal(rf, keep_f)


@pytest.mark.parametrize("seed", range(6))
def test_clean_mesh_lex_meshes_with_iso_valued_nodes(seed):
    from icon_b200 import ops
    rng = np.random.default_rng(seed)
    R = int(rng.integers(7, 21))
    occ = _quantised(R, float(rng.uniform(0.1, 0.5)), seed=seed)
    for order in ("lex", "edge"):
        v, f = ops.marching_cubes(torch.from_numpy(occ).to(_cuda()), 0.5, order=order)
        rv, rf = _oracle(occ, 0.5, order)
        assert np.array_equal(f.cpu().numpy(), rf)
        _clean_check(rv, rf)


@pytest.mark.parametrize("R", [33, 259])
@pytest.mark.parametrize("name", ["slab", "corner_blob_lo", "ramp_x+", "all_inside", "quantised"])
def test_clean_mesh_on_border_and_iso_node_fields(name, R):
    occ = _quantised(R, 0.3, seed=R, box=24 if R > 257 else None) if name == "quantised" else BORDER[name](R)
    rv, rf = _oracle(occ)
    if len(rf) == 0:
        assert name == "all_inside" and R > 257
        return
    assert rv.dtype == (np.float64 if R > 257 else np.float32)
    _clean_check(rv, rf)


def test_clean_mesh_thousands_of_tied_components():
    """isolated voxels on a lattice: one closed 6-vertex surface each, all tied; plus a few equal larger pairs"""
    R = 64
    occ = np.zeros((R, R, R), np.float32)
    occ[2:-1:3, 2:-1:3, 2:-1:3] = 1.0
    occ[47, 47, 48] = occ[11, 11, 12] = 1.0                # two tied 2-voxel bars; the earlier one is kept
    rv, rf = _oracle(occ)
    ncomp, _ = OMesh.face_components(rf)
    assert ncomp > 1000
    cv, cf = _clean_check(rv, rf)
    assert len(cv) == 10


def test_clean_mesh_513_surface_and_determinism():
    """about 10^6 vertices over three components (the union-find under contention); two runs bitwise equal"""
    from icon_b200 import mesh, ops
    dev = _cuda()
    R = 513
    a = torch.linspace(-1, 1, R, device=dev)
    z, y, x = torch.meshgrid(a, a, a, indexing="ij")
    occ = 0.5 + 2.0 * (0.8 - ((x / 1.12) ** 2 + (y / 1.16) ** 2 + (z / 1.08) ** 2).sqrt())
    occ = torch.maximum(occ, 0.5 + 2.0 * (0.05 - ((x - 0.9) ** 2 + (y - 0.9) ** 2 + (z - 0.9) ** 2).sqrt()))
    occ = torch.maximum(occ, 0.5 + 2.0 * (0.05 - ((x + 0.9) ** 2 + (y + 0.9) ** 2 + (z - 0.9) ** 2).sqrt()))
    del x, y, z
    v, f = ops.marching_cubes(occ.float().contiguous(), 0.5)
    assert len(v) > 900_000, len(v)
    cv, cf = mesh.clean_mesh_device(v, f)
    cv2, cf2 = mesh.clean_mesh_device(v, f)
    assert torch.equal(cf, cf2) and _same_bits(cv.cpu().numpy(), cv2.cpu().numpy())
    rv, rf = OMesh.clean_mesh(v.cpu().numpy(), f.cpu().numpy())
    assert np.array_equal(cf.cpu().numpy(), rf) and _same_bits(cv.cpu().numpy(), rv)
    assert len(v) > len(cv) > 0.9 * len(v)
