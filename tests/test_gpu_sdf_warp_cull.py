"""The dense SDF block's warp-level support cull (face_tree.cuh: NearestFace::beats, DESIGN.md 4.2) against the
brute-force kernel, bit for bit.

The cull drops a face for all 32 lanes of a warp at once, from a bound that follows the lanes' own distance bounds
across the warp's box.  It may only drop faces that no lane can take, so rec and the nearest face must equal
icon_sdf_bruteforce exactly: on meshes whose vertices and faces lie on brick and bin boundaries, on flat sheets seen
head-on (where the bound is tightest and exact ties are everywhere), with coincident-corner faces whose distance can
be NaN, with duplicated faces (ties go to the lowest index), on the brick path, on the tree walk and after the lists
overflowed.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402

EYE = torch.eye(4)[None]
BRICK = 2.0 / 32                          # brick edge; bins are a quarter of it


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def dense_policy():
    """PPW = 32 on every call, bricks on with no entry cap; restored afterwards."""
    _cuda()
    from icon_b200 import ops
    ops.set_sdf_policy(32)
    ops.set_sdf_bricks(True)
    yield
    ops.set_sdf_policy(0)
    ops.set_sdf_bricks(True)


def _grid_box(n, lo, hi):
    """Closed, outward-wound surface of the box [lo, hi]^3, each side an n x n grid of quads split in two."""
    t = np.linspace(lo, hi, n + 1)
    verts, faces = [], []
    for axis in range(3):
        for side, val in ((0, lo), (1, hi)):
            u, v = np.meshgrid(t, t, indexing="ij")
            p = np.zeros((n + 1, n + 1, 3))
            p[..., axis], p[..., (axis + 1) % 3], p[..., (axis + 2) % 3] = val, u, v
            base = sum(len(x) for x in verts)
            verts.append(p.reshape(-1, 3))
            idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1) + base
            a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
            q = np.stack([np.stack([a, b, c], -1), np.stack([a, c, d], -1)], 2).reshape(-1, 3)
            faces.append(q if side == 1 else q[:, ::-1])
    return np.concatenate(verts).astype(np.float32), np.concatenate(faces).astype(np.int64)


def _sheet(n, half, z):
    """Open flat sheet z = const over [-half, half]^2, an n x n grid of quads split along one diagonal."""
    t = np.linspace(-half, half, n + 1)
    u, v = np.meshgrid(t, t, indexing="ij")
    verts = np.stack([u, v, np.full_like(u, z)], -1).reshape(-1, 3).astype(np.float32)
    idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
    a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
    faces = np.stack([np.stack([a, b, c], -1), np.stack([a, c, d], -1)], 2).reshape(-1, 3).astype(np.int64)
    return verts, faces


def _body(dev, v, f, seed=0):
    from icon_b200 import ops
    cm, vi = S.body_attributes(v, seed=seed)
    return ops.SmplBody(*(torch.from_numpy(a)[None].to(dev) for a in (v, f, cm, vi)))


def _lattice(res, dev):
    return S.lattice_points(res).permute(0, 2, 1).contiguous().to(dev)


def _assert_equal_brute(body, pts, calib=EYE):
    from icon_b200 import ops
    rec, face = ops.sdf_only(pts, calib, body)
    ref_rec, ref_face = ops.sdf_only(pts, calib, body, brute=True)
    bad = (face != ref_face).sum().item()
    assert bad == 0, f"nearest-face mismatch on {bad} points"
    assert torch.equal(rec, ref_rec), f"rec not bit-exact on {(rec != ref_rec).any(1).sum().item()} points"
    return rec, face


def test_box_on_brick_and_bin_boundaries():
    """Every vertex on a brick corner (sides at +-8 bricks, one quad per brick), every side in a brick plane."""
    from icon_b200 import ops
    dev = _cuda()
    v, f = _grid_box(16, -8 * BRICK, 8 * BRICK)
    body = _body(dev, v, f)
    _assert_equal_brute(body, _lattice(128, dev))
    info = ops.sdf_brick_info(body)
    assert info["built"] == 1 and info["overflow"] == 0
    # bins: a quarter-brick grid, with an off-centre box
    v, f = _grid_box(20, -0.75, 0.5)
    _assert_equal_brute(_body(dev, v, f, seed=1), _lattice(128, dev))


def test_box_rotated_calibration():
    """The warps' boxes no longer line up with the box's faces, so the lanes' distance slope is oblique."""
    dev = _cuda()
    v, f = _grid_box(16, -8 * BRICK, 8 * BRICK)
    body = _body(dev, v, f)
    a, b = math.radians(25.0), math.radians(-35.0)
    rz = torch.tensor([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])
    rx = torch.tensor([[1.0, 0.0, 0.0], [0.0, math.cos(b), -math.sin(b)], [0.0, math.sin(b), math.cos(b)]])
    calib = torch.eye(4)
    calib[:3, :3] = rz @ rx
    calib[:3, 3] = torch.tensor([0.02, -0.01, 0.03])
    _assert_equal_brute(body, _lattice(112, dev), calib=calib[None])


def test_flat_sheet_head_on_with_duplicated_faces():
    """A sheet in a brick plane, seen head-on from the whole lattice, then listed twice: every point ties between
    face i and its copy i + F, and the lower index must win."""
    dev = _cuda()
    v, f = _sheet(24, 12 * BRICK, 4 * BRICK)
    body = _body(dev, v, f)
    _assert_equal_brute(body, _lattice(128, dev))
    F = f.shape[0]
    body2 = _body(dev, v, np.concatenate([f, f]))
    _, face = _assert_equal_brute(body2, _lattice(128, dev))
    assert int(face.max()) < F, "a tie between a face and its copy went to the copy"


def test_coincident_corner_faces():
    """Faces with two equal corners (a NaN distance in the regions that divide by their zero edge, never taken there)
    ahead of and among the box's faces."""
    dev = _cuda()
    v, f = _grid_box(16, -8 * BRICK, 8 * BRICK)
    rng = np.random.RandomState(5)
    pick = rng.choice(len(v), 64, replace=False)
    bad = np.stack([pick, pick, np.roll(pick, 1)], 1)          # corners a == b
    bad2 = np.stack([np.roll(pick, 2), pick, pick], 1)         # corners b == c
    f2 = np.concatenate([bad, f[: len(f) // 2], bad2, f[len(f) // 2:]]).astype(np.int64)
    body = _body(dev, v, f2)
    _assert_equal_brute(body, _lattice(128, dev))


def test_tree_walk_with_bricks_off():
    """The same cull runs in the tree walk at 32 points per warp."""
    from icon_b200 import ops
    dev = _cuda()
    ops.set_sdf_bricks(False)
    v, f = _grid_box(16, -8 * BRICK, 8 * BRICK)
    _assert_equal_brute(_body(dev, v, f), _lattice(128, dev))
    v, f = S.body_mesh(seed=6)
    _assert_equal_brute(_body(dev, v, f, seed=6), _lattice(128, dev))


def test_list_overflow_falls_back_to_tree_walk():
    from icon_b200 import ops
    dev = _cuda()
    ops.set_sdf_bricks(True, max_entries=1000)
    v, f = _sheet(24, 12 * BRICK, 4 * BRICK)
    body = _body(dev, v, np.concatenate([f, f]))
    _assert_equal_brute(body, _lattice(96, dev))
    info = ops.sdf_brick_info(body)
    assert info["built"] == 1 and info["overflow"] == 1
