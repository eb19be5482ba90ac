"""Brick face lists of the dense SDF path (sdf.cu, DESIGN.md 4.2) against the brute-force kernel, bit for bit.

The build culls each brick's faces with a bound that has to hold for every point of the brick, so a face it drops
must be strictly farther than the nearest one everywhere in the brick.  These cases stress that bound: every point of
a 256^3 lattice near the body (where the nearest face changes fastest across a brick), a rotated lattice, and a body
with more faces than the lists' 16-bit positions hold, which must fall back to the tree walk.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def dense_policy():
    _cuda()
    from icon_b200 import ops
    ops.set_sdf_policy(32)
    ops.set_sdf_bricks(True)
    yield
    ops.set_sdf_policy(0)
    ops.set_sdf_bricks(True)


def _body(dev, v, f, seed=0):
    from icon_b200 import ops
    cm, vi = S.body_attributes(v, seed=seed)
    return ops.SmplBody(*(torch.from_numpy(a)[None].to(dev) for a in (v, f, cm, vi)))


def _assert_equal_brute(body, pts, calib=None, rows=None):
    from icon_b200 import ops
    calib = torch.eye(4)[None] if calib is None else calib
    rec, face = ops.sdf_only(pts, calib, body)
    if rows is not None:
        pts, rec, face = pts[:, :, rows].contiguous(), rec[rows], face[rows]
    ref_rec, ref_face = ops.sdf_only(pts, calib, body, brute=True)
    assert (face != ref_face).sum().item() == 0
    assert torch.equal(rec, ref_rec)


def test_lattice_256_near_body():
    """Every 256^3 lattice point within 0.1 of the body, for three bodies."""
    from icon_b200 import ops
    dev = _cuda()
    pts = S.lattice_points(256).permute(0, 2, 1).contiguous().to(dev)
    for seed in (0, 1, 2):
        v, f = S.body_mesh(seed=seed)
        body = _body(dev, v, f, seed)
        rec, _ = ops.sdf_only(pts, torch.eye(4)[None], body)
        rows = (rec[:, 0].abs() * math.sqrt(3.0) < 0.1).nonzero().flatten()
        assert rows.numel() > 100000
        _assert_equal_brute(body, pts, rows=rows)
        info = ops.sdf_brick_info(body)
        assert info["built"] == 1 and info["overflow"] == 0


def test_rotated_lattice():
    dev = _cuda()
    v, f = S.body_mesh(seed=4)
    body = _body(dev, v, f, 4)
    a = math.radians(33.0)
    calib = torch.eye(4)
    calib[:3, :3] = 1.3 * torch.tensor([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0],
                                        [0.0, 0.0, 1.0]])
    _assert_equal_brute(body, S.lattice_points(128).permute(0, 2, 1).contiguous().to(dev), calib=calib[None])


def test_more_faces_than_uint16_falls_back():
    from icon_b200 import ops
    dev = _cuda()
    v, f = S.body_mesh(rings=200, segs=170, seed=0)
    assert len(f) > 65535
    body = _body(dev, v, f)
    _assert_equal_brute(body, S.lattice_points(64).permute(0, 2, 1).contiguous().to(dev))
    info = ops.sdf_brick_info(body)
    assert info["built"] == 1 and info["overflow"] == 1
