"""Brick face lists of the dense SDF path (sdf.cu, DESIGN.md 4.2) against the brute-force kernel, bit for bit.

The brick path only changes which faces a warp looks at, so rec (sdf, cmap, normal, vis) and the nearest face must
equal icon_sdf_bruteforce exactly: on dense lattices, on warps that straddle bricks or leave the cube (tree walk),
when the lists overflow, and with the path switched off.
"""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402

EYE = torch.eye(4)[None]


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def dense_policy():
    """PPW = 32 (the brick path) on every call, bricks on; restored afterwards."""
    _cuda()
    from icon_b200 import ops
    ops.set_sdf_policy(32)
    ops.set_sdf_bricks(True)
    yield
    ops.set_sdf_policy(0)
    ops.set_sdf_bricks(True)


def _tensors(v, f, seed=0):
    cm, vi = S.body_attributes(v, seed=seed)
    return [torch.from_numpy(a)[None] for a in (v, f, cm, vi)]


def _body(dev, seed=0, tensors=None):
    from icon_b200 import ops
    if tensors is None:
        v, f = S.body_mesh(seed=seed)
        tensors = _tensors(v, f, seed)
    return ops.SmplBody(*(t.to(dev) for t in tensors))


def _lattice(res, dev):
    return S.lattice_points(res).permute(0, 2, 1).contiguous().to(dev)


def _assert_equal_brute(body, pts, calib=EYE, rows=None):
    """sdf_only on all of `pts` [1,3,N]; brute force on `rows` of them (all when None)."""
    from icon_b200 import ops
    rec, face = ops.sdf_only(pts, calib, body)
    if rows is not None:
        pts, rec, face = pts[:, :, rows].contiguous(), rec[rows], face[rows]
    ref_rec, ref_face = ops.sdf_only(pts, calib, body, brute=True)
    bad = (face != ref_face).sum().item()
    assert bad == 0, f"nearest-face mismatch on {bad} points"
    assert torch.equal(rec, ref_rec), f"rec not bit-exact on {(rec != ref_rec).any(1).sum().item()} points"
    return rec, face


@pytest.mark.parametrize("res", [64, 128])
def test_dense_lattice_every_point(res):
    from icon_b200 import ops
    body = _body(_cuda())
    _assert_equal_brute(body, _lattice(res, body.ws.device))
    info = ops.sdf_brick_info(body)
    assert info["built"] == 1 and info["overflow"] == 0 and 0 < info["entries"] <= info["capacity"]


def test_dense_lattice_256_seeded_subset():
    dev = _cuda()
    body = _body(dev)
    pts = _lattice(256, dev)
    g = torch.Generator().manual_seed(7)
    rows = torch.randperm(pts.shape[2], generator=g)[: 1 << 19].to(dev)
    _assert_equal_brute(body, pts, rows=rows)


def test_real_scan_body(golden_dir):
    dev = _cuda()
    g = np.load(os.path.join(golden_dir, "scan_body.npz"))
    body = _body(dev, tensors=_tensors(g["verts"], g["faces"].astype(np.int64), seed=3))
    _assert_equal_brute(body, _lattice(96, dev))
    adv = S.adversarial_points(g["verts"], g["faces"].astype(np.int64), n_each=500, seed=1)
    _assert_equal_brute(body, adv.permute(0, 2, 1).contiguous().to(dev))


def test_warps_straddling_bricks():
    """A lattice shifted by half a brick (0.03125) with a spacing that is no divisor of the bins, and a rotating,
    scaling calibration: warps span several bins of different bricks and points leave the cube."""
    dev = _cuda()
    body = _body(dev, seed=1)
    pts = (S.lattice_points(90) + 0.03125).permute(0, 2, 1).contiguous().to(dev)
    _assert_equal_brute(body, pts)
    a = math.radians(20.0)
    calib = torch.eye(4)
    calib[:3, :3] = 1.1 * torch.tensor([[math.cos(a), 0.0, math.sin(a)], [0.0, 1.0, 0.0],
                                        [-math.sin(a), 0.0, math.cos(a)]])
    calib[:3, 3] = torch.tensor([0.01, -0.02, 0.015])
    _assert_equal_brute(body, _lattice(80, dev), calib=calib[None])


def test_points_outside_cube():
    dev = _cuda()
    body = _body(dev)
    g = torch.Generator().manual_seed(3)
    pts = (torch.rand(1, 3, 200000, generator=g) * 2 - 1) * 1.6
    pts[0, 0, :5000] = 1.0
    pts[0, 1, 5000:10000] = -1.0
    _assert_equal_brute(body, pts.to(dev))


def test_forced_list_overflow_falls_back_to_tree():
    from icon_b200 import ops
    dev = _cuda()
    ops.set_sdf_bricks(True, max_entries=1000)
    body = _body(dev)
    _assert_equal_brute(body, _lattice(64, dev))
    info = ops.sdf_brick_info(body)
    assert info["built"] == 1 and info["overflow"] == 1


def test_brick_path_on_equals_off():
    from icon_b200 import ops
    dev = _cuda()
    body = _body(dev, seed=2)
    pts = _lattice(128, dev)
    ops.set_sdf_bricks(False)
    r0, f0 = ops.sdf_only(pts, EYE, body)
    assert ops.sdf_brick_info(body)["built"] == 0
    ops.set_sdf_bricks(True)
    r1, f1 = ops.sdf_only(pts, EYE, body)
    assert ops.sdf_brick_info(body)["built"] == 1
    assert torch.equal(f0, f1) and torch.equal(r0, r1)


def test_lists_built_once_per_body_and_rebuilt_after_new_verts():
    from icon_b200 import config, net, ops
    dev = _cuda()
    netG = net.HGPIFuNet(config.preset("icon-filter")).to(dev).eval()
    v, f = S.body_mesh(seed=4)
    verts, faces, cmap, vis = (t.to(dev) for t in _tensors(v, f, seed=4))
    netG.smpl_feat_dict = {"smpl_verts": verts, "smpl_faces": faces, "smpl_cmap": cmap, "smpl_vis": vis}
    pts = _lattice(64, dev)
    body = netG._prepared_body()
    assert ops.sdf_brick_info(body)["built"] == 0
    ops.sdf_only(pts, EYE, body)
    n0 = ops.sdf_brick_info(body)["builds"]
    assert netG._prepared_body() is body
    ops.sdf_only(pts, EYE, netG._prepared_body())
    assert ops.sdf_brick_info(body)["builds"] == n0              # same prepared body: no second build
    with torch.no_grad():
        verts.mul_(0.9)                                          # a new smpl_verts version -> a new prepared body
    body2 = netG._prepared_body()
    assert body2 is not body
    assert ops.sdf_brick_info(body2)["built"] == 0
    _assert_equal_brute(body2, pts)
    info = ops.sdf_brick_info(body2)
    assert info["built"] == 1 and info["builds"] == n0 + 1
