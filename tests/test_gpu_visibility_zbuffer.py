"""icon_visibility's z-buffer against oracle/visibility.py, pixel by pixel (ops.visibility_zbuffer).

Every case compares pix_to_face exactly, the depth of every pixel as floats (+0 == -0; +inf is background) and the
vertex mask, on the reference configuration -- get_visibility(xy, -z, faces) at 4096^2 as compute_vis_cmap calls it,
on the decimated scan and the synthetic body in four views -- and on the edge scenes of
tests/test_visibility_zbuffer_cpu.py: pixel centres exactly on edges, vertices one ulp either side of a pixel
centre, depth ties in both list orders, signed-zero depths and the camera plane, the 1e-8 area cut, the image border,
vertices far off screen or not finite, overflowing depths, a face over the whole image; image sizes 1 to 16384 (at
16384 the oracle draws a window and the rest of the kernel's buffer must be background).
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as SYN  # noqa: E402
from oracle import visibility as OV  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("_vis_scenes", os.path.join(HERE, "test_visibility_zbuffer_cpu.py"))
SC = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(SC)


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _check(xyz, faces, S, window=None):
    """Kernel z-buffer and mask == oracle's; -> the oracle's (pix_to_face, depth)."""
    from icon_b200 import ops
    dev = _cuda()
    xyz = np.asarray(xyz, np.float32)
    faces = np.asarray(faces, np.int64)
    xt, ft = torch.from_numpy(xyz).to(dev), torch.from_numpy(faces).to(dev)
    p2f, depth = ops.visibility_zbuffer(xt, ft, S)
    assert p2f.shape == (S, S) and p2f.dtype == torch.int64 and depth.dtype == torch.float32
    r_p2f, r_z = OV.rasterize(xyz, faces, S, window)
    if window is not None:
        r0, r1, c0, c1 = window
        outside = torch.ones(S, S, dtype=torch.bool, device=dev)
        outside[r0:r1, c0:c1] = False
        assert bool((p2f[outside] == -1).all()) and bool(torch.isinf(depth[outside]).all()), "drawn outside"
        p2f, depth = p2f[r0:r1, c0:c1], depth[r0:r1, c0:c1]
    p2f, depth = p2f.cpu().numpy(), depth.cpu().numpy()
    bad = p2f != r_p2f
    assert not bad.any(), (f"{int(bad.sum())} of {bad.size} pixels differ; first {np.argwhere(bad)[:3].tolist()}: "
                           f"kernel {p2f[bad][:3].tolist()}, oracle {r_p2f[bad][:3].tolist()}")
    zbad = depth != r_z
    assert not zbad.any(), f"{int(zbad.sum())} depths differ: {depth[zbad][:3]} vs {r_z[zbad][:3]}"
    vis = ops.visibility(xt, ft, S).cpu().numpy()
    ref = OV.vertex_mask(r_p2f if window is None else np.append(r_p2f.ravel(), -1), faces, len(xyz))[:, 0]
    assert np.array_equal(vis, ref), f"{int((vis != ref).sum())} vertices differ"
    return r_p2f, r_z


# ----------------------------------------------------------------------------------- reference configuration
def _body(name):
    if name == "scan":
        g = np.load(os.path.join(HERE, "golden", "scan_body.npz"))
        return g["verts"].astype(np.float32), g["faces"].astype(np.int64)
    return SYN.body_mesh(rings=82, segs=84)


@pytest.mark.parametrize("deg", [0, 90, 180, 35])
@pytest.mark.parametrize("name", ["scan", "body"])
def test_reference_configuration(name, deg):
    """get_visibility(xy, -z, faces) at 4096^2, as TestDataset.compute_vis_cmap calls it, seen from the front, the
    side, the back and at an oblique angle about the vertical axis."""
    _cuda()
    from icon_b200.visibility import get_visibility
    v, f = _body(name)
    a = np.deg2rad(deg)
    v64 = v.astype(np.float64)
    v = np.stack([v64[:, 0] * np.cos(a) + v64[:, 2] * np.sin(a), v64[:, 1],
                  -v64[:, 0] * np.sin(a) + v64[:, 2] * np.cos(a)], 1).astype(np.float32)
    xy, z = v[:, :2], v[:, 2:3]
    vis = get_visibility(torch.from_numpy(xy), torch.from_numpy(-z), torch.from_numpy(f))
    ref = OV.get_visibility(xy, -z, f)
    assert vis.shape == (len(v), 1) and np.array_equal(vis.numpy(), ref), f"{int((vis.numpy() != ref).sum())} differ"
    xyz = (np.concatenate([xy, z], 1) + np.float32(1.0)) / np.float32(2.0)        # = (cat(xy, -(-z)) + 1) / 2
    p2f, _ = _check(xyz, f, 4096)
    assert (p2f >= 0).sum() > 100000 and 0.2 < ref.mean() < 0.9


# -------------------------------------------------------------------------------------------------- the edges
@pytest.mark.parametrize("S,k0", [(64, 8), (256, 100), (250, 37), (4096, 2030), (4096, 0), (16384, 8170),
                                  (16384, 16336)])
def test_pixel_centres_on_edges(S, k0):
    xyz, faces, win = SC.edge_scene(S, k0)
    p2f, _ = _check(xyz, faces, S, win if S == 16384 else None)
    if S in (64, 4096, 16384):                        # power of two: centres on the diagonals are holes in both faces
        d = [k0 + 3, k0 + 4, k0 + 5]                  # the A-C diagonal, clear of the second quad
        sub = p2f if S == 16384 else p2f[k0:k0 + 48, k0:k0 + 48]
        assert (sub[[k - k0 for k in d], [k - k0 for k in d]] == -1).all()
        assert (sub[4:12, 4:12] >= 0).sum() > 30


@pytest.mark.parametrize("z", [0.0, 0.5])
def test_depth_ties(z):
    """Duplicates and the two triangulations of one quad: the kernel's atomicMin order must be the oracle's scan
    order, in both list orders; at z = 0 every depth is exactly +0 and the lowest covering index wins."""
    for rev in (False, True):
        xyz, faces = SC.tie_scene(z, rev)
        p2f, _ = _check(xyz, faces, 64)
        dup = [i for i in range(len(faces)) for j in range(i) if (faces[i] == faces[j]).all()]
        assert dup and not np.isin(p2f, dup).any()
        if z == 0.0:
            cover = np.stack([OV.rasterize(xyz, faces[i:i + 1], 64)[0] == 0 for i in range(len(faces))])
            lowest = np.where(cover.any(0), cover.argmax(0), -1)
            assert np.array_equal(p2f, lowest)


@pytest.mark.parametrize("order", [0, 1])
def test_signed_zero_and_camera_plane(order):
    xyz, faces, idx = SC.zero_scene(order)
    p2f, z = _check(xyz, faces, 64)
    assert (p2f == idx["minus0"]).sum() > 50 and (p2f == min(idx["minus0"], idx["plus0"])).sum() > 50


def test_area_cut():
    xyz, faces = SC.area_scene(4096)
    p2f, _ = _check(xyz, faces, 4096)
    assert [bool((p2f == f).any()) for f in range(len(faces))] == [a > SC.EPS for a in SC.AREAS]


@pytest.mark.parametrize("S", [1, 2, 3, 1023, 4096])
def test_border_and_beyond(S):
    """Faces across the border, off screen, with vertices at 1e6 / 3e6 / 1e30, non-finite, overflowing depths."""
    xyz, faces = SC.border_scene(S)
    _check(xyz, faces, S)


def test_infinite_depth_never_takes_a_pixel():
    S, r, c = SC.INF_DEPTH_PIXEL
    p2f, z = _check(SC.INF_DEPTH_FACE, [[0, 1, 2]], S)
    assert p2f[r, c] == -1 and (p2f == 0).sum() > 1000


@pytest.mark.parametrize("S", [1, 2, 3, 64])
@pytest.mark.parametrize("last_covers", [False, True])
def test_whole_image_face(S, last_covers):
    """No empty pixel: the last face is marked only if it owns a pixel."""
    xyz, faces = SC.whole_scene(last_covers)
    p2f, _ = _check(xyz, faces, S)
    assert (p2f == (1 if last_covers else 0)).all()


# ----------------------------------------------------------------------------------- determinism and inputs
def test_two_calls_are_bitwise_identical():
    dev = _cuda()
    from icon_b200 import ops
    v, f = _body("scan")
    xyz = torch.from_numpy((v + 1) / 2).to(dev)
    ft = torch.from_numpy(f).to(dev)
    a, b = ops.visibility_zbuffer(xyz, ft, 4096), ops.visibility_zbuffer(xyz, ft, 4096)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    assert torch.equal(ops.visibility(xyz, ft, 4096), ops.visibility(xyz, ft, 4096))


def test_cpu_cuda_and_float64_inputs_give_one_mask():
    dev = _cuda()
    from icon_b200.visibility import get_visibility
    v, f = _body("scan")
    v64 = v.astype(np.float64) * 1.0000001
    xy64, z64 = torch.from_numpy(v64[:, :2]), torch.from_numpy(-v64[:, 2:3])
    xy32, z32 = xy64.float(), z64.float()
    ft = torch.from_numpy(f)
    ref = OV.get_visibility(xy32.numpy(), z32.numpy(), f)
    for xy, z, fc in [(xy32, z32, ft), (xy32.to(dev), z32.to(dev), ft.to(dev)), (xy64, z64, ft),
                      (xy64.to(dev), z64.to(dev), ft.int().to(dev))]:
        out = get_visibility(xy, z, fc)
        assert out.device.type == "cpu" and out.dtype == torch.float32 and np.array_equal(out.numpy(), ref)
