"""The face tree (csrc/face_tree.cu) of a prepared SMPL body and of a prepared mesh, bit for bit against a float32 numpy
reconstruction.

The tree's queries are exact for any valid tree, so they cannot tell whether the tree itself changed; this test pins
its contents.  The build is -fmad=false and its divisions and square roots are correctly rounded, so float32 numpy
reproduces them; the sphere radius goes through dot3 (geom.cuh), which is written with fmaf, emulated here with libm's.
  order   Morton codes of the centroids (tools/brick_face_lists.leaf_boxes), sorted by (code, face id);
  tri_s   (a, ab, ac) of each sorted face;
  sph_s   centroid and sqrt(max corner distance^2) * 1.0001 + slack, slack 1e-7 on a body and 1e-7 max(1, |coords|) on
          a mesh, whose frame is its own bounding cube;
  nodes   leaf boxes over a, a + ab and a + ac, then parent boxes over 4 children, level by level.
"""
import ctypes
import ctypes.util

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402
from tools import brick_face_lists as B  # noqa: E402

f32 = np.float32
_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.fmaf.restype = ctypes.c_float
_libm.fmaf.argtypes = [ctypes.c_float] * 3
_fmaf = np.frompyfunc(_libm.fmaf, 3, 1)


def fmaf(x, y, z):
    return _fmaf(x, y, z).astype(f32)


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def reconstruct(v, f, fit):
    tri = v[f]                                                          # float32 [F,3,3]
    if fit:
        lo, hi = tri.reshape(-1, 3).min(0), tri.reshape(-1, 3).max(0)
        ext = (hi - lo).max()
        scale = f32(1024) / ext if ext > 0 else f32(0)
        absmax = max(np.abs(lo).max(), np.abs(hi).max())
        slack = f32(1e-7) * max(f32(1), absmax)
        order = B.leaf_boxes(v, f, lo, scale)[0]
    else:
        slack = f32(1e-7)
        order = B.leaf_boxes(v, f)[0]
    a, b, c = (tri[order, k] for k in range(3))
    ab, ac = b - a, c - a
    F = len(f)
    tri_s = np.concatenate([a, ab, ac, np.zeros((F, 3), f32)], 1)
    sc = (a + b + c) / f32(3)

    def dot3(d):                                                        # fmaf(z, z, fmaf(y, y, x * x))
        return fmaf(d[:, 2], d[:, 2], fmaf(d[:, 1], d[:, 1], d[:, 0] * d[:, 0]))
    r2 = np.maximum(dot3(a - sc), np.maximum(dot3(b - sc), dot3(c - sc)))
    sph_s = np.concatenate([sc, (np.sqrt(r2) * f32(1.0001) + slack)[:, None]], 1)
    corners = np.stack([a, a + ab, a + ac], 1).reshape(-1, 3)          # 3 per sorted face
    starts = np.arange(0, 3 * F, 12)                                    # 4 faces per leaf
    lo, hi = np.minimum.reduceat(corners, starts), np.maximum.reduceat(corners, starts)
    levels = [(lo, hi)]
    while len(lo) > 1:
        starts = np.arange(0, len(lo), 4)
        lo, hi = np.minimum.reduceat(lo, starts), np.maximum.reduceat(hi, starts)
        levels.append((lo, hi))
    lo, hi = (np.concatenate([lv[k] for lv in levels]) for k in range(2))
    z = np.zeros((len(lo), 1), f32)
    nodes = np.stack([np.concatenate([lo, z], 1), np.concatenate([hi, z], 1)], 1)
    return order.astype(np.int32), tri_s, sph_s, nodes


def _prepare(kind, v, f):
    from icon_b200 import metrics, ops
    dev = _cuda()
    if kind == "body":
        cm, vi = S.body_attributes(v, seed=0)
        return ops.SmplBody(*(torch.from_numpy(x)[None].to(dev) for x in (v, f, cm, vi)))
    return metrics.Mesh(v, f, device=dev)


def _bits(x):
    return np.ascontiguousarray(x, f32).view(np.uint32)


def check_tree(kind, v, f):
    from icon_b200 import ops
    v = np.ascontiguousarray(v, f32)
    f = np.ascontiguousarray(f, np.int64)
    got = {k: t.numpy() for k, t in ops.face_tree(_prepare(kind, v, f)).items()}
    order, tri_s, sph_s, nodes = reconstruct(v, f, fit=kind == "mesh")
    assert np.array_equal(got["order"], order)
    assert np.array_equal(_bits(got["tri_s"]), _bits(tri_s))
    assert np.array_equal(_bits(got["sph_s"]), _bits(sph_s))
    # fminf / fmaxf may return either zero of +0 / -0: compare the boxes with the zeros' signs made equal
    assert np.array_equal(_bits(got["nodes"] + f32(0)), _bits(nodes + f32(0)))


def _voxel_units(v):
    return v * f32(256) + f32([300.5, 17.25, 96.0])


def _duplicated(f):                                                     # every face twice: equal centroids
    return np.concatenate([f, f[::-1]])


MESHES = {
    "smpl_13776": lambda: S.body_mesh(seed=0),
    "body_68k": lambda: S.body_mesh(rings=200, segs=170, seed=0),
}


@pytest.mark.parametrize("kind", ["body", "mesh"])
@pytest.mark.parametrize("name", sorted(MESHES))
def test_tree_of_synthetic_bodies(kind, name):
    v, f = MESHES[name]()
    check_tree(kind, v, f)


@pytest.mark.parametrize("kind", ["body", "mesh"])
def test_tree_in_voxel_units(kind):
    """A mesh in voxel units: the slack scales with its coordinates; on a body, far outside the fixed cube, every code
    clamps to one corner so the order is by face id alone."""
    v, f = S.body_mesh(seed=1)
    check_tree(kind, _voxel_units(v), f)


@pytest.mark.parametrize("kind", ["body", "mesh"])
def test_tree_with_duplicate_centroids_and_degenerate_faces(kind):
    v, f = S.body_mesh(seed=2)
    check_tree(kind, v, _duplicated(S.collapse_faces(f, n=64, seed=3)))
    check_tree(kind, v, np.zeros((9, 3), np.int64))                    # nine faces on one point


@pytest.mark.parametrize("kind", ["body", "mesh"])
@pytest.mark.parametrize("F", [1, 2, 3, 4, 5, 7, 17, 4099])
def test_tree_level_edges(kind, F):
    """Partial leaves and partial parents, and a leaf level of one CTA and just over."""
    v, f = S.body_mesh(seed=4)
    rng = np.random.RandomState(F)
    check_tree(kind, v, f[rng.choice(len(f), F, replace=False)])
