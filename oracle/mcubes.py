"""oracle/mcubes.py -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

CPU (numpy) restatement of the mesh-extraction step of the reference,
`Seg3dLossless.export_mesh` (lib/common/seg3d_lossless.py:583-604).

The marching cubes themselves live in un-vendored third-party code:
  * grids <= 256^3: kaolin 0.11.0 `voxelgrids_to_trianglemeshes` (seg3d_lossless.py:599), a
    CUDA port of the NVIDIA-samples marching cubes (classify / scan / compact / generate on a
    grid zero-padded by one voxel, iso 0.5, cube bit set where f < iso, linear edge
    interpolation, Bourke triangle table) followed by a vertex merge;
  * grids  > 256^3: PyMCubes `mcubes.marching_cubes` (seg3d_lossless.py:592), CPU.
Neither source is in /root/reference and neither wheel installs offline: PARITY UNPINNED.
What is restated here is the published algorithm plus an explicit, deterministic indexing
contract that the CUDA kernels reproduce bit for bit:

  contract "padded" (kaolin branch)
    - the volume is zero-padded by one voxel on every side; vertex coordinates are in the
      padded frame (voxel i of the input sits at coordinate i+1), fp32;
    - every vertex lies on a grid edge and is owned by that edge's lower voxel; its position
      is lower + t, t = (iso - f_lo) / (f_hi - f_lo), fp32;
    - vertex ids ascend with key = 3 * linear_index(owner voxel, padded grid, last dim
      fastest) + axis;
    - triangles are emitted cell by cell in linear cell order (last dim fastest), and within a
      cell in triangle-table order.
  contract "plain" (PyMCubes branch): same, without padding, fp64 coordinates; the iso value stays a double
    (PyMCubes' `isovalue`), so the cube test is float64(f) < iso and t is computed in fp64 from it.
  In both, NaN is never below iso; ±inf compare as themselves; t follows IEEE arithmetic (NaN for inf / inf).

`export_mesh` then applies the reference's own `[:, [2,1,0]]` / `[:, [0,2,1]]` permutations.

Second selectable vertex order, `order="lex"` -- what SURVEY 8c believes kaolin's merge does: the triangle soup's
vertices are merged with `torch.unique(dim=0)`, i.e. vertices sorted lexicographically by coordinate row and
coincident ones (an edge vertex landing exactly on a grid node is shared by up to 3 edges) collapsed; triangles keep
soup order.  A user with the kaolin wheel can compare against either order; both are UNPINNED here.

Public algorithm references (sources absent from /root/reference, wheels not installable offline):
  kaolin 0.11.0   kaolin/ops/conversions/voxelgrid.py::voxelgrids_to_trianglemeshes -> unbatched_mcube CUDA op
                  (kaolin/csrc/ops/conversions/unbatched_mcube/unbatched_mcube_cuda.cu: classifyVoxel / compactVoxels /
                  generateTriangles2, after the NVIDIA CUDA-samples marchingCubes), iso default 0.5
  PyMCubes        mcubes/src/marchingcubes.h::marching_cubes (P. Bourke's table, shared vertices created on first
                  use along x-fastest scan), called as mcubes.marching_cubes(arr, isovalue)
"""
import numpy as np

from .mc_table import CORNERS, EDGE_CORNERS, TRI_TABLE, NUM_VERTS      # the checker's own copy of the table


def _edge_owner():
    """edge id -> (corner offset of the owning (lower) voxel, axis)."""
    out = []
    for a, b in EDGE_CORNERS:
        ca, cb = np.array(CORNERS[a]), np.array(CORNERS[b])
        axis = int(np.nonzero(ca != cb)[0][0])
        lo = ca if ca[axis] < cb[axis] else cb
        out.append((tuple(int(v) for v in lo), axis))
    return out


_OWNER = _edge_owner()


def _grid(vol, pad):
    g = np.asarray(vol, dtype=np.float32)
    return np.pad(g, 1) if pad else g


def cube_cases(vol, iso=0.5, pad=True, dtype=np.float32):
    """Cube case (bit c set when corner c is below iso) of every cell of the working grid [X-1, Y-1, Z-1].  The
    comparison runs in the output precision: fp64 iso in the PyMCubes branch, which takes it as a double; NaN is
    never below iso."""
    g = _grid(vol, pad)
    cx, cy, cz = (n - 1 for n in g.shape)
    below = g.astype(dtype) < dtype(iso)
    cube = np.zeros((cx, cy, cz), np.int32)
    for c, (dx, dy, dz) in enumerate(CORNERS):
        cube |= below[dx:dx + cx, dy:dy + cy, dz:dz + cz].astype(np.int32) << c
    return cube


def marching_cubes(vol, iso=0.5, pad=True, dtype=np.float32):
    """vol [X,Y,Z] -> (verts [Nv,3] in vol's index frame (+1 if padded), faces [Nf,3] int64)."""
    g = _grid(vol, pad)
    X, Y, Z = g.shape
    cx, cy, cz = X - 1, Y - 1, Z - 1
    cube = cube_cases(vol, iso, pad, dtype)
    nv = np.asarray(NUM_VERTS, np.int32)[cube]
    act = np.flatnonzero(nv.reshape(-1))           # linear cell order, last dim fastest
    if act.size == 0:
        return np.zeros((0, 3), dtype), np.zeros((0, 3), np.int64)
    ci, cj, ck = np.unravel_index(act, (cx, cy, cz))
    case = cube.reshape(-1)[act]
    tri = np.asarray(TRI_TABLE, np.int32)[case][:, :15]             # [A,15]
    valid = tri >= 0
    own_off = np.asarray([o for o, _ in _OWNER], np.int64)         # [12,3]
    own_axis = np.asarray([a for _, a in _OWNER], np.int64)         # [12]
    e = np.where(valid, tri, 0)
    oi = ci[:, None] + own_off[e, 0]
    oj = cj[:, None] + own_off[e, 1]
    ok = ck[:, None] + own_off[e, 2]
    key = ((oi * Y + oj) * Z + ok) * 3 + own_axis[e]
    keys = key[valid]                                               # soup order
    ukeys, inv = np.unique(keys, return_inverse=True)
    faces = inv.reshape(-1, 3).astype(np.int64)
    lin, axis = ukeys // 3, ukeys % 3
    vi, vj, vk = np.unravel_index(lin, (X, Y, Z))
    f_lo = g[vi, vj, vk].astype(dtype)
    f_hi = g[vi + (axis == 0), vj + (axis == 1), vk + (axis == 2)].astype(dtype)
    t = (dtype(iso) - f_lo) / (f_hi - f_lo)
    verts = np.stack([vi, vj, vk], 1).astype(dtype)
    verts[np.arange(len(verts)), axis] += t
    return verts, faces


def lexicographic_merge(verts, faces):
    """Edge-owned (verts, faces) -> the soup + `unique(dim=0)` order: rows sorted lexicographically, coincident rows
    merged, faces remapped (triangle order unchanged)."""
    if len(verts) == 0:
        return verts, faces
    u, inv = np.unique(verts, axis=0, return_inverse=True)
    return u, inv.reshape(-1)[faces]


def export_mesh(occupancys, balance_value=0.5, order="edge"):
    """seg3d_lossless.py:583-604 restated.  occupancys: [R,R,R] float array indexed [z,y,x].
    The kaolin branch (grid <= 256^3, :599) runs at kaolin's default iso 0.5; PyMCubes (:592) at balance_value."""
    final = np.ascontiguousarray(np.asarray(occupancys)[1:, 1:, 1:])
    if final.shape[0] > 256:
        v, t = marching_cubes(final, balance_value, pad=False, dtype=np.float64)
    else:
        v, t = marching_cubes(final, 0.5, pad=True, dtype=np.float32)
    if order == "lex":
        v, t = lexicographic_merge(v, t)
    return v[:, [2, 1, 0]], t[:, [0, 2, 1]]
