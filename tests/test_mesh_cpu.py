"""oracle/mesh.py (trimesh's split + the component with the most vertices) on hand-built meshes, as known answers.

trimesh joins two faces when they share an edge used by exactly two faces, counts a component's distinct vertices and
keeps the first largest one in smallest-face-index order.  Each mesh below is a configuration where that rule and
"vertices joined by a triangle edge, ties to the smallest vertex id" keep different things.  HAND_MESHES is shared
with the device tests (tests/test_gpu_mc_edges.py): name -> (vertex count, faces, kept vertex ids, kept faces).
"""
import numpy as np
import pytest

from oracle import mesh as OMesh

_TET = [[0, 2, 1], [0, 1, 3], [1, 2, 3], [0, 3, 2]]


def _tet(base):
    return [[base + a for a in f] for f in _TET]


HAND_MESHES = {
    # two triangles touching at vertex 2: two components of 3 vertices, the first face's wins the tie
    "bow_tie": (5, [[0, 1, 2], [2, 3, 4]], [0, 1, 2], [[0, 1, 2]]),
    # two closed tetrahedra sharing vertex 3: 4 vertices each
    "tetra_bow_tie": (7, _tet(0) + _tet(3), [0, 1, 2, 3], _tet(0)),
    # edge (0, 1) used by 3 faces joins nothing; faces 2..4 are a strip over (1, 4) and (4, 5) with 5 vertices
    "edge_of_3": (7, [[0, 1, 2], [0, 1, 3], [0, 1, 4], [1, 4, 5], [4, 5, 6]], [0, 1, 4, 5, 6],
                  [[0, 1, 2], [1, 2, 3], [2, 3, 4]]),
    # edge (0, 1) used by 4 faces: four single-face components of 3 vertices; a 4-vertex pair through (2, 6) wins
    "edge_of_4": (9, [[0, 1, 2], [1, 0, 3], [0, 1, 4], [1, 0, 5], [2, 6, 7], [6, 2, 8]], [2, 6, 7, 8],
                  [[0, 1, 2], [1, 0, 3]]),
    # a duplicated face, joined to its copy by (0, 1) and (0, 2); (1, 2) is used 3 times, so face 2 stays alone
    "duplicate_pair": (4, [[0, 1, 2], [0, 1, 2], [1, 2, 3]], [0, 1, 2], [[0, 1, 2], [0, 1, 2]]),
    # a face repeated three times: every edge used 3 times, three components of 3 vertices, the first one kept
    "duplicate_triple": (3, [[0, 1, 2], [2, 1, 0], [1, 2, 0]], [0, 1, 2], [[0, 1, 2]]),
    # [a, a, b] uses (a, b) twice, [a, a, a] uses (a, a) three times; (0, 1) is used 3 times (faces 0 and 1)
    "repeated_ids": (9, [[0, 1, 2], [0, 0, 1], [5, 5, 5], [3, 3, 4], [2, 1, 6], [6, 1, 7]], [0, 1, 2, 6, 7],
                     [[0, 1, 2], [2, 1, 3], [3, 1, 4]]),
    # vertices 0, 1 and 8 are referenced by no face; vertex ids of the output skip them
    "unreferenced": (9, [[2, 3, 4], [4, 3, 5], [6, 7, 2]], [2, 3, 4, 5], [[0, 1, 2], [2, 1, 3]]),
    # equal vertex counts: the component of face 0 holds the LARGEST vertex ids and must win over the one of face 1
    "tie_face_order": (8, [[5, 6, 7], [0, 1, 2], [2, 1, 3], [6, 5, 4]], [4, 5, 6, 7], [[1, 2, 3], [2, 1, 0]]),
}


def _verts(n):
    return (np.arange(3 * n, dtype=np.float64).reshape(n, 3) * 0.25 + 1.0).astype(np.float32)


@pytest.mark.parametrize("name", sorted(HAND_MESHES))
def test_oracle_clean_mesh_known_answers(name):
    nv, faces, keep_v, keep_f = HAND_MESHES[name]
    v = _verts(nv)
    rv, rf = OMesh.clean_mesh(v, np.asarray(faces, np.int64))
    assert rv.dtype == np.float32 and rf.dtype == np.int32
    assert np.array_equal(rv, v[keep_v])
    assert np.array_equal(rf, np.asarray(keep_f, np.int32))


def test_oracle_face_components_counts():
    counts = {"bow_tie": 2, "tetra_bow_tie": 2, "edge_of_3": 3, "edge_of_4": 5, "duplicate_pair": 2,
              "duplicate_triple": 3, "repeated_ids": 4, "unreferenced": 2, "tie_face_order": 2}
    for name, n in counts.items():
        assert OMesh.face_components(np.asarray(HAND_MESHES[name][1], np.int64))[0] == n, name


def test_oracle_clean_mesh_keeps_first_component_among_equals():
    """Component order is smallest face index: relabelling the faces moves the kept component with them."""
    nv, faces, _, _ = HAND_MESHES["tie_face_order"]
    f = np.asarray(faces, np.int64)
    v = _verts(nv)
    rv, rf = OMesh.clean_mesh(v, f[[1, 0, 3, 2]])
    assert np.array_equal(rv, v[[0, 1, 2, 3]]) and np.array_equal(rf, [[0, 1, 2], [2, 1, 3]])
