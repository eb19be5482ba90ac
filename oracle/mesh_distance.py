"""oracle/mesh_distance.py -- TEST INFRASTRUCTURE ONLY.

Brute-force unsigned point-to-mesh distance (oracle/mesh_oracle.c), the checker of icon_mesh_distance: every point
against every face with sdf_oracle.c's fp32 Ericson distance, lowest face index on ties.  build() compiles it with the
same gcc flags as the other oracle sources (no implicit contraction) into oracle/libmesh_oracle.so.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libmesh_oracle.so")
_SRCS = [os.path.join(_HERE, f) for f in ("mesh_oracle.c", "sdf_oracle.c")]


def build(force=False):
    if (not force and os.path.exists(_SO)
            and all(os.path.getmtime(_SO) >= os.path.getmtime(s) for s in _SRCS)):
        return _SO
    cmd = ["gcc", "-O2", "-shared", "-fPIC", "-fopenmp", "-mfma", "-mavx2", "-ffp-contract=off",
           "-fno-fast-math", "-o", _SO, _SRCS[0], "-lm"]
    subprocess.check_call(cmd)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        _lib = ctypes.CDLL(_SO)
    return _lib


def mesh_distance(points, verts, faces):
    """points [N,3], verts [V,3], faces [F,3] -> (squared distance f32 [N], nearest face i32 [N])"""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    v = np.ascontiguousarray(verts, np.float32)
    f = np.ascontiguousarray(faces, np.int64)
    d = np.empty(len(p), np.float32)
    fi = np.empty(len(p), np.int32)
    P = ctypes.c_void_p
    lib().oracle_mesh_distance(P(p.ctypes.data), ctypes.c_int64(len(p)), P(v.ctypes.data), ctypes.c_int(len(v)),
                               P(f.ctypes.data), ctypes.c_int(len(f)), P(d.ctypes.data), P(fi.ctypes.data))
    return d, fi
