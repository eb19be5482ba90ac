"""oracle/prt.py -- TEST INFRASTRUCTURE ONLY.

The checker of icon_prt (the PRT transfer of lib/renderer/prt_util.py:115-182, computePRT):

* hit_bits: brute-force any-hit ray cast (oracle/prt_oracle.c), every ray against every face with geom.cuh's fp32
  Moller-Trumbore convention; build() compiles it with the same gcc flags as the other oracle sources (no implicit
  contraction) into oracle/libprt_oracle.so.
* sh_basis: the real spherical-harmonic basis up to `order`, restated from its definition (below), in the column
  order the reference's getSHCoeffs uses: degree l = 0..order, order m = -l..l.
* transfer: PRT[v, k] = w sum_d front (1 - hit) dot SH[d, k] in float64, in the reference's order: the terms of a
  block of n directions summed in direction order, the block sums added in block order, then times w; plus the
  matching sum of |terms| for tolerances.

Real SH (with the Condon-Shortley phase in P_l^m, as the reference's Legendre recursion has it):
    Y_l^0 = K_l^0 P_l^0(cos theta),
    Y_l^m = sqrt(2) K_l^m cos(m phi) P_l^m(cos theta),          m > 0,
    Y_l^m = sqrt(2) K_l^|m| sin(|m| phi) P_l^|m|(cos theta),     m < 0,
    K_l^m = sqrt((2l + 1) / (4 pi) (l - m)! / (l + m)!).
"""
import ctypes
import math
import os
import subprocess

import numpy as np
from scipy.special import lpmv

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libprt_oracle.so")
_SRCS = [os.path.join(_HERE, f) for f in ("prt_oracle.c", "sdf_oracle.c")]


def build(force=False):
    if (not force and os.path.exists(_SO)
            and all(os.path.getmtime(_SO) >= os.path.getmtime(s) for s in _SRCS)):
        return _SO
    # -O3: the face loop is written to vectorise; the arithmetic contract is unchanged (no contraction, IEEE fp32)
    cmd = ["gcc", "-O3", "-shared", "-fPIC", "-fopenmp", "-mfma", "-mavx2", "-ffp-contract=off",
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


def ray_origins(origins, normals, delta):
    """fp32(o + delta n): formed in float64 as the reference forms it, rounded once."""
    o = np.asarray(origins, np.float64)
    return (o + delta * np.asarray(normals, np.float64)).astype(np.float32)


def hit_bits(origins32, dirs, verts, faces):
    """origins32 [N,3] f32, dirs [D,3] (rounded to f32), verts [V,3] f32, faces [F,3] -> uint32 [N, ceil(D/32)]."""
    o = np.ascontiguousarray(origins32, np.float32).reshape(-1, 3)
    d = np.ascontiguousarray(dirs, np.float64).astype(np.float32).reshape(-1, 3)
    v = np.ascontiguousarray(verts, np.float32)
    f = np.ascontiguousarray(faces, np.int64)
    out = np.zeros((len(o), (len(d) + 31) // 32), np.uint32)
    P = ctypes.c_void_p
    lib().oracle_prt_hits(P(o.ctypes.data), ctypes.c_int64(len(o)), P(d.ctypes.data), ctypes.c_int(len(d)),
                          P(v.ctypes.data), ctypes.c_int(len(v)), P(f.ctypes.data), ctypes.c_int(len(f)),
                          P(out.ctypes.data))
    return out


def unpack(bits, D):
    """uint32 [N, ceil(D/32)] -> bool [N, D]"""
    b = np.asarray(bits, np.uint32)
    return ((b[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(len(b), -1)[:, :D].astype(bool)


def sh_basis(order, phi, theta):
    """[D, (order+1)^2] float64 real SH of the directions (phi, theta)."""
    phi, theta = np.asarray(phi, np.float64), np.asarray(theta, np.float64)
    x = np.cos(theta)
    cols = []
    for l in range(order + 1):
        for m in range(-l, l + 1):
            a = abs(m)
            k = math.sqrt((2 * l + 1) / (4 * math.pi) * math.factorial(l - a) / math.factorial(l + a))
            p = lpmv(a, l, x)
            if m == 0:
                cols.append(k * p)
            elif m > 0:
                cols.append(math.sqrt(2.0) * k * np.cos(m * phi) * p)
            else:
                cols.append(math.sqrt(2.0) * k * np.sin(a * phi) * p)
    return np.stack(cols, 1)


def transfer(normals, dirs, sh, w, hit, n=None):
    """PRT [V,K] and sum |terms| [V,K] (float64).  normals [V,3], dirs [D,3], sh [D,K], hit bool [V,D]; n: the
    block size (default: sqrt(D) when D is a square, else D)."""
    nrm, d, sh = (np.asarray(a, np.float64) for a in (normals, dirs, sh))
    D = len(d)
    if n is None:
        r = int(round(math.sqrt(D)))
        n = r if r * r == D else D
    dots = (d[None, :, 0] * nrm[:, None, 0] + d[None, :, 1] * nrm[:, None, 1]) + d[None, :, 2] * nrm[:, None, 2]
    lit = np.logical_and(dots > 0.0, np.logical_not(hit)).astype(np.float64)
    acc = absacc = None
    for b0 in range(0, D, n):
        s = None
        for j in range(b0, min(b0 + n, D)):
            term = (lit[:, j] * dots[:, j])[:, None] * sh[None, j]
            s = term if s is None else s + term
            absacc = np.abs(term) if absacc is None else absacc + np.abs(term)
        acc = s if acc is None else acc + s
    return w * acc, abs(w) * absacc
