"""Build tests/golden/prt.npz: the reference's own sphere sampling and SH basis, as its computePRT
(lib/renderer/prt_util.py:115-182) calls them, for the checks of oracle/prt.py and icon_b200/prt.py.

For n in {1, 10, 40}: np.random.seed(0), then sampleSphericalDirections(n) -> dirs_n [n^2,3], phi_n, theta_n, and
getSHCoeffs(order, phi_n, theta_n) -> sh_n_order [n^2,(order+1)^2] for order 0..3.  Both functions need only NumPy,
but prt_util.py imports trimesh at the top, so they are compiled from the checkout's source with `ast` (every other
definition is left out).  Needs the ICON checkout (ICON_REFERENCE_DIR); the fixture is committed.

    ICON_REFERENCE_DIR=/path/to/ICON python tests/golden/make_prt.py
"""
import ast
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = ("factratio", "KVal", "AssociatedLegendre", "SphericalHarmonic", "sampleSphericalDirections", "getSHCoeffs")


def reference_functions(root):
    path = os.path.join(root, "lib", "renderer", "prt_util.py")
    tree = ast.parse(open(path).read(), path)
    defs = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in NAMES]
    assert sorted(n.name for n in defs) == sorted(NAMES), [n.name for n in defs]
    g = {"np": np, "math": math}
    exec(compile(ast.Module(defs, []), path, "exec"), g)
    return g


def main():
    g = reference_functions(os.environ["ICON_REFERENCE_DIR"])
    out = {}
    for n in (1, 10, 40):
        np.random.seed(0)
        dirs, phi, theta = g["sampleSphericalDirections"](n)
        out[f"dirs_{n}"], out[f"phi_{n}"], out[f"theta_{n}"] = dirs, phi, theta
        for order in range(4):
            out[f"sh_{n}_{order}"] = g["getSHCoeffs"](order, phi, theta)
    np.savez_compressed(os.path.join(HERE, "prt.npz"), **out)


if __name__ == "__main__":
    main()
