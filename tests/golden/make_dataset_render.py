"""Build tests/golden/dataset_render.npz: what scripts/render_single.py feeds its renderers, taken from the reference's
own code and sample scan, for the checks of oracle/dataset_render.py and icon_b200/dataset_render.py.

* rotateBand2 / rotateSH (lib/renderer/opengl_util.py) on seeded inputs and make_rotate rotations;
* Camera.get_gl_matrix() (lib/renderer/camera.py with glm.ortho) at the script's settings (ortho_ratio
  0.4 * 512 / size, near / far -100 / 100 for the front view, swapped for the back), at 512^2 and 96 x 64;
* load_calib for the same settings and several rotations y;
* rows 0, 7, 100 and 239 of scripts/env_sh.npy;
* a textured patch of the sample scan (sample_data/thuman2/scans/0525): the faces whose centroid lies in a box on the
  torso, with their vt.  Vertices and uvs are renumbered separately and the uvs of the faces right of a vertical line
  are duplicated (a split seam), so faces_uvs != faces; material0.jpeg is cropped to the patch's uv box and resized
  to 151 x 117 (odd), the uvs remapped into the crop.

The functions need only NumPy but the modules import cv2 / OpenGL at the top, so they are compiled from the checkout's
source with `ast` (every other definition is left out).  Needs the ICON checkout (ICON_REFERENCE_DIR) and OpenCV; the
fixture is committed.

    ICON_REFERENCE_DIR=/path/to/ICON python tests/golden/make_dataset_render.py
"""
import ast
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
Y_ROT = (0, 10, 90, 170, 350)
TEX_W, TEX_H = 151, 117


def _compile(path, names, g):
    tree = ast.parse(open(path).read(), path)
    defs = [n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in names]
    assert sorted(n.name for n in defs) == sorted(names), [n.name for n in defs]
    exec(compile(ast.Module(defs, []), path, "exec"), g)
    return g


def reference_functions(root):
    r = os.path.join(root, "lib", "renderer")
    g = {"np": np, "math": math}
    _compile(os.path.join(r, "glm.py"), ("identity", "ortho"), g)
    _compile(os.path.join(r, "camera.py"), ("Camera",), g)
    _compile(os.path.join(r, "opengl_util.py"), ("make_rotate", "rotateSH", "rotateBand2", "load_calib"), g)
    return g


def textured_patch(root):
    import cv2
    scan = os.path.join(root, "sample_data", "thuman2", "scans", "0525")
    v, vt, f, ft = [], [], [], []
    for line in open(os.path.join(scan, "0525.obj")):
        s = line.split()
        if not s:
            continue
        if s[0] == "v":
            v.append([float(x) for x in s[1:4]])
        elif s[0] == "vt":
            vt.append([float(x) for x in s[1:3]])
        elif s[0] == "f":
            f.append([int(x.split("/")[0]) - 1 for x in s[1:4]])
            ft.append([int(x.split("/")[1]) - 1 for x in s[1:4]])
    v, vt, f, ft = np.array(v), np.array(vt), np.array(f), np.array(ft)
    c = v[f].mean(1)
    lo, hi = np.percentile(v, 40, 0), np.percentile(v, 60, 0)
    sel = np.nonzero((c[:, 0] > lo[0]) & (c[:, 0] < hi[0]) & (c[:, 1] > lo[1]) & (c[:, 1] < hi[1]))[0][:3000]
    f, ft = f[sel], ft[sel]
    uv_v, f_new = np.unique(f, return_inverse=True)
    uv_t, ft_new = np.unique(ft, return_inverse=True)
    verts, faces = v[uv_v], f_new.reshape(-1, 3)
    uvs, faces_uvs = vt[uv_t][::-1].copy(), (len(uv_t) - 1 - ft_new).reshape(-1, 3)       # reversed numbering
    right = verts[faces].mean(1)[:, 0] > np.median(verts[:, 0])                            # the seam
    dup = np.unique(faces_uvs[right])
    remap = np.full(len(uvs), -1)
    remap[dup] = len(uvs) + np.arange(len(dup))
    uvs = np.concatenate([uvs, uvs[dup]])
    faces_uvs[right] = remap[faces_uvs[right]]
    img = cv2.cvtColor(cv2.imread(os.path.join(scan, "material0.jpeg")), cv2.COLOR_BGR2RGB)
    H, W = img.shape[:2]
    u0, v0 = uvs.min(0) - 0.01
    u1, v1 = uvs.max(0) + 0.01
    x0, x1 = int(math.floor(u0 * W)), int(math.ceil(u1 * W))
    y0, y1 = int(math.floor((1 - v1) * H)), int(math.ceil((1 - v0) * H))       # image rows: v = 1 at the top
    crop = img[y0:y1, x0:x1]
    tex = cv2.resize(crop, (TEX_W, TEX_H), interpolation=cv2.INTER_AREA)
    uvs = np.stack([(uvs[:, 0] * W - x0) / (x1 - x0), (uvs[:, 1] * H - (H - y1)) / (y1 - y0)], 1)
    return dict(patch_verts=verts, patch_faces=faces, patch_uvs=uvs, patch_faces_uvs=faces_uvs, patch_tex=tex)


def main():
    root = os.environ["ICON_REFERENCE_DIR"]
    g = reference_functions(root)
    out = {}
    rng = np.random.default_rng(0)
    xs = rng.standard_normal((6, 5))
    shs = rng.standard_normal((6, 9, 3))
    angles = rng.uniform(-math.pi, math.pi, (6, 3))
    out["band2_x"], out["sh_in"], out["angles"] = xs, shs, angles
    b2, rs, Rs = [], [], []
    for k in range(6):
        R = g["make_rotate"](*angles[k])
        Rs.append(R)
        b2.append(g["rotateBand2"](xs[k].copy(), R))
        rs.append(g["rotateSH"](shs[k].copy(), R))
    out["rot"], out["band2_out"], out["rotsh_out"] = np.array(Rs), np.array(b2), np.array(rs)
    for size in ((512, 512), (96, 64)):
        W, H = size
        cam = g["Camera"](width=W, height=H)
        cam.ortho_ratio = 0.4 * (512 / W)
        for side, (near, far) in (("front", (-100, 100)), ("back", (100, -100))):
            cam.near, cam.far = near, far
            cam.sanity_check()
            P, M = cam.get_gl_matrix()
            out[f"persp_{W}x{H}_{side}"], out[f"model_{W}x{H}_{side}"] = P, M
    center = np.array([1.5, 90.0, -3.0])
    for y in Y_ROT:
        R = g["make_rotate"](0, math.radians(y), 0)
        out[f"calib_{y}"] = g["load_calib"]({"ortho_ratio": 0.4, "scale": 0.011, "center": center, "R": R},
                                            render_size=512)
    out["calib_center"] = center
    out["env_sh_rows"] = np.array([0, 7, 100, 239])
    out["env_sh"] = np.load(os.path.join(root, "scripts", "env_sh.npy"))[out["env_sh_rows"]]
    out.update(textured_patch(root))
    np.savez_compressed(os.path.join(HERE, "dataset_render.npz"), **out)


if __name__ == "__main__":
    main()
