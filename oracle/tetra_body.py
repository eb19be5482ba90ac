"""NumPy restatement of PaMIR's tetrahedral body as TestDataset.compute_voxel_verts builds it
(lib/dataset/TestDataset.py:150-192, lib/dataset/body_model.py:344-427), in the order csrc/body_model.cu's tetra
section follows, with an absolute-value companion.

  rotmat_to_aa(R)            -> aa [N,3] float32: pymaf's rotation_matrix_to_angle_axis (eps = 1e-6) op by op in
                                float32, NaN -> 0 (np.arctan2 stands for torch's atan2: equal to a few ulps).
  skin(model, aa, beta)      -> (verts [V + V_added, 3] float64, m): TetraSMPLModel.update's vertices followed by
                                its added vertices; m = sum of |contribution| per component (every factor replaced by
                                its |.|, a difference a - b by |a| + |b|, sin / cos by |sin| / |cos|), the yardstick
                                the tests divide float64 differences by.
  voxel_verts(verts, scale, trans) -> [8000,3] float32: fp32(v scale + trans), zero rows to 8000, x 0.5, z <- -z.
  model_arrays(model)        -> the arrays skin() reads, from a TetraSMPLModel-like object or a tetra_model() dict.

dtype chain (NumPy >= 2, as the reference runs there): the pose and betas arrive float32; theta =
np.linalg.norm(r, axis=(1, 2)) stays float32 (sqrt of the float32 sum (x^2 + y^2) + z^2), np.maximum with the float64
`tiny` widens it, and everything after it is float64 (r / theta, the float64 model arrays dotted with the float32
betas).
"""
import numpy as np

PAD_V = 8000
PAD_F = 25100
EPS = np.float32(1e-6)      # torch compares the float32 rmat[2,2] with the scalar in float32


def rotmat_to_aa(R):
    """pymaf's rotation_matrix_to_angle_axis on R [N,3,3] (float32), restated op by op."""
    f = np.float32
    R = np.asarray(R, np.float32)
    t = np.swapaxes(R, 1, 2)                       # rmat_t[:, a, b] = R[:, b, a]
    one = f(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        d2 = t[:, 2, 2] < EPS
        d0d1 = t[:, 0, 0] > t[:, 1, 1]
        d0nd1 = t[:, 0, 0] < -t[:, 1, 1]
        t0 = ((one + t[:, 0, 0]) - t[:, 1, 1]) - t[:, 2, 2]
        q0 = np.stack([t[:, 1, 2] - t[:, 2, 1], t0, t[:, 0, 1] + t[:, 1, 0], t[:, 2, 0] + t[:, 0, 2]], -1)
        t1 = ((one - t[:, 0, 0]) + t[:, 1, 1]) - t[:, 2, 2]
        q1 = np.stack([t[:, 2, 0] - t[:, 0, 2], t[:, 0, 1] + t[:, 1, 0], t1, t[:, 1, 2] + t[:, 2, 1]], -1)
        t2 = ((one - t[:, 0, 0]) - t[:, 1, 1]) + t[:, 2, 2]
        q2 = np.stack([t[:, 0, 1] - t[:, 1, 0], t[:, 2, 0] + t[:, 0, 2], t[:, 1, 2] + t[:, 2, 1], t2], -1)
        t3 = ((one + t[:, 0, 0]) + t[:, 1, 1]) + t[:, 2, 2]
        q3 = np.stack([t3, t[:, 1, 2] - t[:, 2, 1], t[:, 2, 0] - t[:, 0, 2], t[:, 0, 1] - t[:, 1, 0]], -1)
        m = [(d2 & d0d1), (d2 & ~d0d1), (~d2 & d0nd1), (~d2 & ~d0nd1)]
        m = [x.astype(np.float32)[:, None] for x in m]
        q = ((q0 * m[0] + q1 * m[1]) + q2 * m[2]) + q3 * m[3]
        den = ((t0[:, None] * m[0] + t1[:, None] * m[1]) + t2[:, None] * m[2]) + t3[:, None] * m[3]
        q = q / np.sqrt(den)
        q = q * f(0.5)
        s2 = (q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3]
        st = np.sqrt(s2)
        ct = q[:, 0]
        two = f(2) * np.where(ct < 0, np.arctan2(-st, -ct), np.arctan2(st, ct))
        k = np.where(s2 > 0, two / st, f(2))
        aa = f(0) + q[:, 1:] * k[:, None]
    aa[np.isnan(aa)] = 0
    return aa.astype(np.float32)


def model_arrays(model):
    """{v_template, shapedirs, posedirs, weights (both sets stacked, float64), J_regressor (dense [24,V] float64),
    parents [24] (root -1)} from a TetraSMPLModel or a synthetic.tetra_model() dict."""
    g = (lambda k: model[k]) if isinstance(model, dict) else (lambda k: getattr(model, k))
    jr = g("J_regressor")
    jr = jr.toarray() if hasattr(jr, "toarray") else np.asarray(jr)
    kin = np.asarray(g("kintree_table"))
    col = {int(kin[1, i]): i for i in range(kin.shape[1])}
    parents = [-1] + [col[int(kin[0, i])] for i in range(1, kin.shape[1])]
    cat = lambda a, b: np.concatenate([np.asarray(g(a), np.float64), np.asarray(g(b), np.float64)], 0)  # noqa: E731
    return dict(v_template=cat("v_template", "v_template_added"), shapedirs=cat("shapedirs", "shapedirs_added"),
                posedirs=cat("posedirs", "posedirs_added"), weights=cat("weights", "weights_added"),
                J_regressor=np.asarray(jr, np.float64), parents=parents, V=np.asarray(g("v_template")).shape[0])


def rodrigues(aa, absmode=False):
    """TetraSMPLModel.rodrigues on float32 aa [24,3]: theta the float32 norm, widened; R [24,3,3] float64."""
    x = np.asarray(aa, np.float32)
    th32 = np.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])
    th = np.maximum(th32.astype(np.float64), np.finfo(np.float64).tiny)[:, None]
    rh = x.astype(np.float64) / th
    cs, sn = np.cos(th)[:, :, None], np.sin(th)[:, :, None]
    z = np.zeros(len(x))
    mk = np.stack([z, -rh[:, 2], rh[:, 1], rh[:, 2], z, -rh[:, 0], -rh[:, 1], rh[:, 0], z], -1).reshape(-1, 3, 3)
    dot = rh[:, :, None] * rh[:, None, :]
    if absmode:
        return np.abs(cs) * np.eye(3) + (1.0 + np.abs(cs)) * np.abs(dot) + np.abs(sn) * np.abs(mk)
    return cs * np.eye(3) + (1.0 - cs) * dot + sn * mk


def skin(arr, aa, beta, absmode=False):
    """TetraSMPLModel.update's verts and verts_added, stacked [V + V_added, 3] (trans zero), float64; with absmode,
    the sum-of-|contribution| companion."""
    f = np.abs if absmode else (lambda x: x)
    sub = (lambda a, b: a + b) if absmode else (lambda a, b: a - b)
    beta = f(np.asarray(beta, np.float32).astype(np.float64))
    vs = np.einsum("vck,k->vc", f(arr["shapedirs"]), beta) + f(arr["v_template"])
    Jm = f(arr["J_regressor"]) @ vs[:arr["V"]]
    R = rodrigues(aa, absmode)
    pf = sub(R[1:], np.eye(3)).reshape(-1)
    vp = vs + np.einsum("vcp,p->vc", f(arr["posedirs"]), pf)
    par = arr["parents"]
    G = np.zeros((24, 4, 4))
    for i in range(24):
        rel = Jm[i] if par[i] < 0 else sub(Jm[i], Jm[par[i]])
        L = np.eye(4)
        L[:3, :3], L[:3, 3] = R[i], rel
        G[i] = L if par[i] < 0 else G[par[i]] @ L
    A = G.copy()
    A[:, :3, 3] = sub(G[:, :3, 3], np.einsum("jrc,jc->jr", G[:, :3, :3], Jm))
    T = np.einsum("vj,jrc->vrc", f(arr["weights"]), A)
    return np.einsum("vrc,vc->vr", T[:, :3, :3], vp) + T[:, :3, 3]


def skin_bounds(arr, aa, beta):
    """(verts, m) of skin()."""
    return skin(arr, aa, beta), skin(arr, aa, beta, absmode=True)


def voxel_verts(verts, scale, trans):
    """compute_voxel_verts' epilogue on the stacked float64 vertices: [8000,3] float32."""
    v = np.asarray(verts, np.float64) * float(np.float32(scale)) + np.asarray(trans, np.float32).reshape(1, 3)
    out = np.zeros((PAD_V, 3), np.float32)
    out[:len(v)] = v.astype(np.float32)
    out = out * np.float32(0.5)
    out[:, 2] *= np.float32(-1.0)
    return out
