"""Float64 NumPy restatement of PIXIE's SMPLX.forward (lib/pixielib/models/SMPLX.py:204-294): lbs() with
pose2rot=False (oracle/body_model.py) followed by the landmark and joint heads as the "heads" section of the
csrc/body_model.cu header states them, with an explicit backward and an absolute-value companion.

  lut_row(pose, chain)            -> (row [B], a [B] degrees, tie [B]): the lookup-table row, the head-yaw angle and
                                     the signed distance of min(a, 39) to the nearest half-integer (a test keeps
                                     |tie| clear of 0, where an fp32 and an fp64 evaluation may round apart)
  heads_forward(verts, jt, pose, T) -> (landmarks [B,Ls+Ld,3], joints [B,J+Ls+Ld+E,3], rows [B])
  heads_backward(T, rows, V, J, g_landmarks, g_joints) -> (g_verts [B,V,3], g_J_transformed [B,J,3])
  pixie_bounds(betas, pose, model, T, g_verts, g_landmarks, g_joints)
                                  -> values, gradients of betas and pose, and for each m = sum of |contribution|

T = tables(...) holds the class's buffers as arrays.  Pinned against the reference's own class and head functions by
tests/test_pixie_body_model_cpu.py when a checkout is present, and through tests/golden/pixie_body_model.npz.
"""
import numpy as np

from oracle import body_model as OB

LUT_ROWS = 79


def tables(faces, lmk_faces_idx, lmk_bary_coords, dynamic_lmk_faces_idx, dynamic_lmk_bary_coords, head_kin_chain,
           face_ids, bcs, extra_joint_regressor, source_idxs, target_idxs):
    """The head buffers as arrays (face_ids / bcs empty when the model has no extra joints)."""
    a = lambda x, t: np.asarray(x, t)  # noqa: E731
    return dict(faces=a(faces, np.int64), lmk=a(lmk_faces_idx, np.int64), lmk_bc=a(lmk_bary_coords, np.float64),
                dyn=a(dynamic_lmk_faces_idx, np.int64), dyn_bc=a(dynamic_lmk_bary_coords, np.float64),
                chain=a(head_kin_chain, np.int64), ext=a(face_ids, np.int64).reshape(-1),
                ext_bc=a(bcs, np.float64).reshape(-1, 3), reg=a(extra_joint_regressor, np.float64),
                src=a(source_idxs, np.int64), tgt=a(target_idxs, np.int64))


def lut_row(pose, chain):
    pose = np.asarray(pose, np.float64)
    B = pose.shape[0]
    rel = np.broadcast_to(np.eye(3), (B, 3, 3))
    for c in chain:
        rel = pose[:, c] @ rel
    a = (-np.arctan2(-rel[:, 2, 0], np.sqrt(rel[:, 0, 0] ** 2 + rel[:, 1, 0] ** 2)) * 180.0) / np.pi
    ac = np.minimum(a, 39.0)
    y = np.round(ac)                                     # half to even, as torch.round
    row = np.where(y >= 0, y, np.where(y < -39, 78, 39 - y)).astype(np.int64)
    return row, a, ac - (np.floor(ac) + 0.5)


def _slots(T, rows):
    """Per batch item: corner vertex ids [B,K,3] and weights [B,K,3] of every head entry (K = Ls + Ld + E)."""
    f = T["faces"]
    B = len(rows)
    vid = np.concatenate([np.broadcast_to(f[T["lmk"]], (B, len(T["lmk"]), 3)), f[T["dyn"][rows]],
                          np.broadcast_to(f[T["ext"]], (B, len(T["ext"]), 3))], 1)
    w = np.concatenate([np.broadcast_to(T["lmk_bc"], (B,) + T["lmk_bc"].shape), T["dyn_bc"][rows],
                        np.broadcast_to(T["ext_bc"], (B,) + T["ext_bc"].shape)], 1)
    return vid, w


def heads_forward(verts, jt, pose, T, absmode=False, rows=None):
    """verts [B,V,3], jt [B,J,3] (lbs' outputs; their |.| companions in absmode), pose [B,J,3,3]."""
    verts, jt = np.asarray(verts, np.float64), np.asarray(jt, np.float64)
    B = verts.shape[0]
    if rows is None:
        rows = lut_row(pose, T["chain"])[0]
    vid, w = _slots(T, rows)
    if absmode:
        w = np.abs(w)
    ent = np.einsum("bkq,bkqc->bkc", w, verts[np.arange(B)[:, None, None], vid])
    L = len(T["lmk"]) + T["dyn"].shape[1]
    reg = np.einsum("rv,bvc->brc", np.abs(T["reg"]) if absmode else T["reg"], verts)
    joints = np.concatenate([jt, ent], 1)
    joints[:, T["src"]] = reg[:, T["tgt"]]
    return ent[:, :L].copy(), joints, rows


def heads_backward(T, rows, V, J, g_landmarks=None, g_joints=None, absmode=False):
    f = np.abs if absmode else (lambda x: x)
    B = len(rows)
    L = len(T["lmk"]) + T["dyn"].shape[1]
    K = L + len(T["ext"])
    gj = np.zeros((B, J + K, 3)) if g_joints is None else f(np.asarray(g_joints, np.float64))
    u = gj[:, J:].copy()
    if g_landmarks is not None:
        u[:, :L] += f(np.asarray(g_landmarks, np.float64))
    vid, w = _slots(T, rows)
    w = f(w)
    gv = np.zeros((B, V, 3))
    for b in range(B):
        np.add.at(gv[b], vid[b].reshape(-1), (w[b][..., None] * u[b][:, None, :]).reshape(-1, 3))
    gv += np.einsum("sv,bsc->bvc", f(T["reg"])[T["tgt"]], gj[:, T["src"]])
    gjt = gj[:, :J].copy()
    gjt[:, T["src"]] = 0.0
    return gv, gjt


def pixie_bounds(betas, pose, model, T, g_verts=None, g_landmarks=None, g_joints=None):
    """betas [B,NB] (shape and expression), pose [B,J,3,3], model = (v_template, shapedirs, posedirs, J_regressor,
    parents, lbs_weights).  dict: verts, landmarks, joints, rows, m_* of each and, with an upstream gradient,
    g_betas, g_pose, m_betas, m_pose."""
    pose = np.asarray(pose, np.float64)
    v, jt, sv = OB.forward(betas, pose, *model, pose2rot=False)
    va, ja, sa = OB.forward(betas, pose, *model, pose2rot=False, absmode=True)
    lm, joints, rows = heads_forward(v, jt, pose, T)
    lma, jointsa, _ = heads_forward(va, ja, pose, T, absmode=True, rows=rows)
    out = dict(verts=v, landmarks=lm, joints=joints, rows=rows, m_verts=va, m_landmarks=lma, m_joints=jointsa)
    if g_verts is None and g_landmarks is None and g_joints is None:
        return out
    B, V, J = v.shape[0], v.shape[1], jt.shape[1]
    for absmode, saved, key in ((False, sv, "g_"), (True, sa, "m_")):
        f = np.abs if absmode else (lambda x: x)
        gv, gjt = heads_backward(T, rows, V, J, g_landmarks, g_joints, absmode)
        if g_verts is not None:
            gv = gv + f(np.asarray(g_verts, np.float64))
        out[key + "betas"], out[key + "pose"] = OB.backward(saved, gv, gjt)
    return out
