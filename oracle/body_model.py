"""Float64 NumPy restatement of lbs() (lib/smplx/lbs.py:152-252) as csrc/body_model.cu states it, with an explicit
backward and an absolute-value companion.

  forward(...)        -> (verts [B,V,3], joints [B,J,3], saved)
  backward(saved, g_verts, g_joints) -> (g_betas [B,NB], g_pose: [B,J,3] with pose2rot, else [B,J,3,3])
  lbs_bounds(...)     -> values, gradients and, for every component of each, m = sum of |contribution|: the same
                         expressions evaluated on |.| of every factor (a difference a - b becomes |a| + |b|; sin, cos
                         become |sin|, |cos|), the yardstick the GPU tests divide their errors by.

Pinned against the reference's own lib/smplx (forward and torch autograd) by tests/test_body_model_cpu.py when a
checkout is present, and through tests/golden/body_model.npz on the GPU.
"""
import numpy as np

EPS = 1e-8


def _skew(d):
    z = np.zeros(d.shape[:-1])
    return np.stack([z, -d[..., 2], d[..., 1], d[..., 2], z, -d[..., 0], -d[..., 1], d[..., 0], z],
                    -1).reshape(d.shape[:-1] + (3, 3))


def rodrigues(r, absmode=False):
    """r [...,3] -> (R [...,3,3], (s, theta, d, K)); s = r + 1e-8 per component, theta = |s|, d = r / theta."""
    s = r + EPS
    th = np.sqrt((s * s).sum(-1, keepdims=True))
    d = r / th
    K = _skew(d)
    sn, cs = np.sin(th)[..., None], np.cos(th)[..., None]
    if absmode:
        K, sn, c1 = np.abs(K), np.abs(sn), 1.0 + np.abs(cs)
    else:
        c1 = 1.0 - cs
    R = np.eye(3) + sn * K + c1 * (K @ K)
    return R, (s, th, d, K)


def rodrigues_backward(r, gR, absmode=False):
    s, th, d, K = rodrigues(r)[1]
    sn, cs = np.sin(th)[..., None], np.cos(th)[..., None]
    KK = K @ K
    Kt = np.swapaxes(K, -1, -2)
    if absmode:
        K, KK, Kt, sn, cs, c1, gR = np.abs(K), np.abs(KK), np.abs(Kt), np.abs(sn), np.abs(cs), 1.0 + np.abs(cs), np.abs(gR)
    else:
        c1 = 1.0 - cs
    gK = sn * gR + c1 * (gR @ Kt + Kt @ gR)
    gsin = (gR * K).sum((-1, -2))[..., None]
    gc1 = (gR * KK).sum((-1, -2))[..., None]
    gth = cs[..., 0] * gsin + sn[..., 0] * gc1
    sub = (lambda a, b: a + b) if absmode else (lambda a, b: a - b)
    gd = np.stack([sub(gK[..., 2, 1], gK[..., 1, 2]), sub(gK[..., 0, 2], gK[..., 2, 0]),
                   sub(gK[..., 1, 0], gK[..., 0, 1])], -1)
    ra, sa = (np.abs(r), np.abs(s)) if absmode else (r, s)
    gth = sub(gth, (gd * ra).sum(-1, keepdims=True) / (th * th))
    return gd / th + gth * (sa / th)


def forward(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True,
            absmode=False):
    """All inputs as float64 arrays; betas [B,NB], pose [B,J*3] / [B,J,3] (pose2rot) or [B,J,3,3]."""
    f = np.abs if absmode else (lambda x: x)
    sub = (lambda a, b: a + b) if absmode else (lambda a, b: a - b)
    betas, vt, sd, pd, Jr, W = (f(np.asarray(x, np.float64)) for x in
                                (betas, v_template, shapedirs, posedirs, J_regressor, lbs_weights))
    pose = np.asarray(pose, np.float64)
    par = np.asarray(parents, np.int64)
    B, NB = betas.shape
    V, J = vt.shape[0], Jr.shape[0]
    vs = vt[None] + np.einsum("vck,bk->bvc", sd, betas)
    Jt = np.einsum("jv,bvc->bjc", Jr, vs)
    if pose2rot:
        aa = pose.reshape(B, J, 3)
        R = rodrigues(aa, absmode)[0]
    else:
        aa = None
        R = f(pose.reshape(B, J, 3, 3))
    pf = sub(R[:, 1:], np.eye(3)).reshape(B, -1)
    vp = vs + (pf @ pd).reshape(B, V, 3)
    rel = Jt.copy()
    rel[:, 1:] = sub(Jt[:, 1:], Jt[:, par[1:]])
    G = np.zeros((B, J, 3, 4))
    for j in range(J):
        if par[j] < 0:
            G[:, j, :, :3], G[:, j, :, 3] = R[:, j], rel[:, j]
        else:
            Gp = G[:, par[j]]
            G[:, j, :, :3] = Gp[:, :, :3] @ R[:, j]
            G[:, j, :, 3] = np.einsum("brk,bk->br", Gp[:, :, :3], rel[:, j]) + Gp[:, :, 3]
    A = G.copy()
    A[..., 3] = sub(G[..., 3], np.einsum("bjrk,bjk->bjr", G[..., :3], Jt))
    T = np.einsum("vj,bjrc->bvrc", W, A)
    verts = np.einsum("bvrc,bvc->bvr", T[..., :3], vp) + T[..., 3]
    joints = G[..., 3].copy()
    saved = dict(betas=betas, aa=aa, R=R, vp=vp, Jt=Jt, rel=rel, G=G, T=T, sd=sd, pd=pd, Jr=Jr, W=W, par=par,
                 pose2rot=pose2rot, absmode=absmode)
    return verts, joints, saved


def backward(saved, g_verts=None, g_joints=None):
    s = saved
    absmode = s["absmode"]
    f = np.abs if absmode else (lambda x: x)
    sub = (lambda a, b: a + b) if absmode else (lambda a, b: a - b)
    R, vp, Jt, rel, G, T, sd, pd, Jr, W, par = (s[k] for k in ("R", "vp", "Jt", "rel", "G", "T", "sd", "pd", "Jr",
                                                                 "W", "par"))
    B, V, J = vp.shape[0], vp.shape[1], Jt.shape[1]
    gv = f(np.zeros((B, V, 3)) if g_verts is None else np.asarray(g_verts, np.float64).reshape(B, V, 3))
    gj = f(np.zeros((B, J, 3)) if g_joints is None else np.asarray(g_joints, np.float64).reshape(B, J, 3))
    gT = np.concatenate([gv[..., :, None] * vp[..., None, :], gv[..., None]], -1)        # [B,V,3,4]
    gvp = np.einsum("bvrc,bvr->bvc", T[..., :3], gv)
    gA = np.einsum("vj,bvre->bjre", W, gT)
    gpf = gvp.reshape(B, -1) @ pd.T
    gbeta = np.einsum("vck,bvc->bk", sd, gvp)
    gG = np.zeros((B, J, 3, 4))
    gG[..., :3] = sub(gA[..., :3], gA[..., 3][..., :, None] * Jt[..., None, :])
    gG[..., 3] = gA[..., 3] + gj
    gJ = np.einsum("bjrc,bjr->bjc", G[..., :3], gA[..., 3])
    gJ = gJ if absmode else -gJ
    gR = np.zeros((B, J, 3, 3))
    grel = np.zeros((B, J, 3))
    for j in range(J - 1, -1, -1):
        p = par[j]
        if p < 0:
            gR[:, j], grel[:, j] = gG[:, j, :, :3], gG[:, j, :, 3]
            continue
        GpR = G[:, p, :, :3]
        gR[:, j] = np.swapaxes(GpR, -1, -2) @ gG[:, j, :, :3]
        grel[:, j] = np.einsum("brk,br->bk", GpR, gG[:, j, :, 3])
        gG[:, p, :, :3] += gG[:, j, :, :3] @ np.swapaxes(R[:, j], -1, -2) + gG[:, j, :, 3][..., None] * rel[:, j][
            :, None, :]
        gG[:, p, :, 3] += gG[:, j, :, 3]
    gJ = gJ + grel
    for j in range(1, J):
        gJ[:, par[j]] = sub(gJ[:, par[j]], grel[:, j])
    gR[:, 1:] += gpf.reshape(B, J - 1, 3, 3)
    gvs = np.einsum("jv,bjc->bvc", Jr, gJ)
    gbeta = gbeta + np.einsum("vck,bvc->bk", sd, gvs)
    if s["pose2rot"]:
        gpose = rodrigues_backward(s["aa"], gR, absmode)
    else:
        gpose = gR
    return gbeta, gpose


def lbs_bounds(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True,
               g_verts=None, g_joints=None):
    """dict: verts, joints, m_verts, m_joints and (with an upstream gradient) g_betas, g_pose, m_betas, m_pose."""
    args = (betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot)
    v, j, sv = forward(*args)
    va, ja, sa = forward(*args, absmode=True)
    out = dict(verts=v, joints=j, m_verts=va, m_joints=ja)
    if g_verts is not None or g_joints is not None:
        out["g_betas"], out["g_pose"] = backward(sv, g_verts, g_joints)
        out["m_betas"], out["m_pose"] = backward(sa, g_verts, g_joints)
    return out
