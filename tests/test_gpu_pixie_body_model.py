"""PIXIE's SMPL-X on the kernels (icon_b200.body_model.make_pixie_SMPLX: the skinning plus the landmark and joint
heads of csrc/body_model.cu) against oracle/pixie_body_model.py and against the reference class's own outputs
(tests/golden/pixie_body_model.npz), on the tiny and the real-size synthetic models.

Bars, in units of m = sum of |contribution| per component (the oracle's absolute-value companion): verts, landmarks
and joints within 2^-18 m; gradients of shape, expression and every pose part within 2^-17 m; lookup rows exact
(every case's yaw angle is asserted clear of a rounding tie).  Also: two runs bitwise equal; row b of a B = 3 call
equal to a one-row call; no host sync in a warm forward plus backward; four launches forward and three backward; CPU
and float64 calls reach the reference's forward; the `-hps_type pixie` body-fit iteration of
apps/infer.py:184-197, 200-270 end to end.
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402
from oracle import pixie_body_model as OP  # noqa: E402
from test_pixie_body_model_cpu import (HEADS, MODEL, _oracle_model, _standin_class, golden_full_inputs,  # noqa
                                       golden_grad_parts)

TOL_FWD = 2.0 ** -18
TOL_BWD = 2.0 ** -17
WORST = {}
POSES = (("global_pose", 0, 1), ("body_pose", 1, 22), ("jaw_pose", 22, 23), ("eye_pose", 23, 25),
         ("left_hand_pose", 25, 40), ("right_hand_pose", 40, 55))


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))
    print("pixie body_model worst error / m:", json.dumps(WORST, sort_keys=True))


def _ratio(got, ref, m, tol):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    r = err / np.maximum(m, 1e-300)
    i = np.unravel_index(np.argmax(r), r.shape)
    assert np.all(err <= tol * m), (float(r[i]), i, float(got[i]), float(ref[i]), float(m[i]))
    return float(r.max())


def _module(buf, dev, n_shape=10):
    """synthetic's PIXIE SMPLX stand-in, patched by make_pixie_SMPLX, on `dev`; and the list of the calls that
    reached the stand-in's own (reference) forward."""
    from icon_b200 import body_model as BM
    K, seen = _standin_class(BM, n_shape)
    return K(buf).to(dev), seen


def _args(betas, pose, dev, ns, none=()):
    """SMPLX.forward's keyword arguments (leaves requiring grad) from betas [B,NB] and the full pose [B,55,3,3]."""
    t = lambda x: torch.tensor(np.asarray(x, np.float32), device=dev, requires_grad=True)  # noqa: E731
    args = {"shape_params": t(betas[:, :ns]), "expression_params": t(betas[:, ns:])}
    for k, lo, hi in POSES:
        args[k] = t(pose[:, lo:hi])
    return {k: (None if k in none else v) for k, v in args.items()}


def _inputs(B, seed, ns, ne):
    rng = np.random.RandomState(seed)
    from oracle.body_model import rodrigues
    pose = rodrigues(0.3 * rng.standard_normal((B, 55, 3)))[0] + 0.03 * rng.standard_normal((B, 55, 3, 3))
    pose = pose.astype(np.float32).astype(np.float64)
    betas = rng.standard_normal((B, ns + ne)).astype(np.float32).astype(np.float64)
    return betas, pose, rng


def _compare(key, mod, args, betas, pose, model, T, gv, gl, gj, dev):
    """One forward (+ backward with the upstreams given) against the oracle; returns the outputs."""
    v, lm, jo = mod(**args)
    outs, ups = zip(*[(o, torch.from_numpy(g).to(dev)) for o, g in ((v, gv), (lm, gl), (jo, gj)) if g is not None])
    torch.autograd.backward(list(outs), list(ups))
    out = OP.pixie_bounds(betas, pose, model, T, g_verts=gv, g_landmarks=gl, g_joints=gj)
    assert np.all(np.abs(OP.lut_row(pose, T["chain"])[2]) >= 1e-3), "a yaw angle too close to a rounding tie"
    for k, o in (("verts", v), ("landmarks", lm), ("joints", jo)):
        _note(f"{key}:{k}", _ratio(o.detach().cpu().numpy(), out[k], out["m_" + k], TOL_FWD))
    ns = args["shape_params"].shape[1] if args["shape_params"] is not None else 10
    for k, a in args.items():
        if a is None:
            continue
        if k in ("shape_params", "expression_params"):
            lo, hi = (0, ns) if k == "shape_params" else (ns, betas.shape[1])
            g, m = out["g_betas"][:, lo:hi], out["m_betas"][:, lo:hi]
        else:
            lo, hi = [(p[1], p[2]) for p in POSES if p[0] == k][0]
            g, m = out["g_pose"][:, lo:hi], out["m_pose"][:, lo:hi]
        _note(f"{key}:g_{k}", _ratio(a.grad.cpu().numpy(), g, m, TOL_BWD))
    return v, lm, jo, out


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("kind", ["tiny", "real"])
def test_against_oracle(kind, B):
    dev = _cuda()
    arr = S.pixie_model(kind, 0)
    buf = S.pixie_buffers(arr)
    model, T = _oracle_model(buf)
    mod, seen = _module(buf, dev)
    betas, pose, rng = _inputs(B, 10 + B, arr["n_shape"], arr["n_exp"])
    V = arr["v_template"].shape[0]
    gv, gl, gj = (rng.standard_normal(s).astype(np.float32) for s in ((B, V, 3), (B, 68, 3), (B, 145, 3)))
    for up in ("verts", "all", "heads"):
        args = _args(betas, pose, dev, arr["n_shape"])
        _compare(f"{kind}{B}:{up}", mod, args, betas, pose, model, T, gv if up != "heads" else None,
                 gl if up != "verts" else None, gj if up != "verts" else None, dev)
    from icon_b200 import body_model as BM
    with torch.no_grad():
        sc = torch.tensor(betas, dtype=torch.float32, device=dev)
        rows = BM.pixie_smplx(mod, sc, torch.tensor(pose, dtype=torch.float32, device=dev))[3]
    assert np.array_equal(rows.cpu().numpy(), OP.lut_row(pose, T["chain"])[0])
    assert not seen


def test_against_reference_golden(golden_dir):
    dev = _cuda()
    d = np.load(os.path.join(golden_dir, "pixie_body_model.npz"))
    buf = {k: d["model_" + k] for k in MODEL + HEADS}
    model, T = _oracle_model(buf)
    mod, _ = _module(buf, dev)
    from icon_b200 import body_model as BM
    cases = sorted({k.split("_")[0] for k in d.files if k.startswith("c")})
    assert len(cases) == 4
    for c in cases:
        betas, pose = golden_full_inputs(d, c)
        none = tuple(x for x in str(d[f"{c}_none"]).split(",") if x) + ("eye_pose",)
        with torch.no_grad():
            rows = BM.pixie_smplx(mod, torch.tensor(betas, dtype=torch.float32, device=dev),
                                  torch.tensor(pose, dtype=torch.float32, device=dev))[3]
        assert np.array_equal(rows.cpu().numpy(), d[f"{c}_row"]), c
        for mode in ("v", "all"):
            args = _args(betas, pose, dev, 10, none)
            ups = (d[f"{c}_gv"], d[f"{c}_gl"] if mode == "all" else None, d[f"{c}_gj"] if mode == "all" else None)
            v, lm, jo, out = _compare(f"golden_{c}_{mode}", mod, args, betas, pose, model, T, *ups, dev)
            for k in ("verts", "landmarks", "joints"):
                got = {"verts": v, "landmarks": lm, "joints": jo}[k].detach().cpu().numpy()
                _note(f"golden:{k}", _ratio(got, d[f"{c}_{k}"], out["m_" + k], TOL_FWD))
            for k, (_, m) in golden_grad_parts(d, c, out, mode).items():
                _note(f"golden:g_{k}", _ratio(args[k].grad.cpu().numpy(), d[f"{c}_{mode}_g_{k}"], m, TOL_BWD))


def _real(dev):
    arr = S.pixie_model("real", 0)
    return arr, _module(S.pixie_buffers(arr), dev, arr["n_shape"])[0]


def test_bitwise_repeatable_and_batch_independent():
    dev = _cuda()
    arr, mod = _real(dev)
    betas, pose, rng = _inputs(3, 5, 200, 50)
    gv = torch.from_numpy(rng.standard_normal((3, 10475, 3)).astype(np.float32)).to(dev)
    gl = torch.from_numpy(rng.standard_normal((3, 68, 3)).astype(np.float32)).to(dev)
    gj = torch.from_numpy(rng.standard_normal((3, 145, 3)).astype(np.float32)).to(dev)

    def run(rows):
        args = _args(betas[rows], pose[rows], dev, 200)
        outs = mod(**args)
        torch.autograd.backward(list(outs), [gv[rows], gl[rows], gj[rows]])
        return [o.detach().cpu() for o in outs] + [a.grad.cpu() for a in args.values()]
    a, b = run(slice(0, 3)), run(slice(0, 3))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for r in range(3):
        one = run(slice(r, r + 1))
        assert all(torch.equal(x[r:r + 1], y) for x, y in zip(a, one)), r


def test_launches_and_no_host_sync_in_a_warm_iteration():
    dev = _cuda()
    from icon_b200 import _C
    arr, mod = _real(dev)
    betas, pose, rng = _inputs(1, 2, 200, 50)
    args = _args(betas, pose, dev, 200, none=("eye_pose",))
    gv = torch.randn(1, 10475, 3, device=dev)
    gl, gj = torch.randn(1, 68, 3, device=dev), torch.randn(1, 145, 3, device=dev)

    def iteration():
        outs = mod(**args)
        torch.autograd.backward(list(outs), [gv, gl, gj])
    iteration()                                               # fills the model caches (their one host copy each)
    torch.cuda.synchronize()
    n0 = _C.launch_count()
    outs = mod(**args)
    n1 = _C.launch_count()
    torch.autograd.backward(list(outs), [gv, gl, gj])
    n2 = _C.launch_count()
    assert (n1 - n0, n2 - n1) == (4, 3)
    assert [tuple(o.shape) for o in outs] == [(1, 10475, 3), (1, 68, 3), (1, 145, 3)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        iteration()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_cpu_and_float64_calls_reach_the_reference():
    dev = _cuda()
    buf = S.pixie_buffers(S.pixie_model("tiny", 0))
    mod, seen = _module(buf, dev)
    r = torch.eye(3, device=dev)[None, None]
    assert mod.double()(global_pose=r.double()) == "reference" and len(seen) == 1
    cpu, seen2 = _module(buf, torch.device("cpu"))
    assert cpu(global_pose=r.cpu()) == "reference" and len(seen2) == 1
    mod32, seen3 = _module(buf, dev)
    out = mod32(global_pose=r)                                 # fp32 CUDA: the kernels
    assert len(seen3) == 0 and [tuple(o.shape) for o in out] == [(1, 98, 3), (1, 68, 3), (1, 145, 3)]


# ---------------------------------------------------------------- the -hps_type pixie body-fit iteration

def _fit_colors(w, ft):
    """VF2Mesh's vertex colours through the project's own differentiable area-weighted normals (no float atomics, so
    the whole iteration is deterministic)."""
    from icon_b200 import mesh_views as MV
    return (MV.VertexNormals.apply(w, ft) + 1.0) * 0.5


def pixie_fit(dev, colors=_fit_colors, steps=30, step=1e-3, momentum=0.5):
    """The -hps_type pixie body-fit iteration of apps/infer.py:184-197, 200-270 on the real-size synthetic model:
    returns (losses per step, first-step {name: (kernel gradient, oracle gradient, m)}).

    The optimiser is SGD on the gradient scaled to unit norm at every step (a step of `step` in parameter norm).  On
    this body the L1 image loss is nearly flat at first and its gradient grows once the silhouettes move; with the
    first step's scale kept and momentum 0.9 the later steps overshoot and the loss rose again (measured on an H100:
    0.4864 -> 0.4835 with a minimum of 0.4799 at step 21).  With these settings it fell to 0.4800."""
    import test_gpu_fit_render as FR
    from oracle.body_model import rodrigues
    arr = S.pixie_model("real", 0)
    buf = S.pixie_buffers(arr)
    model, T = _oracle_model(buf)
    mod, seen = _module(buf, dev, arr["n_shape"])
    ft = torch.from_numpy(buf["faces_tensor"]).to(dev)
    rng = np.random.RandomState(21)
    aa = 0.2 * rng.standard_normal((55, 3))
    R0 = rodrigues(aa)[0]
    aa_t = aa.copy()
    aa_t[[1, 2, 16, 17]] += 0.25 * rng.standard_normal((4, 3))
    Rt = rodrigues(aa_t)[0]
    betas0 = 0.5 * rng.standard_normal((1, 200))
    flip = torch.tensor([1.0, -1.0, -1.0], device=dev)
    f32 = lambda x, g=False: torch.tensor(np.asarray(x, np.float32), device=dev, requires_grad=g)  # noqa: E731
    exp, jaw = f32(0.3 * rng.standard_normal((1, 50)), True), f32(R0[None, 22:23], True)
    lh, rh = f32(R0[None, 25:40], True), f32(R0[None, 40:55], True)        # tensor2variable's leaves
    with torch.no_grad():
        vt = mod(shape_params=f32(betas0 + 0.3), expression_params=exp, global_pose=f32(Rt[None, :1]),
                 body_pose=f32(Rt[None, 1:22]), jaw_pose=jaw, left_hand_pose=lh, right_hand_pose=rh)[0]
        w = (vt[0] + 0.02) * 0.9 * flip
        nF, nB = FR._render_obj(w, ft, colors(w, ft)).get_rgb_image()
    betas = f32(betas0, True)
    orient = f32(R0[None, :1], True)
    pose = f32(R0[None, 1:22], True)
    trans = torch.zeros(3, device=dev, requires_grad=True)
    scale = 0.9
    params = [pose, trans, betas, orient]
    opt = torch.optim.SGD(params, lr=step, momentum=momentum)
    losses, first = [], {}
    for it in range(steps):
        opt.zero_grad()
        v, _, _ = mod(shape_params=betas, expression_params=exp, body_pose=pose, global_pose=orient, jaw_pose=jaw,
                      left_hand_pose=lh, right_hand_pose=rh)
        if it == 0:
            v.retain_grad()
        w = (((v + trans) * scale) * flip)[0]
        r = FR._render_obj(w, ft, colors(w, ft))
        T_F, T_B = r.get_rgb_image()
        M_F, M_B = r.get_silhouette_image()
        loss = FR._body_fit_loss(T_F, T_B, M_F, M_B, nF, nB)
        loss.backward()
        if it == 0:
            gv = v.grad.double().cpu().numpy()
            full = np.concatenate([orient.detach().cpu().numpy(), pose.detach().cpu().numpy(),
                                   jaw.detach().cpu().numpy(), np.broadcast_to(np.eye(3), (1, 2, 3, 3)),
                                   lh.detach().cpu().numpy(), rh.detach().cpu().numpy()], 1).astype(np.float64)
            sc = np.concatenate([betas.detach().cpu().numpy(), exp.detach().cpu().numpy()], 1).astype(np.float64)
            out = OP.pixie_bounds(sc, full, model, T, g_verts=gv)
            g = lambda t: t.grad.cpu().numpy()  # noqa: E731
            first = {"g_betas": (g(betas), out["g_betas"][:, :200], out["m_betas"][:, :200]),
                     "g_orient": (g(orient), out["g_pose"][:, :1], out["m_pose"][:, :1]),
                     "g_pose": (g(pose), out["g_pose"][:, 1:22], out["m_pose"][:, 1:22]),
                     "g_trans": (g(trans), gv.sum((0, 1)), np.abs(gv).sum((0, 1))),
                     "g_jaw": (g(jaw), out["g_pose"][:, 22:23], out["m_pose"][:, 22:23])}
        gn = torch.cat([p.grad.reshape(-1) for p in params]).norm()
        for p in params:
            p.grad.div_(gn)
        opt.step()
        losses.append(float(loss.detach()))
    assert not seen
    return losses, first


def test_pixie_body_fit_iteration_end_to_end():
    dev = _cuda()
    losses, first = pixie_fit(dev)
    for k, (got, ref, m) in first.items():
        _note("fit:" + k, _ratio(got, ref, m, TOL_BWD))
    assert np.abs(first["g_pose"][1]).max() > 0
    # every step is deterministic (no float atomics in the body model, the normals or the renders), so this is the
    # same trajectory on every run; the bar is a third of the drop measured on an H100 (0.4864 -> 0.4800)
    assert losses[-1] < losses[0] - 2e-3, losses
