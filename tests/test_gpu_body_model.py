"""The body model's kernels (icon_b200/body_model.py, csrc/body_model.cu) against oracle/body_model.py and against the
reference's own lib/smplx outputs (tests/golden/body_model.npz).

Bars, in units of m = sum of |contribution| per component (the oracle's absolute-value companion): verts and joints
within 2^-18 m, g_betas and g_pose within 2^-17 m.  Every long sum is fp64 in the kernels and every output is rounded
to fp32 once, so the error is the final rounding (2^-24 relative) plus fp64 rounding along the chain (depth <= 10);
the bars leave a wide margin.  Also: two runs bitwise equal; row b of a B = 3 call equal to a one-row call; no host
sync in a warm iteration; the body-fit iteration of apps/infer.py:175-231 end to end (first-step gradients against
the oracle's backward of the renderer's grad_verts, then 30 SGD steps lower the loss); the overlay's dispatcher.
"""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402
from oracle import body_model as OB  # noqa: E402

TOL_FWD = 2.0 ** -18
TOL_BWD = 2.0 ** -17
NAMES = ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights")
WORST = {}


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _note(key, ratio):
    """Keep the worst error / m per key; printed (pytest -s) as one JSON line."""
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))
    print("body_model worst error / m:", json.dumps(WORST, sort_keys=True))


def _ratio(got, ref, m, tol):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    r = err / np.maximum(m, 1e-300)
    i = np.unravel_index(np.argmax(r), r.shape)
    assert np.all(err <= tol * m), (float(r[i]), i, float(got[i]), float(ref[i]), float(m[i]))
    return float(r.max())


def _model(kind, V=None):
    m = S.body_model(kind, 0, V=V) if kind != "tiny" else S.body_model("tiny", 0, V=V)
    return m, [m[k].astype(np.float64) if k != "parents" else m[k] for k in NAMES]


def _inputs(m, pose2rot, B, seed):
    J, NB = len(m["parents"]), m["shapedirs"].shape[2]
    rng = np.random.RandomState(seed)
    betas = rng.standard_normal((B, NB)).astype(np.float32)
    aa = (0.5 * rng.standard_normal((B, J, 3))).astype(np.float32)
    aa[:, 1] = 0.0
    if pose2rot:
        pose = aa.reshape(B, J * 3)
    else:
        pose = (OB.rodrigues(aa.astype(np.float64))[0] + 0.05 * rng.standard_normal((B, J, 3, 3))).astype(np.float32)
    return betas, pose, rng


def _run(model_t, betas_t, pose_t, pose2rot, gv=None, gj=None):
    from icon_b200 import body_model as BM
    v, j = BM.lbs(betas_t, pose_t, *model_t, pose2rot=pose2rot)
    if gv is not None or gj is not None:
        outs, gs = zip(*[(o, g) for o, g in ((v, gv), (j, gj)) if g is not None])
        torch.autograd.backward(list(outs), list(gs))
    return v, j


def _check(key, m, model64, betas, pose, pose2rot, expand, dev, rng, golden=None):
    B = pose.shape[0]
    V, J = m["v_template"].shape[0], len(m["parents"])
    model_t = [torch.from_numpy(m[k]).to(dev) for k in NAMES]
    b1 = torch.from_numpy(betas[:1] if expand else betas).to(dev).requires_grad_(True)
    pt = torch.from_numpy(pose).to(dev)
    betas_full = np.broadcast_to(betas[:1], betas.shape) if expand else betas
    gvn = rng.standard_normal((B, V, 3)).astype(np.float32)
    gjn = rng.standard_normal((B, J, 3)).astype(np.float32)
    for up in ("verts", "joints", "both"):
        gv = gvn if up != "joints" else None
        gj = gjn if up != "verts" else None
        bt = b1.expand(B, -1) if expand else b1
        pr = pt.clone().requires_grad_(True)
        b1.grad = None
        v, j = _run(model_t, bt, pr, pose2rot, None if gv is None else torch.from_numpy(gv).to(dev),
                    None if gj is None else torch.from_numpy(gj).to(dev))
        out = OB.lbs_bounds(betas_full, pose, *model64, pose2rot, g_verts=gv, g_joints=gj)
        _note(f"{key}:verts", _ratio(v.detach().cpu().numpy(), out["verts"], out["m_verts"], TOL_FWD))
        _note(f"{key}:joints", _ratio(j.detach().cpu().numpy(), out["joints"], out["m_joints"], TOL_FWD))
        gb, mb = out["g_betas"], out["m_betas"]
        if expand:
            gb, mb = gb.sum(0, keepdims=True), mb.sum(0, keepdims=True)
        _note(f"{key}:g_betas", _ratio(b1.grad.cpu().numpy(), gb, mb, TOL_BWD))
        _note(f"{key}:g_pose", _ratio(pr.grad.cpu().numpy(), out["g_pose"].reshape(pose.shape),
                                      out["m_pose"].reshape(pose.shape), TOL_BWD))
        if V > 1 or up != "joints":          # one vertex: both joints regress to it, so rel_1 = 0
            assert np.abs(pr.grad.cpu().numpy()).max() > 0
    if golden is not None:
        gvg, gjg = golden["gv"].astype(np.float32), golden["gj"].astype(np.float32)
        b1.grad = None
        pr = pt.clone().requires_grad_(True)
        v, j = _run(model_t, b1.expand(B, -1) if expand else b1, pr, pose2rot, torch.from_numpy(gvg).to(dev),
                    torch.from_numpy(gjg).to(dev))
        out = OB.lbs_bounds(betas_full, pose, *model64, pose2rot, g_verts=gvg, g_joints=gjg)
        mb = out["m_betas"].sum(0, keepdims=True) if expand else out["m_betas"]
        _note("golden:verts", _ratio(v.detach().cpu().numpy(), golden["verts"], out["m_verts"], TOL_FWD))
        _note("golden:joints", _ratio(j.detach().cpu().numpy(), golden["joints"], out["m_joints"], TOL_FWD))
        _note("golden:g_betas", _ratio(b1.grad.cpu().numpy(), golden["g_betas"], mb, TOL_BWD))
        _note("golden:g_pose", _ratio(pr.grad.cpu().numpy(), golden["g_pose"].reshape(pose.shape),
                                      out["m_pose"].reshape(pose.shape), TOL_BWD))


@pytest.mark.parametrize("batch", ["1", "3", "3e"])
@pytest.mark.parametrize("pose2rot", [True, False])
@pytest.mark.parametrize("kind", ["smpl", "smplx", "tiny1", "tiny31", "tiny257"])
def test_against_oracle(kind, pose2rot, batch):
    dev = _cuda()
    m, model64 = _model("tiny", int(kind[4:])) if kind.startswith("tiny") else _model(kind)
    B = int(batch[0])
    betas, pose, rng = _inputs(m, pose2rot, B, 3 + B)
    _check(f"{kind}", m, model64, betas, pose, pose2rot, batch == "3e", dev, rng)


def test_against_reference_golden(golden_dir):
    dev = _cuda()
    import os
    d = np.load(os.path.join(golden_dir, "body_model.npz"))
    cases = sorted({k.split("_")[0] for k in d.files if k.startswith("c")})
    assert len(cases) == 7
    for c in cases:
        mn = str(d[f"{c}_model"])
        m = {k: d[f"{mn}_{k}"] for k in NAMES}
        model64 = [m[k].astype(np.float64) if k != "parents" else m[k] for k in NAMES]
        pose2rot, expand = bool(d[f"{c}_pose2rot"]), bool(d[f"{c}_expand"])
        pose = d[f"{c}_pose"].astype(np.float32)
        B = pose.shape[0]
        betas = np.broadcast_to(d[f"{c}_betas"], (B, d[f"{c}_betas"].shape[1])).astype(np.float32)
        golden = {k: d[f"{c}_{k}"] for k in ("verts", "joints", "gv", "gj", "g_betas", "g_pose")}
        _check(f"golden_{c}", m, model64, betas, pose, pose2rot, expand, dev, np.random.RandomState(1), golden)


@pytest.mark.parametrize("pose2rot", [True, False])
def test_bitwise_repeatable_and_batch_independent(pose2rot):
    dev = _cuda()
    m, _ = _model("smpl")
    model_t = [torch.from_numpy(m[k]).to(dev) for k in NAMES]
    betas, pose, rng = _inputs(m, pose2rot, 3, 9)
    gv = torch.from_numpy(rng.standard_normal((3, 6890, 3)).astype(np.float32)).to(dev)
    gj = torch.from_numpy(rng.standard_normal((3, 24, 3)).astype(np.float32)).to(dev)

    def run(rows):
        bt = torch.from_numpy(betas[rows]).to(dev).requires_grad_(True)
        pt = torch.from_numpy(pose[rows]).to(dev).requires_grad_(True)
        v, j = _run(model_t, bt, pt, pose2rot, gv[rows], gj[rows])
        return [x.detach().cpu() for x in (v, j, bt.grad, pt.grad)]
    a, b = run(slice(0, 3)), run(slice(0, 3))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for r in range(3):
        one = run(slice(r, r + 1))
        assert all(torch.equal(x[r:r + 1], y) for x, y in zip(a, one)), r


def test_no_host_sync_in_a_warm_iteration():
    dev = _cuda()
    m, _ = _model("smpl")
    model_t = [torch.from_numpy(m[k]).to(dev) for k in NAMES]
    betas, pose, rng = _inputs(m, False, 1, 2)
    bt = torch.from_numpy(betas).to(dev).requires_grad_(True)
    pt = torch.from_numpy(pose).to(dev).requires_grad_(True)
    gv = torch.randn(1, 6890, 3, device=dev)
    _run(model_t, bt, pt, False, gv)                          # fills the model cache (its one host copy)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _run(model_t, bt, pt, False, gv)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_model_cache_holds_several_models():
    dev = _cuda()
    from icon_b200 import body_model as BM
    ms = [[torch.from_numpy(S.body_model("tiny", s, V=40)[k]).to(dev) for k in NAMES] for s in range(3)]
    ps = [BM.prepared(*m) for m in ms]
    assert all(BM.prepared(*m) is p for m, p in zip(ms, ps))
    ms[0][0].add_(0.0)                                          # a new version: refilled
    assert BM.prepared(*ms[0]) is not ps[0]


def test_dispatcher_routes_cuda_fp32_to_the_kernels():
    dev = _cuda()
    from icon_b200 import _C, body_model as BM
    calls = []
    lbs = BM.make_lbs(lambda *a, **k: calls.append(1) or "reference")
    m, _ = _model("tiny", 31)
    model_t = [torch.from_numpy(m[k]).to(dev) for k in NAMES]
    betas = torch.zeros(2, 3, device=dev)
    pose = torch.zeros(2, 6, device=dev)
    BM.prepared(*model_t)
    torch.cuda.synchronize()
    n0 = _C.launch_count()
    v, j = lbs(betas, pose, *model_t)
    assert _C.launch_count() - n0 == 2 and not calls
    assert torch.allclose(v, model_t[0].expand(2, -1, -1), atol=1e-6)
    assert lbs(betas, pose, *model_t, return_transformation=True) == "reference"
    assert lbs(betas.double(), pose.double(), *[t.double() if t.is_floating_point() else t for t in model_t]) == \
        "reference"
    model_b = list(model_t)
    model_b[0] = model_t[0][None].expand(2, -1, -1)              # a batched v_template
    assert lbs(betas, pose, *model_b) == "reference" and len(calls) == 3


# ---------------------------------------------------------------- the body-fit iteration, end to end

def _fit_setup(dev):
    import test_gpu_fit_render as FR
    m = S.body_model("smpl", 0)
    model_t = [torch.from_numpy(m[k]).to(dev) for k in NAMES]
    ft = torch.from_numpy(m["faces"]).to(dev)
    rng = np.random.RandomState(21)
    aa = 0.2 * rng.standard_normal((24, 3))
    R0 = OB.rodrigues(aa)[0]
    betas0 = 0.5 * rng.standard_normal((1, 10))
    aa_t = aa.copy()
    aa_t[[1, 2, 16, 17]] += 0.25 * rng.standard_normal((4, 3))         # the targets' perturbed pose
    Rt = OB.rodrigues(aa_t)[0]
    flip = torch.tensor([1.0, -1.0, -1.0], device=dev)
    from icon_b200 import body_model as BM
    with torch.no_grad():
        vt, _ = BM.lbs(torch.tensor(betas0 + 0.3, dtype=torch.float32, device=dev),
                       torch.tensor(Rt[None], dtype=torch.float32, device=dev), *model_t, pose2rot=False)
        w = (vt[0] + 0.02) * 0.9 * flip
        nF, nB = FR._render_obj(w, ft, FR._area_colors(w, ft)).get_rgb_image()
    return FR, m, model_t, ft, R0, betas0, flip, nF, nB


def test_body_fit_iteration_end_to_end():
    dev = _cuda()
    from icon_b200 import body_model as BM
    FR, m, model_t, ft, R0, betas0, flip, nF, nB = _fit_setup(dev)
    betas = torch.tensor(betas0, dtype=torch.float32, device=dev, requires_grad=True)
    orient = torch.tensor(R0[None, :1], dtype=torch.float32, device=dev, requires_grad=True)
    pose = torch.tensor(R0[None, 1:], dtype=torch.float32, device=dev, requires_grad=True)
    trans = torch.zeros(3, device=dev, requires_grad=True)
    scale = 0.9
    params = [pose, trans, betas, orient]
    opt = torch.optim.SGD(params, lr=1e-3, momentum=0.9)
    losses = []
    for it in range(30):
        opt.zero_grad()
        full = torch.cat([orient, pose], 1)
        v, _ = BM.lbs(betas, full, *model_t, pose2rot=False)
        if it == 0:
            v.retain_grad()
        smpl_verts = (v + trans) * scale
        w = (smpl_verts * flip)[0]
        r = FR._render_obj(w, ft, FR._area_colors(w, ft))
        T_F, T_B = r.get_rgb_image()
        M_F, M_B = r.get_silhouette_image()
        loss = FR._body_fit_loss(T_F, T_B, M_F, M_B, nF, nB)
        loss.backward()
        if it == 0:
            gv = v.grad.double().cpu().numpy()
            model64 = [m[k].astype(np.float64) if k != "parents" else m[k] for k in NAMES]
            full_np = full.detach().double().cpu().numpy()
            out = OB.lbs_bounds(betas.detach().double().cpu().numpy(), full_np, *model64, False, g_verts=gv)
            _note("fit:g_betas", _ratio(betas.grad.cpu().numpy(), out["g_betas"], out["m_betas"], TOL_BWD))
            gp, mp = out["g_pose"].reshape(1, 24, 3, 3), out["m_pose"].reshape(1, 24, 3, 3)
            _note("fit:g_orient", _ratio(orient.grad.cpu().numpy(), gp[:, :1], mp[:, :1], TOL_BWD))
            _note("fit:g_pose", _ratio(pose.grad.cpu().numpy(), gp[:, 1:], mp[:, 1:], TOL_BWD))
            _note("fit:g_trans", _ratio(trans.grad.cpu().numpy(), gv.sum((0, 1)), np.abs(gv).sum((0, 1)), TOL_BWD))
            assert np.abs(out["g_pose"]).max() > 0
            # apps/infer.py's SGD (lr 1e-3, momentum 0.9) on the gradient scaled to norm 1: the first step moves the
            # parameters by 1e-3, under a pixel at 512^2, where the L1 image losses are locally linear; on this
            # synthetic body the unscaled step overshoots (the loss rose on the first step)
            g0 = float(torch.cat([p.grad.reshape(-1) for p in params]).norm())
            for group in opt.param_groups:
                group["lr"] = 1e-3 / g0
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0], losses
