"""PyMAF's body estimate on the H100 against the float64 oracle (oracle/pymaf.py) computed live on the CPU from the
same seeded weights: every backbone and deconvolution layer, the max pool and the relu = 2 act, the MAF sampling and
MLP, the regressor and the SMPL tail, each given the oracle's input; end to end from three images; determinism and
graph replay; and the overlay-patched class (icon_b200/hps.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SEEDS = (0, 1, 2)
U19, U24 = 2.0 ** -19, 2.0 ** -24


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs cuda:0")
    from icon_b200 import hps, synthetic as S
    from oracle import pymaf as O
    T = S.pymaf_tables(0)
    sd = S.pymaf_state_dict(0, T)
    jm = [T["joint_map"]] * 3
    dev = torch.device("cuda:0")
    sdc = {k: v.to(dev) for k, v in sd.items()}
    drv = hps.PyMAFDriver(sdc, jm)
    refs = {}
    for seed in SEEDS:
        rec = {}
        x = S.pymaf_image(seed)
        refs[seed] = (x, O.forward(sd, jm, x, rec), rec)
    return dict(hps=hps, S=S, O=O, sd=sd, jm=jm, dev=dev, drv=drv, refs=refs, T=T)


def _nhwc(x, dev):
    return x.permute(0, 2, 3, 1).contiguous().float().to(dev)


def _conv_modules(drv):
    mods = [drv.stem]
    for b in drv.blocks:
        mods += [b["conv1"], b["conv2"], b["conv3"]] + ([b["down"]] if b["down"] is not None else [])
    return mods + list(drv.deconvs)


def test_every_layer_within_the_conv_bar(env):
    from icon_b200 import nhwc
    drv, dev = env["drv"], env["dev"]
    _, _, rec = env["refs"][0]
    mods = _conv_modules(drv)
    assert len(mods) == len(rec["layers"]) == 53 + 3
    worst = 0.0
    for m, (name, x, wf, bf, s, pad, tr) in zip(mods, rec["layers"]):
        x32 = x.float()
        if name == "conv1":
            y = nhwc.stem_conv7(x32.to(dev), m, reflect=False, stats=False).t
        else:
            op, _ = nhwc.act(nhwc.Raw(_nhwc(x32, dev)), s2d=(s == 2 and not tr))
            y = (nhwc.conv_transpose(op, m, stats=False) if tr else nhwc.conv(op, m, stats=False)).t
        # the device weights are the folds rounded to fp32: the bar is on them, as the conv tests state it
        w32, b32 = m.weight.detach().double().cpu(), m.bias.detach().double().cpu()
        assert torch.allclose(w32, wf, rtol=2 ** -23, atol=0), name
        f = F.conv_transpose2d if tr else F.conv2d
        ref = f(x32.double(), w32, b32, s, pad)
        bound = f(x32.double().abs(), w32.abs(), b32.abs(), s, pad)
        got = y.permute(0, 3, 1, 2).double().cpu()
        err = (got - ref).abs()
        bar = U19 * bound + U24 * ref.abs()
        assert bool((err <= bar).all()), f"{name}: max err/bar {(err / bar).max().item():.3f}"
        worst = max(worst, (err / bar).max().item())
    print(f"worst layer err/bar {worst:.3f}")


def test_maxpool_exact(env):
    drv, dev = env["drv"], env["dev"]
    _, _, rec = env["refs"][0]
    pre = rec["layers"][0]
    y = F.conv2d(pre[1].float().double(), pre[2], pre[3], 2, 3).float()     # conv1 + bn1, relu left to the pool
    from icon_b200 import nhwc
    from icon_b200.ops import _p, _stream
    from icon_b200._C import check, lib
    t = _nhwc(y, dev)
    hi = torch.empty(1, 56, 56, 64, dtype=torch.float16, device=dev)
    lo = torch.empty_like(hi)
    check(lib.icon_maxpool3s2_nhwc(_p(t), _p(hi), _p(lo), 1, 112, 112, 64, 64, 1, _stream()), "maxpool")
    ref = F.max_pool2d(torch.relu(y), 3, 2, 1).permute(0, 2, 3, 1).to(dev)
    rh = ref.half()
    assert torch.equal(hi, rh) and torch.equal(lo, (ref - rh.float()).half())
    # without relu: -inf padding, negative values survive
    neg = -torch.rand(1, 5, 7, 64, device=dev) - 1
    hi2 = torch.empty(1, 3, 4, 64, dtype=torch.float16, device=dev)
    lo2 = torch.empty_like(hi2)
    check(lib.icon_maxpool3s2_nhwc(_p(neg), _p(hi2), _p(lo2), 1, 5, 7, 64, 64, 0, _stream()), "maxpool")
    r2 = F.max_pool2d(neg.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(hi2, r2.half()) and bool((r2 < 0).all())
    del nhwc


def test_relu_after_residual(env):
    from icon_b200 import nhwc
    dev = env["dev"]
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(1, 14, 14, 1024, generator=g).to(dev)
    res = torch.randn(1, 14, 14, 1024, generator=g).to(dev)
    op, f32 = nhwc.act(nhwc.Raw(x), relu=2, res=res, f32=True)
    ref = torch.relu(x + res)
    assert torch.equal(f32, ref)
    assert torch.equal(op.hi, ref.half()) and torch.equal(op.lo, (ref - ref.half().float()).half())
    _, f1 = nhwc.act(nhwc.Raw(x), relu=True, res=res, f32=True, operand=False)
    assert torch.equal(f1, torch.relu(x) + res)                             # mode 1 unchanged: ReLU, then the add


def _abs_maf(sd, i, feat, pts):
    m = f"maf_extractor.{i}."
    f = F.grid_sample(feat.abs(), pts.unsqueeze(2), align_corners=True)[..., 0]
    y = f
    for k in range(3):
        w, b = sd[m + f"conv{k}.weight"].double().abs(), sd[m + f"conv{k}.bias"].double().abs()
        y = F.conv1d(y if k == 0 else torch.cat([y, f], 1), w, b)
    return y.reshape(1, -1)


def test_maf_and_regressor_given_oracle_inputs(env):
    O, sd, drv, dev = env["O"], env["sd"], env["drv"], env["dev"]
    _, _, rec = env["refs"][0]
    prev = torch.cat([sd["regressor.0." + k].reshape(1, -1).double() for k in ("init_pose", "init_shape", "init_cam")], 1)
    for i in range(3):
        feat = rec["s_feat"][i].float()
        pts = rec["pts"][i].float()
        prev32 = prev.float()
        xc = drv.maf_row(i, _nhwc(feat, dev), pts[0].t().contiguous().to(dev), prev32[0].to(dev)).cpu().double()
        ref = torch.cat([O.maf(sd, i, feat.double(), pts.double()), prev32.double()], 1)[0]
        bar = U19 * torch.cat([_abs_maf(sd, i, feat.double(), pts.double()), prev32.double().abs()], 1)[0] + U24 * ref.abs()
        err = (xc - ref).abs()
        assert bool((err <= bar).all()), f"maf {i}: max err/bar {(err / bar).max().item():.3f}"
        xc32 = rec["xc"][i].float()
        par = drv.regress(i, xc32[0].to(dev), prev32[0].to(dev)).cpu().double()
        r = f"regressor.{i}."
        refp = O.regress(sd, i, xc32.double(), prev32.double())[0]
        h = F.linear(F.linear(xc32.double().abs(), sd[r + "fc1.weight"].double().abs(), sd[r + "fc1.bias"].double().abs()),
                     sd[r + "fc2.weight"].double().abs(), sd[r + "fc2.bias"].double().abs())
        heads = [F.linear(h, sd[r + n + ".weight"].double().abs(), sd[r + n + ".bias"].double().abs())
                 for n in ("decpose", "decshape", "deccam")]
        barp = U19 * (torch.cat(heads, 1)[0] + prev32[0].double().abs()) + U24 * refp.abs()
        errp = (par - refp).abs()
        assert bool((errp <= barp).all()), f"regressor {i}: max err/bar {(errp / barp).max().item():.3f}"
        prev = rec["par"][i]


def test_tail_given_oracle_inputs(env):
    O, sd, drv, dev, jm = env["O"], env["sd"], env["drv"], env["dev"], env["jm"]
    _, _, rec = env["refs"][0]
    for i in range(3):
        par32 = rec["par"][i].float()
        dmap = drv.dmap[i + 1] if i + 1 < 3 else None
        outs, pts = drv.tail(i, par32[0].contiguous().to(dev), dmap)
        ref = O.smpl_out(sd, i, jm[i], par32.double())
        for k, v in zip(env["hps"].OUT_KEYS, outs):
            r = ref[k]
            err = (v.cpu().double() - r).abs()
            tol = 2.0 ** -18 * torch.clamp(r.abs(), min=1.0)
            assert bool((err <= tol).all()), f"tail {i} {k}: max err {err.max().item():.3e}"
        if dmap is not None:
            ds = torch.einsum("mv,bvc->bmc", sd[f"maf_extractor.{i + 1}.Dmap"].double(), ref["verts"])
            rp = O.projection(ds.float().double(), ref["pred_cam"])[0].t()
            assert (pts.cpu().double() - rp).abs().max().item() <= 2.0 ** -18 * max(1.0, rp.abs().max().item())


def test_end_to_end(env):
    hps, drv, dev = env["hps"], env["drv"], env["dev"]
    report = []
    for seed in SEEDS:
        x, ref, rec = env["refs"][seed]
        out = drv(x.to(dev))
        assert len(out["smpl_out"]) == 4 and out["dp_out"] == []
        for d, rd in zip(out["smpl_out"], ref["smpl_out"]):
            for k in hps.OUT_KEYS:
                assert tuple(d[k].shape) == tuple(rd[k].shape), k
        last, rl = out["smpl_out"][-1], ref["smpl_out"][-1]
        for k in ("pred_pose", "pred_shape", "pred_cam", "rotmat", "verts", "kp_2d", "theta"):
            err = ((last[k].cpu().double() - rl[k]).abs() / torch.clamp(rl[k].abs(), min=1.0)).max().item()
            report.append((seed, k, err))
            assert err <= 1e-4, f"seed {seed} {k}: {err:.3e}"
        _, feats = drv.run(x.to(dev))
        for i in range(3):
            sf = rec["s_feat"][i]
            e = ((feats[i].permute(0, 3, 1, 2).cpu().double() - sf).abs().max() / sf.abs().max()).item()
            report.append((seed, f"s_feat{i}", e))
    print("end-to-end max err / max(1, |ref|): " + ", ".join(f"{s}:{k}={e:.2e}" for s, k, e in report))


def test_deterministic_and_graph_replay(env):
    hps, S, sd, jm, dev = env["hps"], env["S"], env["sd"], env["jm"], env["dev"]
    drv = hps.PyMAFDriver({k: v.to(dev) for k, v in sd.items()}, jm)
    x = S.pymaf_image(1).to(dev)
    eager = drv._forward_eager(x)
    eager2 = drv._forward_eager(x)
    assert all(torch.equal(a, b) for a, b in zip(eager, eager2))
    flat1, _ = drv.run(x)            # first sight: eager
    flat2, _ = drv.run(x)            # captured, then replayed
    flat3, _ = drv.run(x)
    assert drv._graphed.replays >= 2
    for a, b, c, e in zip(flat1, flat2, flat3, eager):
        assert torch.equal(a, e) and torch.equal(b, e) and torch.equal(c, e)


def test_overlay_patched_class(env):
    hps, S, sd, T, dev, drv = env["hps"], env["S"], env["sd"], env["T"], env["dev"], env["drv"]
    cls = hps.make_PyMAF(S.pymaf_standin(sd, T["joint_map"], S.pymaf_cfg()))
    m = cls().eval().to(dev)
    x = S.pymaf_image(2).to(dev)
    with torch.no_grad():
        out = m(x)
    assert cls.calls == []
    ref = drv(x)
    for d, rd in zip(out["smpl_out"], ref["smpl_out"]):
        for k in hps.OUT_KEYS:
            assert torch.equal(d[k], rd[k]), k
    assert m(x.double()) == "reference" and len(cls.calls) == 1


def test_angle_axis_branches_on_the_device(env):
    """Every branch of kornia's rotation_matrix_to_quaternion and the NaN -> 0 mask, through icon_hps_tail."""
    O, dev = env["O"], env["dev"]
    from icon_b200._C import check, lib
    from icon_b200.ops import _p, _stream
    R, _ = O.rotations(0)
    R = np.concatenate([R, np.full((1, 3, 3), np.nan)], 0)
    R32 = torch.from_numpy(R).float()
    J = R32.shape[0]
    m = R32.double().transpose(1, 2)
    d2, d0d1, d0nd1 = m[:, 2, 2] < 1e-6, m[:, 0, 0] > m[:, 1, 1], m[:, 0, 0] < -m[:, 1, 1]
    counts = [int((d2 & d0d1).sum()), int((d2 & ~d0d1).sum()), int((~d2 & d0nd1).sum()), int((~d2 & ~d0nd1).sum())]
    assert all(c > 0 for c in counts), counts
    par = torch.zeros(6 * J + 13, device=dev)
    par[6 * J + 10] = 0.9
    zeros3 = torch.zeros(J, 3, device=dev)
    jmap = torch.zeros(1, dtype=torch.int32, device=dev)
    kp3d, kp2d = torch.empty(1, 3, device=dev), torch.empty(1, 2, device=dev)
    theta = torch.empty(3 + 10 + 3 * J, device=dev)
    rot = R32.to(dev).contiguous()
    check(lib.icon_hps_tail(_p(zeros3), _p(zeros3), J, None, 0, None, 0, _p(jmap), 1, _p(rot), _p(par), 6 * J, 10,
                            _p(kp3d), _p(kp2d), _p(theta), _stream()), "icon_hps_tail")
    got = theta[13:].view(J, 3).cpu().double()
    ref = O.rotmat_to_aa(R32.double())
    assert not torch.isnan(got).any() and torch.equal(got[-1], torch.zeros(3, dtype=torch.float64))
    err = (got - ref).abs() / torch.clamp(ref.abs(), min=1.0)
    assert err.max().item() <= 2.0 ** -22, f"max {err.max().item():.3e}"


def test_each_fallback_condition_reaches_the_reference(env):
    """CUDA input; one condition of on_kernels broken at a time."""
    hps, S, sd, T, dev = env["hps"], env["S"], env["sd"], env["T"], env["dev"]
    cls = hps.make_PyMAF(S.pymaf_standin(sd, T["joint_map"], S.pymaf_cfg()))
    import sys
    mod = sys.modules[cls.__module__]
    m = cls().eval().to(dev)
    x = S.pymaf_image(0).to(dev)

    def routed(fn):
        cls.calls.clear()
        r = fn()
        return r == "reference" and len(cls.calls) == 1

    with torch.no_grad():
        assert not routed(lambda: m(x))                                  # the ported case runs the driver
        assert routed(lambda: m.train()(x))
        m.eval()
        assert routed(lambda: m(x, J_regressor=torch.zeros(17, 6890, device=dev)))
        assert routed(lambda: m(x.double()))
        assert routed(lambda: m(torch.cat([x, x])))
        assert routed(lambda: m(F.interpolate(x, size=(256, 256))))
        assert routed(lambda: m(x.cpu()))
        for path, value in (("N_ITER", 2), ("BACKBONE", "res18")):
            old = getattr(mod.cfg.MODEL.PyMAF, path)
            setattr(mod.cfg.MODEL.PyMAF, path, value)
            try:
                assert routed(lambda: m(x)), path
            finally:
                setattr(mod.cfg.MODEL.PyMAF, path, old)
        old = mod.cfg.RES_MODEL.NUM_DECONV_KERNELS
        mod.cfg.RES_MODEL.NUM_DECONV_KERNELS = [4, 4, 3]
        try:
            assert routed(lambda: m(x))
        finally:
            mod.cfg.RES_MODEL.NUM_DECONV_KERNELS = old
        m64 = cls().eval().to(dev)
        m64.regressor[0].init_cam = m64.regressor[0].init_cam.double()   # a floating tensor not fp32
        assert routed(lambda: m64(x))
        mcpu = cls().eval().to(dev)
        mcpu.points_grid = mcpu.points_grid.cpu()                         # a tensor on another device
        assert routed(lambda: mcpu(x))
    with torch.enable_grad():
        assert any(p.requires_grad for p in m.parameters())
        assert routed(lambda: m(x))                                       # grad mode and grad-requiring parameters
        m.requires_grad_(False)
        assert not routed(lambda: m(x))                                   # grad mode alone is not a reason
