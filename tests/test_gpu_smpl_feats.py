"""The icon prior with every `smpl_feats` subset (icon_query_feats) in both fused gather + MLP kernels, against the fp64
CPU oracle; the full set through the new entry point against icon_query; point-locality of the subsets without cmap;
and the ICON-MVP prior (smpl_feats = ['sdf']) end to end through the engine and marching cubes (run on an H100).

Bar: |out - ref| <= 1e-4 * max(1, |ref|).
"""
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402

EYE = torch.eye(4)[None]
FULL = ("sdf", "cmap", "norm", "vis")
SUBSETS = [("sdf",), ("sdf", "cmap"), ("sdf", "norm"), ("sdf", "vis"), ("sdf", "cmap", "norm"), ("sdf", "cmap", "vis"),
           ("sdf", "norm", "vis")]                     # every subset but the full set, which test_gpu_mlp.py covers


@pytest.fixture(params=["tcgen05", "fp32"], autouse=True)
def mlp_impl(request):
    """Every test runs against both fused gather+MLP kernels (mlp_tc.cu and mlp.cu)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from icon_b200 import ops
    ops.set_mlp_impl(request.param)
    yield request.param
    ops.set_mlp_impl("tcgen05")


def _dev():
    return torch.device("cuda:0")


def _tail(feats):
    return 1 + 3 * ("cmap" in feats) + 3 * ("norm" in feats)


def _c0(feats, C):
    return (C // 2 if "vis" in feats else C) + _tail(feats)


def _assert_close(out, ref):
    out, ref = out.reshape(-1).double(), ref.reshape(-1).double()
    assert out.shape == ref.shape
    assert not torch.isnan(out).any(), f"{torch.isnan(out).sum().item()} NaN outputs"
    tol = 1e-4 * ref.abs().clamp(min=1.0)
    err = (out - ref).abs()
    bad = ~(err <= tol)
    i = int((err / tol).argmax())
    assert not bad.any(), f"{bad.sum().item()} of {out.numel()} points off; worst at {i}: out {out[i]:.6g} ref {ref[i]:.6g}"


@functools.lru_cache(maxsize=None)
def _body():
    v, f = S.body_mesh()
    cm, vi = S.body_attributes(v)
    return (torch.from_numpy(v)[None], torch.from_numpy(f)[None], torch.from_numpy(cm)[None],
            torch.from_numpy(vi)[None])


def _smpl():
    verts, faces, cmap, vis = _body()
    return {"smpl_verts": verts, "smpl_faces": faces, "smpl_cmap": cmap, "smpl_vis": vis}


@functools.lru_cache(maxsize=None)
def _gpu_body():
    from icon_b200 import ops
    return ops.SmplBody(*(t.to(_dev()) for t in _body()))


def _points(n, seed):
    """About a quarter outside the cube; half of the points within ~0.03 of the body, so that non-outliers exist."""
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(1, n, 3, generator=g) * 2 - 1) * 1.1
    verts = _body()[0]
    sel = torch.randint(0, verts.shape[1], (n // 2,), generator=g)
    pts[0, : n // 2] = verts[0][sel] + 0.03 * torch.randn(n // 2, 3, generator=g)
    return pts.permute(0, 2, 1).contiguous()


# ---------------------------------------------------------------------------------------------------- 1. layouts
def _layout_params():
    """Per subset: the smallest C, C = 6 and 12 where c0 <= 15 allows them, the largest C it allows, an odd C without
    vis (feat_select needs an even C with it), and a 2 x 3 map."""
    out = []
    for feats in SUBSETS:
        room = 15 - _tail(feats)                       # image columns that fit under c0 <= 15
        if "vis" in feats:
            Cs = {2, 2 * room} | {c for c in (6, 12) if c // 2 <= room}
        else:
            Cs = {1, room, 7 if room >= 7 else 5} | {c for c in (6, 12) if c <= room}
        name = "-".join(feats)
        for C in sorted(Cs):
            assert _c0(feats, C) <= 15
            out.append(pytest.param(feats, C, 96, 160, id=f"{name}-C{C}-96x160"))
        out.append(pytest.param(feats, 6, 2, 3, id=f"{name}-C6-2x3"))
    return out


@functools.lru_cache(maxsize=None)
def _layout_case(feats, C, H, W, n=10000):
    """Inputs and the fp64 oracle's occupancies for one layout (the same for both kernels)."""
    from oracle import query as OQ
    seed = 1000 + 100 * C + H + 7 * _tail(feats) + 50 * ("vis" in feats)
    g = torch.Generator().manual_seed(seed)
    c0 = _c0(feats, C)
    sd = S.mlp_state_dict(c0=c0, seed=seed)
    feat = torch.randn(1, C, H, W, generator=g)
    samples = _points(n, seed)
    ref = OQ.query(sd, [feat], samples, EYE, prior="icon", smpl=_smpl(), sdf_clip=0.05, smpl_feats=feats,
                   mlp_dtype=torch.float64)[0]
    return sd, c0, feat, samples, ref


@pytest.mark.parametrize("feats,C,H,W", _layout_params())
def test_query_smpl_feats_layout_vs_oracle(feats, C, H, W):
    from icon_b200 import ops
    dev = _dev()
    sd, c0, feat, samples, ref = _layout_case(feats, C, H, W)
    packed = ops.pack_mlp(sd, c0, device=dev)
    out = ops.query("icon", samples.to(dev), EYE, feat.to(dev), packed, body=_gpu_body(), sdf_clip=0.05,
                    smpl_feats=feats).cpu()
    _assert_close(out, ref)
    assert (ref.abs() > 1e-3).float().mean() > 0.5            # the comparison is not vacuous


# ---------------------------------------------------------------------------------------------------- 2. full set
def test_full_set_mask_equals_icon_query():
    """The full set through icon_query_feats is icon_query, bit for bit, on the same call."""
    from icon_b200 import _C, ops
    dev = _dev()
    C, c0, n = 12, 13, 10000
    sd = S.mlp_state_dict(c0=c0, seed=5)
    packed = ops.pack_mlp(sd, c0, device=dev)
    feat = torch.randn(1, C, 96, 160, generator=torch.Generator().manual_seed(6)).to(dev)
    pts = _points(n, 7).to(dev)
    body = _gpu_body()
    a = ops.query("icon", pts, EYE, feat, packed, body=body, smpl_feats=["vis", "norm", "cmap", "sdf"])
    b = torch.full_like(a, float("nan"))
    nbytes = _C.lib.icon_query_workspace_bytes(n, body.F, 0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _C.check(_C.lib.icon_query(0, ops._p(pts), pts.stride(1), pts.stride(2), n, ops._calib_rows(EYE), ops._p(feat), C,
                               96, 160, ops._p(None), 0, ops._p(body.ws), body.V, body.F, ops._p(packed.f32),
                               ops._p(packed.tc), c0, 0.05, ops._p(b), ops._p(ws), nbytes, ops._stream()), "icon_query")
    assert torch.equal(a, b), f"{(a != b).sum().item()} outputs differ"


# ---------------------------------------------------------------------------------------------------- 3. locality
@pytest.mark.parametrize("feats", [f for f in SUBSETS if "cmap" not in f], ids="-".join)
def test_subsets_without_cmap_are_point_local(feats):
    """Without cmap nothing depends on the other points of the call: one call equals two calls that split the points at
    an index off the 128-point tile grid, bit for bit, and the call launches no outlier-rank kernel (its launches are
    the SDF block's plus the MLP; the same call with cmap adds the flag, scan and sign passes).  C = 6 keeps c0 <= 15
    with cmap added."""
    from icon_b200 import _C, ops
    dev = _dev()
    C, n, k = 6, 20000, 5037
    sd = S.mlp_state_dict(c0=_c0(feats, C), seed=8)
    packed = ops.pack_mlp(sd, _c0(feats, C), device=dev)
    feat = torch.randn(1, C, 96, 160, generator=torch.Generator().manual_seed(9)).to(dev)
    pts = _points(n, 10).to(dev)
    body = _gpu_body()
    whole = ops.query("icon", pts, EYE, feat, packed, body=body, smpl_feats=feats)
    parts = torch.cat([ops.query("icon", pts[:, :, :k], EYE, feat, packed, body=body, smpl_feats=feats),
                       ops.query("icon", pts[:, :, k:], EYE, feat, packed, body=body, smpl_feats=feats)], 2)
    assert torch.equal(whole, parts), f"{(whole != parts).sum().item()} outputs differ"

    with_cmap = tuple(feats) + ("cmap",)
    packed_cm = ops.pack_mlp(S.mlp_state_dict(c0=_c0(with_cmap, C), seed=11), _c0(with_cmap, C), device=dev)
    torch.cuda.synchronize()

    def launches(fn):
        l0 = _C.launch_count()
        fn()
        torch.cuda.synchronize()
        return _C.launch_count() - l0

    sdf = launches(lambda: ops.sdf_only(pts, EYE, body))
    assert launches(lambda: ops.query("icon", pts, EYE, feat, packed, body=body, smpl_feats=feats)) == sdf + 1
    assert launches(lambda: ops.query("icon", pts, EYE, feat, packed_cm, body=body, smpl_feats=with_cmap)) >= sdf + 4


# ---------------------------------------------------------------------------------------------------- 4. end to end
@pytest.mark.parametrize("res", [[9, 17, 33], [33, 65, 129]], ids=["9-33", "33-129"])
def test_icon_mvp_end_to_end_vs_oracle(res):
    """preset("icon-mvp"): filter-less, smpl_feats = ['sdf'], sdf_clip 15 / 100; HGPIFuNet.filter on 512^2 normal maps,
    the engine, the fused query and marching cubes against the CPU oracle chain."""
    dev = _dev()
    from icon_b200 import config, net
    from icon_b200.engine import Seg3dLossless
    from oracle import query as OQ
    from oracle import mcubes as OM
    from oracle.engine import Seg3dOracle
    cfg = config.preset("icon-mvp")
    netG = net.HGPIFuNet(cfg).to(dev).eval()
    assert netG.if_regressor.c0 == 7 and netG.sdf_clip == pytest.approx(0.15)
    sd = S.mlp_state_dict(c0=7, seed=31)
    sd["filters.3.bias"] = sd["filters.3.bias"] + 0.5       # the 0.5 level set crosses the volume
    netG.if_regressor.load_state_dict(sd)
    v, f = S.body_mesh(rings=20, segs=24, seed=3)
    cm, vi = S.body_attributes(v, seed=3)
    verts, faces = torch.from_numpy(v)[None], torch.from_numpy(f)[None]
    cmap, vis = torch.from_numpy(cm)[None], torch.from_numpy(vi)[None]
    gen = torch.Generator().manual_seed(32)
    nF = torch.randn(1, 3, 512, 512, generator=gen)
    nB = torch.randn(1, 3, 512, 512, generator=gen)
    batch = {"normal_F": nF.to(dev), "normal_B": nB.to(dev), "smpl_verts": verts.to(dev),
             "smpl_faces": faces.to(dev), "smpl_cmap": cmap.to(dev), "smpl_vis": vis.to(dev)}
    eng = Seg3dLossless(query_func=net.query_func, b_min=[[-1.0, 1.0, -1.0]], b_max=[[1.0, -1.0, 1.0]],
                        resolutions=res, align_corners=True, balance_value=0.5, faster=True).to(dev)
    with torch.no_grad():
        features = netG.filter(batch)
        assert features[0].shape == (1, 6, 512, 512)
        occ = eng(opt=cfg, netG=netG, features=features, proj_matrix=None)
    assert occ is not None
    smpl = {"smpl_verts": verts, "smpl_faces": faces, "smpl_cmap": cmap, "smpl_vis": vis}
    feat_cpu = torch.cat([nF, nB], 1)
    ora = Seg3dOracle([[-1.0, 1.0, -1.0]], [[1.0, -1.0, 1.0]], res)
    ref = ora.forward(lambda p: OQ.query_func(sd, [feat_cpu], p, prior="icon", smpl=smpl, smpl_feats=("sdf",),
                                              sdf_clip=0.15))
    assert ref is not None
    assert [int(c.shape[0]) for c in ora.log] == eng.last_query_counts
    assert (occ.cpu() - ref).abs().max() <= 1e-4
    verts_o, faces_o = eng.export_mesh(occ)
    rv, rf = OM.export_mesh(occ.cpu().numpy(), 0.5)
    assert len(rf) > 0
    assert np.array_equal(faces_o.numpy(), rf)
    assert np.array_equal(verts_o.numpy(), rv)
