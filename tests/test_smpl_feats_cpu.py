"""The icon prior's `smpl_feats` subsets on the host: the ICON-MVP preset, the MLP width of every subset, and the width
checks that run before any kernel (no GPU needed)."""
import ctypes
import itertools

import pytest
import torch

from icon_b200 import synthetic as S  # noqa: F401  (imports the package: the library must be built)


def _subsets():
    """All 8 subsets: sdf plus any of cmap / norm / vis."""
    out = []
    for k in range(4):
        for extra in itertools.combinations(("cmap", "norm", "vis"), k):
            out.append(("sdf",) + extra)
    return out


def test_icon_mvp_preset_restates_the_reference_config():
    from icon_b200 import config, net
    cfg = config.preset("icon-mvp")
    assert cfg.net.smpl_feats == ["sdf"] and cfg.net.smpl_dim == 1 and not cfg.net.use_filter
    assert cfg.sdf_clip == 15.0 and cfg.test_mode
    g = net.HGPIFuNet(cfg)
    assert g.if_regressor.filter_channels == [7, 512, 256, 128, 1]
    assert g.sdf_clip == pytest.approx(0.15)
    assert g.if_regressor.last_op is None


@pytest.mark.parametrize("use_filter", [True, False], ids=["filter", "nofilter"])
@pytest.mark.parametrize("feats", _subsets(), ids="-".join)
def test_every_subset_gets_the_mlp_width_of_the_column_table(feats, use_filter):
    """HGPIFuNet.py:97-104 with smpl_dim = 1 + 3 cmap + 3 norm gives c0 = L + smpl_dim, where L = C/2 with vis and C
    without; C = 2 hourglass_dim = 12 with the filter, 6 (normal_F | normal_B) without."""
    from icon_b200 import config, net, ops
    cm, nm, vis = ("cmap" in feats), ("norm" in feats), ("vis" in feats)
    cfg = config.preset("icon-filter" if use_filter else "icon-nofilter")
    cfg.net.smpl_feats = list(feats)
    cfg.net.smpl_dim = 1 + 3 * cm + 3 * nm
    g = net.HGPIFuNet(cfg)
    C = 12 if use_filter else 6
    want = (C // 2 if vis else C) + 1 + 3 * cm + 3 * nm
    assert g.if_regressor.c0 == want == ops.icon_c0(feats, C)


def test_smpl_feats_mask_ignores_order_and_rejects_unknown_names():
    from icon_b200 import _C, ops
    assert ops.smpl_feats_mask(["sdf", "norm", "vis", "cmap"]) == 7 == ops.smpl_feats_mask(ops.SMPL_FEATS_ALL)
    assert ops.smpl_feats_mask(["vis", "sdf"]) == ops.smpl_feats_mask(["vis"]) == 4
    assert ops.smpl_feats_mask(["sdf"]) == 0
    with pytest.raises(_C.IconError, match="unknown"):
        ops.smpl_feats_mask(["sdf", "normal"])


def test_mismatched_smpl_dim_raises_before_any_kernel():
    """smpl_feats = ['sdf'] with the full set's smpl_dim = 7: the reference fails inside conv1d; here HGPIFuNet.query
    raises before the body is prepared or anything is launched (CPU tensors: nothing could run anyway)."""
    from icon_b200 import _C, config, net
    cfg = config.preset("icon-mvp")
    cfg.net.smpl_dim = 7
    g = net.HGPIFuNet(cfg).eval()
    l0 = _C.launch_count()
    with pytest.raises(RuntimeError, match=r"smpl_feats.*c0 = 7.*c0 = 13 \(smpl_dim = 7\)"):
        g.query([torch.zeros(1, 6, 32, 32)], torch.zeros(1, 3, 10), torch.eye(4)[None])
    assert _C.launch_count() == l0


@pytest.mark.parametrize("mask,C,c0", [(0, 6, 8), (7, 12, 12), (4, 7, 4), (1, 12, 15), (8, 12, 13), (-1, 12, 13)])
def test_icon_query_feats_rejects_layouts_outside_the_table(mask, C, c0):
    """The C entry point checks c0 against the column table (an odd C with vis included, where C/2 would round) and
    the mask's bits before it touches the device.  Every case here is rejected, so the placeholder pointers are never
    used."""
    from icon_b200 import _C
    lib = _C.lib
    fake = ctypes.c_void_p(1 << 20)                     # never dereferenced: the checks fail first
    calib = (ctypes.c_float * 12)()
    n, F = 1000, 100
    nbytes = lib.icon_query_workspace_bytes(n, F, 0)
    rc = lib.icon_query_feats(0, fake, 1, 3, n, calib, fake, C, 8, 8, None, 0, fake, 50, F, fake, fake, c0, 0.05, mask,
                              fake, fake, nbytes, None)
    assert rc == -1
    assert "smpl_feats mask" in lib.icon_last_error().decode()
