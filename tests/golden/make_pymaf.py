"""Generate tests/golden/pymaf.npz by running the REFERENCE's own PyMAF (lib/pymaf/models/pymaf_net.py) live on the
CPU in float64, from an ICON checkout (read-only; path in ICON_REFERENCE_DIR).  The fixture is committed and pins
oracle/pymaf.py (tests/test_pymaf_cpu.py); the GPU tests compare icon_b200/hps.py with the oracle.

    ICON_REFERENCE_DIR=/path/to/ICON python tests/golden/make_pymaf.py

Set-up, with nothing read from the network:
  * `lib.common.config.cfg` and `lib.pymaf.core.cfgs.cfg` are stand-ins holding the shipped
    lib/pymaf/configs/pymaf_config.yaml values (yacs is not a dependency here), and `torchvision.models.resnet` an empty
    module: ResNet_Backbone only touches it for pretrained=True, and the model is built with pretrained=False;
  * `lib.pymaf.core.path_config` points at the files icon_b200.synthetic.pymaf_files(seed 0) writes to a temporary
    directory (SMPL_NEUTRAL.pkl, J_regressor_extra.npy, mesh_downsampling.npz, smpl_mean_params.npz);
  * the module is built by `pymaf_net(SMPL_MEAN_PARAMS, pretrained=False)`, loaded with
    synthetic.pymaf_state_dict(0) under load_state_dict(strict=True), made float64 (torch's default dtype too, which
    perspective_projection's intrinsics take) and run in eval mode.

Stored: the reference's state_dict key names and shapes (dp_head included), the SHA-256 of the synthetic state dict
(synthetic.pymaf_sha256), the reference's own joint_map, smplh vertex ids and J24_TO_J19, and for the images
synthetic.pymaf_image(0, 1, 2): every field of the four smpl_out dicts except `verts`, the last dict's `verts`, and 64
values of each of the three s_feat maps at PROBE_SEED-drawn positions.
"""
import importlib
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
OUT = os.path.join(HERE, "pymaf.npz")
IMAGES = (0, 1, 2)
PROBE_SEED = 64
KEYS = ("theta", "verts", "kp_2d", "kp_3d", "smpl_kp_3d", "rotmat", "pred_cam", "pred_shape", "pred_pose")


def probe_index(shape, n=64, seed=PROBE_SEED):
    """n flat positions of an NCHW map of `shape`, seeded."""
    return np.random.RandomState(seed).choice(int(np.prod(shape)), n, replace=False)


def load_reference(ref, folder):
    from icon_b200 import synthetic as S
    sys.path.insert(0, ref)
    cfg = S.pymaf_cfg()
    for name in ("lib.common.config", "lib.pymaf.core.cfgs"):
        m = types.ModuleType(name)
        m.cfg = cfg
        sys.modules[name] = m
    common = types.ModuleType("lib.common")
    common.__path__ = [os.path.join(ref, "lib", "common")]
    sys.modules["lib.common"] = common
    tv = types.ModuleType("torchvision")
    tv.__path__ = []
    tvm = types.ModuleType("torchvision.models")
    tvm.__path__ = []
    tvr = types.ModuleType("torchvision.models.resnet")
    sys.modules.update({"torchvision": tv, "torchvision.models": tvm, "torchvision.models.resnet": tvr})
    pc = importlib.import_module("lib.pymaf.core.path_config")
    pc.SMPL_MEAN_PARAMS = os.path.join(folder, S.PYMAF_FILES[3])
    pc.SMPL_MODEL_DIR = os.path.dirname(os.path.join(folder, S.PYMAF_FILES[0]))
    pc.MESH_DOWNSAMPLEING = os.path.join(folder, S.PYMAF_FILES[2])
    pc.JOINT_REGRESSOR_TRAIN_EXTRA = os.path.join(folder, S.PYMAF_FILES[1])
    return importlib.import_module("lib.pymaf.models.pymaf_net"), importlib.import_module("lib.pymaf.core.constants")


def make(ref):
    from icon_b200 import synthetic as S
    folder = tempfile.mkdtemp(prefix="pymaf_files_")
    S.pymaf_files(folder, 0)
    P, C = load_reference(ref, folder)
    model = P.pymaf_net(P.SMPL_MEAN_PARAMS, pretrained=False)
    smpl = model.regressor[0].smpl
    out = {"joint_map": smpl.joint_map.numpy().astype(np.int64),
           "vertex_ids": smpl.vertex_joint_selector.extra_joints_idxs.numpy().astype(np.int64),
           "J24_TO_J19": np.asarray(C.J24_TO_J19, np.int64)}
    ref_sd = model.state_dict()
    out["sd_keys"] = np.array(list(ref_sd), dtype=object).astype(str)
    out["sd_shapes"] = np.array([",".join(str(d) for d in t.shape) for t in ref_sd.values()]).astype(str)
    sd = S.pymaf_state_dict(0)
    out["sd_sha256"] = np.array(S.pymaf_sha256(sd))
    model.load_state_dict(sd, strict=True)
    torch.set_default_dtype(torch.float64)
    model = model.double().eval()
    feats = []
    for k in (2, 5, 8):
        model.deconv_layers[k].register_forward_hook(lambda m, i, o: feats.append(o.detach().clone()))
    for seed in IMAGES:
        feats.clear()
        with torch.no_grad():
            res = model(S.pymaf_image(seed).double())
        assert len(res["smpl_out"]) == 4 and res["dp_out"] == []
        for j, d in enumerate(res["smpl_out"]):
            for k in KEYS:
                if k != "verts" or j == 3:
                    out[f"img{seed}_{j}_{k}"] = d[k].numpy()
        for i, f in enumerate(feats):
            out[f"img{seed}_sfeat{i}"] = f.numpy().reshape(-1)[probe_index(f.shape)]
    return out


if __name__ == "__main__":
    out = make(os.environ["ICON_REFERENCE_DIR"])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes,", len(out), "arrays")
