"""Configuration tree for the hot path.

The reference reads a yacs CfgNode (`lib/common/config.py:21-162` defaults merged with
`configs/*.yaml`).  yacs is not a dependency here: `CfgNode` below is a small attribute
dict that is enough for the keys the hot path reads, and any object with the same
attributes (a real yacs node included) can be passed to HGPIFuNet / NormalNet instead.
`preset(name)` restates the four inference YAMLs named by BASELINE.json
(configs/icon-filter.yaml, icon-nofilter.yaml, pamir.yaml, pifu.yaml) and the ICON-MVP prior
(configs/train/icon-mvp.yaml with the test_mode that `apps/train.py -test` forces).
"""
import copy


class CfgNode(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    def clone(self):
        return copy.deepcopy(self)

    def merge(self, other):
        for k, v in other.items():
            if isinstance(v, dict) and isinstance(self.get(k), dict):
                self[k].merge(v)
            else:
                self[k] = copy.deepcopy(v)
        return self


def _to_node(d):
    n = CfgNode()
    for k, v in d.items():
        n[k] = _to_node(v) if isinstance(v, dict) else v
    return n


# defaults the path reads (lib/common/config.py:24-110)
_DEFAULTS = {
    "name": "default", "gpus": [0], "test_gpus": [0], "root": "./data/", "projection_mode": "orthogonal",
    "num_views": 1, "sdf": False, "sdf_clip": 5.0, "overfit": False, "test_mode": True, "mcube_res": 256,
    "clean_mesh": True, "batch_size": 1,
    "net": {
        "gtype": "HGPIFuNet", "norm": "group", "norm_mlp": "group", "hg_down": "ave_pool", "num_views": 1,
        "conv1": [7, 2, 1, 3], "conv3x3": [3, 1, 1, 1], "num_stack": 4, "num_hourglass": 2,
        "hourglass_dim": 256, "voxel_dim": 32, "mlp_dim": [320, 1024, 512, 256, 128, 1],
        "res_layers": [2, 3, 4], "smpl_dim": 3, "prior_type": "icon", "use_filter": True,
        "smpl_feats": ["sdf", "cmap", "norm", "vis"],
        "in_geo": (("normal_F", 3), ("normal_B", 3)),
        "in_nml": (("image", 3), ("T_normal_F", 3), ("T_normal_B", 3)),
    },
}

_COMMON_NET = {"mlp_dim": [256, 512, 256, 128, 1], "res_layers": [2, 3, 4], "num_stack": 2,
               "gtype": "HGPIFuNet", "norm_mlp": "batch",
               "in_nml": (("image", 3), ("T_normal_F", 3), ("T_normal_B", 3))}

_PRESETS = {
    "icon-filter": {"net": dict(_COMMON_NET, prior_type="icon", use_filter=True,
                                in_geo=(("normal_F", 3), ("normal_B", 3)),
                                smpl_feats=["sdf", "norm", "vis", "cmap"], hourglass_dim=6, smpl_dim=7)},
    "icon-nofilter": {"net": dict(_COMMON_NET, prior_type="icon", use_filter=False,
                                  in_geo=(("normal_F", 3), ("normal_B", 3)),
                                  smpl_feats=["sdf", "norm", "vis", "cmap"], hourglass_dim=6, smpl_dim=7)},
    # configs/train/icon-mvp.yaml, the paper's ICON-MVP prior (SMPL sdf only, no filter), evaluated as `-test` runs it
    "icon-mvp": {"net": dict(_COMMON_NET, prior_type="icon", use_filter=False,
                             in_geo=(("normal_F", 3), ("normal_B", 3)), smpl_feats=["sdf"], ctype="resnet34",
                             N_freqs=10, geo_w=0.1, norm_w=0.001, dc_w=1.0, hourglass_dim=6, voxel_dim=32, smpl_dim=1),
                 "sdf_clip": 15.0, "test_mode": True},
    "pamir": {"net": dict(_COMMON_NET, prior_type="pamir", use_filter=True,
                          in_geo=(("image", 3), ("normal_F", 3), ("normal_B", 3)), hourglass_dim=6, voxel_dim=7)},
    "pifu": {"net": dict(_COMMON_NET, prior_type="pifu", use_filter=True,
                         in_geo=(("image", 3), ("normal_F", 3), ("normal_B", 3)), hourglass_dim=12)},
}


def default_cfg():
    return _to_node(copy.deepcopy(_DEFAULTS))


def preset(name, **overrides):
    cfg = default_cfg()
    cfg.merge(_to_node(copy.deepcopy(_PRESETS[name])))
    cfg.name = name
    for k, v in overrides.items():
        cfg[k] = v
    return cfg
