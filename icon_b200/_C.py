"""ctypes binding of libicon_b200.so (include/icon_b200.h).

The product path has no fallback: if the shared library is missing, importing this module
raises with the build command.  `python -m icon_b200.build` (or __graft_entry__.build())
produces it in-tree.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ICON_B200_LIB") or os.path.join(_HERE, "libicon_b200.so")   # override: diagnostics builds only

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: the CUDA extension must be built (python -m icon_b200.build); "
        "icon_b200 has no CPU or PyTorch fallback.")

lib = ctypes.CDLL(LIB_PATH)

_vp, _i, _i64, _f, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_size_t

_SIGS = {
    "icon_version": (_i, []),
    "icon_last_error": (ctypes.c_char_p, []),
    "icon_launch_count": (_i64, []),
    "icon_profile_enable": (_i, [_i]),
    "icon_profile_last_query": (_i, [_vp]),
    "icon_smpl_workspace_bytes": (_sz, [_i, _i]),
    "icon_smpl_prepare": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _sz, _vp]),
    "icon_query_workspace_bytes": (_sz, [_i64, _i, _i]),
    "icon_set_mlp_impl": (_i, [_i]),
    "icon_get_mlp_impl": (_i, []),
    "icon_query": (_i, [_i, _vp, _i64, _i64, _i64, _vp, _vp, _i, _i, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _i, _f,
                        _vp, _vp, _sz, _vp]),
    "icon_query_feats": (_i, [_i, _vp, _i64, _i64, _i64, _vp, _vp, _i, _i, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _i, _f,
                              _i, _vp, _vp, _sz, _vp]),
    "icon_set_sdf_policy": (_i, [_i, _i64, _i64]),
    "icon_set_sdf_bricks": (_i, [_i, _i64]),
    "icon_sdf_brick_info": (_i, [_vp, _i, _i, _vp]),
    "icon_sdf_only": (_i, [_vp, _i64, _i64, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "icon_sdf_bruteforce": (_i, [_vp, _i64, _i64, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "icon_mesh_workspace_bytes": (_sz, [_i, _i]),
    "icon_mesh_prepare": (_i, [_vp, _vp, _i, _i, _vp, _sz, _vp]),
    "icon_mesh_distance": (_i, [_vp, _i64, _vp, _i, _i, _vp, _vp, _vp]),
    "icon_mesh_sample_workspace_bytes": (_sz, [_i]),
    "icon_mesh_sample": (_i, [_vp, _vp, _i, _i, _vp, _i, ctypes.c_uint64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_mlp_only": (_i, [_vp, _i, _i64, _vp, _vp, _vp, _vp]),
    "icon_display": (_i, [_vp, _i, _vp, _vp]),
    "icon_grid_upsample": (_i, [_vp, _vp, _i, _f, _vp, _vp, _vp, _vp]),
    "icon_grid_dilate": (_i, [_vp, _i, _i, _vp, _vp, _vp]),
    "icon_compact_workspace_bytes": (_sz, [_i]),
    "icon_grid_compact": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _sz, _vp]),
    "icon_grid_scatter": (_i, [_vp, _vp, _vp, _i64, _vp]),
    "icon_grid_init_points": (_i, [_i, _i, _vp, _vp, _vp, _vp]),
    "icon_grid_count_above": (_i, [_vp, _i64, _f, _vp, _vp]),
    "icon_conv_nhwc_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "icon_conv_nhwc": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i,
                           _i, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "icon_norm_finalize": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, ctypes.c_double, _f, _vp]),
    "icon_act_nhwc": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _i, _f, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "icon_splitk_instnorm_act": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "icon_col2im7": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "icon_ew_nhwc": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "icon_nchw_to_nhwc": (_i, [_vp, _vp, _vp, _i, _i, _i64, _vp]),
    "icon_nhwc_to_nchw": (_i, [_vp, _vp, _i, _i, _i, _i, _i64, _vp]),
    "icon_stem_pack": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "icon_clean_mesh_workspace_bytes": (_sz, [_i64, _i64]),
    "icon_clean_mesh_count": (_i, [_vp, _i64, _i64, _vp, _sz, _vp, _vp]),
    "icon_clean_mesh_emit": (_i, [_vp, _i, _vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "icon_conv3d": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "icon_normalize_mask": (_i, [_vp, _vp, _vp, _i, _i, _i64, _vp]),
    "icon_voxelize_workspace_bytes": (_sz, [_i]),
    "icon_voxelize": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _f, _vp, _vp, _sz, _vp]),
    "icon_visibility_workspace_bytes": (_sz, [_i]),
    "icon_visibility": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _sz, _vp]),
    "icon_vertex_normals_workspace_bytes": (_sz, [_i, _i]),
    "icon_vertex_normals": (_i, [_vp, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "icon_normal_render_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "icon_normal_render": (_i, [_vp, _vp, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "icon_mc_workspace_bytes": (_sz, [_i, _i]),
    "icon_mc_count": (_i, [_vp, _i, ctypes.c_double, _i, _vp, _sz, _vp, _vp]),
    "icon_mc_emit": (_i, [_vp, _i, ctypes.c_double, _i, _vp, _vp, _vp, _i64, _i64, _vp]),
}

EXPORTS = tuple(_SIGS.keys())

for _name, (_res, _args) in _SIGS.items():
    _fn = getattr(lib, _name)          # AttributeError here = header / library mismatch
    _fn.restype = _res
    _fn.argtypes = _args


class IconError(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        msg = lib.icon_last_error().decode("utf-8", "replace")
        raise IconError(f"{what} failed (code {rc}): {msg}")


def launch_count():
    return int(lib.icon_launch_count())
