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
    "icon_sdf_brick_lists": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "icon_sdf_only": (_i, [_vp, _i64, _i64, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "icon_sdf_bruteforce": (_i, [_vp, _i64, _i64, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "icon_face_tree_read": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp]),
    "icon_mesh_workspace_bytes": (_sz, [_i, _i]),
    "icon_mesh_prepare": (_i, [_vp, _vp, _i, _i, _vp, _sz, _vp]),
    "icon_mesh_distance": (_i, [_vp, _i64, _vp, _i, _i, _vp, _vp, _vp]),
    "icon_mesh_sample_workspace_bytes": (_sz, [_i]),
    "icon_mesh_sample": (_i, [_vp, _vp, _i, _i, _vp, _i, ctypes.c_uint64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_prt_workspace_bytes": (_sz, [_i, _i, _i]),
    "icon_prt": (_i, [_vp, _i, _i, _vp, _vp, _i, ctypes.c_double, _vp, _vp, _i, _i, ctypes.c_double, _vp, _vp, _vp, _sz,
                      _vp]),
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
    "icon_dataset_render_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "icon_dataset_render": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "icon_dataset_texture_bytes": (_sz, [_i, _i]),
    "icon_dataset_texture": (_i, [_vp, _i, _i, _vp, _sz, _vp]),
    "icon_area_vertex_normals_workspace_bytes": (_sz, [_i, _i]),
    "icon_area_vertex_normals": (_i, [_vp, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "icon_area_vertex_normals_backward_workspace_bytes": (_sz, [_i, _i]),
    "icon_area_vertex_normals_backward": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "icon_mesh_topology_workspace_bytes": (_sz, [_i, _i]),
    "icon_mesh_topology_count": (_i, [_vp, _i, _i, ctypes.POINTER(_i64), _vp, _sz, _vp]),
    "icon_mesh_topology_build": (_i, [_vp, _vp, _sz, _vp]),
    "icon_vertex_edges_workspace_bytes": (_sz, [_i, _i]),
    "icon_vertex_edges": (_i, [_vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "icon_mesh_priors_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "icon_mesh_priors_forward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_mesh_priors_backward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_local_affine_forward": (_i, [_vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    "icon_local_affine_backward": (_i, [_vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "icon_mesh_views_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "icon_mesh_views": (_i, [_vp, _vp, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_mesh_render_state_bytes": (_sz, [_i, _i, _i]),
    "icon_mesh_render_workspace_bytes": (_sz, [_i, _i, _i, _i, _i, _i]),
    "icon_mesh_render_forward": (_i, [_i, _vp, _vp, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _sz, _vp, _sz, _vp]),
    "icon_mesh_render_backward": (_i, [_i, _vp, _vp, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _sz, _vp, _vp, _vp, _sz,
                                       _vp]),
    "icon_lbs_prepare_workspace_bytes": (_sz, [_i, _i, _i]),
    "icon_lbs_prepare": (_i, [_vp, _vp, _i, _vp, _sz, _vp]),
    "icon_lbs_state_bytes": (_sz, [_i, _i, _i, _i]),
    "icon_lbs_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "icon_lbs_forward": (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _sz, _vp, _sz, _vp]),
    "icon_lbs_backward": (_i, [_vp, _i, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_smplx_heads_prepare": (_i, [_vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _i, _vp, _i,
                                      _vp]),
    "icon_smplx_heads_state_bytes": (_sz, [_i, _i, _i]),
    "icon_smplx_heads_forward": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_smplx_heads_backward": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "icon_tetra_prepare": (_i, [_vp, _vp, _i, _i, _i]),
    "icon_tetra_state_bytes": (_sz, []),
    "icon_tetra_forward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_remesh_workspace_bytes": (_sz, [_i, _i, _i]),
    "icon_remesh_compact": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_remesh_classify": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "icon_remesh_smooth_step": (_i, [_vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_remesh_midpoints": (_i, [_vp, _vp, _vp, _vp]),
    "icon_remesh_select": (_i, [_i, _vp, _vp, ctypes.c_double, _i, _vp, ctypes.c_double, _vp, _vp, _sz, _vp]),
    "icon_remesh_apply": (_i, [_i, _vp, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "icon_remesh_relax": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "icon_remesh_reproject": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "icon_mc_workspace_bytes": (_sz, [_i, _i]),
    "icon_mc_count": (_i, [_vp, _i, ctypes.c_double, _i, _vp, _sz, _vp, _vp]),
    "icon_mc_emit": (_i, [_vp, _i, ctypes.c_double, _i, _vp, _vp, _vp, _i64, _i64, _vp]),
    "icon_garment_labels_workspace_bytes": (_sz, [_i]),
    "icon_garment_labels": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "icon_garment_face_mask_workspace_bytes": (_sz, [_i, _i]),
    "icon_garment_face_mask": (_i, [_vp, _i, _vp, _i, _vp, ctypes.c_uint32, _vp, _i, _vp, _i, _vp, _vp, _vp, _sz,
                                    _vp]),
    "icon_maxpool3s2_nhwc": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "icon_maf_mlp": (_i, [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp]),
    "icon_hps_gemv": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    "icon_hps_rot6d": (_i, [_vp, _vp, _i, _vp]),
    "icon_hps_regress": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "icon_hps_tail": (_i, [_vp, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
}

EXPORTS = tuple(_SIGS.keys())

for _name, (_res, _args) in _SIGS.items():
    _fn = getattr(lib, _name)          # AttributeError here = header / library mismatch
    _fn.restype = _res
    _fn.argtypes = _args


class MeshTopology(ctypes.Structure):
    """icon_mesh_topology (include/icon_b200.h): device pointers of one mesh's topology arrays."""
    _fields_ = [("V", _i), ("F", _i), ("E", _i), ("faces", _vp), ("edges", _vp), ("face_to_edge", _vp),
                ("vert_off", _vp), ("vert_edges", _vp), ("edge_off", _vp), ("edge_entries", _vp),
                ("corner_off", _vp), ("vert_corners", _vp)]


class LbsModel(ctypes.Structure):
    """icon_lbs_model (include/icon_b200.h): one body model's sizes, parents and device buffers."""
    _fields_ = [("V", _i), ("J", _i), ("NB", _i), ("parents", _i * 64), ("v_template", _vp), ("shapedirs", _vp),
                ("posedirs", _vp), ("J_regressor", _vp), ("lbs_weights", _vp), ("J_template", _vp), ("J_dirs", _vp)]


class SmplxHeads(ctypes.Structure):
    """icon_smplx_heads (include/icon_b200.h): PIXIE's landmark / joint head tables of one SMPL-X model."""
    _fields_ = [("V", _i), ("J", _i), ("R", _i), ("Ls", _i), ("Ld", _i), ("E", _i), ("nchain", _i),
                ("chain", _i * 8), ("regressor", _vp), ("vid", _vp), ("bc", _vp), ("joint_reg", _vp),
                ("reg_joint", _vp), ("inc_off", _vp), ("inc", _vp)]


class TetraModel(ctypes.Structure):
    """icon_tetra_model (include/icon_b200.h): PaMIR's tetrahedral SMPL, both vertex sets, on the device."""
    _fields_ = [("V", _i), ("N", _i), ("T", _i), ("nnz", _i), ("parents", _i * 24), ("v_template", _vp),
                ("shapedirs", _vp), ("posedirs", _vp), ("weights", _vp), ("jr_off", _vp), ("jr_col", _vp),
                ("jr_val", _vp)]


class DatasetMesh(ctypes.Structure):
    """icon_dr_mesh (include/icon_b200.h): one mesh of the dataset renderer, device arrays indexed per face corner."""
    _fields_ = [("mode", _i), ("F", _i), ("V", _i), ("Vn", _i), ("Vt", _i), ("Va", _i), ("pos", _vp), ("nrm", _vp),
                ("uv", _vp), ("attr", _vp), ("f_pos", _vp), ("f_nrm", _vp), ("f_uv", _vp), ("f_attr", _vp),
                ("tex", _vp), ("tex_w", _i), ("tex_h", _i)]


class IconError(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        msg = lib.icon_last_error().decode("utf-8", "replace")
        raise IconError(f"{what} failed (code {rc}): {msg}")


def launch_count():
    return int(lib.icon_launch_count())
