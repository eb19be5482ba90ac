"""Drop-in overlay: make an UNMODIFIED checkout of YuliangXiu/ICON run its hot path on icon_b200.

    import icon_b200.overlay
    icon_b200.overlay.install("/path/to/ICON")      # before `import apps.ICON` / `python -m apps.infer`
    # or, with no code change at all:  ICON_B200_OVERLAY=/path/to/ICON python -m icon_b200.overlay -m apps.infer ...

The reference's `lib` package stays the reference's: every module, helper and constant that is not part of the
accelerated path (`lib.common.render` but for `Render.get_rendered_video`, `lib.dataset.Evaluator` but for
`calculate_chamfer_p2s`, `init_gl` and `_render_normal`, `lib.smplx` but for the `lbs` its body models call,
`lib.pixielib` but for `SMPLX.forward` in `lib/pixielib/models/SMPLX.py`, `lib.renderer` but for `computePRT` and the
GL renderers `PRTRender` / `ColorRender` / `initialize_GL_context`,
`lib.common.config`, the rest of
`train_util` / `mesh_util` / `net_util` ...) is imported from the checkout unchanged.  An import hook on
`sys.meta_path` then does two things, only for the modules listed below:

* REPLACE  -- the module is never executed; a synthetic module exporting the icon_b200 classes takes its place.
              Used where the reference file exists only to reach third-party CUDA wheels
              (`lib/net/HGPIFuNet.py` -> kaolin / pytorch3d / voxelize_cuda, `lib/net/voxelize.py` -> voxelize_cuda,
              `lib/common/seg3d_lossless.py` -> kaolin marching cubes / PyMCubes), or only to reach OpenGL
              (`lib/renderer/gl/prt_render.py`, `color_render.py`, `init_gl.py` -> PyOpenGL and an EGL context).
* PATCH    -- the reference module is executed normally, then the accelerated names are rebound in its namespace
              (`query_func` in `lib/common/train_util.py`, `get_visibility` and `remesh` in `lib/dataset/mesh_util.py`, the
              encoder classes in `lib/net/{NormalNet,MLP,HGFilters,VE}.py`, `define_G` in `lib/net/FBNet.py`,
              `Evaluator.calculate_chamfer_p2s`, `Evaluator.init_gl` and `Evaluator._render_normal` in
              `lib/dataset/Evaluator.py`, `Render.get_rendered_video` in `lib/common/render.py`, and in
              `lib/dataset/TestDataset.py` an `__init__` that rebinds `get_rgb_image` / `get_silhouette_image` /
              `VF2Mesh` on the instance's `self.render` only, `lbs` in `lib/smplx/body_models.py`, `SMPLX` in
              `lib/pixielib/models/SMPLX.py`: the same class, its `forward` patched to run on the kernels,
              `computePRT` in `lib/renderer/prt_util.py`, `extract_cloth` in `lib/common/cloth_extraction.py`), so
              `from lib.common.train_util import *` (apps/ICON.py:20) still finds everything else it uses.

Callers and call sites this serves: apps/ICON.py:17-22, 52-90 (HGPIFuNet, Seg3dLossless, query_func, get_visibility),
apps/infer.py:22-31, apps/ICON.py:634-640 (calculate_chamfer_p2s), apps/ICON.py:527-528, 555-558, 641-643 (init_gl,
render_normal and calculate_normal_consist through _render_normal: no OpenGL context),
apps/infer.py:168-273, 431-505 (the body-fit and cloth loops: differentiable normal / silhouette renders through
TestDataset.render_normal and render.get_silhouette_image),
apps/infer.py:175-180 (the body-fit loop's `dataset.smpl_model(...)`: SMPL / SMPLH / SMPLX.forward call `lbs`
through lib/smplx/body_models.py's namespace; fp32 CUDA calls run the fused skinning kernels, forward and backward;
with `-hps_type pixie` it is PIXIE's SMPLX.forward, whose skinning and landmark / joint heads run on the kernels),
apps/infer.py:402 (`remesh` of the reconstruction: smoothing and isotropic remeshing on the kernels, the same
`_remesh.obj` written),
apps/infer.py:405-476 and apps/ICON.py:483 (the cloth loop's LocalAffine and shape priors; VF2Mesh's differentiable
vertex colours),
apps/infer.py:548-562 (`-export_video`: get_rendered_video's 360 views per mesh, a chunk of views per kernel call),
lib/dataset/mesh_util.py:187-237 (load_checkpoint:
identical state_dict keys),
lib/dataset/TestDataset.py:137 (get_visibility),
scripts/render_single.py:118 (computePRT of the dataset preparation: the rays cast on the kernels, the same
prt/bounce.npy and prt/face.npy written),
scripts/render_single.py:41, 97-141, 144-239 (initialize_GL_context, ColorRender and PRTRender: every render/,
normal_F/B and T_normal_F/B image drawn on the kernels with no GL context; opengl_util's render_result, load_calib,
make_rotate and rotateSH, Camera, load_scan and the script's RNG use stay the reference's),
apps/infer.py:566-605 (`-seg_dir`: extract_cloth's body-part labels and polygon test on the kernels, the mesh cut by
the reference's own trimesh calls; load_segmentation and smpl_to_recon_labels stay the reference's).
"""
import importlib.abc
import importlib.machinery
import importlib.util
import os
import sys
import types

_INSTALLED = None


def _replacements():
    from . import dataset_render, encoders, engine, net, voxelize
    return {
        "lib.net.HGPIFuNet": {"HGPIFuNet": net.HGPIFuNet, "MLP": net.MLP, "BasePIFuNet": net.BasePIFuNet,
                              "NormalNet": encoders.NormalNet, "HGFilter": encoders.HGFilter,
                              "VolumeEncoder": encoders.VolumeEncoder, "Voxelization": voxelize.Voxelization,
                              "init_net": net.init_net},
        "lib.net.voxelize": {"Voxelization": voxelize.Voxelization},
        "lib.common.seg3d_lossless": {"Seg3dLossless": engine.Seg3dLossless},
        # the dataset renderer: each of these imports OpenGL.GL at the top
        "lib.renderer.gl.prt_render": {"PRTRender": dataset_render.PRTRender},
        "lib.renderer.gl.color_render": {"ColorRender": dataset_render.ColorRender},
        "lib.renderer.gl.init_gl": {"initialize_GL_context": dataset_render.initialize_GL_context},
    }


def _patches():
    from . import (body_model, encoders, garments, hps, mesh, mesh_priors, mesh_views, metrics, net, prt, remesh,
                   visibility, voxelize)

    def make_define_G(reference_define_G):
        import torch.nn as nn

        def define_G(input_nc, output_nc, ngf, netG, n_downsample_global=3, n_blocks_global=9, n_local_enhancers=1,
                     n_blocks_local=3, norm="instance", gpu_ids=[], last_op=nn.Tanh()):
            """lib/net/FBNet.py:52-90: the one configuration the path builds (NormalNet.py:67-70: 'global' +
            'instance', ngf 64, at most 3 output channels) returns the icon_b200 generator; everything else is the
            reference's own."""
            if netG == "global" and norm == "instance" and ngf == 64 and output_nc <= 3:
                return encoders.GlobalGenerator(input_nc, output_nc, ngf, n_downsample_global, n_blocks_global, last_op)
            return reference_define_G(input_nc, output_nc, ngf, netG, n_downsample_global, n_blocks_global,
                                      n_local_enhancers, n_blocks_local, norm, gpu_ids, last_op)
        return define_G

    return {
        "lib.common.train_util": {"query_func": net.query_func, "clean_mesh": mesh.clean_mesh,
                                  "get_visibility": visibility.get_visibility},      # duplicate at train_util.py:361
        "lib.dataset.mesh_util": {"get_visibility": visibility.get_visibility, "clean_mesh": mesh.clean_mesh,
                                  "read_smpl_constants": voxelize.read_smpl_constants,
                                  "update_mesh_shape_prior_losses": mesh_priors.update_mesh_shape_prior_losses,
                                  "remesh": remesh.remesh},
        "lib.net.local_affine": {"LocalAffine": mesh_priors.LocalAffine},
        "lib.net.NormalNet": {"NormalNet": encoders.NormalNet},
        "lib.net.MLP": {"MLP": net.MLP},
        "lib.net.HGFilters": {"HGFilter": encoders.HGFilter, "HourGlass": encoders.HourGlass},
        "lib.net.FBNet": {"define_G": make_define_G},          # callable(old value) -> new value
        "lib.net.VE": {"VolumeEncoder": encoders.VolumeEncoder, "Residual3D": encoders.Residual3D},
        "lib.dataset.Evaluator": {"Evaluator": metrics.make_Evaluator},     # chamfer_p2s, init_gl, _render_normal
        "lib.common.render": {"Render": mesh_views.make_Render},            # get_rendered_video
        "lib.dataset.TestDataset": {"TestDataset": mesh_views.make_TestDataset},  # self.render's fit renders, VF2Mesh
        "lib.smplx.body_models": {"lbs": body_model.make_lbs},              # SMPL / SMPLH / SMPLX.forward's skinning
        "lib.pixielib.models.SMPLX": {"SMPLX": body_model.make_pixie_SMPLX},  # PIXIE's SMPL-X: skinning and heads
        "lib.renderer.prt_util": {"computePRT": prt.make_computePRT},       # the dataset renderer's PRT transfer
        "lib.common.cloth_extraction": {"extract_cloth": garments.make_extract_cloth},  # -seg_dir garments
        "lib.pymaf.models.pymaf_net": {"PyMAF": hps.make_PyMAF},           # the body estimate (-hps_type pymaf)
    }


def _rebind(module, names):
    """Rebind `names` in an executed reference module; a value wrapped in make_* style (a function whose name
    starts with 'make_') receives the reference's own object and returns the replacement."""
    for k, v in names.items():
        if callable(v) and getattr(v, "__name__", "").startswith("make_"):
            v = v(module.__dict__.get(k))
        module.__dict__[k] = v
    module.__icon_b200_overlay__ = "patch"


class _ReplaceLoader(importlib.abc.Loader):
    def __init__(self, names):
        self.names = names

    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__doc__ = f"icon_b200 overlay of the reference's {spec.name} (module not executed)"
        return m

    def exec_module(self, module):
        module.__dict__.update(self.names)
        module.__all__ = sorted(self.names)
        module.__icon_b200_overlay__ = "replace"


class _PatchLoader(importlib.abc.Loader):
    def __init__(self, inner, names):
        self.inner, self.names = inner, names

    def create_module(self, spec):
        return self.inner.create_module(spec) if hasattr(self.inner, "create_module") else None

    def exec_module(self, module):
        self.inner.exec_module(module)
        _rebind(module, self.names)

    def __getattr__(self, k):                      # get_code / get_source / is_package ... of the real loader
        return getattr(self.inner, k)


class OverlayFinder(importlib.abc.MetaPathFinder):
    def __init__(self, replace, patch):
        self.replace, self.patch = replace, patch

    def find_spec(self, fullname, path, target=None):
        if fullname in self.replace:
            return importlib.machinery.ModuleSpec(fullname, _ReplaceLoader(self.replace[fullname]),
                                                  origin="icon_b200.overlay")
        if fullname in self.patch:
            spec = importlib.machinery.PathFinder.find_spec(fullname, path)      # the reference's own file
            if spec is None or spec.loader is None:
                return None
            spec.loader = _PatchLoader(spec.loader, self.patch[fullname])
            return spec
        return None


def install(reference_root=None):
    """Activate the overlay (idempotent).  `reference_root` = the ICON checkout; it is put on sys.path so that
    `lib` and `apps` resolve to the reference's packages.  Must run before the reference's modules are imported;
    modules that were imported earlier are patched in place (PATCH set) or swapped (REPLACE set)."""
    global _INSTALLED
    if reference_root is not None:
        root = os.path.abspath(reference_root)
        if not os.path.isdir(os.path.join(root, "lib")):
            raise FileNotFoundError(f"{root} does not look like an ICON checkout (no lib/)")
        if root not in sys.path:
            sys.path.insert(0, root)
    if _INSTALLED is not None:
        return _INSTALLED
    replace, patch = _replacements(), _patches()
    finder = OverlayFinder(replace, patch)
    sys.meta_path.insert(0, finder)
    for name, names in patch.items():                  # already imported: rebind in place
        if name in sys.modules and getattr(sys.modules[name], "__icon_b200_overlay__", None) is None:
            _rebind(sys.modules[name], names)
    for name in replace:
        if name in sys.modules and getattr(sys.modules[name], "__icon_b200_overlay__", None) is None:
            del sys.modules[name]
            parent, _, child = name.rpartition(".")
            if parent in sys.modules and hasattr(sys.modules[parent], child):
                delattr(sys.modules[parent], child)
    _INSTALLED = finder
    return finder


def uninstall():
    global _INSTALLED
    if _INSTALLED is not None and _INSTALLED in sys.meta_path:
        sys.meta_path.remove(_INSTALLED)
    _INSTALLED = None


def _main(argv):
    """python -m icon_b200.overlay [-r ICON_ROOT] -m apps.infer <args...>   (runpy under the overlay)"""
    import runpy
    root = os.environ.get("ICON_B200_OVERLAY")
    args = list(argv)
    if args and args[0] == "-r":
        root, args = args[1], args[2:]
    if not args or args[0] != "-m" or len(args) < 2:
        raise SystemExit(_main.__doc__)
    install(root or os.getcwd())
    sys.argv = [args[1]] + args[2:]
    runpy.run_module(args[1], run_name="__main__", alter_sys=True)


if __name__ == "__main__":
    _main(sys.argv[1:])
