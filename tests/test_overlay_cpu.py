"""The drop-in boundary (icon_b200/overlay.py) on a stand-in ICON checkout written by the test: the modules the
overlay REPLACES are never executed (their stand-ins raise on import, as the real ones would without kaolin /
pytorch3d / voxelize_cuda), the modules it PATCHES run and keep every name off the accelerated path, and a caller
written like apps/ICON.py (`from lib.common.train_util import *`, `from lib.net import HGPIFuNet` ...) receives the
icon_b200 objects.  The stand-in files mirror the reference's module names and import structure only; no reference
source is used.  Runs on the CPU in a fresh interpreter (the overlay installs a process-wide import hook)."""
import os
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHECKOUT = {
    "lib/__init__.py": "",
    "lib/net/__init__.py": """
        from .HGPIFuNet import HGPIFuNet
        from .NormalNet import NormalNet
        from .VE import VolumeEncoder
    """,
    "lib/common/__init__.py": "",
    "lib/dataset/__init__.py": "",
    # replaced: executing any of these is a failure
    "lib/net/HGPIFuNet.py": "raise ImportError('stand-in: needs kaolin / pytorch3d')",
    "lib/net/voxelize.py": "raise ImportError('stand-in: needs voxelize_cuda')",
    "lib/common/seg3d_lossless.py": "raise ImportError('stand-in: needs kaolin marching cubes')",
    # patched: executed, then the accelerated names are rebound
    "lib/common/train_util.py": """
        def query_func(*a): return "reference"
        def clean_mesh(*a): return "reference"
        def get_visibility(*a): return "reference"
        def batch_mean(*a): return "reference"
    """,
    "lib/dataset/mesh_util.py": """
        def get_visibility(*a): return "reference"
        def clean_mesh(*a): return "reference"
        def read_smpl_constants(*a): return "reference"
        def load_checkpoint(*a): return "reference"
    """,
    "lib/net/NormalNet.py": "class NormalNet: pass\n",
    "lib/net/MLP.py": "class MLP: pass\n",
    "lib/net/HGFilters.py": "class HGFilter: pass\nclass HourGlass: pass\nclass ConvBlock: pass\n",
    "lib/net/VE.py": "class VolumeEncoder: pass\nclass Residual3D: pass\n",
    "lib/net/FBNet.py": """
        class LocalEnhancer: pass
        def define_G(input_nc, output_nc, ngf, netG, n_downsample_global=3, n_blocks_global=9, n_local_enhancers=1,
                     n_blocks_local=3, norm="instance", gpu_ids=[], last_op=None):
            return ("reference", netG, norm)
    """,
    "apps/__init__.py": "",
    "apps/caller.py": """
        from lib.common.train_util import *
        from lib.common.seg3d_lossless import Seg3dLossless
        from lib.dataset.mesh_util import get_visibility, load_checkpoint
        from lib.net import HGPIFuNet
        from lib.net.voxelize import Voxelization
    """,
}

SCRIPT = r'''
import sys
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OV
OV.install(REF)
import apps.caller as A
import lib.common.train_util as TU, lib.dataset.mesh_util as MU, lib.net as LN, lib.net.FBNet as FB
import lib.net.HGFilters as HG
HP = sys.modules["lib.net.HGPIFuNet"]              # `lib.net.HGPIFuNet` the attribute is the class
import icon_b200.net, icon_b200.engine, icon_b200.encoders, icon_b200.visibility, icon_b200.mesh, icon_b200.voxelize
assert A.__file__.startswith(REF) and TU.__file__.startswith(REF) and MU.__file__.startswith(REF)
assert HP.__icon_b200_overlay__ == "replace" and TU.__icon_b200_overlay__ == "patch"
assert A.HGPIFuNet is icon_b200.net.HGPIFuNet and LN.HGPIFuNet is icon_b200.net.HGPIFuNet
assert LN.NormalNet is icon_b200.encoders.NormalNet and LN.VolumeEncoder is icon_b200.encoders.VolumeEncoder
assert A.Seg3dLossless is icon_b200.engine.Seg3dLossless and A.Voxelization is icon_b200.voxelize.Voxelization
assert A.query_func is icon_b200.net.query_func and TU.query_func is icon_b200.net.query_func
assert A.get_visibility is icon_b200.visibility.get_visibility and TU.get_visibility is icon_b200.visibility.get_visibility
assert A.clean_mesh is icon_b200.mesh.clean_mesh and MU.clean_mesh is icon_b200.mesh.clean_mesh
assert HG.HGFilter is icon_b200.encoders.HGFilter and HG.ConvBlock.__module__ == "lib.net.HGFilters"
# names off the accelerated path stay the checkout's own objects
assert A.batch_mean() == "reference" and A.batch_mean is TU.batch_mean
assert A.load_checkpoint() == "reference" and MU.load_checkpoint.__module__ == "lib.dataset.mesh_util"
assert FB.LocalEnhancer.__module__ == "lib.net.FBNet"
# define_G: the configuration NormalNet builds -> icon_b200 generator, anything else -> the checkout's define_G
assert isinstance(FB.define_G(6, 3, 64, "global", 2, 1, 1, 3, "instance"), icon_b200.encoders.GlobalGenerator)
assert FB.define_G(6, 3, 8, "global", 2, 1, 1, 3, "instance") == ("reference", "global", "instance")
assert FB.define_G(6, 3, 8, "local", 2, 1, 1, 3, "instance") == ("reference", "local", "instance")
print("OVERLAY_OK")
'''


def test_overlay_replaces_and_patches_a_checkout_and_routes_define_g(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=600, cwd=str(tmp_path))
    assert r.returncode == 0 and "OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
