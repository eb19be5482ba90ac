"""Reference-equivalent single-GPU path (SURVEY.md 8d (b): the ">= 10x" denominator of north_star).

The reference's GPU path = kaolin's two brute-force O(N*F) CUDA kernels (point_to_mesh_distance, check_sign) for
the SMPL block + stock PyTorch ops (grid_sample, gather, cat, Conv1d, BatchNorm1d, LeakyReLU) for everything else.
kaolin is not installable here, so its kernels are stood in for by this repo's own brute-force kernel
(`icon_sdf_bruteforce`: every point against every face, exact distance + ray parity -- the same algorithm class);
the rest is written below with stock torch ops exactly as HGPIFuNet.query / MLP.forward compose them
(lib/net/HGPIFuNet.py:285-365, lib/net/MLP.py:49-72), in chunks of 2^20 points (a dense 256^3 call needs 34 GB for
one [1,512,N] activation otherwise).  Self-contained on purpose: nothing here imports oracle/.

Prints M points/s of that path next to this repo's fused query on the same 256^3 lattice and the max |diff|.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from icon_b200 import config, net, ops, synthetic as S

dev = torch.device("cuda:0")
GRID = int(sys.argv[1]) if len(sys.argv) > 1 else 256
CHUNK = 1 << 20

cfg = config.preset("icon-filter")
netG = net.HGPIFuNet(cfg).to(dev).eval()
sd = S.mlp_state_dict(c0=13, seed=0)
netG.if_regressor.load_state_dict(sd)
sd = {k: v.to(dev) for k, v in sd.items()}
v, f = S.body_mesh(seed=0)
cm, vi = S.body_attributes(v, seed=0)
smpl = {"smpl_verts": torch.from_numpy(v)[None].to(dev), "smpl_faces": torch.from_numpy(f)[None].to(dev),
        "smpl_cmap": torch.from_numpy(cm)[None].to(dev), "smpl_vis": torch.from_numpy(vi)[None].to(dev)}
netG.smpl_feat_dict = smpl
feat = S.feature_map(12, 128, seed=0).to(dev)
pts = S.lattice_points(GRID).to(dev)                       # [1, N, 3]
N = pts.shape[1]
body = ops.SmplBody(smpl["smpl_verts"], smpl["smpl_faces"], smpl["smpl_cmap"], smpl["smpl_vis"])
eye = torch.eye(4)[None]


def torch_mlp(x):
    """lib/net/MLP.py:49-72 with norm='batch' in eval mode, res_layers [2,3,4], no last_op."""
    y, x0 = x, x
    for i in range(4):
        if i in (2, 3):
            y = torch.cat([y, x0], 1)
        y = F.conv1d(y, sd[f"filters.{i}.weight"], sd[f"filters.{i}.bias"])
        if i != 3:
            y = F.batch_norm(y, sd[f"norms.{i}.running_mean"], sd[f"norms.{i}.running_var"], sd[f"norms.{i}.weight"],
                             sd[f"norms.{i}.bias"], training=False, eps=1e-5)
            y = F.leaky_relu(y, 0.01)
    return y


def reference_path():
    """one dense call, as HGPIFuNet.query composes it; returns preds [1,1,N]"""
    p3 = pts.permute(0, 2, 1)                                              # [1,3,N]
    rec, _ = ops.sdf_only(p3, eye, body, brute=True)                       # stands in for kaolin: [N,8]
    sdf, cmap, norm, vis = rec[:, 0:1], rec[:, 1:4].clone(), rec[:, 4:7], rec[:, 7:8]
    # HGPIFuNet.py:296-304, whole-call semantics (the outlier rule depends on the call's outlier count)
    sdf = sdf.clone()[None]
    cmap = cmap[None]
    outlier = sdf.abs() >= 0.05
    sdf[outlier] = torch.sign(sdf[outlier])
    cmap[outlier.repeat(1, 1, 3)] = sdf[outlier].repeat(1, 1, 3)
    smpl_feat = torch.cat([sdf, cmap, norm[None], vis[None]], dim=2).permute(0, 2, 1)          # [1,8,N]
    in_cube = ((p3 > -1.0) & (p3 < 1.0)).all(dim=1, keepdim=True).float()
    out = torch.empty(1, 1, N, device=dev)
    for s in range(0, N, CHUNK):
        e = min(N, s + CHUNK)
        xy = p3[:, :2, s:e]
        samples = F.grid_sample(feat, xy.transpose(1, 2).unsqueeze(2), align_corners=True)[..., 0]    # geometry.py:21-43
        visc = smpl_feat[:, 7:8, s:e]
        dim = samples.shape[1] // 2
        idx = torch.tile(1 - visc, (1, dim, 1)) * dim + torch.arange(dim, device=dev)[None, :, None]
        local = torch.gather(samples, 1, idx.long())                                                   # feat_select
        point_feat = torch.cat([local, smpl_feat[:, :7, s:e]], 1)
        out[:, :, s:e] = torch_mlp(point_feat) * in_cube[:, :, s:e]
    return out


def timed(fn, n, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        r = fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, r


with torch.no_grad():
    ms_ref, ref = timed(reference_path, 2, 1)              # stock settings: cuDNN convolutions may use TF32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ms_ref32, ref32 = timed(reference_path, 1, 0)          # same path forced to fp32 arithmetic
    torch.backends.cudnn.allow_tf32 = True
    ms_sdf, _ = timed(lambda: ops.sdf_only(pts.permute(0, 2, 1), eye, body, brute=True), 2, 0)
    ms_ours, ours = timed(lambda: net.query_func(cfg, netG, [feat], pts), 5, 3)
print(json.dumps({
    "grid": GRID, "points": N,
    "reference_equivalent_gpu_path_ms": ms_ref, "reference_equivalent_Mpts_s": N / ms_ref / 1e3,
    "of_which_bruteforce_sdf_ms (kaolin stand-in)": ms_sdf, "stock_torch_rest_ms": ms_ref - ms_sdf,
    "fused_query_ms": ms_ours, "fused_query_Mpts_s": N / ms_ours / 1e3, "speedup": ms_ref / ms_ours,
    "max_abs_diff_vs_stock_settings (TF32 convs)": float((ref - ours).abs().max()),
    "reference_equivalent_fp32_ms": ms_ref32, "max_abs_diff_vs_fp32": float((ref32 - ours).abs().max())}, indent=1))
