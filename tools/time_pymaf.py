"""PyMAF's body estimate (icon_b200/hps.py, csrc/hps.cu) on one 224 x 224 image with the seeded weights of
icon_b200.synthetic.pymaf_state_dict.

    python tools/time_pymaf.py [--reps 30] [--out results/time_pymaf.json]

Prints one JSON line: CUDA-event medians of the whole forward eager and graph-replayed, of each stage run eagerly
(backbone, the three deconvolutions, the three MAF rows, the three regressors, the four SMPL tails), and of the same
network's backbone + deconvolutions + MAF + regressors as stock torch fp32 on CUDA (cuDNN, TF32 off; the SMPL tail is
not in the stock figure), plus the GPU's name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from icon_b200 import hps, synthetic as S  # noqa: E402
from tools.time_metrics import ev_ms, gpu_info, median  # noqa: E402


def stock(sd, x, pts0):
    """backbone + deconvolutions + MAF + regressors in stock torch fp32 (points of later iterations: pts0)."""
    def bn(y, n):
        return F.batch_norm(y, sd[n + ".running_mean"], sd[n + ".running_var"], sd[n + ".weight"], sd[n + ".bias"],
                            False, 0.0, 1e-5)
    fe = "feature_extractor."
    y = F.max_pool2d(F.relu(bn(F.conv2d(x, sd[fe + "conv1.weight"], None, 2, 3), fe + "bn1")), 3, 2, 1)
    for li, n in enumerate(hps.LAYERS):
        for b in range(n):
            p = f"{fe}layer{li + 1}.{b}."
            s = 2 if (li > 0 and b == 0) else 1
            o = F.relu(bn(F.conv2d(y, sd[p + "conv1.weight"]), p + "bn1"))
            o = F.relu(bn(F.conv2d(o, sd[p + "conv2.weight"], None, s, 1), p + "bn2"))
            o = bn(F.conv2d(o, sd[p + "conv3.weight"]), p + "bn3")
            r = bn(F.conv2d(y, sd[p + "downsample.0.weight"], None, s), p + "downsample.1") if b == 0 else y
            y = F.relu(o + r)
    par = torch.cat([sd["regressor.0." + k].reshape(1, -1) for k in ("init_pose", "init_shape", "init_cam")], 1)
    for i in range(3):
        y = F.relu(bn(F.conv_transpose2d(y, sd[f"deconv_layers.{3 * i}.weight"], None, 2, 1), f"deconv_layers.{3 * i + 1}"))
        pts = pts0[i]
        f = F.grid_sample(y, pts.unsqueeze(2), align_corners=True)[..., 0]
        z = f
        for k in range(3):
            m = f"maf_extractor.{i}.conv{k}"
            z = F.conv1d(z if k == 0 else torch.cat([z, f], 1), sd[m + ".weight"], sd[m + ".bias"])
            z = F.leaky_relu(z) if k < 2 else F.relu(z)
        xc = torch.cat([z.reshape(1, -1), par], 1)
        r = f"regressor.{i}."
        h = F.linear(F.linear(xc, sd[r + "fc1.weight"], sd[r + "fc1.bias"]), sd[r + "fc2.weight"], sd[r + "fc2.bias"])
        par = torch.cat([F.linear(h, sd[r + k + ".weight"], sd[r + k + ".bias"]) for k in ("decpose", "decshape", "deccam")],
                        1) + par
    return par


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    T = S.pymaf_tables(0)
    sd = {k: v.to(dev) for k, v in S.pymaf_state_dict(0, T).items()}
    drv = hps.PyMAFDriver(sd, [T["joint_map"]] * 3)
    x = S.pymaf_image(0).to(dev)

    def reps(fn):
        fn()
        return median([ev_ms(fn) for _ in range(a.reps)])

    res = {"eager_ms": reps(lambda: drv._forward_eager(x))}
    drv.run(x)
    drv.run(x)
    res["graph_ms"] = reps(lambda: drv.run(x))
    op, _ = drv.backbone(x)
    res["backbone_ms"] = reps(lambda: drv.backbone(x))
    ops, feats = [op], []
    for i in range(3):
        o, f = drv.deconv(i, ops[-1])
        ops.append(o)
        feats.append(f)
    res["deconv_ms"] = [reps(lambda i=i: drv.deconv(i, ops[i])) for i in range(3)]
    par = drv.init_par
    pts = [drv.grid]
    xcs, pars = [], [par]
    for i in range(3):
        xcs.append(drv.maf_row(i, feats[i], pts[i], pars[i]))
        pars.append(drv.regress(i, xcs[i], pars[i]))
        _, p = drv.tail(i, pars[-1], drv.dmap[i + 1] if i < 2 else None)
        pts.append(p)
    res["maf_ms"] = [reps(lambda i=i: drv.maf_row(i, feats[i], pts[i], pars[i])) for i in range(3)]
    res["regressor_ms"] = [reps(lambda i=i: drv.regress(i, xcs[i], pars[i])) for i in range(3)]
    res["tail_ms"] = [reps(lambda: drv.tail(0, drv.init_par))] + [
        reps(lambda i=i: drv.tail(i, pars[i + 1], drv.dmap[i + 1] if i < 2 else None)) for i in range(3)]
    pts0 = [p.t().unsqueeze(0).contiguous() for p in pts[:3]]
    with torch.no_grad():
        res["stock_torch_fp32_ms"] = reps(lambda: stock(sd, x, pts0))
    res["gpu"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
