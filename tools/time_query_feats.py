"""icon_query with each smpl_feats subset: one call on the dense 256^3 cell-centre lattice per configuration.

    python tools/time_query_feats.py [--reps 5] [--out FILE]

Configurations: the icon-filter layout (C = 12, 128^2 feature map) with the full set, {sdf, norm, vis}, {sdf, vis} and
{sdf}; icon-mvp (C = 6, 512^2 map, {sdf}).  Each is timed with CUDA events around one call, the configurations
alternating, `--reps` rounds; the median, min and max are reported.  A separate profiled pass, alternating the same
way, gives the median icon_profile_last_query stage split ([0] binning + sort, [1] SDF, [2] outlier rank, [3] gather +
MLP) and the library launches of one call.  The GPU's name, power limit and maximum SM clock are read in the same run.
Prints one JSON line.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from icon_b200 import _C, ops, synthetic as S  # noqa: E402

EYE = torch.eye(4)[None]
CONFIGS = [   # name, image channels C, map size, smpl_feats
    ("filter-full", 12, 128, ("sdf", "cmap", "norm", "vis")),
    ("filter-sdf-norm-vis", 12, 128, ("sdf", "norm", "vis")),
    ("filter-sdf-vis", 12, 128, ("sdf", "vis")),
    ("filter-sdf", 12, 128, ("sdf",)),
    ("mvp-sdf", 6, 512, ("sdf",)),
]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except (OSError, subprocess.SubprocessError, IndexError):
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: power limit unknown)"


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    ops.set_mlp_impl("tcgen05")
    v, f = S.body_mesh(seed=0)
    cm, vi = S.body_attributes(v, seed=0)
    body = ops.SmplBody(*(torch.from_numpy(a)[None].to(dev) for a in (v, f, cm, vi)))
    pts = S.lattice_points(args.grid).permute(0, 2, 1).contiguous().to(dev)
    N = pts.shape[2]
    out = torch.empty(1, 1, N, device=dev)
    calls = {}
    for name, C, size, feats in CONFIGS:
        c0 = ops.icon_c0(feats, C)
        feat = S.feature_map(C, size, seed=1).to(dev)
        mlp = ops.pack_mlp(S.mlp_state_dict(c0=c0, seed=2), c0, device=dev)
        calls[name] = (lambda feat=feat, mlp=mlp, feats=feats:
                       ops.query("icon", pts, EYE, feat, mlp, body=body, sdf_clip=0.05, out=out, smpl_feats=feats))

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def ms(fn):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for fn in calls.values():             # warm-up: module loads, the body's brick lists
        fn(); fn()
    torch.cuda.synchronize()
    times = {name: [] for name in calls}
    for _ in range(args.reps):
        for name, fn in calls.items():
            times[name].append(ms(fn))

    buf = (ctypes.c_float * 4)()
    stages = {name: [] for name in calls}
    launches = {}
    _C.lib.icon_profile_enable(1)
    for _ in range(args.reps):
        for name, fn in calls.items():
            l0 = _C.launch_count()
            fn()
            _C.check(_C.lib.icon_profile_last_query(buf), "icon_profile_last_query")
            launches[name] = _C.launch_count() - l0
            stages[name].append([buf[i] for i in range(4)])
    _C.lib.icon_profile_enable(0)

    res = {"gpu": gpu_info(), "points": N, "reps": args.reps, "configs": {}}
    for name, C, size, feats in CONFIGS:
        t = sorted(times[name])
        split = [median([s[i] for s in stages[name]]) for i in range(4)]
        res["configs"][name] = {
            "C": C, "map": size, "smpl_feats": list(feats), "c0": ops.icon_c0(feats, C),
            "ms": {"median": t[len(t) // 2], "min": t[0], "max": t[-1]},
            "Mpoints_per_s": N / t[len(t) // 2] / 1e3,
            "stages_ms_median": [round(v, 4) for v in split],
            "launches": launches[name],
        }
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
