"""Body preparation and the brick lists of the dense SDF path: SmplBody construction time on the 13,776-face body and a
68k-face one, brick-list build cost, list size, and sdf_only with the path on / off (alternating).

    python tools/time_sdf_bricks.py [--reps 5]

Prints one JSON line.  All times are CUDA-event times of sdf_only (binning + sort + SDF) on the synthetic body.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from icon_b200 import ops, synthetic as S  # noqa: E402

EYE = torch.eye(4)[None]


def body_arrays(dev, seed=0, **mesh):
    v, f = S.body_mesh(seed=seed, **mesh)
    cm, vi = S.body_attributes(v, seed=seed)
    return [torch.from_numpy(a)[None].to(dev) for a in (v, f, cm, vi)]


def body(dev, seed=0):
    return ops.SmplBody(*body_arrays(dev, seed))


def ms(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(dev)}
    ops.set_sdf_policy(32)
    ops.set_sdf_bricks(True)
    out["prepare_ms"] = {}
    for name, mesh in (("faces_13776", {}), ("faces_68k", {"rings": 200, "segs": 170})):
        arrs = body_arrays(dev, 0, **mesh)
        ms(lambda: ops.SmplBody(*arrs), 2)                                  # warm-up
        t = [ms(lambda: ops.SmplBody(*arrs)) for _ in range(4 * args.reps)]
        out["prepare_ms"][name] = {"F": int(arrs[1].shape[1]), "median": median(t), "min": min(t), "max": max(t)}
    tiny = S.lattice_points(4).permute(0, 2, 1).contiguous().to(dev)       # 64 points: the call is the build
    builds = []
    for seed in range(args.reps + 1):
        b = body(dev, seed)
        torch.cuda.synchronize()
        first = ms(lambda: ops.sdf_only(tiny, EYE, b))
        again = ms(lambda: ops.sdf_only(tiny, EYE, b), 3)
        if seed:                                                            # seed 0 warms the kernels up
            builds.append(first - again)
    info = ops.sdf_brick_info(b)
    out["build_ms"] = {"median": median(builds), "min": min(builds), "max": max(builds)}
    # a face-list entry is a uint16 face position and a float key
    out["lists"] = {"entries": info["entries"], "list_bytes": 6 * info["entries"], "overflow": info["overflow"],
                    "workspace_bytes": int(b.ws.numel())}
    ops.set_sdf_policy(0)
    b = body(dev, 0)
    for res in (256, 512):
        pts = S.lattice_points(res).permute(0, 2, 1).contiguous().to(dev)
        if res == 256:                                                      # fresh body: build + one call, honestly
            fresh = body(dev, 100)
            torch.cuda.synchronize()
            out["fresh_body_build_plus_call_256_ms"] = ms(lambda: ops.sdf_only(pts, EYE, fresh))
            del fresh
        t = {True: [], False: []}
        for on in (True, False):
            ops.set_sdf_bricks(on)
            ms(lambda: ops.sdf_only(pts, EYE, b), 2)
        for _ in range(args.reps):
            for on in (True, False):
                ops.set_sdf_bricks(on)
                t[on].append(ms(lambda: ops.sdf_only(pts, EYE, b), 3))
        out[f"sdf_only_{res}"] = {k: {"median": median(v), "min": min(v), "max": max(v)}
                                  for k, v in (("bricks_on", t[True]), ("bricks_off", t[False]))}
        del pts
        torch.cuda.empty_cache()
    ops.set_sdf_bricks(True)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
