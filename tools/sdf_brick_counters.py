"""Per-warp counters of the dense SDF block's brick path (sdf.cu, DESIGN.md 4.2).

    python tools/sdf_brick_counters.py --out DIR [--res 256]

Builds a diagnostics copy of the library into DIR (sdf.cu with -DICON_SDF_STATS, the other objects as
icon_b200/build.py left them; the product build is not touched), runs sdf_only once on the synthetic body (seed 0)
and the res^3 cell-centre lattice, and prints one JSON line: per brick-path warp, the median / p90 / p99 and the
mean of each counter, and the cycle-weighted mean (warps weighted by their total cycles).  Also reports ptxas
registers and spills of both dense instantiations as the product build compiles them.  DIR/warps.npz keeps the raw
records.  The counters' own stores and the scan behind ideal_entries / ideal_faces (what the break and bounding sphere
alone keep at the final bound) run outside the timed segments, but the clocks are those of a build that also counts,
so use them as shares, not as the product kernel's time.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# record layout of sdf.cu (WS_* enum)
FIELDS = ["defer", "entries", "steps", "staged", "sph_pass", "exact", "win", "ray", "cyc_start", "cyc_c", "cyc_ray",
          "cyc_emit", "ub0", "ub_end", "list_len", "ideal_entries", "ideal_faces", "dead_staged"]
WS_N = 20
FLOAT_FIELDS = ("ub0", "ub_end")
PER_LANE = ("sph_pass", "exact", "win", "ray")      # summed over the 32 lanes in the record


def build_stats_lib(out):
    from icon_b200 import build as B
    B.build()
    os.makedirs(out, exist_ok=True)
    src = os.path.join(B.CSRC, "sdf.cu")
    obj = os.path.join(out, "sdf_stats.o")
    subprocess.check_call(["nvcc", "-c", src, "-o", obj, "-DICON_SDF_STATS"] + B.ARCH + B.COMMON
                          + B.SOURCES["sdf.cu"])
    objs = [obj if s == "sdf.cu" else os.path.join(B.OBJ, s.replace(".cu", ".o")) for s in B.SOURCES]
    lib = os.path.join(out, "libicon_b200_stats.so")
    subprocess.check_call(["nvcc", "-shared", "-o", lib] + objs + B.ARCH + ["-lcudart"])
    # registers / spills of the product instantiations
    r = subprocess.run(["nvcc", "-c", src, "-o", os.path.join(out, "sdf_ptxas.o"), "-Xptxas", "-v"] + B.ARCH
                       + B.COMMON + B.SOURCES["sdf.cu"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    ptxas, fn = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"Used (\d+) registers", line)
        if fn and m and "k_sdf_warp" in fn and ("ILi32ELb1E" in fn or "ILi32ELb0E" in fn):
            name = "k_sdf_warp<32,true>" if "ILi32ELb1E" in fn else "k_sdf_warp<32,false>"
            ptxas.setdefault(name, {})["registers"] = int(m.group(1))
        m = re.search(r"(\d+) bytes spill stores", line)
        if fn and m and "k_sdf_warp" in fn and ("ILi32ELb1E" in fn or "ILi32ELb0E" in fn):
            name = "k_sdf_warp<32,true>" if "ILi32ELb1E" in fn else "k_sdf_warp<32,false>"
            ptxas.setdefault(name, {})["spill_store_bytes"] = int(m.group(1))
    for v in ptxas.values():   # 128-thread blocks, 64 K registers and 64 warps per SM
        regs = v.get("registers", 255)
        v["resident_warps_per_sm_by_registers"] = min(64, 4 * (65536 // (regs * 128)))
    return lib, ptxas


def measure(out, res):
    import ctypes
    import numpy as np
    import torch
    from icon_b200 import _C, ops, synthetic as S
    lib = _C.lib
    lib.icon_debug_sdf_warp_stats.argtypes = [ctypes.c_void_p]
    lib.icon_debug_sdf_stats.argtypes = [ctypes.c_void_p, ctypes.c_int]
    dev = torch.device("cuda:0")
    v, f = S.body_mesh(seed=0)
    cm, vi = S.body_attributes(v, seed=0)
    body = ops.SmplBody(*(torch.from_numpy(a)[None].to(dev) for a in (v, f, cm, vi)))
    pts = S.lattice_points(res).permute(0, 2, 1).contiguous().to(dev)
    eye = torch.eye(4)[None]
    ops.set_sdf_policy(32)
    ops.set_sdf_bricks(True)
    ops.sdf_only(pts, eye, body)                      # builds the lists
    torch.cuda.synchronize()
    nw = (pts.shape[2] + 31) // 32
    rec = torch.zeros(nw * WS_N, dtype=torch.int32, device=dev)
    g = (ctypes.c_ulonglong * 8)()
    lib.icon_debug_sdf_stats(ctypes.addressof(g), 1)
    lib.icon_debug_sdf_warp_stats(rec.data_ptr())
    ops.sdf_only(pts, eye, body)
    torch.cuda.synchronize()
    lib.icon_debug_sdf_warp_stats(None)
    lib.icon_debug_sdf_stats(ctypes.addressof(g), 1)
    ops.set_sdf_policy(0)
    r = rec.view(nw, WS_N).cpu().numpy()[:, :len(FIELDS)]
    cols = {}
    for i, k in enumerate(FIELDS):
        c = r[:, i].copy()
        cols[k] = c.view(np.float32).astype(np.float64) if k in FLOAT_FIELDS else c.view(np.uint32).astype(np.float64)
    np.savez_compressed(os.path.join(out, "warps.npz"), **cols)
    brick = cols["defer"] == 0
    cyc = cols["cyc_start"] + cols["cyc_c"] + cols["cyc_ray"] + cols["cyc_emit"]
    cols["cyc_total"] = cyc
    w = cyc[brick] / cyc[brick].sum()
    table = {}
    for k, c in cols.items():
        if k == "defer":
            continue
        x = c[brick] / (32.0 if k in PER_LANE else 1.0)
        table[k + ("_per_lane" if k in PER_LANE else "")] = {
            "median": float(np.median(x)), "p90": float(np.percentile(x, 90)), "p99": float(np.percentile(x, 99)),
            "mean": float(x.mean()), "cycle_weighted": float((x * w).sum())}
    tc = cols["cyc_start"][brick].sum() + cols["cyc_c"][brick].sum() + cols["cyc_ray"][brick].sum() \
        + cols["cyc_emit"][brick].sum()
    return {"gpu": torch.cuda.get_device_name(dev), "res": res, "warps": int(nw),
            "brick_warps": int(brick.sum()), "deferred_warps": int(g[4]),
            "deferred_walk_cycles_mean": float(g[5]) / max(1, int(g[4])),
            "cycle_share": {k: float(cols[k][brick].sum() / tc) for k in ("cyc_start", "cyc_c", "cyc_ray", "cyc_emit")},
            "per_warp": table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--measure", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    out = os.path.abspath(args.out)
    if args.measure:
        print(json.dumps(measure(out, args.res)), flush=True)
        return
    lib, ptxas = build_stats_lib(out)
    env = dict(os.environ, ICON_B200_LIB=lib)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--out", out, "--res", str(args.res), "--measure"],
                       env=env, stdout=subprocess.PIPE, text=True, check=True)
    res = json.loads(r.stdout.strip().splitlines()[-1])
    res["ptxas"] = ptxas
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
