"""The body-fit loop's body model (apps/infer.py:175-180: lbs() through SMPL.forward), B = 1, at SMPL's and SMPL-X's
sizes (icon_b200.synthetic.body_model "smpl": V 6890, J 24, NB 10; "smplx": V 10475, J 55, NB 20).

    python tools/time_body_model.py [--reps 50] [--out results/time_body_model.json]

Prints one JSON line.  Per size:
  fwd / bwd / fwd_bwd   CUDA-event medians (ms) of the kernels: icon_lbs_forward, icon_lbs_backward, and a forward
                        plus backward through the autograd Function;
  wall_kernels          wall-clock per iteration (ms) of forward + backward with the kernels, host included (a device
                        synchronise ends each timed window of `reps` iterations);
  wall_eager            the same for an fp32 stock-torch eager restatement of lbs() with autograd (the reference's
                        sequence of ops, written here; it is a restatement, not the reference's own code).
The GPU's name and power limit are part of the result.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from icon_b200 import body_model as BM, synthetic as S  # noqa: E402
from tools.time_metrics import ev_ms, gpu_info, median  # noqa: E402


def eager_lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights):
    """fp32 torch restatement of lbs(pose2rot=False): shape blend, joint regression, pose blend, the Python chain of
    4x4 matmuls and the skinning, as separate ops."""
    B = pose.shape[0]
    ident = torch.eye(3, dtype=pose.dtype, device=pose.device)
    v_shaped = v_template + torch.einsum("bl,mkl->bmk", betas, shapedirs)
    J = torch.einsum("bik,ji->bjk", v_shaped, J_regressor)
    rot = pose.view(B, -1, 3, 3)
    pose_feature = (rot[:, 1:] - ident).view(B, -1)
    v_posed = v_shaped + torch.matmul(pose_feature, posedirs).view(B, -1, 3)
    joints = J.unsqueeze(-1)
    rel = joints.clone()
    rel[:, 1:] -= joints[:, parents[1:]]
    tm = torch.cat([F.pad(rot.reshape(-1, 3, 3), [0, 0, 0, 1]), F.pad(rel.reshape(-1, 3, 1), [0, 0, 0, 1], value=1)],
                   2).reshape(B, -1, 4, 4)
    chain = [tm[:, 0]]
    for i in range(1, len(parents)):
        chain.append(torch.matmul(chain[parents[i]], tm[:, i]))
    G = torch.stack(chain, 1)
    posed = G[:, :, :3, 3]
    A = G - F.pad(torch.matmul(G, F.pad(joints, [0, 0, 0, 1])), [3, 0, 0, 0, 0, 0, 0, 0])
    T = torch.matmul(lbs_weights.unsqueeze(0).expand(B, -1, -1), A.view(B, -1, 16)).view(B, -1, 4, 4)
    vh = torch.cat([v_posed, torch.ones_like(v_posed[..., :1])], 2)
    return torch.matmul(T, vh.unsqueeze(-1))[:, :, :3, 0], posed


def time_size(kind, reps, dev):
    m = S.body_model(kind, 0)
    names = ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights")
    model = [torch.from_numpy(m[k]).to(dev) for k in names]
    J, NB = len(m["parents"]), m["shapedirs"].shape[2]
    g = torch.Generator().manual_seed(1)
    betas = (0.5 * torch.randn(1, NB, generator=g)).to(dev).requires_grad_(True)
    from oracle.body_model import rodrigues
    R = rodrigues((0.3 * torch.randn(1, J, 3, generator=g)).double().numpy())[0]
    pose = torch.from_numpy(R).float().to(dev).requires_grad_(True)
    gv = torch.randn(1, m["v_template"].shape[0], 3, generator=g).to(dev)
    par_host = [int(p) for p in m["parents"]]

    def kernels():
        v, j = BM.lbs(betas, pose, *model, pose2rot=False)
        torch.autograd.backward([v, j], [gv, torch.zeros_like(j)])

    def eager():
        v, j = eager_lbs(betas, pose, model[0], model[1], model[2], model[3], par_host, model[5])
        torch.autograd.backward([v, j], [gv, torch.zeros_like(j)])

    pm = BM.prepared(*model)
    saved = {}

    def fwd():
        saved["out"] = BM._Lbs.apply(betas, pose, pm, False)

    def bwd():
        torch.autograd.backward(list(saved["out"]), [gv, torch.zeros_like(saved["out"][1])])

    def wall(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / reps

    res = {"V": int(m["v_template"].shape[0]), "J": J, "NB": int(NB), "B": 1}
    for _ in range(5):
        kernels()
    f, b = [], []
    for _ in range(reps):
        f.append(ev_ms(fwd))
        b.append(ev_ms(bwd))
    res["fwd"], res["bwd"] = round(median(f), 4), round(median(b), 4)
    res["fwd_bwd"] = round(median([ev_ms(kernels) for _ in range(reps)]), 4)
    res["wall_kernels"] = round(median([wall(kernels) for _ in range(5)]), 4)
    res["wall_eager"] = round(median([wall(eager) for _ in range(5)]), 4)
    with torch.no_grad():
        v1, j1 = BM.lbs(betas, pose, *model, pose2rot=False)
        v2, j2 = eager_lbs(betas, pose, model[0], model[1], model[2], model[3], par_host, model[5])
    res["max_abs_diff_vs_eager"] = float(max((v1 - v2).abs().max(), (j1 - j2).abs().max()))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_body_model.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"what": "body model lbs(), forward + backward, B = 1 (ms)", "gpu": gpu_info(), "reps": args.reps,
           "eager": "fp32 stock-torch restatement of lbs() with autograd, not the reference's code"}
    for kind in ("smpl", "smplx"):
        res[kind] = time_size(kind, args.reps, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
