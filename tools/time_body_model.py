"""The body-fit loop's body model (apps/infer.py:175-180: lbs() through SMPL.forward), B = 1, at SMPL's and SMPL-X's
sizes (icon_b200.synthetic.body_model "smpl": V 6890, J 24, NB 10; "smplx": V 10475, J 55, NB 20), and PIXIE's SMPL-X
(apps/infer.py:184-197 with -hps_type pixie: SMPLX.forward, the skinning plus the landmark and joint heads) at the real
size ("pixie": icon_b200.synthetic.pixie_model "real", V 10475, F 20908, J 55, NB 200 + 50).

    python tools/time_body_model.py [--reps 50] [--out results/time_body_model.json]

Prints one JSON line.  Per size:
  fwd / bwd / fwd_bwd   CUDA-event medians (ms) of the kernels: icon_lbs_forward, icon_lbs_backward, and a forward
                        plus backward through the autograd Function;
  wall_kernels          wall-clock per iteration (ms) of forward + backward with the kernels, host included (a device
                        synchronise ends each timed window of `reps` iterations);
  wall_eager            the same for an fp32 stock-torch eager restatement of lbs() with autograd (the reference's
                        sequence of ops, written here; it is a restatement, not the reference's own code).
For "pixie", fwd / bwd / fwd_bwd time the whole forward (the two torch.cats, the skinning and the heads) and the
backward with an upstream on all three outputs, wall_eager an fp32 torch restatement of PIXIE's SMPLX.forward
(eager_pixie, written here); skin_bwd_nb250 is icon_lbs_backward alone at NB = 250 and heads_bwd the heads' backward
alone.  Without an ICON checkout, the "pixie" row runs on synthetic.pixie_smplx_standin(): a module with the
class's buffers whose `forward` make_pixie_SMPLX patches, as the overlay patches the reference's class.  The GPU's
name and power limit are part of the result.
"""
import argparse
import ctypes
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from icon_b200 import body_model as BM, synthetic as S  # noqa: E402
from icon_b200.ops import _p, _stream  # noqa: E402
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


def eager_pixie(betas, pose, model, par_host, heads):
    """fp32 torch restatement of PIXIE's SMPLX.forward after its torch.cats: eager_lbs, the head-yaw lookup row (a
    Python loop of 3x3 matmuls, atan2, round, masks, index_select), the landmarks, the extra joints and the J14
    regressor written over its joints through detach() * 0 + reg."""
    B = pose.shape[0]
    verts, jt = eager_lbs(betas, pose, model[0], model[1], model[2], model[3], par_host, model[5])
    f = heads["faces_tensor"]
    rot = torch.index_select(pose.detach(), 1, heads["head_kin_chain"])
    rel = torch.eye(3, device=pose.device, dtype=pose.dtype).unsqueeze(0)
    for i in range(rot.shape[1]):
        rel = torch.matmul(rot[:, i], rel)
    sy = torch.sqrt(rel[:, 0, 0] * rel[:, 0, 0] + rel[:, 1, 0] * rel[:, 1, 0])
    y = torch.round(torch.clamp(-torch.atan2(-rel[:, 2, 0], sy) * 180.0 / 3.141592653589793, max=39)).long()
    neg, low = y.lt(0).long(), y.lt(-39).long()
    y = neg * (low * 78 + (1 - low) * (39 - y)) + (1 - neg) * y
    lf = torch.cat([heads["lmk_faces_idx"][None].expand(B, -1), heads["dynamic_lmk_faces_idx"][y]], 1)
    lb = torch.cat([heads["lmk_bary_coords"][None].expand(B, -1, -1), heads["dynamic_lmk_bary_coords"][y]], 1)
    lv = verts.reshape(-1, 3)[f[lf.reshape(-1)].view(B, -1, 3) + torch.arange(B, device=pose.device).view(-1, 1, 1)
                                                                * verts.shape[1]].view(B, -1, 3, 3)
    lm = torch.einsum("blfi,blf->bli", lv, lb)
    tri = torch.index_select(verts, 1, f[heads["face_ids"]].reshape(-1)).reshape(B, -1, 3, 3)
    extra = (tri * heads["bcs"][None, :, :, None]).sum(2)
    joints = torch.cat([jt, lm, extra], 1)
    reg = torch.einsum("ji,bik->bjk", heads["extra_joint_regressor"], verts)
    src, tgt = heads["source_idxs"], heads["target_idxs"]
    joints[:, src] = joints[:, src].detach() * 0.0 + reg[:, tgt] * 1.0
    return verts, lm, joints


def time_pixie(reps, dev):
    import numpy as np
    from oracle.body_model import rodrigues
    from icon_b200 import _C
    arr = S.pixie_model("real", 0)
    buf = {k: torch.from_numpy(np.asarray(v)) for k, v in S.pixie_buffers(arr).items()}
    SMPLX = BM.make_pixie_SMPLX(S.pixie_smplx_standin())      # PIXIE SMPLX's buffers, its forward patched
    mod = SMPLX(buf, arr["n_shape"]).to(dev)
    g = torch.Generator().manual_seed(2)
    R = torch.from_numpy(rodrigues((0.3 * torch.randn(1, 55, 3, generator=g)).double().numpy())[0]).float().to(dev)
    leaf = lambda x: x.clone().requires_grad_(True)  # noqa: E731
    args = dict(shape_params=leaf((0.5 * torch.randn(1, 200, generator=g)).to(dev)),
                expression_params=leaf((0.5 * torch.randn(1, 50, generator=g)).to(dev)), global_pose=leaf(R[:, :1]),
                body_pose=leaf(R[:, 1:22]), jaw_pose=leaf(R[:, 22:23]), left_hand_pose=leaf(R[:, 25:40]),
                right_hand_pose=leaf(R[:, 40:]))
    ups = [torch.randn(1, 10475, 3, generator=g).to(dev), torch.randn(1, 68, 3, generator=g).to(dev),
           torch.randn(1, 145, 3, generator=g).to(dev)]
    model = [getattr(mod, k) for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "parents",
                                       "lbs_weights")]
    heads = {k: buf[k].to(dev) for k in buf}
    par_host = [int(p) for p in arr["kintree_table"][0]]

    def full_args():
        eye = mod.eye_pose.unsqueeze(0).expand(1, -1, -1, -1)
        return (torch.cat([args["shape_params"], args["expression_params"]], 1),
                torch.cat([args["global_pose"], args["body_pose"], args["jaw_pose"], eye, args["left_hand_pose"],
                           args["right_hand_pose"]], 1))

    def kernels():
        torch.autograd.backward(list(mod(**args)), ups)

    def eager():
        torch.autograd.backward(list(eager_pixie(*full_args(), model, par_host, heads)), ups)

    saved = {}

    def fwd():
        saved["out"] = mod(**args)

    def bwd():
        torch.autograd.backward(list(saved["out"]), ups)

    res = {"V": 10475, "F": 20908, "J": 55, "NB": 250, "B": 1}
    for _ in range(5):
        kernels()
        eager()
    f, b = [], []
    for _ in range(reps):
        f.append(ev_ms(fwd))
        b.append(ev_ms(bwd))
    res["fwd"], res["bwd"] = round(median(f), 4), round(median(b), 4)
    res["fwd_bwd"] = round(median([ev_ms(kernels) for _ in range(reps)]), 4)
    res["wall_kernels"] = round(median([wall(kernels, reps) for _ in range(5)]), 4)
    res["wall_eager"] = round(median([wall(eager, reps) for _ in range(5)]), 4)
    # the NB = 250 skin backward and the heads' backward, each alone
    sc, fp = full_args()
    pm = BM.prepared(*model)
    hd = BM.prepared_heads(mod)
    st = {}

    def lbs_fwd():
        st["vj"] = BM._Lbs.apply(sc.detach().requires_grad_(True), fp.detach().requires_grad_(True), pm, False)

    def lbs_bwd():
        torch.autograd.backward([st["vj"][0]], [ups[0]])
    sk = []
    for _ in range(reps):
        lbs_fwd()
        sk.append(ev_ms(lbs_bwd))
    res["skin_bwd_nb250"] = round(median(sk), 4)
    rows = torch.zeros(1, dtype=torch.int32, device=dev)
    gv = torch.empty(1, 10475, 3, device=dev)
    gjt = torch.empty(1, 55, 3, device=dev)

    def heads_bwd():
        _C.check(_C.lib.icon_smplx_heads_backward(ctypes.byref(hd.c), 1, _p(rows), _p(ups[1]), _p(ups[2]), _p(gv),
                                                   _p(gjt), _stream()), "icon_smplx_heads_backward")
    for _ in range(5):
        heads_bwd()
    res["heads_bwd"] = round(median([ev_ms(heads_bwd) for _ in range(reps)]), 4)
    with torch.no_grad():
        k_out = mod(**args)
        e_out = eager_pixie(*full_args(), model, par_host, heads)
    res["max_abs_diff_vs_eager"] = float(max((a - b).abs().max() for a, b in zip(k_out, e_out)))
    return res


def wall(fn, reps):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


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
    res["pixie"] = time_pixie(args.reps, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
