"""clean_mesh on a 513^3 marching-cubes surface (about 10^6 vertices, three components), CUDA events.

Each repetition times one clean_mesh_device call (count + emit, including its workspace allocation and the
device-to-host read of the kept counts); the median of 5 rounds of 20 calls is printed."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from icon_b200 import mesh, ops
dev = torch.device("cuda:0")
R = 513
a = torch.linspace(-1, 1, R, device=dev)
z, y, x = torch.meshgrid(a, a, a, indexing="ij")
occ = 0.5 + 2.0 * (0.8 - ((x / 1.12) ** 2 + (y / 1.16) ** 2 + (z / 1.08) ** 2).sqrt())
occ = torch.maximum(occ, 0.5 + 2.0 * (0.05 - ((x - 0.9) ** 2 + (y - 0.9) ** 2 + (z - 0.9) ** 2).sqrt()))
occ = torch.maximum(occ, 0.5 + 2.0 * (0.05 - ((x + 0.9) ** 2 + (y + 0.9) ** 2 + (z - 0.9) ** 2).sqrt()))
del x, y, z
v, f = ops.marching_cubes(occ.float().contiguous(), 0.5)
del occ
for _ in range(3):
    cv, cf = mesh.clean_mesh_device(v, f)
rounds = []
for _ in range(5):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        cv, cf = mesh.clean_mesh_device(v, f)
    e1.record(); torch.cuda.synchronize()
    rounds.append(e0.elapsed_time(e1) / 20)
rounds.sort()
print(f"clean_mesh 513^3 surface, V={len(v)} F={len(f)} -> kept V={len(cv)} F={len(cf)}: median {rounds[2]:.3f} ms "
      f"(rounds {', '.join(f'{r:.3f}' for r in rounds)})")
