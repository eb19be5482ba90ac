"""CPU restatement of csrc/mesh_priors.cu and icon_area_vertex_normals_backward -- TEST INFRASTRUCTURE ONLY.

The topology in NumPy; the three shape priors, LocalAffine and the area-weighted vertex normals as float64 torch ops,
with torch.autograd for the gradients.  Each term reads its own gathered copy of the vertices it uses (a leaf per
term), so one backward gives each term's contribution to each vertex: their sum is the gradient and the sum of their
absolute values is m, the scale the device's error is measured against.  The rules restated are the .cu header's;
pytorch3d is not a dependency, so they are unpinned against pytorch3d.
"""
import numpy as np
import torch
import torch.nn.functional as F

COLS = ((1, 2), (2, 0), (0, 1))            # face_to_edge columns e12, e20, e01


class Topology:
    pass


def _csr(own, key, rows):
    order = np.lexsort((key, own))
    off = np.zeros(rows + 1, np.int64)
    off[1:] = np.cumsum(np.bincount(own, minlength=rows))
    return off, key[order]


def topology(faces, V):
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) and (f.min() < 0 or f.max() >= V):
        raise ValueError("face index outside [0, V)")
    pr = np.sort(np.stack([np.stack([f[:, a], f[:, b]], -1) for a, b in COLS], 1), axis=-1)     # [F,3,2]
    edges, inv = np.unique(pr.reshape(-1, 2), axis=0, return_inverse=True)
    t = Topology()
    t.V, t.F, t.E = V, len(f), len(edges)
    t.faces, t.edges, t.face_to_edge = f, edges, inv.reshape(-1, 3)
    t.vert_off, t.vert_edges = _csr(edges.reshape(-1), np.repeat(np.arange(t.E), 2), V)
    t.edge_off, t.edge_entries = _csr(t.face_to_edge.reshape(-1), np.arange(3 * t.F), t.E)
    t.corner_off, t.vert_corners = _csr(f.reshape(-1), np.arange(3 * t.F), V)
    t.degree = np.diff(t.vert_off)
    a, b = [], []
    for e in range(t.E):
        ent = t.edge_entries[t.edge_off[e]:t.edge_off[e + 1]]
        for i in range(len(ent)):
            for j in range(i + 1, len(ent)):
                a.append(ent[i])
                b.append(ent[j])
    t.pairs = np.array([a, b], np.int64).reshape(2, -1).T          # [P,2] entries, per edge ascending
    return t


def edges_unique(faces):
    """pytorch3d's edges_packed restated with torch.unique (a second, independent construction)."""
    f = torch.as_tensor(np.asarray(faces, np.int64))
    e = torch.cat([f[:, [1, 2]], f[:, [2, 0]], f[:, [0, 1]]], 0)
    e, _ = e.sort(dim=1)
    return torch.unique(e, dim=0).numpy()


def _leaf(v, ids):
    return v[torch.as_tensor(ids)].detach().clone().requires_grad_(True)


def _scatter(V, ids, g):
    ids = torch.as_tensor(np.asarray(ids)).reshape(-1)
    g = g.reshape(-1, 3)
    return (torch.zeros(V, 3, dtype=g.dtype).index_add_(0, ids, g),
            torch.zeros(V, 3, dtype=g.dtype).index_add_(0, ids, g.abs()))


def entry_normals(X):
    """n of entries from gathered rows X [..., 5, 3] = (v0, v1, f0, f1, f2)."""
    u = X[..., 1, :] - X[..., 0, :]
    n = torch.zeros_like(u)
    for k in range(3):
        n = n + torch.cross(u, X[..., 2 + k, :] - X[..., 0, :], dim=-1)
    return n


def priors(verts, t, g=(1.0, 1.0, 1.0)):
    """-> values (edge, nc, lap) as floats, and per term (grad [V,3], m [V,3]) for upstream gradients g (None: no
    gradient for that term).  verts: float64 [V,3] (array or tensor)."""
    v = torch.as_tensor(np.asarray(verts), dtype=torch.float64)
    V, E = t.V, t.E
    out, grads = [], []
    # edge
    va, vb = _leaf(v, t.edges[:, 0]), _leaf(v, t.edges[:, 1])
    L = (va - vb).norm(dim=1)
    edge = ((L - 0.0) ** 2).sum() / E
    out.append(edge)
    # nc
    if len(t.pairs):
        ids = []
        for k in range(2):
            ent = t.pairs[:, k]
            e = t.face_to_edge.reshape(-1)[ent]
            ids.append(np.concatenate([t.edges[e], t.faces[ent // 3]], 1))
        ids = np.stack(ids, 1)                                          # [P,2,5]
        X = _leaf(v, ids)
        n = entry_normals(X)
        nc = (1.0 - F.cosine_similarity(n[:, 0], -n[:, 1], dim=1, eps=1e-8)).sum() / len(t.pairs)
    else:
        ids, X, nc = None, None, torch.zeros((), dtype=torch.float64)
    out.append(nc)
    # lap
    own = np.repeat(np.arange(V), t.degree)
    e = t.vert_edges
    other = np.where(t.edges[e, 0] == own, t.edges[e, 1], t.edges[e, 0])
    nb, vi = _leaf(v, other), v.detach().clone().requires_grad_(True)
    deg = torch.as_tensor(t.degree, dtype=torch.float64)
    ell = torch.zeros(V, 3, dtype=torch.float64).index_add(0, torch.as_tensor(own),
                                                          nb / deg[torch.as_tensor(own)][:, None]) - vi
    lap = ell.norm(dim=1).sum() / V
    out.append(lap)
    total = sum(o * gi for o, gi in zip(out, g) if gi is not None and o.requires_grad)
    if torch.is_tensor(total):
        total.backward()
    zero = torch.zeros(V, 3, dtype=torch.float64)
    grads.append(_sum2(_scatter(V, t.edges[:, 0], va.grad), _scatter(V, t.edges[:, 1], vb.grad))
                 if g[0] is not None else (zero, zero))
    grads.append(_scatter(V, ids, X.grad) if g[1] is not None and X is not None and X.grad is not None
                 else (zero, zero))
    grads.append(_sum2(_scatter(V, other, nb.grad), (vi.grad, vi.grad.abs())) if g[2] is not None else (zero, zero))
    values = [float(o.detach()) for o in out]
    return values, grads


def _sum2(p, q):
    return p[0] + q[0], p[1] + q[1]


def cos_grad_example():
    """d cos / dx at x = y = [1e-9, 0, 0], eps 1e-8: the unclamped norm carries the gradient (9e6)."""
    x = torch.tensor([[1e-9, 0.0, 0.0]], dtype=torch.float64, requires_grad=True)
    F.cosine_similarity(x, torch.tensor([[1e-9, 0.0, 0.0]], dtype=torch.float64), dim=1, eps=1e-8).sum().backward()
    return x.grad[0].numpy()


def local_affine(A, b, x, edges, g_out=None, g_diff=None, g_rigid=None):
    """A [N,3,3], b [N,3], x [N,3], edges [E,2] -> (out, w_diff [E,3,4], w_rigid [N]) and, for the given upstream
    gradients, ((grad_A, m_A), (grad_b, m_b), (grad_x, m_x))."""
    A, b, x = (torch.as_tensor(np.asarray(z), dtype=torch.float64) for z in (A, b, x))
    N = A.shape[0]
    edges = np.asarray(edges, np.int64).reshape(-1, 2)
    A1, b1, x1 = (z.clone().requires_grad_(True) for z in (A, b, x))
    out = (A1 @ x1[..., None])[..., 0] + b1
    W = torch.cat([A, b[..., None]], 2)
    Wi, Wj = _leaf(W, edges[:, 0]), _leaf(W, edges[:, 1])
    w_diff = (Wi - Wj) ** 2
    A2 = A.clone().requires_grad_(True)
    a = A2.reshape(N, 9)
    C0 = a[:, 4] * a[:, 8] - a[:, 5] * a[:, 7]
    C1 = -(a[:, 3] * a[:, 8] - a[:, 5] * a[:, 6])
    C2 = a[:, 3] * a[:, 7] - a[:, 4] * a[:, 6]
    det = (a[:, 0] * C0 + a[:, 1] * C1) + a[:, 2] * C2
    w_rigid = (det - 1.0) ** 2
    vals = (out.detach().numpy(), w_diff.detach().numpy(), w_rigid.detach().numpy())
    total = 0
    for val, gg in ((out, g_out), (w_diff, g_diff), (w_rigid, g_rigid)):
        if gg is not None:
            total = total + (val * torch.as_tensor(np.asarray(gg), dtype=torch.float64).reshape(val.shape)).sum()
    if not torch.is_tensor(total):
        return vals, None
    total.backward()
    z9, z3 = torch.zeros(N, 3, 3, dtype=torch.float64), torch.zeros(N, 3, dtype=torch.float64)

    def grad_or(t, z):
        return t.grad if t.grad is not None else z
    gW = torch.zeros(N, 3, 4, dtype=torch.float64)
    mW = torch.zeros(N, 3, 4, dtype=torch.float64)
    if g_diff is not None:
        for idx, leaf in ((edges[:, 0], Wi), (edges[:, 1], Wj)):
            gW.index_add_(0, torch.as_tensor(idx), leaf.grad)
            mW.index_add_(0, torch.as_tensor(idx), leaf.grad.abs())
    gA1, gb1, gA2 = grad_or(A1, z9), grad_or(b1, z3), grad_or(A2, z9)
    grad_A = gA1 + gW[..., :3] + gA2
    m_A = gA1.abs() + mW[..., :3] + gA2.abs()
    grad_b, m_b = gb1 + gW[..., 3], gb1.abs() + mW[..., 3]
    if g_out is not None:
        go = torch.as_tensor(np.asarray(g_out), dtype=torch.float64).reshape(N, 3)
        m_x = (A.abs() * go.abs()[..., None]).sum(1)
    else:
        m_x = z3
    return vals, ((grad_A.numpy(), m_A.numpy()), (grad_b.numpy(), m_b.numpy()),
                  (grad_or(x1, z3).numpy(), m_x.numpy()))


def vertex_normals(verts, faces, g=None):
    """F.normalize(sum of corner products, eps 1e-6) per vertex (float64) and, for upstream g [V,3], (grad, m)."""
    v = torch.as_tensor(np.asarray(verts), dtype=torch.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    V = v.shape[0]
    ids = np.stack([f[:, [c, (c + 1) % 3, (c + 2) % 3]] for c in range(3)], 1).reshape(-1, 3)   # per corner entry
    X = _leaf(v, ids)
    prod = torch.cross(X[:, 1] - X[:, 0], X[:, 2] - X[:, 0], dim=-1)
    s = torch.zeros(V, 3, dtype=torch.float64).index_add(0, torch.as_tensor(ids[:, 0]), prod)
    n = F.normalize(s, eps=1e-6, dim=1)
    if g is None:
        return n.detach().numpy(), None
    (n * torch.as_tensor(np.asarray(g), dtype=torch.float64)).sum().backward()
    grad, m = _scatter(V, ids, X.grad)
    return n.detach().numpy(), (grad.numpy(), m.numpy())
