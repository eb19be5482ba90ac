"""CPU restatement of the dataset renderer's views (PRTRender / ColorRender of scripts/render_single.py) -- TEST
INFRASTRUCTURE ONLY.

PARITY UNPINNED.  The reference draws with OpenGL (lib/renderer/gl/prt_render.py, color_render.py; shaders prt.vs /
prt.fs, color.vs / color.fs); GL is not a dependency of this project.  The rules are the ones written in the header
of csrc/dataset_render.cu, restated here operation for operation in float32 (one rounding per operation, in the
kernel's order; the gamma's pow and the level of detail's log2 in float64, rounded once), so the three attachments are
compared bit for bit.  The raster (1/256-pixel snapping, exact int64 edge functions, top-left rule, 24-bit GL_LESS,
lowest face on a tie) is normal_render's, evaluated at S = 1 or 16 samples per pixel.
"""
import numpy as np

F32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
RANGE = F32(65536.0)
BATCH = 1 << 21

# D3D11 standard 16-sample pattern, in 1/16 pixel from the pixel centre
PATTERN16 = np.array([[1, 1], [-1, -3], [-3, 2], [4, -1], [-5, -2], [2, 5], [5, 3], [3, -5], [-2, 6], [0, -7],
                      [-4, -6], [-6, 4], [-8, 0], [7, -4], [6, 7], [-7, -8]], np.int64)


def sample_offsets(S):
    """[S,2] sample offsets in 1/256 pixel from the pixel's corner (256 p + offset)"""
    if S == 1:
        return np.array([[128, 128]], np.int64)
    assert S == 16
    return 128 + 16 * PATTERN16


# ---------------------------------------------------------------- uniforms

def mat_mul(a, b):
    """fp32 product, entries summed left to right"""
    acc = a[:, 0:1] * b[0:1, :]
    for k in range(1, a.shape[1]):
        acc = acc + a[:, k:k + 1] * b[k:k + 1, :]
    return acc


def uniforms(normalize_matrix, rot_matrix, model_view, projection, sh):
    N = np.asarray(normalize_matrix, np.float64).astype(F32)
    Rm = np.asarray(rot_matrix, np.float64).astype(F32)
    M = np.asarray(model_view, np.float64).astype(F32)
    P = np.asarray(projection, np.float64).astype(F32)
    assert np.array_equal(P[3], np.array([0, 0, 0, 1], F32)), "orthographic only"
    return dict(N=N, Rot=Rm, MP=mat_mul(P, M), R=mat_mul(M[:3, :3], Rm), SH=np.asarray(sh, np.float64).astype(F32))


# ---------------------------------------------------------------- PRT band rotation (GLSL indexing, copy-in)

def band1(x, R):
    """OptRotateBand1 with GLSL R[i][j] = R_rowmajor[j][i]; x [...,3] -> new array (no aliasing)"""
    G = lambda i, j: R[j][i]     # noqa: E731
    x0, x1, x2 = x[..., 0], x[..., 1], x[..., 2]
    return np.stack([(G(1, 1) * x0 + (-G(1, 2)) * x1) + G(1, 0) * x2,
                     ((-G(2, 1)) * x0 + G(2, 2) * x1) + (-G(2, 0)) * x2,
                     (G(0, 1) * x0 + (-G(0, 2)) * x1) + G(0, 0) * x2], -1)


def band2(x, R, dtype=F32):
    """OptRotateBand2 (prt.vs) in `dtype` with GLSL indexing; constants formed in `dtype` as GLSL forms them in float.
    With dtype float64 and R given row-major as the reference's NumPy rotateBand2 takes it (R[0][1] = row 0), pass
    R transposed so that G(i, j) reads R[i][j]."""
    t = dtype
    G = lambda i, j: R[j][i]     # noqa: E731
    s_c3, s_c4, s_c5 = t(0.94617469575), t(-0.31539156525), t(0.54627421529)
    s_c_scale, s_c_scale_inv = t(1.0) / t(0.91529123286551084), t(0.91529123286551084)
    s_rc2 = t(1.5853309190550713) * s_c_scale
    s_c4_div_c3, s_c4_div_c3_x2 = s_c4 / s_c3, (s_c4 / s_c3) * t(2.0)
    s_scale_dst2, s_scale_dst4 = s_c3 * s_c_scale_inv, s_c5 * s_c_scale_inv
    x = [x[..., k] for k in range(5)]
    sh0 = ((x[3] + x[4]) + x[4]) - x[1]
    sh1 = ((x[0] + s_rc2 * x[2]) + x[3]) + x[4]
    sh2, sh3, sh4 = x[0], -x[3], -x[1]
    r2x, r2y, r2z = G(0, 0) + G(0, 1), G(1, 0) + G(1, 1), G(2, 0) + G(2, 1)
    r3x, r3y, r3z = G(0, 0) + G(0, 2), G(1, 0) + G(1, 2), G(2, 0) + G(2, 2)
    r4x, r4y, r4z = G(0, 1) + G(0, 2), G(1, 1) + G(1, 2), G(2, 1) + G(2, 2)
    sh0_x, sh0_y = sh0 * G(0, 0), sh0 * G(1, 0)
    d0 = sh0_x * G(1, 0)
    d1 = sh0_y * G(2, 0)
    d2 = sh0 * (G(2, 0) * G(2, 0) + s_c4_div_c3)
    d3 = sh0_x * G(2, 0)
    d4 = sh0_x * G(0, 0) - sh0_y * G(1, 0)
    sh1_x, sh1_y = sh1 * G(0, 2), sh1 * G(1, 2)
    d0 = d0 + sh1_x * G(1, 2)
    d1 = d1 + sh1_y * G(2, 2)
    d2 = d2 + sh1 * (G(2, 2) * G(2, 2) + s_c4_div_c3)
    d3 = d3 + sh1_x * G(2, 2)
    d4 = d4 + (sh1_x * G(0, 2) - sh1_y * G(1, 2))
    for shk, rx, ry, rz in ((sh2, r2x, r2y, r2z), (sh3, r3x, r3y, r3z), (sh4, r4x, r4y, r4z)):
        sx, sy = shk * rx, shk * ry
        d0 = d0 + sx * ry
        d1 = d1 + sy * rz
        d2 = d2 + shk * (rz * rz + s_c4_div_c3_x2)
        d3 = d3 + sx * rz
        d4 = d4 + (sx * rx - sy * ry)
    return np.stack([d0, -d1, d2 * s_scale_dst2, -d3, d4 * s_scale_dst4], -1)


# ---------------------------------------------------------------- albedo texture

def mip_levels(image):
    """set_albedo: [h,w,3] u8 -> [level 0..3] of [h_L, w_L, 3] u8, row 0 = GL's bottom row"""
    t = np.asarray(image, np.uint8)[::-1].astype(np.int64)
    out = [t.astype(np.uint8)]
    for _ in range(3):
        h, w = t.shape[:2]
        hd, wd = max(1, h // 2), max(1, w // 2)
        i, j = np.arange(wd), np.arange(hd)
        x0, x1 = np.minimum(2 * i, w - 1), np.minimum(2 * i + 1, w - 1)
        y0, y1 = np.minimum(2 * j, h - 1), np.minimum(2 * j + 1, h - 1)
        s = t[y0][:, x0] + t[y0][:, x1] + t[y1][:, x0] + t[y1][:, x1]
        t = (s + 2) >> 2
        out.append(t.astype(np.uint8))
    return out


def _lerp(p, q, a):
    return p + a * (q - p)


def bilinear(level, u, v):
    """level [h,w,3] u8, u, v [n] f32 -> [n,3] f32"""
    h, w = level.shape[:2]
    x = np.fmin(np.fmax(u * F32(w) - F32(0.5), F32(-1.0)), F32(w))
    y = np.fmin(np.fmax(v * F32(h) - F32(0.5), F32(-1.0)), F32(h))
    xf, yf = np.floor(x), np.floor(y)
    a, b = (x - xf)[:, None], (y - yf)[:, None]
    xi, yi = xf.astype(np.int64), yf.astype(np.int64)
    i0, i1 = np.clip(xi, 0, w - 1), np.clip(xi + 1, 0, w - 1)
    j0, j1 = np.clip(yi, 0, h - 1), np.clip(yi + 1, 0, h - 1)
    T = level.astype(F32) / F32(255.0)
    return _lerp(_lerp(T[j0, i0], T[j0, i1], a), _lerp(T[j1, i0], T[j1, i1], a), b)


def trilinear(levels, lam, u, v):
    out = bilinear(levels[0], u, v)
    mn = lam > 0
    if not mn.any():
        return out
    lc = np.fmin(lam[mn], F32(3.0))
    d = np.floor(lc)
    fr = (lc - d)[:, None]
    res = np.empty((mn.sum(), 3), F32)
    um, vm = u[mn], v[mn]
    for L in range(4):
        sel = d == L
        if not sel.any():
            continue
        c1 = bilinear(levels[L], um[sel], vm[sel])
        res[sel] = c1 if L == 3 else _lerp(c1, bilinear(levels[L + 1], um[sel], vm[sel]), fr[sel])
    out[mn] = res
    return out


# ---------------------------------------------------------------- raster

def _r3(m, r, x, y, z):
    return (m[r, 0] * x + m[r, 1] * y) + m[r, 2] * z


def vertex_stage(mesh, U, W, H):
    """per corner [3F]: X, Y (1/256 px), z_w, ok, z_ndc, rotated normal [3F,3], attribute [3F,k], uv [3F,2]"""
    fp, fn, fa = (np.asarray(mesh[k], np.int64).reshape(-1) for k in ("f_pos", "f_nrm", "f_attr"))
    pos, nrm, attr = (np.asarray(mesh[k], np.float64).astype(F32) for k in ("pos", "nrm", "attr"))
    tex = mesh.get("tex") is not None
    ok = (fp >= 0) & (fp < len(pos)) & (fn >= 0) & (fn < len(nrm)) & (fa >= 0) & (fa < len(attr))
    if tex:
        uvs = np.asarray(mesh["uv"], np.float64).astype(F32)
        fu = np.asarray(mesh["f_uv"], np.int64).reshape(-1)
        ok &= (fu >= 0) & (fu < len(uvs))
        uv = uvs[np.where(ok, fu, 0)]
    else:
        uv = np.zeros((len(fp), 2), F32)
    p = pos[np.where(ok, fp, 0)]
    N, Rot, MP, R = U["N"], U["Rot"], U["MP"], U["R"]
    px, py, pz = (_r3(N, r, p[:, 0], p[:, 1], p[:, 2]) + N[r, 3] for r in range(3))
    q = [_r3(Rot, r, px, py, pz) for r in range(3)]
    gx, gy, gz = (_r3(MP, r, *q) + MP[r, 3] for r in range(3))
    hw, hh = F32(W) * F32(0.5), F32(H) * F32(0.5)
    with np.errstate(invalid="ignore", over="ignore"):
        xw, yw = gx * hw + hw, gy * hh + hh
        zw = (gz + F32(1.0)) * F32(0.5)
        ok &= (np.abs(xw) <= RANGE) & (np.abs(yw) <= RANGE) & np.isfinite(zw)
    X = np.rint(np.where(ok, xw, F32(0)) * F32(256.0)).astype(np.int64)
    Y = np.rint(np.where(ok, yw, F32(0)) * F32(256.0)).astype(np.int64)
    n = nrm[np.where(ok, fn, 0)]
    nr = np.stack([_r3(R, r, n[:, 0], n[:, 1], n[:, 2]) for r in range(3)], 1)
    a = attr[np.where(ok, fa, 0)]
    if mesh["mode"] == "prt":
        a = np.concatenate([a[:, :1], band1(a[:, 1:4], R), band2(a[:, 4:9], R)], 1)
    return dict(X=X, Y=Y, zw=zw, ok=ok, z=gz, n=nr, a=a, uv=uv)


def _setup(c, F, W, H, lo, hi):
    X, Y, ok = c["X"].reshape(F, 3), c["Y"].reshape(F, 3), c["ok"].reshape(F, 3).all(1)
    area = (X[:, 1] - X[:, 0]) * (Y[:, 2] - Y[:, 0]) - (Y[:, 1] - Y[:, 0]) * (X[:, 2] - X[:, 0])
    sw = area < 0
    order = np.where(sw[:, None], np.array([0, 2, 1]), np.array([0, 1, 2]))
    Xi, Yi = np.take_along_axis(X, order, 1), np.take_along_axis(Y, order, 1)
    bx0 = np.maximum(-((hi - Xi.min(1)) >> 8), 0)
    bx1 = np.minimum((Xi.max(1) - lo) >> 8, W - 1)
    by0 = np.maximum(-((hi - Yi.min(1)) >> 8), 0)
    by1 = np.minimum((Yi.max(1) - lo) >> 8, H - 1)
    draw = ok & (area != 0) & (bx0 <= bx1) & (by0 <= by1)
    return dict(Xi=Xi, Yi=Yi, area=np.abs(area), sw=sw, bx0=bx0, bx1=bx1, by0=by0, by1=by1, draw=draw)


def _edges(s, f, Px, Py):
    """internal-order edge functions [n,3] and their dx, dy"""
    Xi, Yi = s["Xi"][f], s["Yi"][f]
    E, DX, DY = [], [], []
    for k in range(3):
        a, b = (k + 1) % 3, (k + 2) % 3
        dx, dy = Xi[:, b] - Xi[:, a], Yi[:, b] - Yi[:, a]
        E.append(dx * (Py - Yi[:, a]) - dy * (Px - Xi[:, a]))
        DX.append(dx)
        DY.append(dy)
    return np.stack(E, 1), np.stack(DX, 1), np.stack(DY, 1)


def _orig(s, f, Ei):
    sw = s["sw"][f]
    return np.stack([Ei[:, 0], np.where(sw, Ei[:, 2], Ei[:, 1]), np.where(sw, Ei[:, 1], Ei[:, 2])], 1)


def _weights(s, f, E):
    fa = s["area"][f].astype(np.float64).astype(F32)
    return E.astype(np.float64).astype(F32) / fa[:, None]


def _interp(l, a):
    """l [n,3], a [n,3(corners),...] -> (l0 a0 + l1 a1) + l2 a2"""
    sh = (slice(None),) + (None,) * (a.ndim - 2)
    return (l[:, 0][sh] * a[:, 0] + l[:, 1][sh] * a[:, 1]) + l[:, 2][sh] * a[:, 2]


def zbuffer(c, F, W, H, S):
    lo, hi = (128, 128) if S == 1 else (0, 240)
    s = _setup(c, F, W, H, lo, hi)
    offs = sample_offsets(S)
    zw = c["zw"].reshape(F, 3)
    zbuf = np.full(W * H * S, EMPTY, np.uint64)
    ids = np.nonzero(s["draw"])[0]
    nx = (s["bx1"] - s["bx0"] + 1)[ids]
    cnt = nx * (s["by1"] - s["by0"] + 1)[ids] * S
    i = 0
    while i < len(ids):
        j = i + max(1, int(np.searchsorted(np.cumsum(cnt[i:]), BATCH, side="right")))
        f, n = np.repeat(ids[i:j], cnt[i:j]), np.repeat(nx[i:j], cnt[i:j])
        start = np.repeat(np.cumsum(cnt[i:j]) - cnt[i:j], cnt[i:j])
        t = np.arange(len(f)) - start
        smp, pp = t % S, t // S
        px, py = s["bx0"][f] + pp % n, s["by0"][f] + pp // n
        Px, Py = px * 256 + offs[smp, 0], py * 256 + offs[smp, 1]
        Ei, DX, DY = _edges(s, f, Px, Py)
        tl = (DY < 0) | ((DY == 0) & (DX < 0))
        cov = ((Ei > 0) | ((Ei == 0) & tl)).all(1)
        l = _weights(s, f, _orig(s, f, Ei))
        with np.errstate(invalid="ignore", over="ignore"):
            z = _interp(l, zw[f])
            keep = cov & (z >= 0) & (z <= 1)
            q = np.rint(np.where(keep, z, F32(0)) * F32(16777215.0)).astype(np.uint64)
        keep &= q < 16777215
        key = (q << np.uint64(32)) | f.astype(np.uint64)
        np.minimum.at(zbuf, ((py * W + px) * S + smp)[keep], key[keep])
        i = j
    return zbuf.reshape(H * W, S), s


def shade(mesh, c, s, U, levels, f, px, py):
    """the three attachments of faces f at pixel centres (px, py): [n,4] each"""
    Ei, DX, DY = _edges(s, f, px * 256 + 128, py * 256 + 128)
    l = _weights(s, f, _orig(s, f, Ei))
    corner = 3 * f[:, None] + np.arange(3)
    z = _interp(l, c["z"][corner])
    one = np.ones(len(f), F32)
    a2 = np.stack([z, z, z, one], 1)
    n = _interp(l, c["n"][corner])
    r = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    with np.errstate(invalid="ignore", divide="ignore"):
        nn = (n / r[:, None] + F32(1.0)) * F32(0.5)
    nn[r == 0] = F32(0.5)
    a1 = np.concatenate([nn, one[:, None]], 1)
    p = _interp(l, c["a"][corner])
    if mesh["mode"] != "prt":
        return np.concatenate([p, one[:, None]], 1), a1, a2
    SH = U["SH"]
    g = np.empty((len(f), 3), F32)
    for ch in range(3):
        acc = np.zeros(len(f), F32)
        for k in range(9):
            acc = acc + p[:, k] * SH[k, ch]
        pos = acc >= 0
        g[:, ch] = np.where(pos, np.power(np.where(pos, acc, 0).astype(np.float64),
                                          np.float64(F32(1.0) / F32(2.2))).astype(F32), F32(0))
    alb = np.ones((len(f), 3), F32)
    if levels is not None:
        h0, w0 = levels[0].shape[:2]
        ex = _orig(s, f, -DY * 256)
        ey = _orig(s, f, DX * 256)
        gx, gy = _weights(s, f, ex), _weights(s, f, ey)
        uv = c["uv"][corner]
        us, vs = uv[..., 0], uv[..., 1]
        dudx, dvdx = _interp(gx, us) * F32(w0), _interp(gx, vs) * F32(h0)
        dudy, dvdy = _interp(gy, us) * F32(w0), _interp(gy, vs) * F32(h0)
        rho = np.fmax(np.sqrt(dudx * dudx + dvdx * dvdx), np.sqrt(dudy * dudy + dvdy * dvdy))
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = np.log2(rho.astype(np.float64)).astype(F32)
        alb = trilinear(levels, lam, _interp(l, us), _interp(l, vs))
    a0 = np.concatenate([np.fmin(np.fmax(alb * g, F32(0)), F32(1)), one[:, None]], 1)
    return a0, a1, a2


def render(mesh, normalize_matrix, rot_matrix, model_view, projection, sh, W, H, S):
    """mesh: dict(mode='prt'|'color', pos, nrm, attr, f_pos, f_nrm, f_attr[, uv, f_uv, tex (an [h,w,3] u8 image)]) ->
    float32 [3,H,W,4]: attachments 0-2 in get_color's layout"""
    U = uniforms(normalize_matrix, rot_matrix, model_view, projection, sh if sh is not None else np.zeros((9, 3)))
    F = np.asarray(mesh["f_pos"]).reshape(-1, 3).shape[0]
    c = vertex_stage(mesh, U, W, H)
    zbuf, s = zbuffer(c, F, W, H, S)
    levels = mip_levels(mesh["tex"]) if mesh.get("tex") is not None else None
    hit = zbuf != EMPTY
    pix, smp = np.nonzero(hit)
    f = (zbuf[pix, smp] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    out = np.zeros((3, H * W, 4), F32)
    if len(f):
        uk, inv = np.unique(pix * F + f, return_inverse=True)
        up, uf = uk // F, uk % F
        vals = shade(mesh, c, s, U, levels, uf, up % W, up // W)
        for a in range(3):
            per = np.zeros((H * W, S, 4), F32)
            per[pix, smp] = vals[a][inv]
            acc = np.zeros((H * W, 4), F32)
            for k in range(S):
                acc = acc + per[:, k]
            out[a] = acc * F32(1.0 / S)
    return out.reshape(3, H, W, 4)[:, ::-1].copy()
