"""Independent numpy rasteriser of the mesh-overlay contract (DESIGN.md section 6 "Mesh overlay") -- TEST INFRASTRUCTURE ONLY.

It restates reference render_demo.py:58-153 (pyrender 0.1.45 + trimesh, requirements.txt:18) the way csrc/render.cu does:
24.8 fixed-point window coordinates, int64 edge functions with the top-left rule in image coordinates (rows down), back-face
culling in window space, per-fragment near/far discard, double-precision depth rounded to fp32 with the lower face id
winning a tie, the 1x / 4x sample patterns, and float64 shading.  The geometric part is evaluated with the same operations
in the same order as the kernel, so the winning face of every sample agrees bit for bit.  It never touches a GPU.
"""
import numpy as np

GUARD = float(2 ** 20)
OFFSETS = {1: np.array([[0, 0]], dtype=np.int64),
           4: np.array([[-2, -6], [6, -2], [-6, 2], [2, 6]], dtype=np.int64) * 16}     # 1/256 pixel
LIGHTS = np.array([[0.0, -1.0, 1.0], [0.0, 1.0, 1.0], [1.0, 1.0, 2.0]])


def transform(verts, cam4, rot, W, H):
    """Render-frame positions p (NV,3), fixed-point window coordinates X, Y, ndc_z and the guard-band mask."""
    v = np.asarray(verts, dtype=np.float32).astype(np.float64)
    q = np.stack([v[:, 0], -v[:, 1], -v[:, 2]], 1)
    if rot is None:
        p = q
    else:
        R = np.asarray(rot, dtype=np.float32).astype(np.float64).reshape(3, 3)
        p = np.stack([(R[k, 0] * q[:, 0] + R[k, 1] * q[:, 1]) + R[k, 2] * q[:, 2] for k in range(3)], 1)
    sx, sy, tx, ty = (float(c) for c in np.asarray(cam4, dtype=np.float32))
    u = (1.0 + sx * (p[:, 0] + tx)) * 0.5 * float(W)
    r = (1.0 - sy * (p[:, 1] - ty)) * 0.5 * float(H)
    with np.errstate(invalid='ignore'):
        ok = (np.abs(u) <= GUARD) & (np.abs(r) <= GUARD)
    X = np.where(ok, np.rint(np.where(ok, u, 0.0) * 256.0), 0).astype(np.int64)
    Y = np.where(ok, np.rint(np.where(ok, r, 0.0) * 256.0), 0).astype(np.int64)
    return p, X, Y, -p[:, 2], ok


def vertex_normals(p, faces):
    """trimesh's angle-weighted vertex normals; zero-area faces contribute nothing."""
    P = p[faces]
    u, v, w = P[:, 1] - P[:, 0], P[:, 2] - P[:, 0], P[:, 2] - P[:, 1]
    n = np.cross(u, v)
    nn = np.sqrt((n * n).sum(1))
    good = nn > 0
    with np.errstate(invalid='ignore', divide='ignore'):
        uu = u / np.sqrt((u * u).sum(1))[:, None]
        vv = v / np.sqrt((v * v).sum(1))[:, None]
        ww = w / np.sqrt((w * w).sum(1))[:, None]
        a0 = np.arccos(np.clip((uu * vv).sum(1), -1, 1))
        a1 = np.arccos(np.clip(-(uu * ww).sum(1), -1, 1))
        fn = n / nn[:, None]
    a2 = np.pi - a0 - a1
    ang = np.stack([a0, a1, a2], 1)
    good &= (ang >= 1e-8).all(1)
    acc = np.zeros_like(p)
    for k in range(3):
        np.add.at(acc, faces[good, k], ang[good, k, None] * fn[good])
    ln = np.sqrt((acc * acc).sum(1))
    return np.where(ln[:, None] > 0, acc / np.where(ln > 0, ln, 1.0)[:, None], 0.0)


def _edge(px, py, qx, qy, sx, sy):
    return (qx - px) * (sy - py) - (qy - py) * (sx - px)


def _top_left(px, py, qx, qy):
    return (qy < py) | ((qy == py) & (qx > px))


def depth_key(d):
    """Order-preserving unsigned bits of an fp32 depth (-0 counted as +0)."""
    d = np.where(d == 0, np.float32(0), d).astype(np.float32)
    b = d.view(np.uint32).astype(np.uint64)
    return np.where(b & 0x80000000, ~b & 0xFFFFFFFF, b | 0x80000000)


def rasterise(faces, X, Y, z, ok, W, H, samples):
    """face_ids (H, W, samples) int32, -1 where nothing is covered."""
    off = OFFSETS[samples]
    keys = np.full(H * W * samples, np.iinfo(np.uint64).max, dtype=np.uint64)
    for f, (a, b, c) in enumerate(np.asarray(faces, dtype=np.int64)):
        if not (ok[a] and ok[b] and ok[c]):
            continue
        area = (X[b] - X[a]) * (Y[c] - Y[a]) - (Y[b] - Y[a]) * (X[c] - X[a])
        if area >= 0:
            continue
        i0, i1, i2 = a, c, b                                     # raster order: positive area in image coordinates
        x0, y0, x1, y1, x2, y2 = X[i0], Y[i0], X[i1], Y[i1], X[i2], Y[i2]
        xs, ys = (x0, x1, x2), (y0, y1, y2)
        c0, c1 = max(0, -((224 - min(xs)) // 256)), min(W - 1, (max(xs) - 32) // 256)
        r0, r1 = max(0, -((224 - min(ys)) // 256)), min(H - 1, (max(ys) - 32) // 256)
        if c0 > c1 or r0 > r1:
            continue
        cc, rr = np.meshgrid(np.arange(c0, c1 + 1, dtype=np.int64), np.arange(r0, r1 + 1, dtype=np.int64))
        cc, rr = cc.reshape(-1, 1), rr.reshape(-1, 1)
        sx, sy = 256 * cc + 128 + off[None, :, 0], 256 * rr + 128 + off[None, :, 1]
        w0, w1, w2 = _edge(x1, y1, x2, y2, sx, sy), _edge(x2, y2, x0, y0, sx, sy), _edge(x0, y0, x1, y1, sx, sy)
        inside = (((w0 > 0) | ((w0 == 0) & _top_left(x1, y1, x2, y2))) & ((w1 > 0) | ((w1 == 0) & _top_left(x2, y2, x0, y0)))
                  & ((w2 > 0) | ((w2 == 0) & _top_left(x0, y0, x1, y1))))
        if not inside.any():
            continue
        A = np.float64(_edge(x0, y0, x1, y1, x2, y2))
        w0, w1, w2 = w0[inside].astype(np.float64), w1[inside].astype(np.float64), w2[inside].astype(np.float64)
        d = (((w0 * z[i0] + w1 * z[i1]) + w2 * z[i2]) / A).astype(np.float32)
        keep = (d >= -1) & (d <= 1)
        idx = ((rr * W + cc) * samples + np.arange(samples)[None, :])[inside][keep]
        key = (depth_key(d[keep]) << np.uint64(32)) | np.uint64(f)
        keys[idx] = np.minimum(keys[idx], key)
    fid = np.where(keys == np.iinfo(np.uint64).max, -1, (keys & np.uint64(0xFFFFFFFF)).astype(np.int64))
    return fid.reshape(H, W, samples).astype(np.int32)


def shade(p, nrm, X, Y, faces, fid, rows, cols, color):
    """Bytes (n, 3) of face fid[i] shaded at the centre of pixel (cols[i], rows[i])."""
    F = np.asarray(faces, dtype=np.int64)[fid]
    i0, i1, i2 = F[:, 0], F[:, 2], F[:, 1]
    sx, sy = 256 * cols.astype(np.int64) + 128, 256 * rows.astype(np.int64) + 128
    A = _edge(X[i0], Y[i0], X[i1], Y[i1], X[i2], Y[i2]).astype(np.float64)
    l0 = _edge(X[i1], Y[i1], X[i2], Y[i2], sx, sy).astype(np.float64) / A
    l1 = _edge(X[i2], Y[i2], X[i0], Y[i0], sx, sy).astype(np.float64) / A
    l2 = _edge(X[i0], Y[i0], X[i1], Y[i1], sx, sy).astype(np.float64) / A
    pp = (l0[:, None] * p[i0] + l1[:, None] * p[i1]) + l2[:, None] * p[i2]
    n = (l0[:, None] * nrm[i0] + l1[:, None] * nrm[i1]) + l2[:, None] * nrm[i2]
    ln = np.sqrt((n * n).sum(1, keepdims=True))
    n = np.where(ln > 0, n / np.where(ln > 0, ln, 1.0), 0.0)
    pl = np.sqrt((pp * pp).sum(1, keepdims=True))
    v = np.where(pl > 0, -pp / np.where(pl > 0, pl, 1.0), np.array([0.0, 0.0, 1.0]))
    nv = np.clip((n * v).sum(1), 0, 1)
    base = np.asarray(color, dtype=np.float32).astype(np.float64)
    col = np.zeros((len(fid), 3))
    for L in LIGHTS:
        l = L[None] - pp
        d2 = (l * l).sum(1)
        l = l / np.sqrt(d2)[:, None]
        h = l + v
        hl = np.sqrt((h * h).sum(1, keepdims=True))
        h = np.where(hl > 0, h / np.where(hl > 0, hl, 1.0), 0.0)
        nl = np.clip((n * l).sum(1), 0, 1)
        vh = np.clip((v * h).sum(1), 0, 1)
        Fr = 0.04 + 0.96 * (1.0 - vh) ** 5
        G = (2 * nl / (nl + 1)) * (2 * nv / (nv + 1))
        spec = Fr * G * (1 / np.pi) / (4 * nl * nv + 0.001)
        col += (nl / d2)[:, None] * ((1 - Fr)[:, None] * (0.96 * base)[None] / np.pi + spec[:, None])
    c = np.clip((col + 0.3 * base[None]) ** (1 / 2.2), 0, 1)
    return np.floor(255.0 * c + 0.5).astype(np.int64)


def render(img, verts, faces, cam4, rot=None, color=(1.0, 1.0, 0.9), samples=4):
    """(out (H,W,3) uint8, face_ids (H,W,samples) int32) of the contract for one mesh over one frame."""
    img = np.asarray(img)
    H, W = img.shape[:2]
    faces = np.asarray(faces, dtype=np.int64)
    p, X, Y, z, ok = transform(verts, cam4, rot, W, H)
    fid = rasterise(faces, X, Y, z, ok, W, H, samples)
    nrm = vertex_normals(p, faces) if len(faces) else np.zeros_like(p)
    rr, cc, _ = np.nonzero(fid >= 0)
    byt = np.zeros((H, W, samples, 3), dtype=np.int64)
    if len(rr):
        byt[fid >= 0] = shade(p, nrm, X, Y, faces, fid[fid >= 0], rr, cc, color)
    k = (fid >= 0).sum(2)
    val = (byt.sum(2) + samples // 2) // samples
    out = np.where(k[..., None] > 0, val, img).astype(np.uint8)
    return out, fid
