"""ORACLE -- test infrastructure, not product code (only tests/ and tools/ may import it).

numpy float64 z-buffer of the map renderer (vista_slam_b200/render.py, csrc/render.cu): the same float32 inputs,
unprojected (K^-1 [col row 1]^T depth scale, then R p + t), projected into each camera (K (w2c p), u / w, v / w) and
splatted over the (2 r + 1)^2 pixels centred on floor(u / w + 0.5), floor(v / w + 0.5); segments are clipped to
z >= near, then to the image grown by r + 0.5 (Liang-Barsky), and stepped max(|du|, |dv|) times with perspective-correct z.
Each pixel keeps the smallest (z, id).

Where float32 and float64 can disagree, a pixel is marked ambiguous: a candidate point whose u / w + 0.5 or
v / w + 0.5 lies within `boundary` px of an integer (its footprint may shift by one pixel; both footprints are
candidates), or two nearest candidates whose depths differ by less than `tie` relative.  `accept[c, y, x]` then holds the
ids a float32 renderer may show there (-1 for empty when a shifted footprint may leave the pixel uncovered)."""
import numpy as np


def points(maps, conf_thres):
    """World points (float64) and ids v H W + row W + col of the pixels with conf > conf_thres."""
    depth = np.asarray(maps["depth"], np.float32)
    V, H, W = depth.shape
    conf = np.asarray(maps["conf"], np.float32)
    pose = np.asarray(maps["pose"], np.float64)
    scale = np.asarray(maps["scale"], np.float32).reshape(V)
    intri = np.asarray(maps["intri"], np.float64)
    ids = np.flatnonzero(conf.reshape(-1) > np.float32(conf_thres))
    v, pix = ids // (H * W), ids % (H * W)
    row, col = pix // W, pix % W
    d = (depth.reshape(-1)[ids] * scale[v]).astype(np.float64)  # the float32 product the kernel forms
    ray = np.einsum("nij,nj->ni", np.linalg.inv(intri)[v], np.stack([col, row, np.ones_like(col)], -1).astype(np.float64))
    cam = ray * d[:, None]
    world = np.einsum("nij,nj->ni", pose[v, :3, :3], cam) + pose[v, :3, 3]
    return world, ids


def _clip_axis(p, d, lo, hi, t0, t1):
    if d == 0:
        return (lo <= p <= hi), t0, t1
    a, b = sorted(((lo - p) / d, (hi - p) / d))
    t0, t1 = max(t0, a), min(t1, b)
    return t0 <= t1, t0, t1


def segment_samples(a, b, w2c, K, Ho, Wo, r, near):
    """(x, y, z) float64 samples of world segment a-b seen through w2c and K, as the kernel steps it."""
    qa, qb = w2c[:3, :3] @ a + w2c[:3, 3], w2c[:3, :3] @ b + w2c[:3, 3]
    ina, inb = qa[2] >= near, qb[2] >= near
    if not ina and not inb:
        return []
    if not (ina and inb):
        f, k = (qa, qb) if ina else (qb, qa)
        m = f + (near - f[2]) / (k[2] - f[2]) * (k - f)
        m[2] = near
        qa, qb = (qa, m) if ina else (m, qb)
    ua, ub = K @ qa, K @ qb
    xa, ya, xb, yb = ua[0] / ua[2], ua[1] / ua[2], ub[0] / ub[2], ub[1] / ub[2]
    du, dv = xb - xa, yb - ya
    rr = r + 0.5
    ok, t0, t1 = _clip_axis(xa, du, -rr, Wo - 1 + rr, 0.0, 1.0)
    ok = ok and _clip_axis(ya, dv, -rr, Ho - 1 + rr, t0, t1)[0]
    if not ok:
        return []
    _, t0, t1 = _clip_axis(ya, dv, -rr, Ho - 1 + rr, t0, t1)
    x0, y0, cu, cv = xa + t0 * du, ya + t0 * dv, (t1 - t0) * du, (t1 - t0) * dv
    n = int(np.ceil(max(abs(cu), abs(cv))))
    za, zb = qa[2], qb[2]
    out = []
    for k in range(n + 1):
        f = k / n if n else 0.0
        s = t0 + f * (t1 - t0)
        z = max(za + za * s * (zb - za) / (zb + s * (za - zb)), near)
        out.append((x0 + cu * f, y0 + cv * f, z))
    return out


def render(maps, conf_thres, w2c, K, size, radius=0, near=1e-3, segs=None, seg_colors=None, background=(1.0, 1.0, 1.0),
           boundary=1e-3, tie=1e-5):
    """The oracle's images and ambiguity record: {rgb [C,Ho,Wo,3], depth [C,Ho,Wo], index [C,Ho,Wo], ambiguous
    [C,Ho,Wo] bool, accept {(c, y, x): set of ids}} for world-to-camera w2c [C,4,4] and K [C,3,3]."""
    Ho, Wo = size
    w2c, K = np.asarray(w2c, np.float64), np.asarray(K, np.float64)
    C = len(w2c)
    depth_in = np.asarray(maps["depth"])
    V, H, W = depth_in.shape
    imgs = np.asarray(maps["images"], np.float32)
    world, ids = points(maps, conf_thres)
    nseg = 0 if segs is None else len(segs)
    # candidates per pixel: (z, id, primary, sure); primary False for a shifted footprint, sure False for both
    # footprints of a point near a pixel boundary
    cand = {}

    def add(c, x, y, z, i, primary, sure):
        cx, cy = int(np.floor(x + 0.5)), int(np.floor(y + 0.5))
        for yy in range(max(0, cy - radius), min(Ho - 1, cy + radius) + 1):
            for xx in range(max(0, cx - radius), min(Wo - 1, cx + radius) + 1):
                cand.setdefault((c, yy, xx), []).append((z, i, primary, sure))

    def near_boundary(x):
        f = (x + 0.5) - np.floor(x + 0.5)
        return min(f, 1 - f) < boundary

    for c in range(C):
        q = world @ w2c[c, :3, :3].T + w2c[c, :3, 3]
        uvw = q @ K[c].T
        with np.errstate(divide="ignore", invalid="ignore"):
            xs, ys = uvw[:, 0] / uvw[:, 2], uvw[:, 1] / uvw[:, 2]
        for k in np.flatnonzero(q[:, 2] >= near):
            x, y, z, i = xs[k], ys[k], q[k, 2], int(ids[k])
            if not (np.isfinite(x) and np.isfinite(y)) or abs(x) > 1e9 or abs(y) > 1e9:
                continue
            bx, by = near_boundary(x), near_boundary(y)
            add(c, x, y, z, i, True, not (bx or by))
            for sx in ((-1, 1) if bx else (0,)):
                for sy in ((-1, 1) if by else (0,)):
                    if sx or sy:
                        add(c, x + sx * 2 * boundary, y + sy * 2 * boundary, z, i, False, False)
        for l in range(nseg):
            for x, y, z in segment_samples(np.asarray(segs[l][0], np.float64), np.asarray(segs[l][1], np.float64), w2c[c],
                                           K[c], Ho, Wo, radius, near):
                add(c, x, y, z, V * H * W + l, True, True)
    rgb = np.empty((C, Ho, Wo, 3), np.float32)
    rgb[:] = np.asarray(background, np.float32)
    depth = np.zeros((C, Ho, Wo), np.float64)
    index = np.full((C, Ho, Wo), -1, np.int64)
    ambiguous = np.zeros((C, Ho, Wo), bool)
    accept = {}
    for (c, y, x), lst in cand.items():
        prim = sorted({(z, i) for z, i, p, _ in lst if p})
        if prim:
            z, i = prim[0]
            index[c, y, x], depth[c, y, x] = i, z
            if i < V * H * W:
                v, pix = divmod(i, H * W)
                rgb[c, y, x] = (imgs[v, :, pix // W, pix % W] + np.float32(1)) / np.float32(2)
            else:
                rgb[c, y, x] = np.asarray(seg_colors[i - V * H * W], np.float32)
        if not all(sure for *_, sure in lst):
            ambiguous[c, y, x] = True
            accept[(c, y, x)] = {i for _, i, _, _ in lst} | {-1}
        elif len(prim) > 1 and prim[1][0] - prim[0][0] < tie * prim[0][0]:
            ambiguous[c, y, x] = True
            accept[(c, y, x)] = {i for z, i in prim if z - prim[0][0] < tie * prim[0][0]}
    return {"rgb": rgb, "depth": depth, "index": index, "ambiguous": ambiguous, "accept": accept}

