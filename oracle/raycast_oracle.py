"""float64 oracle of the ray casting of vista_slam_b200/fusion.py (csrc/raycast.cu), written from the semantics in
raycast.cu's header comment and fusion.raycast's docstring.

raycast(keys, tsdf, weight, color, voxel, c2w, K, size, min_weight, near, background) -> {rgb, color, depth, normal,
hit, ambiguous}, over a volume given as arrays: keys [B] (sorted, distinct), tsdf / weight [B,8,8,8] ([b, z, y, x]),
color [B,8,8,8,3]; cameras c2w [C,4,4], K [C,3,3]; images [C,Ho,Wo(,3)].

  Ray       pixel (col, row): o + z R ((col - cx) / fx, (row - cy) / fy, 1), z the camera depth.
  Field     point p lies in cell floor(p / v); the cell is valid when its 8 corner samples (lattice points, sample
            (i, j, k) at (i v, j v, k v)) exist with weight >= min_weight; there T and the colour are trilinear in
            the fractions p / v - floor(p / v).
  March     over the ray's overlap with the bricks' box [8 bmin v, 8 (bmax + 1) v] per axis from z >= near, samples
            z_k = za + k dz, dz = (v / 2) / |R d|.  The device jumps over absent bricks; no valid cell has its lower
            corner in one, so the oracle simply visits every sample, those in absent bricks being invalid.
  Hit       the first k with valid samples k - 1 and k and T_{k-1} > 0 >= T_k, refined by 16 bisection steps on
            [z_{k-1}, z_k] (an invalid midpoint replaces the far end, keeping its T), then the bracket's secant
            point.  Normal (normalised gradient of the interpolant) and colour in that point's cell, or in the near
            end's cell when that cell is invalid.  rgb = color (0.3 + 0.7 max(0, -n . r)), r the unit ray direction.
            depth 0, normal 0, color and rgb the background on a miss.

`ambiguous` marks the pixels where float32 rounding may legitimately change the hit or miss: a sample up to the hit
within 1e-3 v (world distance along the ray) of a zero of the field, a sample within 1e-3 v of a face across which
cell validity changes where the change could make or break the hit pair, the hit within 1e-3 v of such a face, a
grazing hit (|dT/ds| v < 1e-3, s world length along the ray, or the ray within 0.05 rad of the surface's tangent
plane, where the rounding of a float32 position moves the hit twenty-fold along the ray), or more than one
crossing (or an invalid point) inside the hit's step."""
import numpy as np

BRICK = 8
BIAS = 1 << 20
AMBIENT = 0.3
REFINE = 16
_EPS = 1e-3
_GRAZE = 0.05


def _unkey(k):
    k = np.asarray(k, np.int64)
    return np.stack([(k >> s) & ((1 << 21) - 1) for s in (0, 21, 42)], -1) - BIAS


def _key(b):
    b = np.asarray(b, np.int64) + BIAS
    return (b[..., 2] << 42) | (b[..., 1] << 21) | b[..., 0]


class _Volume:
    def __init__(self, keys, tsdf, weight, color, voxel, min_weight):
        self.keys = np.asarray(keys, np.int64)
        self.T = np.asarray(tsdf, np.float64).reshape(-1)
        self.W = np.asarray(weight, np.float64).reshape(-1)
        self.C = np.asarray(color, np.float64).reshape(-1, 3)
        self.v = float(voxel)
        self.mw = float(min_weight)

    def corners(self, p):
        """Cells of points p [..., 3]: (valid [...], sample indices [..., 8], fractions [..., 3])."""
        s = p / self.v
        i = np.floor(s)
        f = s - i
        i = np.clip(i, -8 * BIAS - 8, 8 * BIAS).astype(np.int64)
        off = np.array([[c & 1, c >> 1 & 1, c >> 2] for c in range(8)], np.int64)
        q = i[..., None, :] + off  # [..., 8, 3]
        b = np.floor_divide(q, BRICK)
        inr = ((b >= -BIAS) & (b < BIAS)).all(-1)
        k = _key(np.clip(b, -BIAS, BIAS - 1))
        j = np.searchsorted(self.keys, k)
        jc = np.minimum(j, max(len(self.keys) - 1, 0))
        found = inr & (j < len(self.keys))
        if len(self.keys):
            found &= self.keys[jc] == k
        loc = q - BRICK * b
        g = jc * 512 + loc[..., 2] * 64 + loc[..., 1] * 8 + loc[..., 0]
        g = np.where(found, g, 0)
        ok = found & (self.W[g] >= self.mw) if len(self.keys) else found
        return ok.all(-1), g, f

    def valid(self, p):
        return self.corners(p)[0]

    def field(self, p):
        """(valid, T, gradient in cell units [..., 3], colour [..., 3]) at points p [..., 3]."""
        ok, g, f = self.corners(p)
        v = self.T[g] if len(self.keys) else np.zeros(g.shape)
        fx, fy, fz = f[..., 0:1], f[..., 1:2], f[..., 2:3]
        wx = np.concatenate([1 - fx, fx], -1)
        wy = np.concatenate([1 - fy, fy], -1)
        wz = np.concatenate([1 - fz, fz], -1)
        w = (wz[..., :, None, None] * wy[..., None, :, None] * wx[..., None, None, :]).reshape(f.shape[:-1] + (8,))
        T = (w * v).sum(-1)
        dwx = np.array([-1.0, 1.0])
        gx = (wz[..., :, None, None] * wy[..., None, :, None] * dwx).reshape(f.shape[:-1] + (8,))
        gy = (wz[..., :, None, None] * dwx[:, None] * wx[..., None, None, :]).reshape(f.shape[:-1] + (8,))
        gz = (dwx[:, None, None] * wy[..., None, :, None] * wx[..., None, None, :]).reshape(f.shape[:-1] + (8,))
        grad = np.stack([(gx * v).sum(-1), (gy * v).sum(-1), (gz * v).sum(-1)], -1)
        col = (w[..., None] * self.C[g]).sum(-2) if len(self.keys) else np.zeros(f.shape)
        return ok, T, grad, col


def _validity_change_near(vol, p):
    """True where a face across which cell validity changes lies within 1e-3 v of p [n,3]."""
    near = np.zeros(len(p), bool)
    if not len(p):
        return near
    ok = vol.valid(p)
    for a in range(3):
        for sgn in (-1.0, 1.0):
            q = p.copy()
            q[:, a] += sgn * _EPS * vol.v
            near |= vol.valid(q) != ok
    return near


def raycast(keys, tsdf, weight, color, voxel, c2w, K, size, min_weight=1, near=1e-3, background=(1.0, 1.0, 1.0),
            block=16):
    vol = _Volume(keys, tsdf, weight, color, voxel, min_weight)
    v = vol.v
    P = np.asarray(c2w, np.float64).reshape(-1, 4, 4)
    Ks = np.broadcast_to(np.asarray(K, np.float64), (len(P), 3, 3))
    C = len(P)
    Ho, Wo = size
    row, col = np.mgrid[0:Ho, 0:Wo]
    dc = np.stack([(col[None] - Ks[:, 0, 2, None, None]) / Ks[:, 0, 0, None, None],
                   (row[None] - Ks[:, 1, 2, None, None]) / Ks[:, 1, 1, None, None], np.ones((C, Ho, Wo))], -1)
    d = np.einsum("cij,chwj->chwi", P[:, :3, :3], dc).reshape(-1, 3)
    o = np.broadcast_to(P[:, None, None, :3, 3], (C, Ho, Wo, 3)).reshape(-1, 3)
    n = len(d)
    dn = np.linalg.norm(d, axis=1)
    rdir = d / dn[:, None]
    za = np.full(n, float(near))
    zb = np.full(n, np.inf)
    inside = np.full(n, len(vol.keys) > 0)
    if len(vol.keys):
        bb = _unkey(vol.keys)
        lo, hi = BRICK * bb.min(0) * v, BRICK * (bb.max(0) + 1) * v
        for a in range(3):
            zero = d[:, a] == 0
            inside &= ~zero | ((o[:, a] >= lo[a]) & (o[:, a] <= hi[a]))
            with np.errstate(divide="ignore", invalid="ignore"):
                t1, t2 = (lo[a] - o[:, a]) / d[:, a], (hi[a] - o[:, a]) / d[:, a]
            za = np.where(zero, za, np.maximum(za, np.minimum(t1, t2)))
            zb = np.where(zero, zb, np.minimum(zb, np.maximum(t1, t2)))
    inside &= za <= zb
    dz = 0.5 * v / dn
    nk = np.where(inside, np.floor((np.where(inside, zb, za) - za) / dz) + 1, 0).astype(np.int64)

    hit = np.zeros(n, bool)
    amb = np.zeros(n, bool)
    hk = np.zeros(n, np.int64)  # k of the hit pair's far sample
    T_prev = np.zeros(n)
    ok_prev = np.zeros(n, bool)
    vflip_prev = np.zeros(n, bool)
    active = nk > 0
    k0 = 0
    while active.any():
        idx = np.nonzero(active)[0]
        ks = k0 + np.arange(block)
        z = za[idx, None] + ks[None] * dz[idx, None]
        live = ks[None] < nk[idx, None]
        p = o[idx, None] + z[..., None] * d[idx, None]
        ok, T, grad, _ = vol.field(p)
        ok &= live
        okp = np.concatenate([ok_prev[idx, None], ok[:, :-1]], 1)
        Tp = np.concatenate([T_prev[idx, None], T[:, :-1]], 1)
        pair = okp & ok & (Tp > 0) & (T <= 0)
        first = np.where(pair.any(1), pair.argmax(1), block)
        upto = ks[None] - k0 <= first[:, None]
        # ambiguity of the samples up to the hit: near a zero of the field, or near a validity change
        dTds = np.abs((grad * rdir[idx, None]).sum(-1)) / v
        with np.errstate(divide="ignore", invalid="ignore"):
            zero_near = ok & upto & (np.abs(T) < _EPS * v * dTds)
        cand = live & upto
        pn = p[cand]
        facey = np.zeros(len(pn), bool)
        if len(pn):
            fr = pn / v - np.floor(pn / v)
            close = (np.minimum(fr, 1 - fr) < _EPS).any(1)
            facey[close] = _validity_change_near(vol, pn[close])
        vnear = np.zeros(cand.shape, bool)
        vnear[cand] = facey
        # a validity flip matters where it can make or break a hit pair: a valid sample of the hit pair turning
        # invalid, or an invalid sample turning valid beside a neighbour that would pair with it
        j = np.arange(block)[None]
        okn = np.concatenate([ok[:, 1:], np.ones((len(idx), 1), bool)], 1)
        Tn = np.concatenate([T[:, 1:], np.full((len(idx), 1), -1.0)], 1)  # unknown beyond the block: assume it pairs
        pairs = np.where(ok, (j == first[:, None]) | (j == first[:, None] - 1),
                         (okp & (Tp > 0)) | (okn & (Tn <= 0)))
        amb[idx] |= (zero_near | (vnear & pairs)).any(1)
        amb[idx] |= (first == 0) & vflip_prev[idx]
        got = first < block
        hit[idx[got]] = True
        hk[idx[got]] = k0 + first[got]
        vflip_prev[idx] = vnear[:, -1] & ok[:, -1]
        ok_prev[idx] = ok[:, -1]
        T_prev[idx] = T[:, -1]
        active[idx[got]] = False
        active &= k0 + block < nk
        k0 += block

    out_depth = np.zeros(n)
    out_normal = np.zeros((n, 3))
    out_color = np.tile(np.asarray(background, np.float64), (n, 1))
    out_rgb = out_color.copy()
    h = np.nonzero(hit)[0]
    if len(h):
        z1 = za[h] + hk[h] * dz[h]
        z0 = za[h] + (hk[h] - 1) * dz[h]
        oh, dh = o[h], d[h]
        f0 = vol.field(oh + z0[:, None] * dh)[1]
        f1 = vol.field(oh + z1[:, None] * dh)[1]
        # more than one crossing, or an invalid point, inside the step
        s = np.linspace(0, 1, 17)
        zs = z0[:, None] + s[None] * (z1 - z0)[:, None]
        oks, Ts, _, _ = vol.field(oh[:, None] + zs[..., None] * dh[:, None])
        changes = ((Ts[:, 1:] > 0) != (Ts[:, :-1] > 0)).sum(1)
        amb[h] |= (changes > 1) | ~oks.all(1)
        for _ in range(REFINE):
            m = 0.5 * (z0 + z1)
            okm, fm, _, _ = vol.field(oh + m[:, None] * dh)
            far = ~okm | ~(fm > 0)
            f1 = np.where(far & okm, fm, f1)
            z1 = np.where(far, m, z1)
            f0 = np.where(far, f0, fm)
            z0 = np.where(far, z0, m)
        zh = z0 + (z1 - z0) * (f0 / (f0 - f1))
        ph = oh + zh[:, None] * dh
        okh = vol.valid(ph)
        pe = np.where(okh[:, None], ph, oh + z0[:, None] * dh)
        _, _, g, c = vol.field(pe)
        gn = np.linalg.norm(g, axis=1)
        nrm = np.where(gn[:, None] > 0, g / np.where(gn > 0, gn, 1)[:, None], 0.0)
        amb[h] |= _validity_change_near(vol, ph)
        # grazing: |dT/ds| v (the gradient in cell units along the ray) below 1e-3, or the ray within 1/20 rad of the
        # surface's tangent plane, where a float32 position's rounding moves the zero along the ray twenty-fold
        gr = np.abs((g * rdir[h]).sum(1))
        amb[h] |= (gr < _EPS) | (gr < _GRAZE * gn)
        shade = AMBIENT + (1 - AMBIENT) * np.maximum(0.0, -(nrm * rdir[h]).sum(1))
        out_depth[h] = zh
        out_normal[h] = nrm
        out_color[h] = c
        out_rgb[h] = c * shade[:, None]
    return {"depth": out_depth.reshape(C, Ho, Wo), "normal": out_normal.reshape(C, Ho, Wo, 3),
            "color": out_color.reshape(C, Ho, Wo, 3), "rgb": out_rgb.reshape(C, Ho, Wo, 3),
            "hit": hit.reshape(C, Ho, Wo), "ambiguous": amb.reshape(C, Ho, Wo)}
