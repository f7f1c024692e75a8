"""float64 oracle of the TSDF fusion and marching cubes of vista_slam_b200/fusion.py (csrc/fusion.cu), written from the
semantics in fusion.py's docstring.  Marching cubes reads the generated table, vista_slam_b200/csrc/mc_table.h.

fuse(maps, conf_thres, voxel, trunc) -> volume dict; marching_cubes(bricks, tsdf, weight, color, voxel, min_weight)
-> mesh dict with vertex_keys [Nv,4] (i, j, k, axis of the lattice edge each vertex lies on).  Brick lists are sorted
by key (z, then y, then x).  Besides the values, fuse reports what float32 rounding may legitimately change:
`sure` and `maybe` brick sets (cube faces within 1e-4 v of a brick boundary), and per sample `ambiguous` (a projection
within 1e-4 px of a pixel rounding boundary, or an sdf within 1e-5 relative of -trunc, in some view)."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BRICK = 8
BIAS = 1 << 20


def mc_table():
    """(num_tris [256], tris [256][3 max]) parsed from csrc/mc_table.h."""
    with open(os.path.join(ROOT, "vista_slam_b200", "csrc", "mc_table.h")) as f:
        text = f.read()
    num = re.search(r"kMcNumTris\[256\] = \{(.*?)\};", text, re.S).group(1)
    tris = re.search(r"kMcTris\[256\]\[\d+\] = \{(.*?)\n\};", text, re.S).group(1)
    num = np.array([int(x) for x in re.findall(r"-?\d+", num)], np.int64)
    rows = [[int(x) for x in re.findall(r"-?\d+", r.split("//")[0])] for r in tris.strip().splitlines()]
    return num, np.array(rows, np.int64)


def key(b):
    b = np.asarray(b, np.int64) + BIAS
    return (b[..., 2] << 42) | (b[..., 1] << 21) | b[..., 0]


def unkey(k):
    k = np.asarray(k, np.int64)
    return np.stack([(k >> s) & ((1 << 21) - 1) for s in (0, 21, 42)], -1) - BIAS


def _used(maps, conf_thres):
    d = maps["depth"].astype(np.float64) * maps["scale"].reshape(-1, 1, 1).astype(np.float64)
    return d, (maps["conf"] > conf_thres) & (d > 0)


def _points(maps, conf_thres):
    """World points [n,3] of the used pixels (float64)."""
    d, used = _used(maps, conf_thres)
    V, H, W = d.shape
    out = []
    for v in range(V):
        K = maps["intri"][v].astype(np.float64)
        P = maps["pose"][v].astype(np.float64)
        r, c = np.nonzero(used[v])
        with np.errstate(invalid="ignore"):  # an infinite depth gives NaN coordinates, skipped by fuse
            cam = (np.linalg.inv(K) @ np.stack([c, r, np.ones_like(c)]).astype(np.float64)) * d[v, r, c]
            out.append((P[:3, :3] @ cam).T + P[:3, 3])
    return np.concatenate(out) if out else np.zeros((0, 3))


def _brick_set(p, tau, bs, grow):
    lo = np.floor((p - tau - grow) / bs).astype(np.int64)
    hi = np.floor((p + tau + grow) / bs).astype(np.int64)
    keys = set()
    for q in range(len(p)):
        for bz in range(lo[q, 2], hi[q, 2] + 1):
            for by in range(lo[q, 1], hi[q, 1] + 1):
                for bx in range(lo[q, 0], hi[q, 0] + 1):
                    keys.add(int(key((bx, by, bz))))
    return keys


def fuse(maps, conf_thres, voxel, trunc=None):
    maps = {k: np.asarray(v) for k, v in maps.items()}
    v32 = np.float32(voxel)
    v = float(v32)
    tau = 4 * v if trunc is None else float(np.float32(trunc))
    bs = BRICK * v
    p = _points(maps, conf_thres)
    ok = np.isfinite(p).all(1)
    with np.errstate(invalid="ignore"):
        ok &= (np.floor((p - tau) / bs) >= -BIAS).all(1) & (np.floor((p + tau) / bs) <= BIAS - 1).all(1)
    p = p[ok]
    keys = np.array(sorted(_brick_set(p, tau, bs, 0.0)), np.int64)
    sure = _brick_set(p, tau, bs, -1e-4 * v)
    maybe = _brick_set(p, tau, bs, 1e-4 * v)
    vol = integrate(maps, conf_thres, v32, tau, keys)
    vol.update(bricks=unkey(keys).astype(np.int32), keys=keys, sure=sure, maybe=maybe)
    return vol


def sample_coords(keys):
    """Lattice (i, j, k) [B,8,8,8,3] of every sample of the bricks."""
    b = unkey(keys)
    z, y, x = np.meshgrid(np.arange(BRICK), np.arange(BRICK), np.arange(BRICK), indexing="ij")
    loc = np.stack([x, y, z], -1)
    return b[:, None, None, None, :] * BRICK + loc[None]


def integrate(maps, conf_thres, voxel, tau, keys):
    v32 = np.float32(voxel)
    ijk = sample_coords(keys)
    X = (ijk.astype(np.float32) * v32).astype(np.float64).reshape(-1, 3)  # the float32 lattice
    n = len(X)
    T, Wt, C = np.zeros(n), np.zeros(n), np.zeros((n, 3))
    amb = np.zeros(n, bool)
    d, used = _used(maps, conf_thres)
    V, H, W = d.shape
    for vv in range(V):
        P = maps["pose"][vv].astype(np.float64)
        w2c = np.linalg.inv(P)
        K = maps["intri"][vv].astype(np.float64)
        c = X @ w2c[:3, :3].T + w2c[:3, 3]
        front = c[:, 2] > 0
        with np.errstate(divide="ignore", invalid="ignore"):
            u = (c @ K[0]) / c[:, 2]
            r = (c @ K[1]) / c[:, 2]
            fu, fr = np.floor(u + 0.5), np.floor(r + 0.5)
            near_edge = (np.abs(u + 0.5 - np.round(u + 0.5)) < 1e-4) | (np.abs(r + 0.5 - np.round(r + 0.5)) < 1e-4)
            inside = front & (fu >= 0) & (fu < W) & (fr >= 0) & (fr < H)
            amb |= front & near_edge & (fu >= -1) & (fu <= W) & (fr >= -1) & (fr <= H)
        idx = np.flatnonzero(inside)
        col, row = fu[idx].astype(np.int64), fr[idx].astype(np.int64)
        ok = used[vv, row, col]
        idx, col, row = idx[ok], col[ok], row[ok]
        sdf = d[vv, row, col] - c[idx, 2]
        amb[idx] |= np.abs(sdf + tau) <= 1e-5 * tau
        keep = sdf >= -tau
        idx, col, row, sdf = idx[keep], col[keep], row[keep], sdf[keep]
        t = np.minimum(1.0, sdf / tau)
        rgb = (maps["images"][vv][:, row, col].T.astype(np.float64) + 1.0) / 2.0
        T[idx] = (T[idx] * Wt[idx] + t) / (Wt[idx] + 1)
        C[idx] = (C[idx] * Wt[idx, None] + rgb) / (Wt[idx, None] + 1)
        Wt[idx] += 1
    B = len(keys)
    return {"tsdf": T.reshape(B, 8, 8, 8), "weight": Wt.reshape(B, 8, 8, 8), "color": C.reshape(B, 8, 8, 8, 3),
            "ambiguous": amb.reshape(B, 8, 8, 8)}


def _edge_lower(e):
    axis, o0, o1 = e >> 2, e & 1, e >> 1 & 1
    return [(0, o0, o1), (o0, 0, o1), (o0, o1, 0)][axis], axis


def marching_cubes(bricks, tsdf, weight, color, voxel, min_weight=1):
    """The mesh of fusion.marching_cubes in float64 (float32 lattice positions), and vertex_keys [Nv,4] and, per face,
    the lattice cube it came from (face_cubes [Nf,3])."""
    num, tris = mc_table()
    bricks = np.asarray(bricks, np.int64)
    keys = key(bricks)
    assert (np.diff(keys) > 0).all()
    B = len(keys)
    T = np.asarray(tsdf, np.float64).reshape(-1)
    Wt = np.asarray(weight, np.float64).reshape(-1)
    Cl = np.asarray(color, np.float64).reshape(-1, 3)
    v32 = np.float32(voxel)
    ijk = sample_coords(keys).reshape(-1, 3)

    def lookup(q):  # global sample index of lattice points q [n,3], -1 when missing
        b = np.floor_divide(q, BRICK)
        inr = ((b >= -BIAS) & (b < BIAS)).all(1)
        k = key(np.where(inr[:, None], b, 0))
        pos = np.searchsorted(keys, k)
        pos_c = np.minimum(pos, max(B - 1, 0))
        hit = inr & (pos < B) & (keys[pos_c] == k) if B else np.zeros(len(q), bool)
        loc = q - b * BRICK
        return np.where(hit, pos_c * 512 + loc[:, 2] * 64 + loc[:, 1] * 8 + loc[:, 0], -1)

    n = B * 512
    corners = np.stack([lookup(ijk + np.array([c & 1, c >> 1 & 1, c >> 2])) for c in range(8)], 1)  # [n,8]
    valid = (corners >= 0).all(1)
    safe = np.where(corners >= 0, corners, 0)
    valid &= (Wt[safe] >= min_weight).all(1)
    case = ((T[safe] < 0).astype(np.int64) << np.arange(8)).sum(1)
    case = np.where(valid, case, 0)
    ntri = num[case]
    bits = np.zeros(n, np.int64)
    for e in range(12):
        (ox, oy, oz), axis = _edge_lower(e)
        lc = ox | oy << 1 | oz << 2
        uc = lc | 1 << axis
        cross = (ntri > 0) & (((case >> lc) ^ (case >> uc)) & 1).astype(bool)
        np.bitwise_or.at(bits, corners[cross, lc], 1 << axis)
    cnt = sum((bits >> a) & 1 for a in range(3))
    vbase = np.concatenate([[0], np.cumsum(cnt)[:-1]]) if n else np.zeros(0, np.int64)
    verts, vcols, vkeys = [], [], []
    for s in np.flatnonzero(bits):
        for axis in range(3):
            if not bits[s] >> axis & 1:
                continue
            q = ijk[s].copy()
            q[axis] += 1
            nb = lookup(q[None])[0]
            f = T[s] / (T[s] - T[nb])
            pa = (ijk[s].astype(np.float32) * v32).astype(np.float64)
            pb = (q.astype(np.float32) * v32).astype(np.float64)
            verts.append(pa + f * (pb - pa))
            vcols.append(Cl[s] + f * (Cl[nb] - Cl[s]))
            vkeys.append((*ijk[s], axis))
    faces, fcubes = [], []
    for s in np.flatnonzero(ntri):
        cs = case[s]
        for k in range(ntri[s]):
            tri = []
            for j in range(3):
                (ox, oy, oz), axis = _edge_lower(tris[cs, 3 * k + j])
                g = corners[s, ox | oy << 1 | oz << 2]
                tri.append(vbase[g] + bin(bits[g] & ((1 << axis) - 1)).count("1"))
            faces.append(tri)
            fcubes.append(ijk[s])
    return {"vertices": np.array(verts, np.float64).reshape(-1, 3), "vertex_colors": np.array(vcols).reshape(-1, 3),
            "faces": np.array(faces, np.int64).reshape(-1, 3), "vertex_keys": np.array(vkeys, np.int64).reshape(-1, 4),
            "face_cubes": np.array(fcubes, np.int64).reshape(-1, 3)}
