"""Float64 restatement of the multi-view depth consistency check (view_consistency_check,
vista_slam/utils/slam_utils.py:346-419), written from its description, with a per-test ambiguity flag.

For view i, pixel (x, y) and each neighbour j in [max(0, i - 4), min(n - 1, i + 4)], j != i:
    p = T_i [K_i^-1 [x y 1]^T d_i; 1],   c = (T_j^-1 [p; 1])_xyz,   z = max(c_z, 1e-6 in float32)
    (u, v) = (K_j c)_xy / (K_j c)_z                  (the unclamped c)
    s = bilinear sample of depth j at (u, v) with zero padding (grid_sample, align_corners=True)
    agree = |s - z| < threshold and z > 0
Quirks kept: a finite (u, v) outside the image samples 0 (so an off-image point agrees when z < threshold); a
coordinate that float32 makes NaN or infinite -- a zero third component, or a value whose grid_sample unnormalisation
(g + 1) (W - 1) / 2 overflows -- samples NaN and never agrees.

Ambiguity.  Every float32 implementation (the reference on the CPU, the kernel) computes each quantity q with a
rounding error bounded to first order by err(q) = 8 u m(q), u = 2^-24, where m(q) is q's magnitude sum (the same
expression over absolute values): a dot product of k terms errs by at most about k u times its magnitude sum, the
inverses of K and T add a few u relative to their entries, and the factor 8 covers the op count of each stage and
the inputs' propagated errors, which are carried stage by stage:
    cam      m = |K_i^-1| [x y 1] |d|                 err = 8 u m
    p        m = |T_i| [m_cam; 1]                     err = |T_i| err_cam + 8 u m
    c        m = |T_j^-1| [m_p; 1]                    err = |T_j^-1| err_p + 8 u m
    (uu, vv, ww) = K_j c alike; u = uu / ww errs by (err_uu + |u| err_ww) / |ww| + 8 u (|u| + W)
The sample is continuous in (u, v) (zero padding included) with slope at most L, the spread of depth j over the 4 x 4
corners around the cell (zeros outside), so it errs by L (err_u + err_v) + 8 u max|corner|.  A test is ambiguous when
  * | |s - z| - threshold | <= err_s + err_z + 8 u threshold  (the comparison could go either way), or
  * |ww| <= err_ww with a nonzero err_ww (float32 may or may not divide by zero), or |u|, |v| near the float32 overflow of
    the unnormalisation, or
  * |c_z - 1e-6| <= err_z (the clamp may or may not apply).
For the scenes of the tests err is of the order of 1e-6 to 1e-5 times (threshold + |z|); far below the 1e-4 scale."""
import numpy as np

U = 2.0 ** -24
CLAMP = float(np.float32(1e-6))
FMAX = float(np.finfo(np.float32).max)


def _window(i, n):
    return [j for j in range(max(0, i - 4), min(n, i + 5)) if j != i]


def _bilinear(d, u, v):
    """Sample of map d [H,W] at (u, v) with zero padding (align_corners=True pixel coordinates), the spread of the 4 x 4
    corners around the cell and their largest magnitude; u, v finite float64 arrays."""
    H, W = d.shape
    pad = np.zeros((H + 4, W + 4))
    pad[2:H + 2, 2:W + 2] = d
    big = 1e9
    u = np.clip(u, -big, big)
    v = np.clip(v, -big, big)
    x0, y0 = np.floor(u), np.floor(v)
    fx, fy = u - x0, v - y0
    # cell corners (x0 .. x0 + 1, y0 .. y0 + 1) and the ring around them, in the padded map; far-off cells read zeros
    xi = np.clip(x0, -2, W + 1).astype(np.int64) + 2
    yi = np.clip(y0, -2, H + 1).astype(np.int64) + 2
    far = (x0 < -2) | (x0 > W) | (y0 < -2) | (y0 > H)

    def at(dy, dx):
        yy, xx = np.clip(yi + dy, 0, H + 3), np.clip(xi + dx, 0, W + 3)
        return np.where(far, 0.0, pad[yy, xx])
    s = (at(0, 0) * (1 - fx) * (1 - fy) + at(0, 1) * fx * (1 - fy) + at(1, 0) * (1 - fx) * fy + at(1, 1) * fx * fy)
    ring = np.stack([at(dy, dx) for dy in (-1, 0, 1, 2) for dx in (-1, 0, 1, 2)])
    return s, ring.max(0) - ring.min(0), np.abs(ring).max(0)


def view_consistency(depth, intrinsics, poses, threshold=0.05):
    """depth [n,H,W], intrinsics [n,3,3], poses [n,4,4] (camera-to-world) -> (count int32 [n,H,W], ambiguous bool
    [n,H,W,8]: per pixel and window slot (the neighbours in increasing index, then False))."""
    depth = np.asarray(depth, np.float64)
    K = np.asarray(intrinsics, np.float64)
    T = np.asarray(poses, np.float64)
    n, H, W = depth.shape
    thr = float(np.float32(threshold))
    count = np.zeros((n, H, W), np.int32)
    amb = np.zeros((n, H, W, 8), bool)
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    pix = np.stack([xx, yy, np.ones_like(xx)], -1).reshape(-1, 3)
    for i in range(n):
        d = depth[i].reshape(-1, 1)
        Ki = np.linalg.inv(K[i])
        cam = (pix @ Ki.T) * d
        m_cam = (pix @ np.abs(Ki).T) * np.abs(d)
        e_cam = 8 * U * m_cam
        Ti = T[i]
        p = cam @ Ti[:3, :3].T + Ti[:3, 3]
        m_p = m_cam @ np.abs(Ti[:3, :3]).T + np.abs(Ti[:3, 3])
        e_p = e_cam @ np.abs(Ti[:3, :3]).T + 8 * U * m_p
        with np.errstate(all="ignore"):
            for slot, j in enumerate(_window(i, n)):
                Tj = np.linalg.inv(T[j])
                c = p @ Tj[:3, :3].T + Tj[:3, 3]
                m_c = m_p @ np.abs(Tj[:3, :3]).T + np.abs(Tj[:3, 3])
                e_c = e_p @ np.abs(Tj[:3, :3]).T + 8 * U * m_c
                z = np.maximum(c[:, 2], CLAMP)
                e_z = e_c[:, 2]
                q = c @ K[j].T
                m_q = m_c @ np.abs(K[j]).T
                e_q = e_c @ np.abs(K[j]).T + 8 * U * m_q
                ww = q[:, 2]
                u, v = q[:, 0] / ww, q[:, 1] / ww
                e_u = (e_q[:, 0] + np.abs(u) * e_q[:, 2]) / np.abs(ww) + 8 * U * (np.abs(u) + W)
                e_v = (e_q[:, 1] + np.abs(v) * e_q[:, 2]) / np.abs(ww) + 8 * U * (np.abs(v) + H)
                # float32 finiteness of the grid_sample coordinate: u itself, u / (W - 1) * 2 and the unnormalised value
                lim_u = FMAX * min(1.0, (W - 1) / 2.0)
                lim_v = FMAX * min(1.0, (H - 1) / 2.0)
                fin = np.isfinite(u) & np.isfinite(v) & (np.abs(u) < lim_u) & (np.abs(v) < lim_v)
                near_lim = (np.abs(np.abs(u) - lim_u) <= 1e-5 * lim_u) | (np.abs(np.abs(v) - lim_v) <= 1e-5 * lim_v)
                s = np.full(H * W, np.nan)
                L = np.zeros(H * W)
                big = np.zeros(H * W)
                if fin.any():
                    s[fin], L[fin], big[fin] = _bilinear(depth[j], u[fin], v[fin])
                err = np.abs(s - z)
                agree = fin & (err < thr) & (z > 0)
                e_s = L * (np.nan_to_num(e_u, posinf=np.inf) + np.nan_to_num(e_v, posinf=np.inf)) + 8 * U * big
                a = fin & (np.abs(err - thr) <= e_s + e_z + 8 * U * thr)
                a |= (np.abs(ww) <= e_q[:, 2]) & (e_q[:, 2] > 0)
                a |= near_lim
                a |= np.abs(c[:, 2] - CLAMP) <= e_z
                count[i] += agree.reshape(H, W).astype(np.int32)
                amb[i, :, :, slot] = a.reshape(H, W)
    return count, amb


def _rot(axis_angle):
    a = np.asarray(axis_angle, np.float64)
    t = np.linalg.norm(a)
    if t == 0:
        return np.eye(3)
    k = a / t
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(t) * Kx + (1 - np.cos(t)) * Kx @ Kx


def raycast_scene(seed, n, H, W, holes=True):
    """n views of a box room [-2, 2] x [-1.5, 1.5] x [-1, 6] with a sphere in it, ray cast along a wobbling path
    that looks down +z: depth [n,H,W] (camera z of the first hit), intrinsics [n,3,3] with non-square pixels and
    non-integer principal points, poses [n,4,4] camera-to-world; float32.  With holes, a few depth-0 blocks per view."""
    rng = np.random.default_rng(seed)
    depth = np.zeros((n, H, W), np.float32)
    K = np.zeros((n, 3, 3), np.float32)
    T = np.zeros((n, 4, 4), np.float32)
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    centre, radius = np.array([0.3, 0.2, 3.5]), 0.8
    for v in range(n):
        fx = W * (0.8 + 0.2 * rng.random())
        fy = fx * (1.1 + 0.1 * rng.random())
        cx, cy = (W - 1) / 2 + rng.uniform(-1.3, 1.3), (H - 1) / 2 + rng.uniform(-1.3, 1.3)
        Kv = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
        a = 0.15 * v
        R = _rot([0.05 * np.sin(a) + 0.02 * rng.standard_normal(), 0.25 * np.sin(0.7 * a) + 0.02 * rng.standard_normal(),
                  0.03 * rng.standard_normal()])
        t = np.array([0.6 * np.sin(a), 0.2 * np.cos(1.3 * a), -0.5 + 0.08 * v + 0.02 * rng.standard_normal()])
        Tv = np.eye(4)
        Tv[:3, :3], Tv[:3, 3] = R, t
        Tv = Tv.astype(np.float32)
        Kd, Td = Kv.astype(np.float64), Tv.astype(np.float64)
        ray = np.stack([xx, yy, np.ones_like(xx)], -1) @ np.linalg.inv(Kd).T  # camera rays with z = 1
        dirs = ray @ Td[:3, :3].T
        o = Td[:3, 3]
        best = np.full((H, W), np.inf)
        lo, hi = np.array([-2.0, -1.5, -1.0]), np.array([2.0, 1.5, 6.0])
        for ax in range(3):
            for plane in (lo[ax], hi[ax]):
                with np.errstate(all="ignore"):
                    s = (plane - o[ax]) / dirs[..., ax]
                best = np.where((s > 1e-3) & (s < best), s, best)
        oc = o - centre
        b = (dirs * oc).sum(-1)
        a2 = (dirs * dirs).sum(-1)
        disc = b * b - a2 * ((oc * oc).sum() - radius * radius)
        with np.errstate(invalid="ignore"):
            s = (-b - np.sqrt(disc)) / a2
        best = np.where((disc > 0) & (s > 1e-3) & (s < best), s, best)
        d = best.astype(np.float32)  # rays have camera z = 1, so the ray parameter is the camera z
        if holes:
            for _ in range(2):
                r0, c0 = rng.integers(0, H - 3), rng.integers(0, W - 3)
                d[r0:r0 + 3, c0:c0 + 3] = 0
        depth[v], K[v], T[v] = d, Kv, Tv
    return depth, K, T
