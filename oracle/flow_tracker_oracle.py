"""TEST INFRASTRUCTURE -- numpy restatement of the SLAM keyframe flow tracker.  Only tests/ and tools/ may import this
module; the product path is the CUDA library (vista_slam_b200/csrc/flow.cu).

Restates, with the reference's fixed constants:
  * FlowTracker.compute_disparity / initialize_keyframe      vista_slam/flow_tracker.py:15-66
  * cv2.goodFeaturesToTrack(maxCorners=1000, qualityLevel=0.01, minDistance=8, blockSize=7), gradient size 3,
    no Harris -- OpenCV imgproc/featureselect.cpp + corner.cpp (cornerMinEigenVal)
  * cv2.calcOpticalFlowPyrLK(winSize=(21, 21), maxLevel=3, criteria=(EPS|COUNT, 30, 0.01)), flags 0,
    minEigThreshold 1e-4 -- OpenCV video/lkpyramid.cpp (buildOpticalFlowPyramid, pyrDown, calcSharrDeriv,
    LKTrackerInvoker)

Integer work (pyramids, Scharr and Sobel derivatives, box sums, the LK window sums) is exact.  The float steps are
single correctly-rounded fp32 operations in a fixed order, which the CUDA kernels reproduce bit for bit.  OpenCV sums
the box filter and the LK normal equations in float; those sums are exact here, so the oracle is bounded against
cv2 (tests/test_flow_tracker.py) rather than bit-equal to it.

Also holds the seeded frame generator of the goldens (numpy only, so a machine without cv2 regenerates the inputs)."""
import numpy as np

WIN = 21                      # winSize (21, 21)
HALF = np.float32(10.0)       # (winSize - 1) / 2
MAX_LEVEL = 3
MAX_CORNERS = 1000
MIN_DIST2 = 64                # minDistance 8, squared
QUALITY = 0.01
MIN_EIG = 1e-4                # minEigThreshold (double in OpenCV)
MAX_ITERS = 30
EPS2 = 0.01 * 0.01            # criteria.epsilon squared in double, as calcOpticalFlowPyrLK does
W_BITS = 14
FLT_EPSILON = np.float32(np.finfo(np.float32).eps)
LK_SCALE = np.float32(1.0 / (1 << 20))
# cornerMinEigenVal: Sobel scale 1 / (2^(3-1) * blockSize * 255) -> the covariance entries carry its square
EIG_SCALE2 = np.float32(1.0 / (7140.0 * 7140.0))
F32 = np.float32


def reflect101(i, n):
    """BORDER_REFLECT_101 index for -n < i < 2n - 1."""
    i = np.abs(i)
    return np.where(i >= n, 2 * (n - 1) - i, i)


# ---------------------------------------------------------------- pyramid / derivatives
def pyr_down(src):
    """cv2.pyrDown on uint8: 5x5 [1 4 6 4 1]^2 / 256 with rounding, BORDER_REFLECT_101, size ((w+1)/2, (h+1)/2)."""
    h, w = src.shape
    dh, dw = (h + 1) // 2, (w + 1) // 2
    k = np.array([1, 4, 6, 4, 1], np.int64)
    xs = reflect101(2 * np.arange(dw)[:, None] + np.arange(-2, 3)[None, :], w)
    ys = reflect101(2 * np.arange(dh)[:, None] + np.arange(-2, 3)[None, :], h)
    rows = (src.astype(np.int64)[:, xs] * k).sum(-1)           # (h, dw)
    tot = (rows[ys] * k[None, :, None]).sum(1)                  # (dh, dw)
    return ((tot + 128) >> 8).astype(np.uint8)


def num_levels(h, w):
    """Levels buildOpticalFlowPyramid keeps for winSize 21, maxLevel 3: level L exists while both sides are > 21."""
    n = 1
    while n <= MAX_LEVEL:
        w, h = (w + 1) // 2, (h + 1) // 2
        if w <= WIN or h <= WIN:
            break
        n += 1
    return n


def pyramid(img):
    levels = [np.ascontiguousarray(img, np.uint8)]
    for _ in range(num_levels(*img.shape) - 1):
        levels.append(pyr_down(levels[-1]))
    return levels


def scharr(img):
    """calcSharrDeriv: int16 (h, w, 2) = (dI/dx, dI/dy), 3-10-3 smoothing, BORDER_REFLECT_101."""
    h, w = img.shape
    s = img.astype(np.int32)
    yi, xi = np.arange(h), np.arange(w)
    up, dn = s[reflect101(yi - 1, h)], s[reflect101(yi + 1, h)]
    t0 = (up + dn) * 3 + s * 10
    t1 = dn - up
    xl, xr = reflect101(xi - 1, w), reflect101(xi + 1, w)
    dx = t0[:, xr] - t0[:, xl]
    dy = (t1[:, xr] + t1[:, xl]) * 3 + t1 * 10
    return np.stack([dx, dy], -1).astype(np.int16)


# ---------------------------------------------------------------- Shi-Tomasi corners
def sobel3(img):
    """Integer 3x3 Sobel (dx, dy), BORDER_REFLECT_101."""
    h, w = img.shape
    s = img.astype(np.int64)
    yu, yd = reflect101(np.arange(h) - 1, h), reflect101(np.arange(h) + 1, h)
    xl, xr = reflect101(np.arange(w) - 1, w), reflect101(np.arange(w) + 1, w)
    hd = s[:, xr] - s[:, xl]
    sx = hd[yu] + 2 * hd + hd[yd]
    vd = s[yd] - s[yu]
    sy = vd[:, xl] + 2 * vd + vd[:, xr]
    return sx, sy


def box7(a):
    """Unnormalised 7x7 box sum, BORDER_REFLECT_101 (exact, integer)."""
    h, w = a.shape
    r = sum(a[:, reflect101(np.arange(w) + d, w)] for d in range(-3, 4))
    return sum(r[reflect101(np.arange(h) + d, h)] for d in range(-3, 4))


def min_eigen(img):
    """cornerMinEigenVal(blockSize=7, ksize=3) with exact box sums, scaled once:
    a = sum(dx^2)/2, b = sum(dx dy), c = sum(dy^2)/2, lambda_min = (a + c) - sqrt((a - c)^2 + b^2), fp32."""
    sx, sy = sobel3(img)
    sxx, sxy, syy = box7(sx * sx), box7(sx * sy), box7(sy * sy)
    a = (sxx.astype(F32) * EIG_SCALE2) * F32(0.5)
    b = sxy.astype(F32) * EIG_SCALE2
    c = (syy.astype(F32) * EIG_SCALE2) * F32(0.5)
    d = a - c
    return (a + c) - np.sqrt(d * d + b * b)


def corner_candidates(img):
    """Thresholded local maxima of goodFeaturesToTrack, ranked: -> (ys, xs, vals) in (value desc, index desc) order."""
    h, w = img.shape
    eig = min_eigen(img)
    thr = F32(np.float64(eig.max()) * QUALITY)
    e = np.where(eig > thr, eig, F32(0))
    dil = e.copy()
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            dil[1:-1, 1:-1] = np.maximum(dil[1:-1, 1:-1], e[1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx])
    m = np.zeros((h, w), bool)
    m[1:-1, 1:-1] = (e[1:-1, 1:-1] != 0) & (e[1:-1, 1:-1] == dil[1:-1, 1:-1])
    ys, xs = np.nonzero(m)
    vals = e[ys, xs]
    order = np.lexsort((-(ys * w + xs), -vals.astype(np.float64)))
    return ys[order], xs[order], vals[order]


def _disc():
    d = np.arange(-7, 8)
    return (d[:, None] ** 2 + d[None, :] ** 2) < MIN_DIST2


DISC = _disc()


def good_features(img):
    """cv2.goodFeaturesToTrack with the reference's constants -> (N, 1, 2) float32, or None when there is no corner.
    The minimum-distance selection is the sequential greedy loop of featureselect.cpp."""
    h, w = img.shape
    ys, xs, _ = corner_candidates(img)
    acc = np.zeros((h + 14, w + 14), bool)
    out = []
    for y, x in zip(ys.tolist(), xs.tolist()):
        if (acc[y:y + 15, x:x + 15] & DISC).any():
            continue
        acc[y + 7, x + 7] = True
        out.append((x, y))
        if len(out) == MAX_CORNERS:
            break
    if not out:
        return None
    return np.array(out, np.float32).reshape(-1, 1, 2)


# ---------------------------------------------------------------- pyramidal Lucas-Kanade
def _weights(frac):
    """Bilinear fixed-point weights (W_BITS = 14): iw00..iw10 = cvRound(...) (half to even), iw11 = 2^14 - rest."""
    a, b = frac[:, 0], frac[:, 1]
    one = F32(1.0)
    s = F32(1 << W_BITS)
    w00 = np.rint(((one - a) * (one - b)) * s).astype(np.int64)
    w01 = np.rint((a * (one - b)) * s).astype(np.int64)
    w10 = np.rint(((one - a) * b) * s).astype(np.int64)
    w11 = (1 << W_BITS) - w00 - w01 - w10
    return [v[:, None, None] for v in (w00, w01, w10, w11)]


def _gather(pad, ipt):
    """Window corners (00, 01, 10, 11) at integer top-left ipt (m, 2) of a level padded by WIN on each side."""
    r = np.arange(WIN)
    yy = ipt[:, 1, None, None] + WIN + r[None, :, None]
    xx = ipt[:, 0, None, None] + WIN + r[None, None, :]
    return pad[yy, xx], pad[yy, xx + 1], pad[yy + 1, xx], pad[yy + 1, xx + 1]


def _interp(c, w, shift):
    v = c[0].astype(np.int64) * w[0] + c[1] * w[1] + c[2] * w[2] + c[3] * w[3]
    return (v + (1 << (shift - 1))) >> shift


def lk_track(prev_pyr, next_pyr, pts, prev_derivs=None):
    """cv2.calcOpticalFlowPyrLK with the reference's constants.  pts (n, 1, 2) or (n, 2) float32 ->
    (next_pts (n, 1, 2) float32, status (n, 1) uint8).  A failure clears status only at level 0; at a coarser level
    it skips that level and leaves the point's guess as it was."""
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    n = len(pts)
    status = np.ones(n, bool)
    next_pts = np.zeros((n, 2), np.float32)
    nlev = min(len(prev_pyr), len(next_pyr))
    if prev_derivs is None:
        prev_derivs = [scharr(l) for l in prev_pyr[:nlev]]
    for L in range(nlev - 1, -1, -1):
        h, w = prev_pyr[L].shape
        Ipad = np.pad(prev_pyr[L], WIN, mode="reflect").astype(np.int64)          # numpy 'reflect' = REFLECT_101
        Jpad = np.pad(next_pyr[L], WIN, mode="reflect").astype(np.int64)
        Dpad = np.pad(prev_derivs[L], ((WIN, WIN), (WIN, WIN), (0, 0))).astype(np.int64)  # zero border
        prev = pts * F32(1.0 / (1 << L))
        guess = prev.copy() if L == nlev - 1 else next_pts * F32(2.0)
        next_pts = guess.copy()
        pp = prev - HALF
        ip = np.floor(pp).astype(np.int64)
        ok = (ip[:, 0] >= -WIN) & (ip[:, 0] < w) & (ip[:, 1] >= -WIN) & (ip[:, 1] < h)
        if L == 0:
            status &= ok
        idx = np.nonzero(ok)[0]
        if len(idx) == 0:
            continue
        wts = _weights(pp[idx] - ip[idx].astype(np.float32))
        ival = _interp(_gather(Ipad, ip[idx]), wts, W_BITS - 5)
        dc = _gather(Dpad, ip[idx])
        ix = _interp([c[..., 0] for c in dc], wts, W_BITS)
        iy = _interp([c[..., 1] for c in dc], wts, W_BITS)
        A11 = (ix * ix).sum((1, 2)).astype(F32) * LK_SCALE
        A12 = (ix * iy).sum((1, 2)).astype(F32) * LK_SCALE
        A22 = (iy * iy).sum((1, 2)).astype(F32) * LK_SCALE
        D = A11 * A22 - A12 * A12
        dd = A11 - A22
        min_eig = (A22 + A11 - np.sqrt(dd * dd + (F32(4.0) * A12) * A12)) / F32(2 * WIN * WIN)
        good = ~((min_eig.astype(np.float64) < MIN_EIG) | (D < FLT_EPSILON))
        if L == 0:
            status[idx[~good]] = False
        idx, A11, A12, A22, D = idx[good], A11[good], A12[good], A22[good], D[good]
        ival, ix, iy = ival[good], ix[good], iy[good]
        Dinv = F32(1.0) / D
        nxt = next_pts[idx] - HALF
        pdelta = np.zeros_like(nxt)
        run = np.ones(len(idx), bool)
        for j in range(MAX_ITERS):
            r = np.nonzero(run)[0]
            if len(r) == 0:
                break
            inx = np.floor(nxt[r]).astype(np.int64)
            inb = (inx[:, 0] >= -WIN) & (inx[:, 0] < w) & (inx[:, 1] >= -WIN) & (inx[:, 1] < h)
            if L == 0:
                status[idx[r[~inb]]] = False
            run[r[~inb]] = False
            r, inx = r[inb], inx[inb]
            if len(r) == 0:
                break
            wj = _weights(nxt[r] - inx.astype(np.float32))
            diff = _interp(_gather(Jpad, inx), wj, W_BITS - 5) - ival[r]
            b1 = (diff * ix[r]).sum((1, 2)).astype(F32) * LK_SCALE
            b2 = (diff * iy[r]).sum((1, 2)).astype(F32) * LK_SCALE
            delta = np.stack([(A12[r] * b2 - A22[r] * b1) * Dinv[r], (A12[r] * b1 - A11[r] * b2) * Dinv[r]], -1)
            nxt[r] = nxt[r] + delta
            next_pts[idx[r]] = nxt[r] + HALF
            d64 = delta.astype(np.float64)
            conv = (d64[:, 0] * d64[:, 0] + d64[:, 1] * d64[:, 1]) <= EPS2
            s = delta + pdelta[r]
            osc = ~conv & (j > 0) & (np.abs(s[:, 0]).astype(np.float64) < 0.01) & (np.abs(s[:, 1]).astype(np.float64) < 0.01)
            next_pts[idx[r[osc]]] = next_pts[idx[r[osc]]] - delta[osc] * F32(0.5)
            run[r[conv | osc]] = False
            pdelta[r] = delta
    return next_pts.reshape(-1, 1, 2), status.astype(np.uint8).reshape(-1, 1)


# ---------------------------------------------------------------- the tracker
def mean_disparity(kf_pts, next_pts, status):
    """flow_tracker.py:41-51 as written.  kf_pts / next_pts are (N, 1, 2), so norm(axis=1) runs over the axis of size
    1 and returns |dx| and |dy| as an (M, 2) array: the result is the mean of the 2M absolute components, not the
    mean Euclidean displacement.  -> (M, mean) with mean None when M == 0."""
    st = np.asarray(status).flatten()
    good_kf, good_next = kf_pts[st == 1], next_pts[st == 1]
    if len(good_kf) == 0:
        return 0, None
    return len(good_kf), float(np.mean(np.linalg.norm(good_next - good_kf, axis=1)))


class FlowTrackerOracle:
    """flow_tracker.py's FlowTracker on the restated kernels; keeps the keyframe pyramid and derivatives."""

    def __init__(self, min_disparity):
        self.min_disparity = min_disparity
        self.reset()

    def reset(self):
        self.last_kf = None
        self.kf_pts = None
        self.kf_gray = None
        self.last_mean_disparity = None
        self.last_track = None

    def initialize_keyframe(self, image):
        self.last_kf = image
        self.kf_gray = image
        self.kf_pyr = pyramid(image)
        self.kf_derivs = [scharr(l) for l in self.kf_pyr]
        self.kf_pts = good_features(image)

    def compute_disparity(self, image):
        self.last_mean_disparity = None
        self.last_track = None
        if self.last_kf is None or self.kf_pts is None or len(self.kf_pts) < 10:
            self.initialize_keyframe(image)
            return True
        nxt, st = lk_track(self.kf_pyr, pyramid(image), self.kf_pts, self.kf_derivs)
        self.last_track = (nxt, st)
        m, mean = mean_disparity(self.kf_pts, nxt, st)
        if m < 10:
            self.initialize_keyframe(image)
            return True
        self.last_mean_disparity = mean
        if mean > self.min_disparity:
            self.initialize_keyframe(image)
            return True
        return False


# ---------------------------------------------------------------- seeded frames
def _upsample(a, H, W):
    """Bilinear resize of a coarse grid to (H, W) (align corners)."""
    h, w = a.shape
    y = np.linspace(0, h - 1, H)
    x = np.linspace(0, w - 1, W)
    y0 = np.minimum(np.floor(y).astype(int), h - 2)
    x0 = np.minimum(np.floor(x).astype(int), w - 2)
    fy, fx = (y - y0)[:, None], (x - x0)[None, :]
    a00, a01 = a[y0][:, x0], a[y0][:, x0 + 1]
    a10, a11 = a[y0 + 1][:, x0], a[y0 + 1][:, x0 + 1]
    return (a00 * (1 - fy) * (1 - fx) + a01 * (1 - fy) * fx + a10 * fy * (1 - fx) + a11 * fy * fx)


def make_scene(seed, H, W, octaves=(24, 12, 6, 3), gains=(1.0, 0.7, 0.5, 0.35)):
    """A textured float64 scene in [16, 240]: octaves of bilinearly upsampled Gaussian noise (cell size in pixels)."""
    rng = np.random.default_rng(seed)
    img = np.zeros((H, W))
    for cell, g in zip(octaves, gains):
        img += g * _upsample(rng.standard_normal((H // cell + 2, W // cell + 2)), H, W)
    img -= img.min()
    return 16.0 + 224.0 * img / img.max()


def warp_frame(scene, H, W, tx=0.0, ty=0.0, rot=0.0, zoom=1.0):
    """Frame (H, W) uint8 sampled from the scene around its centre: p_scene = c + zoom R(rot) (p - c_frame) + t,
    bilinear, rounded half to even."""
    Hs, Ws = scene.shape
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    u, v = xx - (W - 1) / 2.0, yy - (H - 1) / 2.0
    cr, sr = np.cos(rot), np.sin(rot)
    sx = (Ws - 1) / 2.0 + zoom * (cr * u - sr * v) + tx
    sy = (Hs - 1) / 2.0 + zoom * (sr * u + cr * v) + ty
    assert sx.min() >= 0 and sy.min() >= 0 and sx.max() < Ws - 1 and sy.max() < Hs - 1, "warp leaves the scene"
    x0, y0 = np.floor(sx).astype(int), np.floor(sy).astype(int)
    fx, fy = sx - x0, sy - y0
    val = (scene[y0, x0] * (1 - fx) * (1 - fy) + scene[y0, x0 + 1] * fx * (1 - fy) + scene[y0 + 1, x0] * (1 - fx) * fy
           + scene[y0 + 1, x0 + 1] * fx * fy)
    return np.clip(np.rint(val), 0, 255).astype(np.uint8)


def tie_frame():
    """64x64 zero frame with a 6x6 square of 200 at (30, 30): four exactly tied maxima at (32..33, 32..33)."""
    f = np.zeros((64, 64), np.uint8)
    f[30:36, 30:36] = 200
    return f


def checker_frame(H, W, shift=0, ramp=False):
    """A checkerboard of 4-pixel cells in the middle of a flat frame: corner candidates 4 px apart, so the greedy
    minimum-distance selection is one long chain.  ramp=True varies the contrast across x, so the chain's values
    strictly decrease instead of tying."""
    f = np.full((H, W), 96, np.float64)
    yy, xx = np.mgrid[0:H, 0:W]
    cell = (((yy + shift) // 4) + ((xx + shift) // 4)) % 2
    amp = 60.0 + (40.0 * xx / W if ramp else 0.0)
    inside = (yy >= H // 4) & (yy < 3 * H // 4) & (xx >= W // 4) & (xx < 3 * W // 4)
    f = np.where(inside, 96 + amp * (2 * cell - 1) * 0.5, f)
    return np.clip(np.rint(f), 0, 255).astype(np.uint8)


def _drift(seed, H, W, steps, margin=40, octaves=(24, 12, 6, 3), gains=(1.0, 0.7, 0.5, 0.35)):
    scene = make_scene(seed, H + 2 * margin, W + 2 * margin, octaves, gains)
    return [warp_frame(scene, H, W, *p) for p in steps]


def sequences():
    """The golden sequences: name -> list of uint8 frames (deterministic, numpy only)."""
    seqs = {}
    # (a) 224x224, slow drift crossing the 5.0 threshold several times
    steps = [(1.35 * t, 0.5 * t, 0.002 * t, 1.0 + 0.001 * t) for t in range(14)]
    seqs["a_224x224"] = _drift(11, 224, 224, steps)
    # (b) 192x256 (the non-square resolution=(256, 192) frame)
    steps = [(-1.3 * t, 0.9 * t, -0.003 * t, 1.0) for t in range(10)]
    seqs["b_192x256"] = _drift(12, 192, 256, steps)
    # (c) 168x224: only 2 pyramid levels above the base
    steps = [(1.1 * t, -0.7 * t, 0.0, 1.0 - 0.002 * t) for t in range(10)]
    seqs["c_168x224"] = _drift(13, 168, 224, steps)
    # (d) 384x512 high texture: more than 1000 uncapped corners
    steps = [(1.7 * t, 0.6 * t, 0.001 * t, 1.0) for t in range(6)]
    seqs["d_384x512"] = _drift(14, 384, 512, steps, octaves=(8, 4, 2), gains=(1.0, 0.8, 0.6))
    # (e) a large jump (points leave the frame or fall below the eigenvalue threshold), a flat frame (no corners), a
    # low-contrast pair (fewer than 10 points tracked), then a frame with a small textured patch only (a keyframe with
    # fewer than 10 corners)
    scene = make_scene(15, 224 + 240, 224 + 240)
    fr = [warp_frame(scene, 224, 224, 0.0, 0.0), warp_frame(scene, 224, 224, 2.0, 1.0),
          warp_frame(scene, 224, 224, 70.0, 55.0), warp_frame(scene, 224, 224, 71.0, 56.0)]
    soft = np.full((224, 224), 120, np.uint8)
    soft[100:124, 100:124] = warp_frame(scene, 24, 24, 0.0, 0.0)
    # a low-contrast copy of the scene: corners (the quality level is relative) whose LK windows fall below the
    # absolute eigenvalue threshold, so tracking from it leaves fewer than 10 points
    low = [np.clip(np.rint(120 + (warp_frame(scene, 224, 224, d, d) - 128.0) / 40.0), 0, 255).astype(np.uint8)
           for d in (0.0, 1.0)]
    fr += [np.full((224, 224), 120, np.uint8)] + low + [soft, soft, warp_frame(scene, 224, 224, 0.5, 0.5)]
    seqs["e_jump_224x224"] = fr
    # (f) flat frames (no corners), then tied eigenvalues and candidate chains
    flat = np.full((128, 160), 77, np.uint8)
    seqs["f_flat_ties_128x160"] = [flat, flat, checker_frame(128, 160), checker_frame(128, 160, ramp=True),
                                   checker_frame(128, 160, shift=1, ramp=True)]
    return seqs
