"""numpy restatement of vista_slam/loop_detector.py::LoopDetector: cv2.ORB_create() defaults, DBoW3's vocabulary files,
BowVector transform / L1 normalisation, L1Scoring::score and detect_loop.

Every stage is written the way the library computes it, so the CUDA kernels (csrc/orb.cu, csrc/bow.cu) can be compared
with it bit for bit, and it is compared with cv2 4.13 / the reference through tests/golden/loop.npz.

ORB (OpenCV modules/features2d/src/orb.cpp, detectAndCompute(gray, None), nfeatures 500, scaleFactor 1.2, nlevels 8,
edgeThreshold 31, firstLevel 0, WTA_K 2, HARRIS_SCORE, patchSize 31, fastThreshold 20):
  1. level sizes cvRound(side / 1.2f^l); level l > 0 is resize(level l-1, INTER_LINEAR_EXACT): 8-bit fixed-point
     weights from a double source coordinate, (sum + 2^15) >> 16;
  2. FAST-9 (threshold 20) with 3x3 non-max suppression on the FAST score, on each level;
  3. points closer than 31 px to a level's border are dropped;
  4. retainBest(2 n_l) on the FAST score, Harris response (7x7 block of Sobel products, k = 0.04, fp32 expression),
     retainBest(n_l) on it.  retainBest keeps every point tied with the n-th best, so the kept set is deterministic;
  5. intensity-centroid angle over the radius-15 disc of the unsmoothed level, cv::fastAtan2;
  6. each level is smoothed by GaussianBlur(7x7, sigma 2, REFLECT_101).  The level is a view into ORB's padded pyramid
     buffer, so OpenCV does not take the fixed-point path a whole 8-bit image gets but its generic separable filter
     with the fp32 kernel getGaussianKernel(7, 2): a row pass accumulated left to right with fused multiply-adds, and a
     symmetric column pass (centre tap, then (above + below) * tap with fused multiply-adds), rounded half to even
     (cv2.sepFilter2D gives the same image);
  7. rBRIEF: 256 pair tests of the smoothed level at the pattern points rotated by the angle, fp32 products and
     cvRound, packed LSB first into 32 bytes.
Output order is canonical: (level, y, x) ascending (cv2's order is libstdc++ nth_element's).
"""
import math
import os
import re
import struct

import numpy as np

NFEATURES, NLEVELS, EDGE_THRESHOLD, PATCH_SIZE, FAST_THRESHOLD = 500, 8, 31, 31, 20
SCALE_FACTOR = float(np.float32(1.2))  # ORB::create takes the scale factor as a float
HARRIS_K = np.float32(0.04)
HALF_PATCH = PATCH_SIZE // 2
# cv::getGaussianKernel(7, 2, CV_32F)
GAUSS_F32 = np.array([float.fromhex(h) for h in ("0x1.1f5f62p-4", "0x1.0c70fcp-3", "0x1.869472p-3", "0x1.ba95c0p-3",
                                                 "0x1.869472p-3", "0x1.0c70fcp-3", "0x1.1f5f62p-4")], np.float32)

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATTERN_H = os.path.join(_HERE, "..", "vista_slam_b200", "csrc", "orb_pattern.h")

f32 = np.float32


def orb_pattern():
    """(512, 2) int32 pattern points (x, y), read from the committed header."""
    with open(_PATTERN_H) as f:
        body = f.read().split("{", 1)[1].split("}", 1)[0]
    return np.array([int(v) for v in re.findall(r"-?\d+", body)], np.int32).reshape(512, 2)


def level_scales():
    return [f32(math.pow(SCALE_FACTOR, l)) for l in range(NLEVELS)]


def level_sizes(H, W):
    out = []
    for s in level_scales():
        out.append((int(np.rint(f32(H) / s)), int(np.rint(f32(W) / s))))
    return out


def features_per_level(nfeatures=NFEATURES):
    factor = f32(1.0 / SCALE_FACTOR)
    nd = f32(f32(nfeatures) * (f32(1) - factor)) / f32(f32(1) - f32(math.pow(float(factor), NLEVELS)))
    out, total = [], 0
    for _ in range(NLEVELS - 1):
        n = int(np.rint(nd))
        out.append(n)
        total += n
        nd = f32(nd * factor)
    out.append(max(nfeatures - total, 0))
    return out


# ---- primitives ---------------------------------------------------------------------------------------------------

def _linear_exact_coeffs(src, dst):
    """(offset, w0, w1) per output sample of resize_bitExact / interpolationLinear: 8-bit fixed-point weights."""
    scale = 1.0 / (float(dst) / float(src))
    ofs = np.zeros(dst, np.int64)
    w = np.zeros((dst, 2), np.int64)
    for i in range(dst):
        fval = scale * (float(i) + 0.5) - 0.5
        iv = math.floor(fval)
        if iv >= 0 and src > 1 and iv < src - 1:
            c1 = int(np.rint((fval - iv) * 256.0))
            ofs[i], w[i] = iv, (256 - c1, c1)
        elif iv >= 0 and src > 1:
            ofs[i], w[i] = src - 1, (256, 0)
        else:
            ofs[i], w[i] = 0, (256, 0)
    return ofs, w


def resize_linear_exact(img, h, w):
    """cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR_EXACT) for a uint8 single-channel image."""
    H, W = img.shape
    if (h, w) == (H, W):
        return img.copy()
    xo, xw = _linear_exact_coeffs(W, w)
    yo, yw = _linear_exact_coeffs(H, h)
    src = img.astype(np.int64)
    xo1 = np.minimum(xo + 1, W - 1)
    rows = src[:, xo] * xw[:, 0] + src[:, xo1] * xw[:, 1]            # (H, w), scale 2^8
    yo1 = np.minimum(yo + 1, H - 1)
    v = rows[yo] * yw[:, 0:1] + rows[yo1] * yw[:, 1:2]                # (h, w), scale 2^16
    return np.minimum((v + (1 << 15)) >> 16, 255).astype(np.uint8)


def _reflect101(i, n):
    i = np.abs(i)
    return np.where(i >= n, 2 * (n - 1) - i, i)


def _fma(a, b, c):
    """fp32 fused multiply-add, correctly rounded.  a * b is exact in fp64 (two 24-bit significands); the fp64 sum
    s = p + c is rounded, with the exact error e from TwoSum.  Rounding s to fp32 gives the correct result unless s
    lies exactly halfway between two fp32 values (fp32 midpoints are fp64 numbers, so the exact sum cannot cross one
    without s landing on it); then e != 0 decides the side."""
    p = np.asarray(a, np.float64) * np.float64(b)
    c = np.asarray(c, np.float64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    d = s - r.astype(np.float64)
    toward = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf))).astype(np.float32)
    tie = (d != 0) & (np.abs(d) * 2 == np.abs(toward.astype(np.float64) - r.astype(np.float64)))
    return np.where(tie & (e != 0) & ((e > 0) == (d > 0)), toward, r).astype(np.float32)


def gaussian_blur_orb(img):
    """ORB's in-pyramid GaussianBlur(7x7, 2, REFLECT_101) of one level (see the module docstring, step 6)."""
    H, W = img.shape
    src = img.astype(np.float32)
    xs, ys = np.arange(W), np.arange(H)
    R = f32(GAUSS_F32[0] * src[:, _reflect101(xs - 3, W)])
    for i in range(1, 7):
        R = _fma(src[:, _reflect101(xs + i - 3, W)], GAUSS_F32[i], R)
    S = f32(R * GAUSS_F32[3])
    for d in range(1, 4):
        S = _fma(f32(R[_reflect101(ys + d, H)] + R[_reflect101(ys - d, H)]), GAUSS_F32[3 + d], S)
    return np.clip(np.rint(S), 0, 255).astype(np.uint8)


def fast_atan2(y, x):
    """cv::fastAtan2 in fp32 (degrees in [0, 360))."""
    y, x = f32(y), f32(x)
    c180 = f32(180.0 / math.pi)
    p1, p3, p5, p7 = (f32(f32(v) * c180) for v in (0.9997878412794807, -0.3258083974640975, 0.1555786518463281,
                                                   -0.04432655554792128))
    ax, ay = np.abs(x), np.abs(y)
    eps = f32(np.finfo(np.float64).eps)
    big = ax >= ay
    with np.errstate(invalid="ignore", divide="ignore"):
        c = np.where(big, ay / f32(ax + eps), ax / f32(ay + eps)).astype(np.float32)
    c2 = f32(c * c)
    a = f32(f32(f32(f32(f32(f32(f32(p7 * c2) + p5) * c2) + p3) * c2) + p1) * c)
    a = np.where(big, a, f32(f32(90) - a)).astype(np.float32)
    a = np.where(x < 0, f32(180) - a, a).astype(np.float32)
    a = np.where(y < 0, f32(360) - a, a).astype(np.float32)
    return a


_CIRCLE = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1),
           (-3, 0), (-3, 1), (-2, 2), (-1, 3)]  # (dx, dy), OpenCV's makeOffsets(pixel, step, 16)


def fast_scores(img, threshold=FAST_THRESHOLD):
    """FAST-9 score map: cornerScore<16> at corners, 0 elsewhere (and in the 3-pixel frame)."""
    H, W = img.shape
    out = np.zeros((H, W), np.int32)
    if H < 7 or W < 7:
        return out
    v = img[3:H - 3, 3:W - 3].astype(np.int32)
    d = np.stack([v - img[3 + dy:H - 3 + dy, 3 + dx:W - 3 + dx].astype(np.int32) for dx, dy in _CIRCLE])
    dd = np.concatenate([d, d[:8]])
    A = np.full(v.shape, -1 << 20, np.int32)
    B = np.full(v.shape, -1 << 20, np.int32)
    for k in range(16):
        A = np.maximum(A, dd[k:k + 9].min(0))
        B = np.maximum(B, (-dd[k:k + 9]).min(0))
    corner = (A > threshold) | (B > threshold)
    score = np.maximum(np.maximum(A, B), threshold) - 1
    out[3:H - 3, 3:W - 3] = np.where(corner, score, 0)
    return out


def fast_nms(scores):
    """Corners whose score is strictly larger than all 8 neighbours' -> (ys, xs, score)."""
    H, W = scores.shape
    p = np.pad(scores, 1)
    keep = scores > 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dy or dx:
                keep &= scores > p[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]
    ys, xs = np.nonzero(keep)
    return ys, xs, scores[ys, xs]


def retain_best_mask(resp, n):
    """KeyPointsFilter::retainBest as a set: keep every point whose response is >= the n-th largest."""
    resp = np.asarray(resp)
    if len(resp) <= n:
        return np.ones(len(resp), bool)
    greater = (resp[None, :] > resp[:, None]).sum(1)
    return greater < n


def harris_responses(img, ys, xs):
    """HarrisResponses(blockSize 7, k 0.04): int sums, fp32 final expression."""
    ys, xs = np.asarray(ys), np.asarray(xs)
    I = img.astype(np.int32)
    a = np.zeros(len(ys), np.int64)
    b = np.zeros(len(ys), np.int64)
    c = np.zeros(len(ys), np.int64)
    for i in range(-3, 4):
        for j in range(-3, 4):
            y, x = ys + i, xs + j
            Ix = (I[y, x + 1] - I[y, x - 1]) * 2 + (I[y - 1, x + 1] - I[y - 1, x - 1]) + (I[y + 1, x + 1] - I[y + 1, x - 1])
            Iy = (I[y + 1, x] - I[y - 1, x]) * 2 + (I[y + 1, x - 1] - I[y - 1, x - 1]) + (I[y + 1, x + 1] - I[y - 1, x + 1])
            a += Ix * Ix
            b += Iy * Iy
            c += Ix * Iy
    scale = f32(f32(1) / f32(f32(4 * 7) * f32(255)))
    s4 = f32(f32(f32(scale * scale) * scale) * scale)
    fa, fb, fc = a.astype(np.float32), b.astype(np.float32), c.astype(np.float32)
    t1 = f32(fa * fb)
    t2 = f32(fc * fc)
    sab = f32(fa + fb)
    t3 = f32(f32(HARRIS_K * sab) * sab)
    return f32(f32(f32(t1 - t2) - t3) * s4)


def _umax():
    vmax = math.floor(HALF_PATCH * math.sqrt(2.0) / 2 + 1)
    vmin = math.ceil(HALF_PATCH * math.sqrt(2.0) / 2)
    u = [0] * (HALF_PATCH + 2)
    for v in range(vmax + 1):
        u[v] = int(np.rint(math.sqrt(float(HALF_PATCH * HALF_PATCH - v * v))))
    v0 = 0
    for v in range(HALF_PATCH, vmin - 1, -1):
        while u[v0] == u[v0 + 1]:
            v0 += 1
        u[v] = v0
        v0 += 1
    return u


UMAX = _umax()


def ic_angles(img, ys, xs):
    """Intensity-centroid angle (ICAngles) in degrees, cv::fastAtan2(m01, m10)."""
    I = img.astype(np.int64)
    ys, xs = np.asarray(ys), np.asarray(xs)
    m01 = np.zeros(len(ys), np.int64)
    m10 = np.zeros(len(ys), np.int64)
    for u in range(-HALF_PATCH, HALF_PATCH + 1):
        m10 += u * I[ys, xs + u]
    for v in range(1, HALF_PATCH + 1):
        vs = np.zeros(len(ys), np.int64)
        d = UMAX[v]
        for u in range(-d, d + 1):
            p, m = I[ys + v, xs + u], I[ys - v, xs + u]
            vs += p - m
            m10 += u * (p + m)
        m01 += v * vs
    return fast_atan2(m01.astype(np.float32), m10.astype(np.float32))


def rbrief(blurred, cy, cx, angle_deg, pattern=None):
    """(N, 32) uint8 rBRIEF descriptors sampled from the smoothed level around (cy, cx)."""
    pat = orb_pattern() if pattern is None else pattern
    ang = f32(np.asarray(angle_deg, np.float32) * f32(math.pi / 180.0))
    ca = np.cos(ang.astype(np.float64)).astype(np.float32)
    sa = np.sin(ang.astype(np.float64)).astype(np.float32)
    px, py = pat[:, 0].astype(np.float32), pat[:, 1].astype(np.float32)
    x = f32(f32(px[None] * ca[:, None]) - f32(py[None] * sa[:, None]))
    y = f32(f32(px[None] * sa[:, None]) + f32(py[None] * ca[:, None]))
    ix, iy = np.rint(x).astype(np.int64), np.rint(y).astype(np.int64)
    vals = blurred[np.asarray(cy)[:, None] + iy, np.asarray(cx)[:, None] + ix].astype(np.int32)  # (N, 512)
    bits = (vals[:, 0::2] < vals[:, 1::2]).astype(np.uint8).reshape(-1, 32, 8)
    return (bits << np.arange(8, dtype=np.uint8)).sum(2).astype(np.uint8)


# ---- ORB -----------------------------------------------------------------------------------------------------------

def orb_pyramid(gray):
    levels = [np.ascontiguousarray(gray, np.uint8)]
    for (h, w) in level_sizes(*gray.shape)[1:]:
        levels.append(resize_linear_exact(levels[-1], h, w))
    return levels


def orb_detect_and_compute(gray, with_stages=False):
    """cv2.ORB_create().detectAndCompute(gray, None) in canonical (level, y, x) order.

    Returns dict: pts (N, 2) fp32 (x, y) in level-0 pixels, level (N,), angle (N,) fp32 degrees, response (N,) fp32
    (Harris), desc (N, 32) uint8; with_stages adds the pyramid, FAST maps, candidate lists and blurred levels."""
    gray = np.asarray(gray)
    assert gray.dtype == np.uint8 and gray.ndim == 2
    levels = orb_pyramid(gray)
    scales = level_scales()
    quota = features_per_level()
    out = {k: [] for k in ("x", "y", "level", "response", "angle")}
    stages = {"pyramid": levels, "fast": [], "blurred": [], "cand": []}
    for l, img in enumerate(levels):
        H, W = img.shape
        sc = fast_scores(img)
        ys, xs, s = fast_nms(sc)
        b = EDGE_THRESHOLD
        inside = (xs >= b) & (ys >= b) & (xs < W - b) & (ys < H - b) if (H > 2 * b and W > 2 * b) else np.zeros(len(xs), bool)
        ys, xs, s = ys[inside], xs[inside], s[inside]
        m = retain_best_mask(s, 2 * quota[l])
        ys, xs, s = ys[m], xs[m], s[m]
        r = harris_responses(img, ys, xs) if len(ys) else np.zeros(0, np.float32)
        stages["fast"].append(sc)
        stages["cand"].append((ys, xs, s, r))
        m = retain_best_mask(r, quota[l])
        ys, xs, r = ys[m], xs[m], r[m]
        out["x"].append(xs)
        out["y"].append(ys)
        out["level"].append(np.full(len(xs), l, np.int32))
        out["response"].append(r)
        out["angle"].append(ic_angles(img, ys, xs) if len(ys) else np.zeros(0, np.float32))
    desc = []
    for l, img in enumerate(levels):
        bl = gaussian_blur_orb(img)
        stages["blurred"].append(bl)
        xs, ys = out["x"][l], out["y"][l]
        sc = scales[l]
        # the keypoint is scaled to level 0 and back, as orb.cpp does (cvRound(pt * (1 / scale)))
        inv = f32(f32(1) / sc)
        cx = np.rint(f32(f32(xs.astype(np.float32) * sc) * inv)).astype(np.int64)
        cy = np.rint(f32(f32(ys.astype(np.float32) * sc) * inv)).astype(np.int64)
        desc.append(rbrief(bl, cy, cx, out["angle"][l]) if len(xs) else np.zeros((0, 32), np.uint8))
    lvl = np.concatenate(out["level"])
    res = {
        "level": lvl,
        "pts": np.stack([np.concatenate(out["x"]).astype(np.float32) * np.array(scales, np.float32)[lvl],
                         np.concatenate(out["y"]).astype(np.float32) * np.array(scales, np.float32)[lvl]], 1)
        .astype(np.float32).reshape(-1, 2),
        "xy_level": np.stack([np.concatenate(out["x"]), np.concatenate(out["y"])], 1).astype(np.int32).reshape(-1, 2),
        "angle": np.concatenate(out["angle"]).astype(np.float32),
        "response": np.concatenate(out["response"]).astype(np.float32),
        "desc": np.concatenate(desc).reshape(-1, 32),
    }
    if with_stages:
        res["stages"] = stages
    return res


# ---- DBoW3 vocabulary -----------------------------------------------------------------------------------------------

TF_IDF, TF, IDF, BINARY = 0, 1, 2, 3  # WeightingType; ScoringType L1_NORM is 0
SCORING_NAMES = ["L1_NORM", "L2_NORM", "CHI_SQUARE", "KL", "BHATTACHARYYA", "DOT_PRODUCT"]


class Vocabulary:
    """A DBoW3 tree: node arrays indexed by node id, children in file order."""

    def __init__(self, k, L, scoring, weighting, parent, desc, weight, word_id):
        self.k, self.L, self.scoring, self.weighting = k, L, scoring, weighting
        self.parent = np.asarray(parent, np.int64)       # parent[0] = -1
        self.desc = np.asarray(desc, np.uint8)           # (N, 32)
        self.weight = np.asarray(weight, np.float64)
        self.word_id = np.asarray(word_id, np.int64)     # -1 for non-words
        self.children = [[] for _ in range(len(self.parent))]

    @property
    def n_nodes(self):
        return len(self.parent)

    @property
    def n_words(self):
        return int((self.word_id >= 0).sum())


def load_vocab_txt(path):
    """Vocabulary::load_fromtxt: header 'k L scoring weighting', then one node per line: parent, leaf flag, descriptor
    bytes, weight (all parsed as float)."""
    with open(path) as f:
        head = f.readline().split()
        k, L, sc, wt = (int(v) for v in head[:4])
        parent, desc, weight, word = [-1], [np.zeros(32, np.uint8)], [0.0], [-1]
        order = []
        nw = 0
        for line in f:
            t = line.split()
            if not t:
                break
            pid, leaf = int(t[0]), int(t[1])
            if not 0 <= pid < len(parent):
                raise ValueError("node %d names a parent that does not precede it" % len(parent))
            vals = np.array([float(v) for v in t[2:]], np.float32)
            parent.append(pid)
            weight.append(float(vals[-1]))
            desc.append(vals[:-1].astype(np.uint8))
            if leaf > 0:
                word.append(nw)
                nw += 1
            else:
                word.append(-1)
            order.append((pid, len(parent) - 1))
    desc = np.stack([d if len(d) == 32 else np.resize(d, 32) for d in desc])
    v = Vocabulary(k, L, sc, wt, parent, desc, weight, word)
    for pid, nid in order:
        v.children[pid].append(nid)
    return v


def save_vocab_txt(v, path):
    """The text format load_fromtxt reads: node ids are line numbers (the root is 0), so nodes are written in
    breadth-first order and renumbered; weights are printed as the float they parse back to."""
    order = _file_order(v)
    new_id = {0: 0}
    for i, nid in enumerate(order):
        new_id[nid] = i + 1
    with open(path, "w") as f:
        f.write("%d %d %d %d\n" % (v.k, v.L, v.scoring, v.weighting))
        for nid in order:
            d = " ".join(str(int(b)) for b in v.desc[nid])
            f.write("%d %d %s %s\n" % (new_id[int(v.parent[nid])], 1 if v.word_id[nid] >= 0 else 0, d,
                                         repr(float(f32(v.weight[nid])))))


def _file_order(v):
    """Nodes in breadth-first order of the children lists (what a writer emits; a parent precedes its children)."""
    out, q = [], [0]
    while q:
        n = q.pop(0)
        for c in v.children[n]:
            out.append(c)
            q.append(c)
    return out


def save_vocab_bin(v, path):
    """Vocabulary::toStream, uncompressed: magic, compressed = 0, node count, k, L, scoring, weighting, then per node
    (id, parent, weight f64, descriptor cols/rows/type/bytes) in file order, then the words (word id, node id)."""
    with open(path, "wb") as f:
        f.write(struct.pack("<Q?I", 88877711233, False, v.n_nodes))
        f.write(_bin_body(v))


def _bin_body(v):
    out = [struct.pack("<iiii", v.k, v.L, v.scoring, v.weighting)]
    for nid in _file_order(v):
        out.append(struct.pack("<IId", nid, v.parent[nid], v.weight[nid]))
        out.append(struct.pack("<iii", 32, 1, 0) + v.desc[nid].tobytes())
    words = [(int(v.word_id[n]), n) for n in range(v.n_nodes) if v.word_id[n] >= 0]
    out.append(struct.pack("<I", len(words)))
    for wid, nid in sorted(words):
        out.append(struct.pack("<II", wid, nid))
    return b"".join(out)


def load_vocab_bin(path):
    """Vocabulary::fromStream: a plain stream, or QuickLZ level-1 chunks (toStream(compressed=true))."""
    with open(path, "rb") as f:
        data = f.read()
    sig, compressed, nnodes = struct.unpack_from("<Q?I", data, 0)
    if sig != 88877711233:
        raise ValueError("not a DBoW3 binary vocabulary")
    pos = 13
    if compressed:
        nchunks, = struct.unpack_from("<I", data, pos)
        pos += 4
        parts = []
        for _ in range(nchunks):
            used, chunk = qlz1_chunk(data, pos)
            parts.append(chunk)
            pos += used
        body, pos = b"".join(parts), 0
    else:
        body = data
    k, L, sc, wt = struct.unpack_from("<iiii", body, pos)
    pos += 16
    parent = np.full(nnodes, -1, np.int64)
    desc = np.zeros((nnodes, 32), np.uint8)
    weight = np.zeros(nnodes, np.float64)
    word = np.full(nnodes, -1, np.int64)
    order = []
    for _ in range(nnodes - 1):
        nid, pid, w = struct.unpack_from("<IId", body, pos)
        cols, rows, typ = struct.unpack_from("<iii", body, pos + 16)
        pos += 28
        if typ != 0 or rows != 1:
            raise ValueError("only binary (CV_8U) descriptors are supported")
        desc[nid, :min(cols, 32)] = np.frombuffer(body, np.uint8, cols, pos)[:32]
        pos += cols
        parent[nid], weight[nid] = pid, w
        order.append((pid, nid))
    nw, = struct.unpack_from("<I", body, pos)
    pos += 4
    for _ in range(nw):
        wid, nid = struct.unpack_from("<II", body, pos)
        pos += 8
        word[nid] = wid
    v = Vocabulary(k, L, sc, wt, parent, desc, weight, word)
    for pid, nid in order:
        v.children[pid].append(nid)
    return v


def qlz1_chunk(buf, pos):
    """One QuickLZ 1.5 chunk (level 1, streaming buffer 0) at buf[pos:] -> (compressed size, bytes); the format is
    described at qlz1_chunk in csrc/bow.cu."""
    flag = buf[pos]
    if flag & 2:
        csize, dsize = struct.unpack_from("<II", buf, pos + 1)
        hdr = 9
    else:
        csize, dsize, hdr = buf[pos + 1], buf[pos + 2], 3
    if not flag & 1:
        return csize, bytes(buf[pos + hdr:pos + hdr + dsize])
    src, dst = pos + hdr, bytearray(dsize)
    table = [0] * 4096
    d, last_hashed, cword = 0, -1, 1
    last_matchstart = dsize - 1 - 6 - 4

    def hash_upto(upto):
        nonlocal last_hashed
        while last_hashed < upto:
            last_hashed += 1
            v = dst[last_hashed] | (dst[last_hashed + 1] << 8) | (dst[last_hashed + 2] << 16)
            table[((v >> 12) ^ v) & 0xFFF] = last_hashed

    while d < dsize:
        if cword == 1:
            cword, = struct.unpack_from("<I", buf, src)
            src += 4
        if cword & 1:
            cword >>= 1
            fetch = buf[src] | (buf[src + 1] << 8) | (buf[src + 2] << 16)
            start = table[(fetch >> 4) & 0xFFF]
            if fetch & 0xF:
                n, src = (fetch & 0xF) + 2, src + 2
            else:
                n, src = buf[src + 2], src + 3
            for k in range(n):
                dst[d + k] = dst[start + k]
            hash_upto(d)
            d += n
            last_hashed = d - 1
        elif d < last_matchstart:
            dst[d] = buf[src]
            d, src, cword = d + 1, src + 1, cword >> 1
            hash_upto(d - 3)
        else:
            while d < dsize:
                if cword == 1:
                    src, cword = src + 4, 1 << 31
                dst[d] = buf[src]
                d, src, cword = d + 1, src + 1, cword >> 1
    return csize, bytes(dst)


# ---- bag of words ----------------------------------------------------------------------------------------------------

def check_supported(v):
    if v.scoring != 0:
        raise ValueError("only L1 scoring is supported, the vocabulary uses %s" % SCORING_NAMES[v.scoring])


def transform_words(v, desc):
    """Per descriptor (word id, weight): descend from the root to the first child of minimal Hamming distance."""
    desc = np.asarray(desc, np.uint8)
    words = np.zeros(len(desc), np.int64)
    weights = np.zeros(len(desc), np.float64)
    pc = np.unpackbits(v.desc, axis=1)
    for i, d in enumerate(desc):
        db = np.unpackbits(d)
        node = 0
        while v.children[node]:
            ch = v.children[node]
            dist = (pc[ch] != db).sum(1)
            node = ch[int(np.argmin(dist))]
        words[i], weights[i] = v.word_id[node], v.weight[node]
    return words, weights


def bow_vector(v, desc):
    """Vocabulary::transform -> (word ids ascending, values) after BowVector::normalize(L1); None for no descriptor."""
    if desc is None or len(desc) == 0:
        return None
    words, weights = transform_words(v, desc)
    acc = {}
    for w, x in zip(words.tolist(), weights.tolist()):
        if not x > 0:
            continue
        if v.weighting in (TF, TF_IDF):
            acc[w] = acc[w] + x if w in acc else x
        elif w not in acc:
            acc[w] = x
    ids = np.array(sorted(acc), np.int64)
    vals = np.array([acc[i] for i in ids.tolist()], np.float64)
    norm = 0.0
    for x in vals.tolist():
        norm += abs(x)
    if norm > 0.0:
        vals = vals / norm
    return ids, vals


def l1_score(a, b):
    """L1Scoring::score over the common words in ascending word id."""
    ia, va = a
    ib, vb = b
    common, pa, pb = np.intersect1d(ia, ib, assume_unique=True, return_indices=True)
    s = 0.0
    for x, y in zip(va[pa].tolist(), vb[pb].tolist()):
        s += (abs(x - y) - abs(x)) - abs(y)
    return -s / 2.0


def detect_loop(bow_feats, i, farthest_neighbor, loop_dist_min, loop_nms, loop_cand_thresh_neighbor):
    """loop_detector.py:23-50 for view i (its vector already in bow_feats[i])."""
    fi = bow_feats[i]
    lo = max(0, i - loop_cand_thresh_neighbor)
    sims = [l1_score(fi, bow_feats[j]) for j in range(lo, i) if fi is not None and bow_feats[j] is not None]
    thresh = 1.0 if not sims else min(sims)
    last = farthest_neighbor
    cands = []
    for j in reversed(range(0, farthest_neighbor)):
        if last - j > loop_nms and i - j > loop_dist_min:
            if fi is None or bow_feats[j] is None:
                continue
            s = l1_score(fi, bow_feats[j])
            if s > thresh:
                cands.append((j, s))
                last = j
    return sorted(cands, key=lambda c: c[1], reverse=True)


# ---- seeded test frames ------------------------------------------------------------------------------------------------

def _texture(rng, H, W):
    """A smooth-plus-edges 8-bit texture: blobs, rectangles and noise (plenty of FAST corners at several scales)."""
    img = np.zeros((H, W), np.float64)
    for s in (64, 24, 9):
        g = rng.random((H // s + 2, W // s + 2))
        img += np.kron(g, np.ones((s, s)))[:H, :W] * (s / 32.0)
    for _ in range(H * W // 900):
        y, x = rng.integers(0, H), rng.integers(0, W)
        h, w = rng.integers(4, 40, size=2)
        img[y:y + h, x:x + w] += rng.uniform(-1.5, 1.5)
    img += rng.normal(0, 0.08, (H, W))
    img = (img - img.min()) / (img.max() - img.min())
    return np.clip(img * 255, 0, 255).astype(np.uint8)


def make_sequence(seed, n_frames, H=224, W=224, revisit_after=44):
    """Integer crops of a large seeded texture along a loop that returns to its start after `revisit_after` frames,
    with a flat frame (no descriptor), a low-texture frame and a near-duplicate (tied similarities) mixed in."""
    rng = np.random.default_rng(seed)
    big = _texture(rng, 3 * H, 3 * W)
    frames = []
    for t in range(n_frames):
        a = 2 * math.pi * (t % revisit_after) / revisit_after
        y = int(H + 0.8 * H * math.sin(a))
        x = int(W + 0.8 * W * (1 - math.cos(a)) / 2)
        f = big[y:y + H, x:x + W].copy()
        if t % 17 == 9:
            f[:] = 128                                       # flat: ORB finds nothing
        elif t % 17 == 13:
            f = (f // 64 * 8 + 100).astype(np.uint8)         # low texture: few corners
        elif t % 17 == 15 and frames:
            f = frames[-1].copy()                            # duplicate of the previous frame
        frames.append(f)
    return frames
