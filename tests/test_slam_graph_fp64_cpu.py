"""CPU companion of tests/test_slam_graph_fp64_gpu.py: a numpy mirror of the device pose graph's algebra
(csrc/slam_graph.cu, cloud.cuh, pointmap.cuh), the planted cases that steer it through each of its branches, and the
per-element bounds the GPU test applies, shown here to accept the fp32 arithmetic and to reject planted mistakes.

  * rot_to_quat, sim3_mul, the export's quaternion -> matrix, inv3_f32 + unproject_f32 and the scale_partial /
    scale_finalize partition are restated statement for statement, with the same branch tests; the fp64 forms also
    return the magnitude of each result (the same expression with every term replaced by its absolute value).
  * The case lists name the branch each case must reach; the test asserts them, so the lists cannot drift away from the
    branches they are meant to cover.
  * The mirror is pinned to the oracle (oracle/pose_graph_oracle.py, oracle/slam_oracle.py), which takes other routes:
    sim3_mul through 4x4 matrices, quat_to_rot with a normalisation.

Bounds (u = 2^-24, the fp32 unit roundoff; S the magnitude of a result):
  * edge quaternion: 2^-23 |ref| per component of the fp64 mirror (one rounding of an fp64 result; the fp64 arithmetic of
    the device may differ from numpy's by FMA contraction: 4 fp64 ulps of the unit norm are allowed on top);
  * node pose: C_SIM3 u S per component, S of the fp64 product of the stored parent and the stored measurement.  The
    deepest path has 6 fp32 roundings (u x t_b, 2 w (u x t_b) + ..., t_b + ..., s_a r, t_a + ...); 16 leaves room for
    FMA contraction and is still about 10^4 times tighter than the 1e-4 of tests/test_slam_gpu.py on O(1) poses;
  * exported rotation: C_ROT u of the magnitude of the un-normalised formula (3 roundings on the deepest path);
  * scale edge sums: (m + 8) u of the magnitude sum, m = terms per thread (m - 1 additions in the thread, 5 shuffle
    levels, 3 product roundings: ci cj, w Di, (w Di) Dj or the square root), then one final rounding of the ratio;
  * points: C_PT u S_p, S_p = |P| |K^-1| |pix| |d s| + |t| in absolute values.  The deepest path of unproject_f32 has 10
    roundings: K^-1 to fp32, Ki0 u, + Ki1 r, + Ki2, x d, d = depth s (6), P0 cx, + P1 cy, + P2 cz, + t (4); the fp64
    adjugate of inv3_f32 adds about 10^-16 relative.  C_PT = 12.
"""
import numpy as np
import pytest

from oracle import pose_graph_oracle as pg
from oracle import slam_oracle as so

F32 = 2.0 ** -24  # fp32 unit roundoff
SO3_TOL = 1e-3  # rot_to_quat's acceptance of the Gram entries and the determinant (pp.mat2SE3(atol=1e-3))
C_SIM3, C_ROT, C_PT = 16, 8, 12
Q_ABS = 4 * 2.0 ** -53  # fp64 noise of the unit-norm quaternion on top of its fp32 rounding
STAT_BLOCKS, STAT_THREADS = 64, 256  # pointmap.cuh kStatBlocks, threads per block
CLAMP = float(np.float32(1e-6))  # fmaxf(ci cj, 1e-6f)
f32 = np.float32


# ------------------------------------------------------------------------------- mirror of csrc/slam_graph.cu
def so3_deviation(M):
    """rot_to_quat's SO(3) check on the fp32 rotation block: the largest Gram deviation on and off the diagonal and
    |det - 1|, evaluated in fp64 as the device does."""
    R = np.asarray(M, np.float32)[:3, :3].astype(np.float64)
    G = np.array([[R[r, 0] * R[c, 0] + R[r, 1] * R[c, 1] + R[r, 2] * R[c, 2] - (1.0 if r == c else 0.0) for c in range(3)]
                  for r in range(3)])
    det = (R[0, 0] * (R[1, 1] * R[2, 2] - R[1, 2] * R[2, 1]) - R[0, 1] * (R[1, 0] * R[2, 2] - R[1, 2] * R[2, 0]) +
           R[0, 2] * (R[1, 0] * R[2, 1] - R[1, 1] * R[2, 0]))
    off = np.abs(G - np.diag(np.diag(G))).max()
    return {"gram_diag": float(np.abs(np.diag(G)).max()), "gram_off": float(off), "det": float(abs(det - 1.0))}


def rot_to_quat(M, mistake=None):
    """slam_graph.cu rot_to_quat on the rotation block of a [4,4] fp32 matrix, statement for statement, in fp64.
    Returns (q fp64 before its rounding to fp32, ok, branch, flipped); branch is "trace" or "diag<i>".
    mistake: "swap_jk" (j and k exchanged in the diagonal branch), "transpose" (R^T read), "no_flip"."""
    R = np.asarray(M, np.float32)[:3, :3].astype(np.float64)
    if mistake == "transpose":
        R = R.T
    ok = all(v <= SO3_TOL for v in so3_deviation(M).values())
    x = np.zeros(4)
    t = R[0, 0] + R[1, 1] + R[2, 2]
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        x[:] = (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s
        branch = "trace"
    else:
        i = 0
        if R[1, 1] > R[i, i]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        if mistake == "swap_jk":
            j, k = k, j
        s = np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k]) * 2
        x[i] = 0.25 * s
        x[j] = (R[j, i] + R[i, j]) / s
        x[k] = (R[k, i] + R[i, k]) / s
        x[3] = (R[k, j] - R[j, k]) / s
        branch = "diag%d" % i
    flipped = bool(x[3] < 0)
    sg = -1.0 if flipped and mistake != "no_flip" else 1.0
    nrm = np.sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + x[3] * x[3])
    return sg * x / nrm, ok, branch, flipped


def _sim3_mul(a, b, sub, mistake=None):
    """The expression of slam_graph.cu sim3_mul in its evaluation order over scalars of one type; `sub` is x - y, or
    x + y for the magnitude (with |a|, |b| as inputs).  Returns (o[8] before the sign, q_w of the product)."""
    ax, ay, az, aw = a[3], a[4], a[5], a[6]
    bx, by, bz, bw = b[3], b[4], b[5], b[6]
    tx, ty, tz = b[0], b[1], b[2]
    two = type(ax)(2)
    ux, uy, uz = (-ax, -ay, -az) if mistake == "RaT_tb" else (ax, ay, az)  # R_a^T t_b: the conjugate rotation
    cx, cy, cz = sub(uy * tz, uz * ty), sub(uz * tx, ux * tz), sub(ux * ty, uy * tx)
    rx = tx + two * sub(aw * cx + uy * cz, uz * cy)
    ry = ty + two * sub(aw * cy + uz * cx, ux * cz)
    rz = tz + two * sub(aw * cz + ux * cy, uy * cx)
    q = [sub(aw * bx + ax * bw + ay * bz, az * by), sub(aw * by, ax * bz) + ay * bw + az * bx,
         sub(aw * bz + ax * by, ay * bx) + az * bw, sub(sub(sub(aw * bw, ax * bx), ay * by), az * bz)]
    sa = {"scale_twice": a[7] * a[7], "scale_none": type(ax)(1)}.get(mistake, a[7])
    o = [a[0] + sa * rx, a[1] + sa * ry, a[2] + sa * rz] + q + [a[7] * b[7]]
    return o, q[3]


def sim3_mul_f32(a, b, mistake=None):
    """sim3_mul in fp32, operation by operation (no FMA contraction).  mistake: "no_flip", "RaT_tb", "scale_twice",
    "scale_none"."""
    a, b = [f32(v) for v in np.asarray(a, np.float32)], [f32(v) for v in np.asarray(b, np.float32)]
    o, w = _sim3_mul(a, b, lambda x, y: x - y, mistake)
    sg = f32(-1) if w < 0 and mistake != "no_flip" else f32(1)
    return np.array([o[0], o[1], o[2]] + [sg * v for v in o[3:7]] + [o[7]], np.float32)


def sim3_mul64(a, b):
    """sim3_mul in fp64 on the (fp32) inputs: (product [8], magnitude S [8], flipped)."""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    o, w = _sim3_mul(list(a64), list(b64), lambda x, y: x - y)
    S, _ = _sim3_mul(list(np.abs(a64)), list(np.abs(b64)), lambda x, y: x + y)
    o = np.array(o)
    if w < 0:
        o[3:7] = -o[3:7]
    return o, np.array(S), bool(w < 0)


def _ratio(err, bound):
    """max of err / bound, where a zero bound admits only a zero error."""
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(r.max())


def sim3_err(got, a, b):
    """max over components of |got - ref| / (C_SIM3 u S) against the fp64 product of a and b.  Where the reference's
    q_w is within its bound of 0, the sign the fp32 product chose is not determined: the closer sign is taken."""
    ref, S, _ = sim3_mul64(a, b)
    bound = C_SIM3 * F32 * S
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    if abs(ref[6]) <= bound[6]:
        alt = ref.copy()
        alt[3:7] = -alt[3:7]
        err = np.minimum(err, np.abs(got - alt))
    return _ratio(err, bound)


def quat_to_rot_export(q, dtype=np.float32):
    """export_gather_kernel's LieTensor.rotation().matrix(): the quaternion is not normalised.  Returns (R [3,3],
    magnitude [3,3]); dtype np.float32 evaluates it as the device does, np.float64 gives the reference."""
    x, y, z, w = [dtype(v) for v in np.asarray(q)]
    one, two = dtype(1), dtype(2)
    R = np.array([[one - two * (y * y + z * z), two * (x * y - z * w), two * (x * z + y * w)],
                  [two * (x * y + z * w), one - two * (x * x + z * z), two * (y * z - x * w)],
                  [two * (x * z - y * w), two * (y * z + x * w), one - two * (x * x + y * y)]])
    x, y, z, w = abs(x), abs(y), abs(z), abs(w)
    M = np.array([[one + two * (y * y + z * z), two * (x * y + z * w), two * (x * z + y * w)],
                  [two * (x * y + z * w), one + two * (x * x + z * z), two * (y * z + x * w)],
                  [two * (x * z + y * w), two * (y * z + x * w), one + two * (x * x + y * y)]])
    return R, M


# ------------------------------------------------------------------------------- mirror of cloud.cuh
def inv3(K):
    """inv3_f32's adjugate / det in fp64 over the entries of K [..., 3, 3] (numpy or torch, fp64): a list of the 9
    entries of K^-1, row-major, not yet rounded to fp32."""
    k = [[K[..., r, c] for c in range(3)] for r in range(3)]
    (k00, k01, k02), (k10, k11, k12), (k20, k21, k22) = k
    det = k00 * (k11 * k22 - k12 * k21) - k01 * (k10 * k22 - k12 * k20) + k02 * (k10 * k21 - k11 * k20)
    return [(k11 * k22 - k12 * k21) / det, (k02 * k21 - k01 * k22) / det, (k01 * k12 - k02 * k11) / det,
            (k12 * k20 - k10 * k22) / det, (k00 * k22 - k02 * k20) / det, (k02 * k10 - k00 * k12) / det,
            (k10 * k21 - k11 * k20) / det, (k01 * k20 - k00 * k21) / det, (k00 * k11 - k01 * k10) / det]


def unproject_ref(Ki, P, u, r, ds):
    """fp64 P (K^-1 [u r 1]^T ds) + t and its magnitude S_p, elementwise over numpy or torch arrays.  Ki: the 9 entries
    of K^-1, P: [..., 3, 4] (or 4 x 4) fp64, ds = depth x scale."""
    cam = [(Ki[3 * c] * u + Ki[3 * c + 1] * r + Ki[3 * c + 2]) * ds for c in range(3)]
    mag = [(abs(Ki[3 * c]) * abs(u) + abs(Ki[3 * c + 1]) * abs(r) + abs(Ki[3 * c + 2])) * abs(ds) for c in range(3)]
    out, S = [], []
    for c in range(3):
        out.append(P[..., c, 0] * cam[0] + P[..., c, 1] * cam[1] + P[..., c, 2] * cam[2] + P[..., c, 3])
        S.append(abs(P[..., c, 0]) * mag[0] + abs(P[..., c, 1]) * mag[1] + abs(P[..., c, 2]) * mag[2] + abs(P[..., c, 3]))
    return out, S


def unproject_f32(K, P, x, row, depth, s, mistake=None):
    """export_scatter_kernel's point of column x, row `row`: inv3_f32 then unproject_f32 in fp32 (no FMA contraction).
    mistake: "K_T" (K^T inverted), "next_column" (the depth of column x + 1 at column x)."""
    K = np.asarray(K, np.float32).astype(np.float64)
    Ki = [f32(v) for v in inv3(K.T if mistake == "K_T" else K)]
    P = np.asarray(P, np.float32)
    d = f32(depth[x + 1] if mistake == "next_column" else depth[x]) * f32(s)
    u, rr = f32(x), f32(row)
    cx = (Ki[0] * u + Ki[1] * rr + Ki[2]) * d
    cy = (Ki[3] * u + Ki[4] * rr + Ki[5]) * d
    cz = (Ki[6] * u + Ki[7] * rr + Ki[8]) * d
    return np.array([P[c, 0] * cx + P[c, 1] * cy + P[c, 2] * cz + P[c, 3] for c in range(3)], np.float32)


def point_err(got, K, P, x, row, depth, s):
    """max over the 3 coordinates of |got - ref| / (C_PT u S_p)."""
    Ki = inv3(np.asarray(K, np.float32).astype(np.float64))
    ref, S = unproject_ref(Ki, np.asarray(P, np.float32).astype(np.float64), float(x), float(row),
                           float(np.float32(depth[x])) * float(np.float32(s)))
    return _ratio([abs(float(got[c]) - ref[c]) for c in range(3)], [C_PT * F32 * S[c] for c in range(3)])


# ------------------------------------------------------------------------------- mirror of pointmap.cuh
def scale_stats_f32(Di, Dj, ci, cj):
    """scale_partial over kStatBlocks blocks of 256 threads (each thread summing its ceil(n / 16384) strided terms in
    fp32, then 5 shuffle levels in fp32), the block records and the 64 of them summed in fp64 in order, and
    scale_finalize: (scale, scale_conf) as fp32."""
    Di, Dj, ci, cj = (np.asarray(v, np.float32).reshape(-1) for v in (Di, Dj, ci, cj))
    n = Di.size
    span = STAT_BLOCKS * STAT_THREADS
    m = -(-n // span)
    pad = m * span - n  # zero terms: x + 0 = x in fp32

    def grid(v):
        return np.concatenate([v, np.zeros(pad, np.float32)]).reshape(m, STAT_BLOCKS, STAT_THREADS)

    a, b, c1, c2 = grid(Di), grid(Dj), grid(ci), grid(cj)
    s = np.zeros((3, STAT_BLOCKS, STAT_THREADS), np.float32)
    for it in range(m):
        cc = c1[it] * c2[it]
        w = np.maximum(cc, f32(1e-6))
        s[0] += w * a[it] * b[it]
        s[1] += w * a[it] * a[it]
        s[2] += np.sqrt(cc)
    s = s.reshape(3, STAT_BLOCKS, 8, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lane ^ o]
    t = [0.0, 0.0, 0.0]
    for blk in range(STAT_BLOCKS):
        for i in range(3):
            rec = 0.0
            for w in range(8):
                rec += float(s[i, blk, w, 0])
            t[i] += rec
    return f32(t[0] / t[1]), f32(t[2] / float(n))


def scale_stats_ref(Di, Dj, ci, cj, xp=np):
    """fp64 sums of the reduction on the fp32 maps and their magnitudes: (T0, T1, T2, S0, S1, S2, n), where
    T0 = sum w Di Dj, T1 = sum w Di^2, T2 = sum sqrt(ci cj), w = max(ci cj, 1e-6f).  xp: numpy or torch (fp64 inputs)."""
    cc = ci * cj
    w = xp.maximum(cc, xp.full_like(cc, CLAMP)) if xp is not np else np.maximum(cc, CLAMP)
    t0, t1, t2 = w * Di * Dj, w * Di * Di, xp.sqrt(cc)
    return (float(t0.sum()), float(t1.sum()), float(t2.sum()), float(abs(t0).sum()), float(t1.sum()), float(t2.sum()),
            int(Di.numel() if xp is not np else Di.size))


def scale_errs(got_scale, got_conf, stats):
    """(err / bound) of the scale and of the scale confidence against the fp64 sums of scale_stats_ref."""
    T0, T1, T2, S0, S1, S2, n = stats
    m = -(-n // (STAT_BLOCKS * STAT_THREADS))
    e = (m + 8) * F32
    r = T0 / T1
    b_scale = e * (S0 + abs(r) * S1) / (T1 * (1 - e)) + F32 * abs(r)
    b_conf = (e * S2 + F32 * T2) / n
    return abs(float(got_scale) - r) / b_scale, abs(float(got_conf) - T2 / n) / b_conf


# ------------------------------------------------------------------------------- cases
def rot(axis, angle):
    """Rotation by angle about axis: cos I + sin [n]x + (1 - cos) n n^T, fp64 (equal n_i give equal R_ii)."""
    n = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    c, s = np.cos(angle), np.sin(angle)
    return c * np.eye(3) + s * pg.hat(n) + (1 - c) * np.outer(n, n)


def pose44(R, t=(0.3, -0.2, 0.5)):
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = R, t
    return M.astype(np.float32)


_G = rot([1, 2, 3], 0.7)  # a generic rotation (trace branch) carrying the SO(3) deviations
_NEAR_PI = np.pi - 1e-3


def _deviated(kind, target):
    """_G with one kind of deviation from SO(3) of size target: a row scaled ("gram_diag"), two rows sheared into each
    other ("gram_off": Gram = I + 2e (E01 + E10) + e^2 (E00 + E11)), or every row scaled ("det": the Gram diagonal
    stays at 2/3 of the determinant's deviation)."""
    if kind == "gram_diag":
        A = np.diag([np.sqrt(1 + target), 1.0, 1.0])
    elif kind == "gram_off":
        A = np.eye(3)
        A[0, 1] = A[1, 0] = target / 2
    else:
        A = np.cbrt(1 + target) * np.eye(3)
    return A @ _G


# name, [4,4] fp32 pose, (branch, flipped before canonicalisation, accepted as SO(3)), [diagonal tie]
ROT_CASES = [
    ("identity", pose44(np.eye(3)), ("trace", False, True)),
    ("generic_0.7", pose44(_G), ("trace", False, True)),
    ("trace>0_2pi/3-1e-3", pose44(rot([1, 3, 2], 2 * np.pi / 3 - 1e-3)), ("trace", False, True)),
    ("trace<0_2pi/3+1e-3", pose44(rot([1, 3, 2], 2 * np.pi / 3 + 1e-3)), ("diag1", False, True)),
    ("trace=0_tie012", pose44(np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0.0]])), ("diag0", False, True)),
    ("near_pi+x", pose44(rot([1, 0, 0], _NEAR_PI)), ("diag0", False, True)),
    ("near_pi+y", pose44(rot([0, 1, 0], _NEAR_PI)), ("diag1", False, True)),
    ("near_pi+z", pose44(rot([0, 0, 1], _NEAR_PI)), ("diag2", False, True)),
    ("near_pi-x", pose44(rot([-1, 0, 0], _NEAR_PI)), ("diag0", True, True)),
    ("near_pi-y", pose44(rot([0, -1, 0], _NEAR_PI)), ("diag1", True, True)),
    ("near_pi-z", pose44(rot([0, 0, -1], _NEAR_PI)), ("diag2", True, True)),
    ("near_pi_generic", pose44(rot([0.3, -0.5, -0.8], _NEAR_PI)), ("diag2", True, True)),
    ("pi_x_w=0", pose44(np.diag([1.0, -1.0, -1.0])), ("diag0", False, True)),
    ("pi_y_w=0", pose44(np.diag([-1.0, 1.0, -1.0])), ("diag1", False, True)),
    ("pi_z_w=0", pose44(np.diag([-1.0, -1.0, 1.0])), ("diag2", False, True)),
    ("pi_110_tie01", pose44(rot([1, 1, 0], np.pi)), ("diag0", False, True)),
    ("pi-0.2_110_tie01", pose44(rot([1, 1, 0], np.pi - 0.2)), ("diag0", False, True)),
    ("pi-0.2_-1-10_tie01", pose44(rot([-1, -1, 0], np.pi - 0.2)), ("diag0", True, True)),
    ("pi-0.2_011_tie12", pose44(rot([0, 1, 1], np.pi - 0.2)), ("diag1", False, True)),
    ("pi-0.2_101_tie02", pose44(rot([1, 0, 1], np.pi - 0.2)), ("diag0", False, True)),
    ("gram_diag_0.9e-3", pose44(_deviated("gram_diag", 0.9e-3)), ("trace", False, True)),
    ("gram_diag_1.1e-3", pose44(_deviated("gram_diag", 1.1e-3)), ("trace", False, False)),
    ("gram_off_0.9e-3", pose44(_deviated("gram_off", 0.9e-3)), ("trace", False, True)),
    ("gram_off_1.1e-3", pose44(_deviated("gram_off", 1.1e-3)), ("trace", False, False)),
    ("det_0.9e-3", pose44(_deviated("det", 0.9e-3)), ("trace", False, True)),
    ("det_1.1e-3", pose44(_deviated("det", 1.1e-3)), ("trace", False, False)),
    ("reflection_det-1", pose44(np.diag([1.0, 1.0, -1.0])), ("trace", False, False)),
]
ROT_IDS = [c[0] for c in ROT_CASES]


def _diag_tie(M):
    d = np.asarray(M, np.float32)[:3, :3].astype(np.float64).diagonal()
    return int(np.sum(d == d.max())) > 1


def _unit_quat(axis, angle):
    n = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([np.sin(angle / 2) * n, [np.cos(angle / 2)]])


def sim3(t, axis, angle, s):
    return np.concatenate([t, _unit_quat(axis, angle), [s]]).astype(np.float32)


# name, a, b, whether the product's raw q_w < 0 (sim3_mul's sign flip)
SIM3_CASES = [
    ("identity_b", sim3([0.3, -1.0, 2.0], [1, 2, 3], 0.7, 1.3), sim3([0, 0, 0], [1, 0, 0], 0.0, 1.0), False),
    ("scale_edge", sim3([0.3, -1.0, 2.0], [1, 2, 3], 0.7, 1.3), np.array([0, 0, 0, 0, 0, 0, 1, 0.87], np.float32), False),
    ("flip_z150x2", sim3([0.5, 0.2, -0.1], [0, 0, 1], np.radians(150), 1.0), sim3([1.0, -2.0, 0.5], [0, 0, 1], np.radians(150), 1.0),
     True),
    ("flip_generic", sim3([2.0, 1.0, -3.0], [1, 2, 3], np.radians(170), 0.8), sim3([-1.0, 4.0, 0.2], [1, 2, 2.5], np.radians(120), 1.1),
     True),
    ("flip_t1e3_s1e2", sim3([1e3, -7e2, 4e2], [2, -1, 1], np.radians(160), 1e2), sim3([-9e2, 3e2, 1e3], [2, -1, 1.5], np.radians(140), 1e-2),
     True),
    ("t1e3_s1e-2", sim3([1e3, 5e2, -8e2], [0.3, 0.4, -0.5], 1.1, 1e-2), sim3([-6e2, 1e3, 2e2], [-1, 0.2, 0.1], 0.9, 1e2), False),
    ("t1e3_s1e2", sim3([-1e3, 2e2, 9e2], [1, 1, 0.2], 2.0, 1e2), sim3([7e2, -1e3, 3e2], [0.5, -1, 2], 0.4, 1e-2), False),
    ("s1e-2_chain", sim3([1.0, 2.0, 3.0], [0, 1, 0], 0.3, 1e-2), sim3([1e3, 1e3, -1e3], [1, 0, 0], 0.2, 1e-2), False),
]
SIM3_IDS = [c[0] for c in SIM3_CASES]


def random_pairs(n, seed=0):
    """fp32 Sim(3) pairs: translations up to 1e3, scales log-uniform in [1e-2, 1e2], uniform unit quaternions."""
    r = np.random.default_rng(seed)

    def one(k):
        q = r.standard_normal((k, 4))
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        q[q[:, 3] < 0] *= -1
        t = r.uniform(-1e3, 1e3, (k, 3)) * 10.0 ** r.uniform(-3, 0, (k, 1))
        return np.concatenate([t, q, 10.0 ** r.uniform(-2, 2, (k, 1))], 1).astype(np.float32)

    return one(n), one(n)


def chain(n, seed=1):
    """A chain of n fp32 Sim(3) measurements from a root at t ~ 1e2: every node is the fp32 product of its stored
    parent and its measurement (what the device stores), and the fp64 chain of the oracle's poses over the same
    measurements.  Returns (root, measurements, stored nodes, oracle poses)."""
    a, b = random_pairs(n, seed)
    b[:, 7] = 10.0 ** np.random.default_rng(seed).uniform(-0.1, 0.1, n)
    root = a[0].copy()
    root[:3] = [120.0, -80.0, 45.0]
    stored, oracle = [root], [root.astype(np.float64)]
    for m in b:
        stored.append(sim3_mul_f32(stored[-1], m))
        oracle.append(pg.sim3_mul(oracle[-1], m.astype(np.float64)))
    return root, b, stored, oracle


def scale_maps(n, seed, plant=True):
    """fp32 depth / confidence maps of n pixels (Di, Dj, ci, cj): positive depths around 2 and confidences in [1, 8];
    planted: pixels with ci cj < 1e-6 (the clamp binds), and negative depths so that sum w Di Dj partly cancels."""
    r = np.random.default_rng(seed)
    Di, Dj = r.uniform(0.5, 3.5, n), r.uniform(0.5, 3.5, n)
    ci, cj = r.uniform(1.0, 8.0, n), r.uniform(1.0, 8.0, n)
    if plant:
        tiny = r.random(n) < 0.05
        ci[tiny], cj[tiny] = r.uniform(0, 1e-3, tiny.sum()), r.uniform(0, 1e-3, tiny.sum())
        neg = r.random(n) < 0.4
        Dj[neg] = -Dj[neg]
    return tuple(v.astype(np.float32) for v in (Di, Dj, ci, cj))


SCALE_SIZES = [1000, 37 * 1001, 224 * 224]


# ------------------------------------------------------------------------------- tests: branches
@pytest.mark.parametrize("case", ROT_CASES, ids=ROT_IDS)
def test_rotation_cases_reach_their_branches(case):
    name, M, want = case
    _, ok, branch, flipped = rot_to_quat(M)
    assert (branch, flipped, ok) == want, (name, branch, flipped, ok)
    dev = so3_deviation(M)
    for kind in ("gram_diag", "gram_off", "det"):
        if name.startswith(kind):  # the planted kind is the one at the limit, the others are within it
            lo, hi = (0.85e-3, 0.95e-3) if name.endswith("0.9e-3") else (1.05e-3, 1.15e-3)
            assert lo <= dev[kind] <= hi and all(v <= SO3_TOL for k, v in dev.items() if k != kind), dev
    if "tie" in name:
        assert _diag_tie(M), name


def test_case_lists_cover_every_branch():
    got = [rot_to_quat(M) + (M,) for _, M, _ in ROT_CASES]
    assert {g[2] for g in got} == {"trace", "diag0", "diag1", "diag2"}
    for b in ("diag0", "diag1", "diag2"):
        assert any(g[2] == b and g[3] for g in got) and any(g[2] == b and not g[3] for g in got), b
    assert any(g[2] != "trace" and _diag_tie(g[4]) and abs(g[0][3]) > 0.05 for g in got)  # a tie where w matters
    traces = [float(np.trace(M[:3, :3].astype(np.float64))) for _, M, _ in ROT_CASES]
    assert min(t for t in traces if t > 0) < 0.01 and max(t for t in traces if t < 0) > -0.01 and 0.0 in traces
    assert sum(g[0][3] == 0.0 for g in got) >= 3  # w = 0 exactly
    for kind in ("gram_diag", "gram_off", "det"):
        acc = [c for c in ROT_CASES if c[0].startswith(kind)]
        assert sorted(c[2][2] for c in acc) == [False, True], kind
    flips = [c for c in SIM3_CASES if c[3]]
    assert flips and all(sim3_mul64(a, b)[2] == want for _, a, b, want in SIM3_CASES)
    assert all(abs(sim3_mul64(a, b)[0][6]) > 0.05 for _, a, b, _ in flips)  # clear of the sign's ambiguity


# ------------------------------------------------------------------------------- tests: the oracle
@pytest.mark.parametrize("case", ROT_CASES, ids=ROT_IDS)
def test_rot_to_quat_pinned_to_the_oracle(case):
    q, _, _, _ = rot_to_quat(case[1])
    want = pg.rot_to_quat(case[1][:3, :3].astype(np.float64))
    assert np.abs(q - want).max() <= 1e-12


def test_sim3_mul_and_quat_to_rot_pinned_to_the_oracle():
    a, b = random_pairs(2000)
    pairs = [(x, y) for _, x, y, _ in SIM3_CASES] + list(zip(a, b))
    for x, y in pairs:
        # sim3_mul rotates t_b by the unit-quaternion formula: pinned on unit quaternions (fp32 ones are not exactly)
        x, y = x.astype(np.float64), y.astype(np.float64)
        x[3:7] /= np.linalg.norm(x[3:7])
        y[3:7] /= np.linalg.norm(y[3:7])
        o, S, _ = sim3_mul64(x, y)
        want = pg.sim3_mul(x, y)
        assert (np.abs(o - want) <= 1e-12 * S).all()
        q = o[3:7] / np.linalg.norm(o[3:7])
        R, _ = quat_to_rot_export(q, np.float64)
        assert np.abs(R - pg.quat_to_rot(q)).max() <= 1e-12


@pytest.mark.parametrize("n", SCALE_SIZES)
def test_depth_scale_pinned_to_the_oracle(n):
    maps = scale_maps(n, n)
    T0, T1, T2, _, _, _, _ = scale_stats_ref(*(v.astype(np.float64) for v in maps))
    s, c = so.depth_scale(*maps)
    for got, want in ((s, T0 / T1), (c, T2 / n)):
        assert abs(float(got) - want) <= (F32 + 1e-12) * abs(want)  # the oracle rounds its fp64 result to fp32


# ------------------------------------------------------------------------------- tests: bounds accept the fp32 mirror
@pytest.mark.parametrize("case", ROT_CASES, ids=ROT_IDS)
def test_edge_quaternion_bound_accepts_one_rounding(case):
    q, _, _, _ = rot_to_quat(case[1])
    assert (np.abs(q.astype(np.float32) - q) <= 2.0 ** -23 * np.abs(q) + Q_ABS).all()


def test_sim3_bound_accepts_the_fp32_product():
    a, b = random_pairs(20000)
    worst = max(sim3_err(sim3_mul_f32(x, y), x, y) for x, y in [(x, y) for _, x, y, _ in SIM3_CASES] + list(zip(a, b)))
    assert worst <= 0.5, worst  # about 3.3 u S measured: half the bound is left for FMA contraction
    _, meas, stored, _ = chain(60)
    assert max(sim3_err(stored[k + 1], stored[k], meas[k]) for k in range(60)) <= 0.5


def test_export_rotation_bound_accepts_fp32():
    a, _ = random_pairs(5000, seed=3)
    qs = np.concatenate([a[:, 3:7], a[:2500, 3:7] * np.float32(1.0 + 1e-3)])  # stored quaternions need not be unit
    for q in qs:
        got, _ = quat_to_rot_export(q, np.float32)
        ref, mag = quat_to_rot_export(q, np.float64)
        assert (np.abs(got.astype(np.float64) - ref) <= C_ROT * F32 * mag).all()


def _camera(seed, W=257, H=5):
    r = np.random.default_rng(seed)
    K = np.array([[W * r.uniform(0.8, 1.2), 0.3, W / 2 + r.uniform(-5, 5)],
                  [0, W * r.uniform(0.8, 1.2), H / 2 + r.uniform(-2, 2)], [0, 0, 1]], np.float32)
    R, _ = quat_to_rot_export(random_pairs(1, seed)[0][0, 3:7], np.float32)
    P = np.eye(4, dtype=np.float32)
    P[:3, :3], P[:3, 3] = R, r.uniform(-50, 50, 3)
    depth = r.uniform(-0.5, 4.0, (H, W)).astype(np.float32)
    return K, P, depth, f32(10.0 ** r.uniform(-1, 1))


def test_point_bound_accepts_the_fp32_unprojection():
    worst = 0.0
    for seed in range(8):
        K, P, depth, s = _camera(seed)
        for row in range(depth.shape[0]):
            for x in range(0, depth.shape[1] - 1):
                worst = max(worst, point_err(unproject_f32(K, P, x, row, depth[row], s), K, P, x, row, depth[row], s))
    assert worst <= 0.75, worst


@pytest.mark.parametrize("n", SCALE_SIZES)
@pytest.mark.parametrize("plant", [True, False], ids=["planted", "plain"])
def test_scale_bound_accepts_the_fp32_partition(n, plant):
    maps = scale_maps(n, n + plant, plant)
    s, c = scale_stats_f32(*maps)
    es, ec = scale_errs(s, c, scale_stats_ref(*(v.astype(np.float64) for v in maps)))
    assert es <= 1 and ec <= 1, (es, ec)


# ------------------------------------------------------------------------------- tests: bounds reject planted mistakes
def _rot_fails(mistake):
    for _, M, _ in ROT_CASES:
        q, _, _, _ = rot_to_quat(M)
        bad, _, _, _ = rot_to_quat(M, mistake)
        if (np.abs(bad.astype(np.float32) - q) > 2.0 ** -23 * np.abs(q) + Q_ABS).any():
            return True
    return False


def _sim3_fails(mistake):
    return any(sim3_err(sim3_mul_f32(a, b, mistake), a, b) > 1 for _, a, b, _ in SIM3_CASES)


def _point_fails(mistake):
    K, P, depth, s = _camera(0)
    return any(point_err(unproject_f32(K, P, x, 2, depth[2], s, mistake), K, P, x, 2, depth[2], s) > 1 for x in range(8))


def _chain_from_oracle_fails():
    """Nodes derived from the oracle's parent poses (the fp64 chain, rounded to fp32) instead of the stored parents,
    judged per step against the stored parent: the drift of the chain shows."""
    _, meas, stored, oracle = chain(60)
    return any(sim3_err(sim3_mul_f32(oracle[k].astype(np.float32), meas[k]), stored[k], meas[k]) > 1 for k in range(60))


MISTAKES = {
    "rot_to_quat:swap_jk": lambda: _rot_fails("swap_jk"),
    "rot_to_quat:transposed_R": lambda: _rot_fails("transpose"),
    "rot_to_quat:no_flip": lambda: _rot_fails("no_flip"),
    "sim3_mul:no_flip": lambda: _sim3_fails("no_flip"),
    "sim3_mul:RaT_tb": lambda: _sim3_fails("RaT_tb"),
    "sim3_mul:scale_twice": lambda: _sim3_fails("scale_twice"),
    "sim3_mul:scale_none": lambda: _sim3_fails("scale_none"),
    "unproject:K_T": lambda: _point_fails("K_T"),
    "unproject:next_column": lambda: _point_fails("next_column"),
    "chain_from_oracle_poses": _chain_from_oracle_fails,
}


@pytest.mark.parametrize("mistake", sorted(MISTAKES))
def test_planted_mistake_is_rejected(mistake):
    assert MISTAKES[mistake]()
