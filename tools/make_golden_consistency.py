"""Golden vectors for view_consistency_check: runs the UNMODIFIED reference function of
vista_slam/utils/slam_utils.py on the CPU (loaded as tools/make_golden_slam_utils.py does, with colorama shimmed) on
seeded scenes and stores inputs and counts in tests/golden/consistency.npz.

Scenes (name: what it pins):
  ray_<n>_<H>x<W>   ray-cast room views (oracle.consistency_oracle.raycast_scene), n in 1, 3, 9, 14 at 24x32 and
                    17x41: non-square pixels, non-integer principal points, depth holes, clipped windows;
  patch             ray_9_24x32 with a planted wrong-depth patch (x 1.3) in view 4;
  flipped           7 ray-cast views with view 3 turned 180 degrees about y: its neighbours see behind themselves, and
                    points that land off-image agree (z clamps to 1e-6, the sample is 0);
  coincident        exact arithmetic: K with power-of-two focal lengths, views 0 and 1 share a camera centre and view 0
                    has depth-0 pixels, which land at (K c)_z = 0 in view 1 (NaN, never agree);
  border            exact arithmetic: a fronto-parallel plane seen by cameras moved along x by whole pixels, so
                    projections fall exactly on the first and last columns and one column beyond them;
  overflow          exact arithmetic: a point with a tiny but nonzero (K c)_z, whose coordinate is finite in float32 but
                    overflows in grid_sample's unnormalisation (NaN there, so it never agrees), next to one that stays
                    finite and lands far off-image (samples 0, agrees: its clamped z is below the threshold).
The `exact` list names the scenes where every float32 operation of both implementations is exact."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_slam_utils import load_reference  # noqa: E402

from oracle import consistency_oracle as co  # noqa: E402

THRESHOLD = 0.05


def _pose(R, t):
    T = np.eye(4, dtype=np.float32)
    T[:3, :3], T[:3, 3] = R, t
    return T


def scenes():
    out = {}
    for H, W in ((24, 32), (17, 41)):
        for n in (1, 3, 9, 14):
            out["ray_%d_%dx%d" % (n, H, W)] = co.raycast_scene(100 * n + H, n, H, W)
    d, K, T = co.raycast_scene(909, 9, 24, 32)
    d = d.copy()
    d[4, 6:14, 10:20] *= np.float32(1.3)
    out["patch"] = (d, K, T)
    d, K, T = co.raycast_scene(707, 7, 24, 32)
    T = T.copy()
    T[3, :3, :3] = T[3, :3, :3] @ np.diag([-1, 1, -1]).astype(np.float32)
    out["flipped"] = (d, K, T)
    # exact scenes: K = [[8, 0, 4], [0, 8, 2], [0, 0, 1]] on 6 x 10 images
    H, W = 6, 10
    K = np.tile(np.array([[8, 0, 4], [0, 8, 2], [0, 0, 1]], np.float32), (3, 1, 1))
    d = np.full((3, H, W), 2.0, np.float32)
    d[0, 1:3, 2:5] = 0.0
    d[2, 4, 7] = 0.0
    T = np.stack([_pose(np.eye(3), [0.5, 0, 0]), _pose(np.eye(3), [0.5, 0, 0]), _pose(np.eye(3), [0.75, 0, 0])])
    out["coincident"] = (d, K, T)
    # a plane at z = 4: a shift of 0.5 along x moves projections by one pixel (f / z = 2 per unit)
    d = np.full((5, H, W), 4.0, np.float32)
    d[1] = 4.03125
    T = np.stack([_pose(np.eye(3), [0.5 * s, 0, 0]) for s in (0, 2, 5, 9, 10)])
    K = np.tile(np.array([[8, 0, 4], [0, 8, 2], [0, 0, 1]], np.float32), (5, 1, 1))
    out["border"] = (d, K, T)
    # overflow, on 2 x 2 images: view 1 sits at z = 2, behind view 0's points at z = 1, so c = (x, y, -1) and z clamps
    # to 1e-6.  K_1 = diag(1.5 2^99, 2^72, 2^-28): pixel (1, 0) gets u = -1.5 2^127, finite, but grid_sample's
    # (u / 1) * 2 overflows to -inf (NaN sample, no agreement); pixel (0, 1) gets v = -2^100, finite all the way, far
    # off-image (sample 0, agrees); pixel (0, 0) lands on the image and samples depth 1 (disagrees).
    d = np.ones((2, 2, 2), np.float32)
    K = np.stack([np.eye(3, dtype=np.float32), np.diag([1.5 * 2.0 ** 99, 2.0 ** 72, 2.0 ** -28]).astype(np.float32)])
    T = np.stack([_pose(np.eye(3), [0, 0, 0]), _pose(np.eye(3), [0, 0, 2])])
    out["overflow"] = (d, K, T)
    return out


def main():
    ref = load_reference()
    out = {"threshold": np.float32(THRESHOLD)}
    names = []
    for name, (d, K, T) in scenes().items():
        cnt = ref.view_consistency_check(torch.from_numpy(d), torch.from_numpy(K), torch.from_numpy(T), THRESHOLD)
        out[name + "_depth"], out[name + "_intri"], out[name + "_pose"] = d, K, T
        out[name + "_count"] = cnt.numpy()
        names.append(name)
        oc, amb = co.view_consistency(d, K, T, THRESHOLD)
        unamb = ~amb.any(-1)
        print("%-14s n=%2d %dx%d  ambiguous tests %.4f%%  oracle != reference on unambiguous pixels: %d  counts %s" % (
            name, d.shape[0], d.shape[1], d.shape[2], 100 * amb.sum() / max(1, d.size * min(8, d.shape[0] - 1)),
            int(((oc != out[name + "_count"]) & unamb).sum()), np.bincount(out[name + "_count"].ravel(), minlength=9)))
    out["names"] = np.array(names)
    out["exact"] = np.array(["coincident", "border", "overflow"])
    path = os.path.join(ROOT, "tests", "golden", "consistency.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
