"""Per-frame cost of keyframe selection on a seeded 224x224 stream.

    python tools/flow_stream.py [--frames 300] [--warmup 20] [--out result.json]

Each RGB frame is preprocessed on the device (SLAM_image_only.process_image) and its fp32 gray goes straight to
vista_slam_b200.flow_tracker.FlowTracker.compute_disparity; the timed span is that call, including its one host
synchronisation.  In the same run, if cv2 imports, the reference tracker (the flow_tracker.py algorithm with
cv2.goodFeaturesToTrack + cv2.calcOpticalFlowPyrLK, the reference's constants) is timed on this host's CPU on the
same uint8 frames; its span includes the device-to-host copy of the gray that the reference's call site needs.
Reports median and p90 ms split by keyframe and non-keyframe calls, with the GPU name and power limit and the CPU
count."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = [v.strip() for v in out[0].split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % type(e).__name__, "unknown"


def summarise(ms, kf):
    ms, kf = np.asarray(ms), np.asarray(kf, bool)
    out = {}
    for label, sel in (("all", np.ones_like(kf)), ("keyframe", kf), ("non_keyframe", ~kf)):
        v = ms[sel]
        out[label] = {"n": int(sel.sum()), "median_ms": float(np.median(v)) if len(v) else None,
                      "p90_ms": float(np.percentile(v, 90)) if len(v) else None}
    return out


class ReferenceTracker:
    """vista_slam/flow_tracker.py's FlowTracker.compute_disparity restated on cv2 for timing (visualize=False)."""

    def __init__(self, cv2, min_disparity):
        self.cv2, self.min_disparity = cv2, min_disparity
        self.kf_gray = self.kf_pts = None

    def init(self, img):
        self.kf_gray = img
        self.kf_pts = self.cv2.goodFeaturesToTrack(img, maxCorners=1000, qualityLevel=0.01, minDistance=8, blockSize=7)

    def compute_disparity(self, img):
        cv2 = self.cv2
        if self.kf_gray is None or self.kf_pts is None or len(self.kf_pts) < 10:
            self.init(img)
            return True
        nxt, st, _ = cv2.calcOpticalFlowPyrLK(self.kf_gray, img, self.kf_pts, None, winSize=(21, 21), maxLevel=3,
                                              criteria=(cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, 30, 0.01))
        st = st.flatten()
        good_kf, good_next = self.kf_pts[st == 1], nxt[st == 1]
        if len(good_kf) < 10 or np.mean(np.linalg.norm(good_next - good_kf, axis=1)) > self.min_disparity:
            self.init(img)
            return True
        return False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--threshold", type=float, default=5.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from oracle.flow_tracker_oracle import make_scene, warp_frame
    from vista_slam_b200.datasets.slam_images_only import SLAM_image_only
    from vista_slam_b200.flow_tracker import FlowTracker

    if not torch.cuda.is_available():
        raise SystemExit("flow_stream.py times the CUDA tracker: no CUDA device")
    n = args.warmup + args.frames
    scene = make_scene(7, 480 + 160, 640 + 400)
    # a camera drifting ~0.9 px / frame at 224x224 (about 2.1 px at 480x640), so keyframes come every few frames
    rgb = []
    for t in range(n):
        g = warp_frame(scene, 480, 640, 1.5 * (t % 200) - 150.0, 0.8 * np.sin(t / 9.0), 0.003 * np.sin(t / 17.0))
        rgb.append(torch.from_numpy(np.stack([g, np.roll(g, 2, 0), 255 - g], -1)).cuda())
    ds = SLAM_image_only([], resolution=(224, 224))
    tr = FlowTracker(args.threshold)
    ms, kf, grays = [], [], []
    for t in range(n):
        gray = ds.process_image(rgb[t])["gray"]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        is_kf = tr.compute_disparity(gray)
        t1 = time.perf_counter()
        if t >= args.warmup:
            ms.append((t1 - t0) * 1e3)
            kf.append(is_kf)
            grays.append(gray)
    name, power = gpu_info()
    try:
        cpus = len(os.sched_getaffinity(0))
    except AttributeError:
        cpus = os.cpu_count()
    res = {"frames": args.frames, "size": "224x224", "gpu": name, "power_limit": power,
           "device": summarise(ms, kf)}
    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is not None:
        ref = ReferenceTracker(cv2, args.threshold)
        rms, rkf = [], []
        for g in grays:
            t0 = time.perf_counter()
            img = (g.squeeze(0).cpu().numpy() * 255).astype(np.uint8)
            is_kf = ref.compute_disparity(img)
            rms.append((time.perf_counter() - t0) * 1e3)
            rkf.append(is_kf)
        res["host_cv2"] = dict(summarise(rms, rkf), cpus=cpus, cv2_threads=cv2.getNumThreads(), cv2=cv2.__version__)
        res["decisions_equal"] = bool(rkf == kf)
    else:
        res["host_cv2"] = "not measured (cv2 not importable)"
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
