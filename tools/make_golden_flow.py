"""Golden vectors for the keyframe flow tracker: runs the UNMODIFIED reference vista_slam/flow_tracker.py::FlowTracker
(numpy + cv2 only) on the seeded sequences of oracle/flow_tracker_oracle.py::sequences() and stores its outputs only
(the inputs are regenerated from the seeds) in tests/golden/flow.npz.

Per sequence <s> and frame t:
  <s>__decision [T] bool           compute_disparity's return value
  <s>__mean [T] float64            mean_disparity of the call, NaN when the call did not reach it
  <s>__tracked [T] int32           number of keyframe corners tracked by the call, -1 when it did not track
  <s>__next_pts [T][1000][2] fp32  calcOpticalFlowPyrLK's nextPts of the call (first `tracked` rows), NaN padding
  <s>__status [T][1000] uint8      its status, 255 padding
  <s>__ncorners [T] int32          corners of the keyframe after the call (0 when kf_pts is None)
  <s>__corners [T][1000][2] fp32   those corners, NaN padding
The LK outputs are the same cv2 call the tracker makes, repeated on the keyframe state before the call.  Every stored
mean is at least 2 % away from the threshold, so a decision cannot flip on rounding."""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
REFERENCE = "/root/reference/vista_slam/flow_tracker.py"
THRESHOLD = 5.0   # configs: flow_thres


def load_reference():
    spec = importlib.util.spec_from_file_location("reference_flow_tracker", REFERENCE)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    import cv2
    ref = load_reference()
    from oracle.flow_tracker_oracle import MAX_CORNERS, sequences
    out = {}
    for name, frames in sequences().items():
        T = len(frames)
        dec = np.zeros(T, bool)
        mean = np.full(T, np.nan)
        tracked = np.full(T, -1, np.int32)
        nxt = np.full((T, MAX_CORNERS, 2), np.nan, np.float32)
        st = np.full((T, MAX_CORNERS), 255, np.uint8)
        ncor = np.zeros(T, np.int32)
        cor = np.full((T, MAX_CORNERS, 2), np.nan, np.float32)
        tr = ref.FlowTracker(THRESHOLD)
        for t, img in enumerate(frames):
            kf_gray, kf_pts = tr.kf_gray, tr.kf_pts
            dec[t] = tr.compute_disparity(img)
            if tr.kf_pts is not None:
                ncor[t] = len(tr.kf_pts)
                cor[t, :ncor[t]] = tr.kf_pts.reshape(-1, 2)
            if tr.last_kf is None or kf_pts is None or len(kf_pts) < 10 or kf_gray is None:
                continue
            n, s, _ = cv2.calcOpticalFlowPyrLK(kf_gray, img, kf_pts, None, winSize=(21, 21), maxLevel=3,
                                               criteria=(cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, 30, 0.01))
            tracked[t] = len(kf_pts)
            nxt[t, :len(kf_pts)] = n.reshape(-1, 2)
            st[t, :len(kf_pts)] = s.flatten()
            good = s.flatten() == 1
            if good.sum() >= 10:
                mean[t] = float(np.mean(np.linalg.norm(n[good] - kf_pts[good], axis=1)))
                assert dec[t] == (mean[t] > THRESHOLD)
                assert abs(mean[t] - THRESHOLD) >= 0.02 * THRESHOLD, (name, t, mean[t])
            else:
                assert dec[t]
        for k, v in (("decision", dec), ("mean", mean), ("tracked", tracked), ("next_pts", nxt), ("status", st),
                     ("ncorners", ncor), ("corners", cor)):
            out[name + "__" + k] = v
        print(name, "decisions", dec.astype(int).tolist(), "mean", np.round(mean, 3).tolist(), "corners", ncor.tolist(),
              "tracked", [int((st[t] == 1).sum()) for t in range(T)])
    path = os.path.join(ROOT, "tests", "golden", "flow.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%.0f kB" % (os.path.getsize(path) / 1e3))


if __name__ == "__main__":
    main()
