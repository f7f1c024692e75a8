"""Time LoopDetector.detect_loop per keyframe on the GPU beside the host path (cv2 ORB + the compiled unmodified DBoW3
of oracle/_ref/, scored view by view as vista_slam/loop_detector.py does), with a synthetic full-size vocabulary.

    python tools/loop_stream.py [--views 100 400] [--keyframes 40] [--out DIR]

The vocabulary is a complete k = 10, L = 6 tree (1 111 111 nodes, 10^6 words, random descriptors and TF-IDF weights),
written as an uncompressed DBoW3 binary stream to a temporary directory.  For each database size N, N seeded 224x224
keyframes are added first (untimed), then `--keyframes` more are timed one detect_loop each, with farthest_neighbor =
i - 3; each GPU timing includes the call's one host synchronisation.  The host path runs when cv2 and oracle/_ref/ are
present and is reported as not measured otherwise.  Prints one JSON line (also written to DIR/loop_stream.json)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import loop_detector_oracle as O  # noqa: E402


def write_full_vocab(path, k=10, L=6, seed=0):
    rng = np.random.default_rng(seed)
    n = (k ** (L + 1) - 1) // (k - 1)
    first_leaf = (k ** L - 1) // (k - 1)
    rec = np.zeros(n - 1, np.dtype([("nid", "<u4"), ("pid", "<u4"), ("w", "<f8"), ("cols", "<i4"), ("rows", "<i4"),
                                     ("type", "<i4"), ("d", "u1", 32)]))
    ids = np.arange(1, n, dtype=np.uint32)
    rec["nid"], rec["pid"] = ids, (ids - 1) // k
    rec["w"] = np.where(ids >= first_leaf, rng.random(n - 1) * 5, 0.0)
    rec["cols"], rec["rows"], rec["type"] = 32, 1, 0
    rec["d"] = rng.integers(0, 256, (n - 1, 32), dtype=np.uint8)
    words = np.zeros(n - first_leaf, np.dtype([("wid", "<u4"), ("nid", "<u4")]))
    words["wid"] = np.arange(n - first_leaf)
    words["nid"] = np.arange(first_leaf, n)
    with open(path, "wb") as f:
        f.write(np.array([88877711233], "<u8").tobytes() + b"\0" + np.array([n], "<u4").tobytes())
        f.write(np.array([k, L, 0, O.TF_IDF], "<i4").tobytes())
        f.write(rec.tobytes())
        f.write(np.array([len(words)], "<u4").tobytes())
        f.write(words.tobytes())


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": round(float(np.median(ms)), 4), "p90_ms": round(float(np.percentile(ms, 90)), 4),
            "n": int(len(ms))}


def host_detect(ref, orb, feats, img, farthest, dist_min=40, nms=40, thresh_neighbor=5):
    """The reference's detect_loop (loop_detector.py:23-50) over cv2 ORB and the compiled DBoW3."""
    _, des = orb.detectAndCompute(img, None)
    feats.append(ref.transform(des) if des is not None else None)
    i = len(feats) - 1
    fi = feats[i]
    sims = [ref.score(fi, feats[j]) for j in range(max(0, i - thresh_neighbor), i)
            if fi is not None and feats[j] is not None]
    th = min(sims) if sims else 1.0
    last, out = farthest, []
    for j in reversed(range(farthest)):
        if last - j > nms and i - j > dist_min and fi is not None and feats[j] is not None:
            s = ref.score(fi, feats[j])
            if s > th:
                out.append((j, s))
                last = j
    return sorted(out, key=lambda c: c[1], reverse=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="+", default=[100, 400])
    ap.add_argument("--keyframes", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("loop_stream.py measures the GPU path: no CUDA device")
    from vista_slam_b200.loop_detector import LoopDetector
    try:
        import cv2
        from oracle.dbow3_ref import RefVocabulary, build as dbow3_ref
        lib = dbow3_ref.load()
    except ImportError:
        cv2, lib = None, None
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    result = {"gpu": gpu, "vocab": "k=10 L=6 synthetic, 1111111 nodes", "frame": "224x224 uint8"}
    with tempfile.TemporaryDirectory() as tmp:
        vpath = os.path.join(tmp, "voc.bin")
        write_full_vocab(vpath)
        total = max(args.views) + args.keyframes
        frames = O.make_sequence(3, total, 224, 224, revisit_after=60)
        dev = [torch.from_numpy(f).cuda() for f in frames]
        ref = None
        if lib is not None and cv2 is not None:
            ref = RefVocabulary(lib)
            t0 = time.perf_counter()
            ref.load(vpath)
            result["host_vocab_load_s"] = round(time.perf_counter() - t0, 2)
        for nv in args.views:
            det = LoopDetector(vpath, 40, 40, 5)
            for t in range(nv):
                det.compute_bow_feat(dev[t])
            ms = []
            for t in range(nv, nv + args.keyframes):
                torch.cuda.synchronize()
                a = time.perf_counter()
                det.detect_loop(dev[t], t - 3)
                ms.append((time.perf_counter() - a) * 1e3)
            entry = {"gpu": stats(ms)}
            if ref is not None:
                orb, feats = cv2.ORB_create(), []
                for t in range(nv):
                    _, des = orb.detectAndCompute(frames[t], None)
                    feats.append(ref.transform(des) if des is not None else None)
                hms = []
                for t in range(nv, nv + args.keyframes):
                    a = time.perf_counter()
                    host_detect(ref, orb, feats, frames[t], t - 3)
                    hms.append((time.perf_counter() - a) * 1e3)
                entry["host"] = stats(hms)
            else:
                entry["host"] = "not measured (cv2 or oracle/_ref/libdbow3_ref.so missing)"
            result["views_%d" % nv] = entry
            del det
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "loop_stream.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
