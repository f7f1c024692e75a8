"""Cost of per-frame poses (OnlineSLAM.track, SLAMSessions.track, frame_trajectory) on a live-shaped stream.

A seeded 224 x 224 synthetic textured stream of --frames frames (a camera panning over a texture), OnlineSLAM's
defaults, random-init weights of the reference architecture and the golden DBoW3 vocabulary.  Keyframes are chosen by
FlowTracker.compute_disparities over the whole stream, as run.py would choose them one frame at a time.  Arms, in one
process, each after a warm-up run of its own, each timed segment ending in a device synchronise:
  keyframes      step on the keyframes only (what run.py does today);
  per_frame      step on the keyframes and track([frame]) on every other frame against the last keyframe; frames that
                 arrive before view 1 has been stepped are buffered and tracked right after it;
  chunk16        the same with the other frames buffered and tracked 16 at a time (and before each keyframe's step);
  sessions_S     S = 1, 4, 8 sessions stepped through the first 20 keyframes, then SLAMSessions.track with 16 frames
                 per session per call;
  trajectory     frame_trajectory() of the per_frame run after a pose_graph_optimize().
Per tracked frame: the call's time over its frames, p50 / p90 in ms.  Totals in s.  Prints the card's name and power
limit, read in the same run, and one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % r.stderr.strip())
    return r.stdout.strip()


def stats(v):
    v = np.sort(np.asarray(v) * 1e3)
    q = lambda p: float(v[int(p * (len(v) - 1))])
    return {"p50_ms": q(0.5), "p90_ms": q(0.9), "n": int(len(v))}


def stream(n, seed=0):
    H = W = 224
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand(1, 3, H // 8, 3 * W // 8, generator=g), size=(H, 3 * W),
                                           mode="bilinear")
    frames = []
    for i in range(n):
        x0 = int(round(i * 0.6)) % (2 * W)  # a slow pan: 0.6 pixel per frame
        img = (base[..., x0:x0 + W] * 2 - 1 + 0.03 * torch.randn(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        frames.append({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                       "view_name": "%05d" % i})
    return frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--warmup", type=int, default=120)
    a = ap.parse_args()
    from vista_slam_b200.flow_tracker import FlowTracker
    from vista_slam_b200.sessions import SLAMSessions
    from vista_slam_b200.slam import OnlineSLAM
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    torch.manual_seed(0)
    model = STA().cuda().eval()
    vocab = os.path.join(ROOT, "tests", "golden", "loop_vocab.txt")

    class Live(OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return model

    frames = stream(a.frames)
    is_kf = FlowTracker(5.0).compute_disparities(torch.stack([f["gray"][None] for f in frames]))

    def run(n, chunk):
        """Keyframes stepped, the other frames tracked `chunk` at a time (0: not tracked).  Returns (session, per-frame
        times of the track calls, total seconds)."""
        slam = Live("unused", vocab)
        per, buf = [], []

        def flush():
            if buf and slam.view_num >= 2:
                t0 = time.perf_counter()
                slam.track(buf)
                torch.cuda.synchronize()
                per.extend([(time.perf_counter() - t0) / len(buf)] * len(buf))
                buf.clear()

        torch.cuda.synchronize()
        t_all = time.perf_counter()
        for i in range(n):
            if is_kf[i]:
                flush()
                slam.step(frames[i])
            elif chunk:
                buf.append(frames[i])
                if len(buf) >= chunk:
                    flush()
        flush()
        torch.cuda.synchronize()
        return slam, per, time.perf_counter() - t_all

    print("card:", card(), flush=True)
    res = {"card": card(), "size": "224x224", "frames": a.frames, "keyframes": int(sum(is_kf))}
    for name, chunk in (("keyframes", 0), ("per_frame", 1), ("chunk16", 16)):
        run(a.warmup, chunk)
        slam, per, total = run(a.frames, chunk)
        res[name] = {"total_s": total, "tracked": len(per)}
        if per:
            res[name]["track_per_frame"] = stats(per)
        if name == "per_frame":
            slam.pose_graph_optimize()
            times = []
            for _ in range(20):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                slam.frame_trajectory()
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
            res["trajectory"] = dict(stats(times), frames=len(per))
        print(name, json.dumps(res[name]), flush=True)
        del slam
        torch.cuda.empty_cache()

    kfs = [f for f, k in zip(frames, is_kf) if k][:20]
    others = [f for f, k in zip(frames, is_kf) if not k]
    for S in (1, 4, 8):
        group = SLAMSessions("unused", vocab, S, frontend=model)
        group.step({k: kfs for k in range(S)})
        per = []
        for c in range(6):
            vals = {k: others[(16 * (c + k)) % (len(others) - 16):][:16] for k in range(S)}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            group.track(vals)
            torch.cuda.synchronize()
            if c:  # the first call warms the shapes up
                per.append((time.perf_counter() - t0) / (16 * S))
        res["sessions_%d" % S] = {"track_per_frame": stats(per), "frames_per_call": 16 * S}
        print("sessions_%d" % S, json.dumps(res["sessions_%d" % S]), flush=True)
        del group
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
