"""Cost of batched keyframe selection on seeded 224x224 streams, against the one-frame calls, in one process.

    python tools/flow_batch_stream.py [--frames 600] [--warmup 40] [--cam-frames 200] [--reps 3] [--out result.json]

The stream is tools/flow_stream.py's (a textured scene from oracle.flow_tracker_oracle.make_scene / warp_frame,
preprocessed to the 224x224 fp32 gray on the device).  Every timing ends in a device synchronise; the arms alternate
within each repetition and the medians over repetitions are reported.
  (a) FlowTracker.compute_disparity per frame over the stream (also its per-call latency, split by keyframe);
  (b) FlowTracker.compute_disparities over the whole stream, for each round length in --rounds (the module constant
      ROUND set for the arm);
  (c) S = 1 / 2 / 4 / 8 cameras, each with its own seeded 224x224 uint8 stream: per-camera compute_disparity against
      compute_disparities_group with one frame per camera per call (the live case: latency of one time step, p50 /
      p90), and the same over whole streams;
  (d) the offline flow pass from RGB frames on the device: process_image + compute_disparity per frame against
      process_images in chunks of --chunk + compute_disparities.
Every arm's decisions must equal the one-frame calls'; the tool stops otherwise.  The GPU name, power limit and SM
clocks are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))


def gpu_info():
    fields = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return dict(zip(fields.split(","), [v.strip() for v in out[0].split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"name": "unknown (%s)" % type(e).__name__}


def pct(v, q):
    return float(np.percentile(np.asarray(v), q)) if len(v) else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--cam-frames", type=int, default=200)
    ap.add_argument("--cams", default="1,2,4,8")
    ap.add_argument("--rounds", default="4,8,16,32")
    ap.add_argument("--chunk", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threshold", type=float, default=5.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from oracle.flow_tracker_oracle import make_scene, warp_frame
    from vista_slam_b200 import flow_tracker as ft
    from vista_slam_b200.datasets.slam_images_only import SLAM_image_only

    if not torch.cuda.is_available():
        raise SystemExit("flow_batch_stream.py times the CUDA tracker: no CUDA device")
    sync = torch.cuda.synchronize
    thr = args.threshold
    n = args.warmup + args.frames
    scene = make_scene(7, 480 + 160, 640 + 400)
    # flow_stream.py's camera: ~0.9 px / frame at 224x224, keyframes every few frames
    rgb = torch.stack([torch.from_numpy(np.stack([g, np.roll(g, 2, 0), 255 - g], -1)) for g in (
        warp_frame(scene, 480, 640, 1.5 * (t % 200) - 150.0, 0.8 * np.sin(t / 9.0), 0.003 * np.sin(t / 17.0))
        for t in range(n))]).cuda()
    ds = SLAM_image_only([], resolution=(224, 224))
    grays = torch.cat([ds.process_images(rgb[i:i + args.chunk])["gray"] for i in range(0, n, args.chunk)])
    warm, timed = grays[:args.warmup], grays[args.warmup:]
    rounds = [int(r) for r in args.rounds.split(",")]
    default_round = ft.ROUND

    def one_frame(frames, lat=None):
        tr = ft.FlowTracker(thr)
        dec = []
        sync()
        t0 = time.perf_counter()
        for i in range(frames.shape[0]):
            if lat is not None:
                sync()
                c0 = time.perf_counter()
            dec.append(tr.compute_disparity(frames[i]))
            if lat is not None:
                lat.append((time.perf_counter() - c0) * 1e3)
        sync()
        return dec, (time.perf_counter() - t0) * 1e3

    def batched(frames, R):
        ft.ROUND = R
        try:
            tr = ft.FlowTracker(thr)
            sync()
            t0 = time.perf_counter()
            dec = tr.compute_disparities(frames)
            sync()
            return dec, (time.perf_counter() - t0) * 1e3
        finally:
            ft.ROUND = default_round

    # warm-up of every shape
    one_frame(warm)
    for R in rounds:
        batched(warm, R)
    ref, _ = one_frame(timed)

    # (a) / (b)
    a_ms, a_lat, b_ms = [], [], {R: [] for R in rounds}
    for _ in range(args.reps):
        lat = []
        dec, ms = one_frame(timed, lat)
        assert dec == ref
        a_ms.append(ms)
        a_lat += lat
        for R in rounds:
            dec, ms = batched(timed, R)
            assert dec == ref, "round %d: decisions differ from compute_disparity" % R
            b_ms[R].append(ms)
    kf = np.array(ref * args.reps, bool)
    lat = np.asarray(a_lat)
    res = {"frames": args.frames, "size": "224x224", "keyframes": int(sum(ref)), "gpu": gpu_info(), "reps": args.reps,
           "default_round": default_round,
           "a_one_frame": {"stream_ms": float(np.median(a_ms)),
                           "per_frame_ms": float(np.median(a_ms)) / args.frames,
                           "call_p50_ms": {"keyframe": pct(lat[kf], 50), "non_keyframe": pct(lat[~kf], 50)},
                           "call_p90_ms": {"keyframe": pct(lat[kf], 90), "non_keyframe": pct(lat[~kf], 90)}},
           "b_batched": {str(R): {"stream_ms": float(np.median(b_ms[R])), "per_frame_ms": float(np.median(b_ms[R])) / args.frames,
                                  "speedup_vs_a": float(np.median(a_ms) / np.median(b_ms[R]))} for R in rounds}}

    # (c) cameras
    cams = [int(c) for c in args.cams.split(",")]
    S_max = max(cams)
    streams = []
    for k in range(S_max):
        sc = make_scene(200 + k, 224 + 200, 224 + 400)
        fr = [warp_frame(sc, 224, 224, 0.9 * (t % 150) - 60.0 + 3 * k, 0.6 * np.sin(t / (7.0 + k)), 0.002 * np.sin(t / 13.0))
              for t in range(args.cam_frames)]
        streams.append(torch.from_numpy(np.stack(fr)).cuda())
    cam_ref = []
    for k in range(S_max):
        dec, _ = one_frame(streams[k])
        cam_ref.append(dec)
    res["c_cameras"] = {}
    for S in cams:
        live_one, live_grp, whole_one, whole_grp = [], [], [], []
        for rep in range(args.reps + 1):  # the first repetition warms up
            trs = [ft.FlowTracker(thr) for _ in range(S)]
            dec = [[] for _ in range(S)]
            steps = []
            for t in range(args.cam_frames):
                sync()
                c0 = time.perf_counter()
                for k in range(S):
                    dec[k].append(trs[k].compute_disparity(streams[k][t]))
                sync()
                steps.append((time.perf_counter() - c0) * 1e3)
            assert dec == cam_ref[:S]
            trs = [ft.FlowTracker(thr) for _ in range(S)]
            dec = [[] for _ in range(S)]
            gsteps = []
            for t in range(args.cam_frames):
                sync()
                c0 = time.perf_counter()
                got = ft.compute_disparities_group(trs, [streams[k][t:t + 1] for k in range(S)])
                sync()
                gsteps.append((time.perf_counter() - c0) * 1e3)
                for k in range(S):
                    dec[k] += got[k]
            assert dec == cam_ref[:S], "group, one frame per camera: decisions differ"
            trs = [ft.FlowTracker(thr) for _ in range(S)]
            sync()
            c0 = time.perf_counter()
            dec = [[trs[k].compute_disparity(streams[k][t]) for t in range(args.cam_frames)] for k in range(S)]
            sync()
            w1 = (time.perf_counter() - c0) * 1e3
            trs = [ft.FlowTracker(thr) for _ in range(S)]
            sync()
            c0 = time.perf_counter()
            got = ft.compute_disparities_group(trs, streams[:S])
            sync()
            w2 = (time.perf_counter() - c0) * 1e3
            assert dec == cam_ref[:S] and got == cam_ref[:S], "whole streams: decisions differ"
            if rep:
                live_one += steps
                live_grp += gsteps
                whole_one.append(w1)
                whole_grp.append(w2)
        res["c_cameras"][str(S)] = {
            "live_step_ms": {"per_camera_calls": {"p50": pct(live_one, 50), "p90": pct(live_one, 90)},
                             "group": {"p50": pct(live_grp, 50), "p90": pct(live_grp, 90)}},
            "whole_stream_ms": {"per_camera_calls": float(np.median(whole_one)), "group": float(np.median(whole_grp)),
                                "frames": S * args.cam_frames}}

    # (d) offline flow pass from RGB
    rgb_t = rgb[args.warmup:]
    d_one, d_bat = [], []
    for rep in range(args.reps + 1):
        tr = ft.FlowTracker(thr)
        sync()
        t0 = time.perf_counter()
        dec = [tr.compute_disparity(ds.process_image(rgb_t[i])["gray"]) for i in range(rgb_t.shape[0])]
        sync()
        m1 = (time.perf_counter() - t0) * 1e3
        assert dec == ref
        tr = ft.FlowTracker(thr)
        sync()
        t0 = time.perf_counter()
        dec = []
        for i in range(0, rgb_t.shape[0], args.chunk):
            dec += tr.compute_disparities(ds.process_images(rgb_t[i:i + args.chunk])["gray"])
        sync()
        m2 = (time.perf_counter() - t0) * 1e3
        assert dec == ref, "offline pass: decisions differ"
        if rep:
            d_one.append(m1)
            d_bat.append(m2)
    res["d_offline_from_rgb"] = {"per_frame_calls_ms": float(np.median(d_one)), "chunked_ms": float(np.median(d_bat)),
                                 "chunk": args.chunk, "speedup": float(np.median(d_one) / np.median(d_bat))}
    res["decisions_equal"] = True
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
