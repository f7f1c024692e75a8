"""Time the SLAM evaluation at an evaluation run's size: the synthetic room of oracle/eval_oracle.py rendered at 400
views x 224 x 224 (about 20 M ground-truth points), written in save_data_all's format, then
  * GPU: eval_recon_from_saved_data and full_traj_eval of vista_slam_b200.eval, per stage (load, clouds, align,
    downsample, ICP, Chamfer) with a device synchronisation after each, after one warm-up run;
  * host: the oracle (numpy, scipy cKDTree with workers=-1) on the same files, per stage.
Prints the card's name and power limit and the host's CPU count, and one JSON line.

    python tools/eval_stream.py [--views 400] [--size 224] [--reps 3] [--host-reps 1] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from oracle import eval_oracle as eo  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = "%s (power limit unknown: %s)" % (torch.cuda.get_device_name(), e)
    return q


def gpu_run(folder):
    from vista_slam_b200.eval import eval_recon as R
    from vista_slam_b200.eval.eval_traj import full_traj_eval
    times = {}
    t = [time.perf_counter()]

    def tick(name):
        torch.cuda.synchronize()
        now = time.perf_counter()
        times[name] = now - t[0]
        t[0] = now

    est = list(np.load(os.path.join(folder, "trajectory.npy")))
    ref = list(np.load(os.path.join(folder, "gt_poses.npy")))
    t0 = time.perf_counter()
    _, _, r, tr, s, ape = full_traj_eval(est, ref, os.path.join(folder, "plots"), "traj")
    times["traj"] = time.perf_counter() - t0
    t[0] = time.perf_counter()
    acc, comp, ch, gp, ep = R._from_saved_data(folder, [r, tr, s], tick)
    times["total_recon"] = sum(v for k, v in times.items() if k != "traj")
    return times, {"rmse_acc": acc, "rmse_comp": comp, "chamfer": ch, "n_gt": len(gp), "n_est": len(ep), "ape_rmse": ape["rmse"]}


def host_run(folder):
    times = {}
    t0 = time.perf_counter()
    est = list(np.load(os.path.join(folder, "trajectory.npy")))
    ref = list(np.load(os.path.join(folder, "gt_poses.npy")))
    _, _, r, tr, s, ape = eo.full_traj_eval(est, ref)
    times["traj"] = time.perf_counter() - t0
    t = time.perf_counter()
    d = eo.load(folder)
    times["load"] = time.perf_counter() - t
    t = time.perf_counter()
    gt, e = eo.clouds(torch.from_numpy(d["gt_depths"]), torch.from_numpy(d["gt_poses"]).float(),
                      torch.from_numpy(d["gt_intrinsic"]), torch.from_numpy(d["unscaled_depths"] * d["scales"]).float(),
                      torch.from_numpy(d["poses"]).float(), torch.from_numpy(d["intrinsics"]).float(),
                      torch.from_numpy(d["confs"] > d["conf_thres"]).float())
    times["clouds"] = time.perf_counter() - t
    t = time.perf_counter()
    e = eo.transform(e, eo.initial_alignment(r, tr, s))
    times["align"] = time.perf_counter() - t
    t = time.perf_counter()
    ed, gd = eo.voxel_down(e, eo.VOXEL), eo.voxel_down(gt, eo.VOXEL)
    times["downsample"] = time.perf_counter() - t
    t = time.perf_counter()
    reg = eo.icp(ed, gd)
    times["icp"] = time.perf_counter() - t
    t = time.perf_counter()
    e = eo.transform(e, reg["transformation"])
    ch, acc, comp, _, _ = eo.chamfer(gt.astype(np.float64), e, eo.MAX_ERROR, workers=-1)
    times["chamfer"] = time.perf_counter() - t
    times["total_recon"] = sum(v for k, v in times.items() if k != "traj")
    return times, {"rmse_acc": acc, "rmse_comp": comp, "chamfer": ch, "n_gt": len(gt), "n_est": len(e), "ape_rmse": ape["rmse"],
                   "icp_iterations": reg["iterations"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=400)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_stream.py times the GPU path and needs a CUDA device")
    from vista_slam_b200 import build
    build.build()
    card = _card()
    cpus = len(os.sched_getaffinity(0))
    print("card:", card, "| host CPUs:", cpus, flush=True)
    with tempfile.TemporaryDirectory() as d:
        t = time.perf_counter()
        eo.write_scene(eo.make_scene(n_views=a.views, H=a.size, W=a.size, seed=0, nan_view=7), d)
        print("rendered %d views at %dx%d in %.1f s" % (a.views, a.size, a.size, time.perf_counter() - t), flush=True)
        gpu_run(d)  # warm-up
        gpu = [gpu_run(d) for _ in range(a.reps)]
        for k, (tm, res) in enumerate(gpu):
            print("gpu rep %d:" % k, json.dumps({x: round(v * 1e3, 2) for x, v in tm.items()}), "ms", res, flush=True)
        host = [host_run(d) for _ in range(a.host_reps)]
        for k, (tm, res) in enumerate(host):
            print("host rep %d:" % k, json.dumps({x: round(v * 1e3, 1) for x, v in tm.items()}), "ms", res, flush=True)
    med = {k: float(np.median([g[0][k] for g in gpu])) * 1e3 for k in gpu[0][0]}
    hmed = {k: float(np.median([h[0][k] for h in host])) * 1e3 for k in host[0][0]}
    rec = {"card": card, "host_cpus": cpus, "views": a.views, "size": a.size, "gpu_ms_median": med, "host_ms_median": hmed,
           "gpu_result": gpu[0][1], "host_result": host[0][1]}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
