"""S SLAM sessions on one H100: SLAMSessions against sessions stepped one after another, at 224 x 224.

Each session runs its own seeded textured stream (the frames of tools/slam_batch_stream.py, one seed per session) with
OnlineSLAM's defaults, random-init weights of the reference architecture and the golden DBoW3 vocabulary.  For
S in --sessions, one process alternates whole runs of four arms after a warm-up run of each:

  (a) step:           for every keyframe index t, sessions[k].step(frame t) for k = 0 .. S-1;
  (b) group_step:     SLAMSessions.step({k: [frame t]}) for every t (the live case: one keyframe per session per call);
  (c) step_many:      for every chunk of 32, sessions[k].step_many(chunk) for k = 0 .. S-1;
  (d) group_step_32:  SLAMSessions.step({k: chunk of 32}) for every chunk.

Every run is timed from its first call to a device synchronise after its last; (b) also times each call to a device
synchronise for its latency percentiles.  Device memory in use (cudaMemGetInfo, after emptying PyTorch's cache, less
the memory in use before any model was built) is read with one keyframe stepped in each session, for SLAMSessions on one
shared model and for S independent OnlineSLAM objects, each with its own model and vocabulary.  Prints the card's name
and power limit, then one JSON line.  --profile writes a torch.profiler table of arm (b) at the largest S instead."""
import argparse
import copy
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
VOCAB = os.path.join(ROOT, "tests", "golden", "loop_vocab.txt")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def stream(seed, n, H=224, W=224):
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(1, 3, H // 8, W // 4, generator=g)
    values = []
    for i in range(n):
        img = torch.nn.functional.interpolate(base.roll(i % (W // 4), dims=3)[..., :W // 8], size=(H, W), mode="bilinear")
        img = ((img * 2 - 1) + 0.05 * torch.randn(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        values.append({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                       "view_name": "%05d" % i})
    return values


def used_bytes():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    return total - free


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="1,2,4,8")
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--chunk", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--profile", default=None, help="write a torch.profiler table of arm (b) at the largest S here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vista_slam_b200.sessions import SLAMSessions
    from vista_slam_b200.slam import OnlineSLAM
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    sizes = [int(s) for s in a.sessions.split(",")]
    n, C, Smax = a.views, a.chunk, max(sizes)
    print("card:", card(), flush=True)

    torch.manual_seed(0)
    template = STA().eval()  # host copy of the random-init weights
    res = {"card": card(), "size": "224x224", "views_per_session": n, "chunk": C, "rounds": a.rounds, "memory_gb": {},
           "arms": {}}
    if a.profile is None:
        # memory: S independent OnlineSLAM objects (own model and vocabulary each), then SLAMSessions on one model
        base = used_bytes()
        first = stream(99, 1)

        class Own(OnlineSLAM):
            def load_frontend(self, ckpt_path):
                return copy.deepcopy(template).cuda()

        own, mem_own = [], {}
        for S in range(1, Smax + 1):
            own.append(Own("unused", VOCAB))
            own[-1].step(first[0])
            if S in sizes:
                mem_own[S] = used_bytes() - base
        del own
        model = copy.deepcopy(template).cuda()
        mem_ses = {}
        for S in sizes:
            ses = SLAMSessions("unused", VOCAB, S, frontend=model)
            ses.step({k: first for k in range(S)})
            mem_ses[S] = used_bytes() - base
            del ses
        for S in sizes:
            res["memory_gb"][S] = {"sessions": round(mem_ses[S] / 2**30, 2), "independent": round(mem_own[S] / 2**30, 2)}
        print(json.dumps({"memory_gb": res["memory_gb"]}), flush=True)
    else:
        model = copy.deepcopy(template).cuda()
    del template
    streams = [stream(1 + k, n) for k in range(Smax)]

    def run(arm, S, views, lat=None):
        ses = SLAMSessions("unused", VOCAB, S, frontend=model)
        vs = [s[:views] for s in streams[:S]]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if arm == "step":
            for t in range(views):
                for k in range(S):
                    ses[k].step(vs[k][t], force_pgo=(t == views - 1))
        elif arm == "group_step":
            for t in range(views):
                c0 = time.perf_counter()
                ses.step({k: [vs[k][t]] for k in range(S)}, force_pgo=range(S) if t == views - 1 else ())
                if lat is not None:
                    torch.cuda.synchronize()
                    lat.append(time.perf_counter() - c0)
        elif arm == "step_many":
            for c in range(0, views, C):
                for k in range(S):
                    ses[k].step_many(vs[k][c:c + C], force_pgo=(c + C >= views))
        else:
            for c in range(0, views, C):
                ses.step({k: vs[k][c:c + C] for k in range(S)}, force_pgo=range(S) if c + C >= views else ())
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        tables = [s._graph.edges[:s.num_edges].cpu().numpy() for s in ses.sessions]
        del ses
        gc.collect()
        return dt, tables

    arms = ["step", "group_step", "step_many", "group_step_32"]
    if a.profile is not None:
        from torch.profiler import ProfilerActivity, profile
        run("group_step", Smax, min(n, 40))
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            dt, _ = run("group_step", Smax, min(n, 40))
        os.makedirs(os.path.dirname(os.path.abspath(a.profile)), exist_ok=True)
        with open(a.profile, "w") as f:
            f.write("group_step S=%d, %d calls, %.3f s (profiled)\n" % (Smax, min(n, 40), dt))
            f.write(prof.key_averages().table(sort_by="cpu_time_total", row_limit=40))
            f.write("\n")
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
        print("profile written to", a.profile, flush=True)
        return
    for S in sizes:  # warm-up: every shape and CUDA graph of every arm
        for arm in arms:
            run(arm, S, min(n, 2 * C + 8))
    times = {S: {arm: [] for arm in arms} for S in sizes}
    lat = {S: [] for S in sizes}
    agree = {S: {} for S in sizes}
    for _ in range(a.rounds):
        for S in sizes:
            ref = None
            for arm in arms:
                dt, tables = run(arm, S, n, lat[S] if arm == "group_step" else None)
                times[S][arm].append(dt)
                ref = tables if ref is None else ref
                agree[S][arm] = all(x.shape == y.shape and np.array_equal(x, y) for x, y in zip(tables, ref))
    for S in sizes:
        r = {}
        for arm in arms:
            best = min(times[S][arm])
            r[arm] = {"keyframes_per_s": round(S * n / best, 1), "seconds_all": [round(x, 3) for x in times[S][arm]],
                      "edges_equal_step": agree[S][arm]}
        ms = 1e3 * np.array(lat[S])
        r["group_step"].update(call_ms_p50=round(float(np.percentile(ms, 50)), 2),
                               call_ms_p90=round(float(np.percentile(ms, 90)), 2))
        for arm in arms[1:]:
            r[arm]["speedup_vs_step"] = round(r[arm]["keyframes_per_s"] / r["step"]["keyframes_per_s"], 3)
        res["arms"][S] = r
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
