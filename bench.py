"""STA image-pairs/s benchmark (BASELINE.json metric) -- contract: see the task statement / DESIGN.md.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference] [--pairs P] [--height H] [--width W]
                    [--dump-outputs DIR]

* b200 arm (default): one process per GPU (torchrun sets RANK/LOCAL_RANK/WORLD_SIZE).  Rank 0 initialises the
  weights, one NCCL broadcast of the packed weight arena, then every rank runs `--pairs` synthetic
  512x384 bf16 pairs per step, independently (weak scaling, no data-path collective).
  `value`   = whole-job pairs/s with the inputs resident in HBM (CUDA events, max over ranks).
  `e2e`     = the same metric through the host-buffer C-ABI call sta_forward_pairs_host: pinned-host ->
              device copies of both image batches and device -> host copies of all four outputs are
              inside the timed region.
  `roofline`= tensor-pipe roofline of the dominant kernel family (wgmma GEMM / implicit-GEMM conv),
              timed live with CUDA events on the launch stream (sta_profile).
  `--dump-outputs DIR` writes what the last timed step returned on rank 0 -- with --gpus N > 1 that is rank 0's own
              pair shard only -- as DIR/<view>_<output>.npy, float32: the
              pose outputs whole, the dense maps as a fixed seeded sample (DUMP_SAMPLE elements each), so that two
              builds can be compared output for output on identical inputs (seeded images and weights).
  `cpu_baseline` = the oracle (PyTorch fp32 CPU port of the reference, oracle/sta_oracle.py) timed on the
              host cores on a bounded sample (rank 0, N=1 only).
* reference arm (`--impl reference`): the reference's own CPU implementation of the path = the oracle
  port (a Python reference cannot travel to the GPU box), all host threads, one 512x384 pair per step.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "sta_image_pairs_per_sec"
UNIT = "pairs/s"


def make_config(P, world, H, W, total=None):
    from vista_slam_b200.flops import flops_per_pair
    if total is not None:  # cfg-5: a fixed global batch split contiguously over the ranks (strong scaling)
        from vista_slam_b200.dist import pair_shard
        shards = [pair_shard(total, r, world) for r in range(world)]
        return {"workload": "cfg-5: %d synthetic %dx%d bf16 pairs per step in total, contiguous B/R shard per rank (%s pairs), "
                            "STA forward only, random-init weights" % (total, W, H, "/".join(str(b - a) for a, b in shards)),
                "pairs_per_gpu": max(b - a for a, b in shards), "global_pairs": total, "height": H, "width": W,
                "parallelism": "contiguous pair shard per rank (vista_slam_b200/dist.py::pair_shard), 1 NCCL weight broadcast, "
                               "no data-path collective",
                "l2_policy": "no explicit flush: weights (0.88 GB) + activations exceed the 50 MB L2",
                "gflop_per_pair": flops_per_pair(H, W) / 1e9}
    return {"workload": "cfg-2: %d synthetic %dx%d bf16 pairs per GPU per step, STA forward only "
                        "(2 enc + symmetric dec + 2 DPT + 2 pose heads per pair), random-init weights" % (P, W, H),
            "pairs_per_gpu": P, "global_pairs": P * world, "height": H, "width": W,
            "parallelism": "pair shard per rank, 1 NCCL weight broadcast, no data-path collective",
            "l2_policy": "no explicit flush: per-step working set (0.88 GB weights + >2 GB activations) "
                         "exceeds the 50 MB L2",
            "gflop_per_pair": flops_per_pair(H, W) / 1e9}


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"bf16_burst": d.get("bf16_tflops"), "bf16_sustained": d.get("bf16_tflops_sustained"),
                "hbm_gbs": d.get("hbm_gbs"), "source": "measured (MEASURED_PEAKS.json)"}
    # NVIDIA H100 SXM data sheet (700 W card): dense BF16 989 TFLOP/s, HBM3 3.35 TB/s -- not a measured rate
    return {"bf16_burst": 989.0, "bf16_sustained": None, "hbm_gbs": 3350.0, "source": "H100 SXM data sheet (dense BF16)"}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index = index
        self.lines = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "200"], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
            import atexit
            atexit.register(self._kill)  # never leave the sampling process behind (an exception before stop())
        except Exception:
            self.proc = None

    def _kill(self):
        try:
            if self.proc is not None and self.proc.poll() is None:
                self.proc.kill()
        except Exception:
            pass

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def mark(self):
        """Index of the next sample: call right before / after the timed region (the process is started BEFORE the warm-up,
        because a cold `nvidia-smi` start-up takes driver locks for tens of milliseconds and would stall the first launches
        of the timed region -- measured: +66..82 ms on a 170 ms region in the first process on a fresh box)."""
        return len(self.lines)

    def stop(self, first=0, last=None):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        if last is not None:
            last = max(last, first) + 1  # the sample that was being taken when the region ended
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, smax, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in (self.lines[first:last] or self.lines[-1:]):  # samples taken during the timed region
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                smax = float(f[1])
            except ValueError:
                continue
            for nm, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": smax, "reasons": sorted(reasons),
                "samples": len(sm)}


DUMP_SAMPLE = 1 << 20  # elements kept of each dense output by --dump-outputs


def dump_outputs(out_dir, views):
    """Write the outputs of one forward_pairs call ((view1, view2) dicts of tensors) as float32 .npy files.  Outputs with
    more than DUMP_SAMPLE elements are sampled at DUMP_SAMPLE flat indices drawn once from a fixed seed (sorted), so the
    files of two runs with the same arguments line up element for element; at most ~4 MB per file, ~17 MB in all at cfg-2."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    written = {}
    for v, d in enumerate(views):
        for key in sorted(d):
            a = d[key].detach().float().cpu().numpy().reshape(-1)
            if a.size > DUMP_SAMPLE:
                idx = np.sort(np.random.default_rng(20240917).choice(a.size, DUMP_SAMPLE, replace=False))
                a = a[idx]
            name = "view%d_%s" % (v + 1, key)
            np.save(os.path.join(out_dir, name + ".npy"), np.ascontiguousarray(a, dtype=np.float32))
            written[name] = int(a.size)
    return written


def cpu_port_baseline(H, W, budget_s=45.0):
    """Time the oracle (fp32 CPU port of the reference path) with BASELINE.md section 3's protocol -- 1 warm-up + 3 timed
    repetitions, median -- at (B=1, 224x224), (B=1, HxW) and, if the budget allows, (B=4, HxW).  `value` is the
    (B=1, HxW) median, the same measurement the `--impl reference` arm makes."""
    import torch

    from oracle.sta_oracle import StaOracle, flops_per_pair, make_images, make_state_dict, usable_cpus
    torch.set_num_threads(usable_cpus())
    cores = torch.get_num_threads()
    orc = StaOracle(make_state_dict(0), emulate_bf16=False)
    t_start = time.perf_counter()

    def med(B, h, w, reps=3):
        a, b = make_images(B, h, w, 1234)
        with torch.no_grad():
            orc.forward_pair(a, b)  # warm-up
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                orc.forward_pair(a, b)
                ts.append(time.perf_counter() - t0)
        t = statistics.median(ts)
        return {"pairs_per_s": B / t, "s_per_call": t, "gflops": B * flops_per_pair(h, w) / t / 1e9, "reps": reps}

    detail = {"b1_224x224": med(1, 224, 224)}
    full = med(1, H, W)
    detail["b1_%dx%d" % (W, H)] = full
    spent = time.perf_counter() - t_start
    if spent + 4 * 4 * full["s_per_call"] < budget_s:
        detail["b4_%dx%d" % (W, H)] = med(4, H, W)
    return {"value": full["pairs_per_s"], "unit": UNIT, "cores": cores, "kind": "port",
            "sample": "oracle port (PyTorch fp32 CPU restatement of the reference), %d threads: 1 warm-up + 3 timed single-pair "
                      "forwards at %dx%d, median (%.2f s each); other shapes in `detail`" % (cores, W, H, full["s_per_call"]),
            "detail": detail}


def run_reference_arm(args, rank, world):
    if rank != 0:
        return
    H, W = args.height, args.width
    import torch

    from oracle.sta_oracle import StaOracle, make_images, make_state_dict, usable_cpus
    torch.set_num_threads(usable_cpus())
    orc = StaOracle(make_state_dict(0), emulate_bf16=False)
    img1, img2 = make_images(1, H, W, 1234)
    with torch.no_grad():
        for _ in range(args.warmup):
            orc.forward_pair(img1, img2)
        t0 = time.perf_counter()
        for _ in range(args.steps):
            orc.forward_pair(img1, img2)
        dt = time.perf_counter() - t0
    v = args.steps / dt
    cores = torch.get_num_threads()
    line = {
        "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "fp32", "data": "synthetic", "impl": "reference",
        "config": make_config(args.pairs, args.gpus, H, W),  # identical to the b200 arm's (the sample is described below)
        "cpu_baseline": {"value": v, "unit": UNIT, "cores": cores, "kind": "port",
                         "sample": "reference CPU path = oracle port (PyTorch fp32, %d threads); each step is a bounded sample "
                                   "of the workload: 1 pair of the %d-pair batch at %dx%d; %d timed steps after %d warm-up"
                                   % (cores, args.pairs, W, H, args.steps, args.warmup)},
        "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def run_b200_arm(args, rank, local_rank, world):
    import torch
    import torch.distributed as dist

    from vista_slam_b200.flops import attention_flops_per_pair, flops_per_pair
    from vista_slam_b200 import _lib
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    H, W, P = args.height, args.width, args.pairs
    total = args.total_pairs
    if total is not None:  # cfg-5 strong scaling: this rank's contiguous block of the global batch
        from vista_slam_b200.dist import pair_shard
        lo, hi = pair_shard(total, rank, world)
        P = hi - lo
        if P == 0:
            raise SystemExit("--total-pairs %d leaves rank %d without work" % (total, rank))
    sampler = ClockSampler(local_rank)  # started long before the timed region (see ClockSampler.mark)
    if rank == 0:
        sampler.start()
    model = STA()  # random-init weights of the reference architecture (no network for the checkpoint)
    model.eval()
    if world > 1:
        model.broadcast_weights(src=0, device=dev)  # one NCCL broadcast of the packed arena over NVLink
    else:
        model._ready(torch.empty(1, device=dev))
    g = torch.Generator().manual_seed(1234 + rank)
    h1 = (torch.rand(P, 3, H, W, generator=g) * 2 - 1).bfloat16().pin_memory()
    h2 = (torch.rand(P, 3, H, W, generator=g) * 2 - 1).bfloat16().pin_memory()
    d1, d2 = h1.to(dev), h2.to(dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        if world == 1:
            return x
        t = torch.tensor([x], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # ---------------- device-resident throughput (`value`) ----------------
    for _ in range(args.warmup):
        model.forward_pairs(d1, d2)
    barrier()
    s_first = sampler.mark()
    l0 = model.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = model.forward_pairs(d1, d2)
    e1.record()
    barrier()
    ms_total = max_over_ranks(e0.elapsed_time(e1))
    launches = model.launch_count - l0
    clocks = sampler.stop(s_first, sampler.mark()) if rank == 0 else None
    ms_step = ms_total / args.steps
    global_pairs = total if total is not None else world * P
    value = global_pairs / (ms_step / 1e3)
    ok = bool(torch.isfinite(out[0]["pts3d_pred"]).all()) and bool(torch.isfinite(out[1]["relative_pose"]).all())
    dumped = dump_outputs(args.dump_outputs, out) if (args.dump_outputs and rank == 0) else None

    # ---------------- end-to-end through the host-buffer C-ABI call (`e2e`) ----------------
    hout = {"pts3d": torch.empty(2, P, H, W, 3).pin_memory(), "conf": torch.empty(2, P, H, W).pin_memory(),
            "pose": torch.empty(2, P, 4, 4).pin_memory(), "pose_conf": torch.empty(2, P).pin_memory()}
    for _ in range(max(1, min(args.warmup, 2))):
        model.forward_pairs_host(h1, h2, hout)
    barrier()
    t0 = time.perf_counter()
    e0.record()
    for _ in range(args.steps):
        model.forward_pairs_host(h1, h2, hout)  # H2D + forward + D2H + stream sync inside
    e1.record()
    barrier()
    e2e_ms = max_over_ranks(max(e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3)) / args.steps
    e2e_value = global_pairs / (e2e_ms / 1e3)
    h2d = 2 * h1.numel() * h1.element_size()
    d2h = sum(t.numel() * t.element_size() for t in hout.values())

    # ---------------- roofline of the dominant kernel family (live CUDA-event timing) ----------------
    L = _lib.lib()
    L.sta_profile(model._handle, 1)
    prof_steps = min(args.steps, 3)
    for _ in range(prof_steps):
        model.forward_pairs(d1, d2)
    ms4, cnt4, fl4 = (ctypes.c_double * 4)(), (ctypes.c_int64 * 4)(), (ctypes.c_double * 4)()
    _lib.check(L.sta_profile_read(model._handle, ms4, cnt4, fl4))
    L.sta_profile(model._handle, 0)
    peaks = load_peaks()
    flop_pair = flops_per_pair(H, W)
    # algorithmic FLOPs handled by the GEMM family per pair = total - attention (SURVEY.md 8(d))
    attn_flops_pair = attention_flops_per_pair(H, W)
    gemm_flops_pair = flop_pair - attn_flops_pair
    gemm_ms = (ms4[0] + ms4[1]) / prof_steps
    gemm_launches = (cnt4[0] + cnt4[1]) // prof_steps
    achieved = P * gemm_flops_pair / (gemm_ms / 1e3) / 1e12
    peak = peaks["bf16_sustained"] or peaks["bf16_burst"]
    roofline = {
        "bound": "tensor", "kernel": "gemm_wg_kernel (wgmma GEMM + implicit-GEMM 3x3 conv family)",
        "achieved": achieved, "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak,
        "peak_source": peaks["source"],
        "launches_per_step": int(gemm_launches), "avg_launch_ms": gemm_ms / max(1, gemm_launches),
        "algorithmic_gflop_per_launch_avg": P * gemm_flops_pair / max(1, gemm_launches) / 1e9,
        "family_ms_per_step": {"gemm_linear": ms4[0] / prof_steps, "gemm_conv3x3": ms4[1] / prof_steps,
                               "attention": ms4[2] / prof_steps, "layernorm": ms4[3] / prof_steps},
        "attention_tflops": P * attn_flops_pair / (ms4[2] / prof_steps / 1e3) / 1e12 if ms4[2] > 0 else None,
        # rank 0's own work over the max-over-ranks time
        "whole_step_tflops": P * flop_pair / (ms_step / 1e3) / 1e12,
        "whole_step_frac": P * flop_pair / (ms_step / 1e3) / 1e12 / peak,
    }

    # ---------------- CPU baseline beside it (rank 0, N = 1 only) ----------------
    cpu_baseline = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cpu_baseline = cpu_port_baseline(H, W)
    if world > 1:
        dist.barrier()
    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_step, "higher_is_better": True, "scaling": "strong" if total is not None else "weak",
            "vs_baseline": None, "dtype": "bf16", "data": "synthetic", "impl": "b200",
            "config": make_config(P, world, H, W, total),
            "clocks": clocks, "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": h2d,
                                      "d2h_bytes_per_step": d2h, "ms_per_step": e2e_ms,
                                      # copy time not hidden behind the kernels (H2D of the first chunk, D2H tail)
                                      "exposed_copy_ms": max(0.0, e2e_ms - ms_step)},
            "gpu_launches": int(launches), "roofline": roofline, "cpu_baseline": cpu_baseline, "outputs_finite": ok,
        }
        if dumped is not None:
            line["dumped_outputs"] = {"dir": args.dump_outputs, "elements": dumped}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--pairs", type=int, default=16, help="pairs per GPU per step (cfg-2: 16)")
    ap.add_argument("--height", type=int, default=384)
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--total-pairs", type=int, default=None,
                    help="cfg-5: global batch split contiguously over the ranks (strong scaling); overrides --pairs")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the outputs of the last timed step as DIR/<name>.npy (float32, dense maps sampled); "
                         "with --gpus N > 1, rank 0's pair shard only")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        run_reference_arm(args, rank, world)
        return
    if world != args.gpus:
        if args.gpus > 1 and world == 1:
            # convenience: re-launch under torchrun
            cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus),
                   "--master-addr", "127.0.0.1", "--master-port", "29517", os.path.abspath(__file__)] + sys.argv[1:]
            sys.exit(subprocess.call(cmd))
    run_b200_arm(args, rank, local_rank, world)


if __name__ == "__main__":
    main()
