"""The FP8 mode against bf16 on one card, in one process: cfg-2 throughput, per-family kernel time, and OnlineSLAM.

  * cfg-2: 16 bf16 512x384 pairs per forward_pairs call; both models (the same random-init weights) are warmed up, then
    timed in alternation, `--rounds` windows of `--steps` calls each, every window from a device synchronise to a device
    synchronise; pairs/s of the best window per mode.
  * sta_profile: one profiled call per mode, milliseconds per kernel family (linear GEMM, conv GEMM, attention,
    LayerNorm + the FP8 quantisers) -- in a separate pass, as the events slow the host.
  * OnlineSLAM at 224 x 224 on the stream of tools/slam_batch_stream.py: `step` per keyframe and `step_many` in chunks of
    32, each mode's frontend built by a load_frontend subclass; ms per keyframe of the best run after a warm-up run.
Prints the card's name and power limit, then one JSON line (also written to --out when given)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--views", type=int, default=400)
    ap.add_argument("--slam-rounds", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vista_slam_b200 import _lib
    from vista_slam_b200.slam import OnlineSLAM
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA

    torch.manual_seed(0)
    ref = STA()
    sd = ref.state_dict()
    models = {}
    for prec in ("bf16", "fp8"):
        m = STA(precision=prec)
        m.load_state_dict(sd)
        models[prec] = m.cuda().eval()
    print("card:", card(), flush=True)

    # ---- cfg-2 ----
    B, H, W = 16, 384, 512
    g = torch.Generator().manual_seed(3)
    i1 = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).bfloat16().cuda()
    i2 = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).bfloat16().cuda()
    for m in models.values():
        for _ in range(3):
            m.forward_pairs(i1, i2)
    torch.cuda.synchronize()
    win = {p: [] for p in models}
    for _ in range(a.rounds):
        for p, m in models.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                m.forward_pairs(i1, i2)
            torch.cuda.synchronize()
            win[p].append(time.perf_counter() - t0)
    cfg2 = {p: {"pairs_per_s": round(B * a.steps / min(win[p]), 2), "ms_per_step": round(1e3 * min(win[p]) / a.steps, 3),
                "ms_per_step_all": [round(1e3 * t / a.steps, 3) for t in win[p]]} for p in models}
    cfg2["fp8_speedup"] = round(cfg2["bf16"]["ms_per_step"] / cfg2["fp8"]["ms_per_step"], 4)

    # ---- per-family device time (separate pass) ----
    L = _lib.lib()
    fam = {}
    for p, m in models.items():
        L.sta_profile(m._handle, 1)
        m.forward_pairs(i1, i2)
        ms, cnt, fl = (ctypes.c_double * 4)(), (ctypes.c_int64 * 4)(), (ctypes.c_double * 4)()
        _lib.check(L.sta_profile_read(m._handle, ms, cnt, fl), "sta_profile_read")
        L.sta_profile(m._handle, 0)
        fam[p] = {n: {"ms": round(ms[i], 3), "launches": cnt[i], "tflops": round(fl[i] / max(ms[i], 1e-9) / 1e9, 1)}
                  for i, n in enumerate(("gemm_linear", "gemm_conv", "attention", "layernorm_quant"))}

    # ---- OnlineSLAM ----
    HS = WS = 224
    gs = torch.Generator().manual_seed(1)
    base = torch.rand(1, 3, HS // 8, WS // 4, generator=gs)
    values = []
    for i in range(a.views):
        img = torch.nn.functional.interpolate(base.roll(i % (WS // 4), dims=3)[..., :WS // 8], size=(HS, WS), mode="bilinear")
        img = ((img * 2 - 1) + 0.05 * torch.randn(1, 3, HS, WS, generator=gs)).clamp(-1, 1).cuda()
        values.append({"rgb": img, "shape": torch.tensor([[HS, WS]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                       "view_name": "%05d" % i})
    vocab = os.path.join(ROOT, "tests", "golden", "loop_vocab.txt")
    n = a.views

    def run(prec, chunk):
        class Slam(OnlineSLAM):
            def load_frontend(self, ckpt_path):
                return models[prec]

        slam = Slam("unused", vocab, pgo_every=500)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if chunk is None:
            for i, v in enumerate(values):
                slam.step(v, force_pgo=(i == n - 1))
        else:
            for c in range(0, n, chunk):
                slam.step_many(values[c:c + chunk], force_pgo=(c + chunk >= n))
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        nodes = slam.num_nodes
        del slam
        torch.cuda.empty_cache()
        return dt, nodes

    slam_res = {}
    for chunk in (None, 32):
        for p in models:
            run(p, chunk)  # warm-up: every shape and CUDA graph
    for chunk in (None, 32):
        name = "step" if chunk is None else "step_many_32"
        ts = {p: [] for p in models}
        nodes = {}
        for _ in range(a.slam_rounds):
            for p in models:
                dt, nodes[p] = run(p, chunk)
                ts[p].append(dt)
        slam_res[name] = {p: {"ms_per_keyframe": round(1e3 * min(ts[p]) / n, 3), "nodes": nodes[p]} for p in models}

    res = {"card": card(), "cfg2": cfg2, "families_ms_one_step": fam, "slam_224": slam_res, "views": n}
    print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
