"""Measured parity of the CUDA path on every golden case (run under gpurun); writes gpurun_out/parity_report*.json.

    python tools/parity_report.py [--precision bf16|x3] [--no-emu]

For each committed reference golden (tests/golden/pair_*.npz, produced by the UNMODIFIED reference in fp32 on CPU) the
same seeded inputs go through `forward_pairs` on the GPU.  Per output the report holds
  max-normalised error  max|a-b| / max|b|      and      median-normalised error  median|a-b| / max|b|
of (1) cuda vs fp32 reference golden, (2) cuda vs the oracle in bf16-operand emulation, (3) emulation oracle vs the
fp32 golden -- so that |cuda - fp32| can be compared with the noise floor |emu - fp32| of the same operand precision.
The cfg-2 case is also run as pair 0 of a 16-pair batch (the production tile routes: full GEMM grids, 128-row attention
tiles) next to the single-pair call (small-problem routes).
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from oracle.sta_oracle import StaOracle, make_images, make_state_dict, usable_cpus  # noqa: E402

KEYS = (("pts3d_pred", "pts3d"), ("conf", "conf"), ("relative_pose", "pose"), ("relative_pose_conf", "pose_conf"))
CASES = ("pair_64x80", "pair_b2_48x64", "pair_224x224", "pair_384x512")


def err(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    d = (a - b).abs()
    s = float(b.abs().max().clamp_min(1e-30))
    return {"maxn": float(d.max()) / s, "medn": float(d.median()) / s}


def golden_inputs(g):
    meta = json.loads(str(g["meta"]))
    img1, img2 = make_images(meta["B"], meta["H"], meta["W"], meta["image_seed"])
    if meta.get("bf16_images"):
        img1, img2 = img1.bfloat16().float(), img2.bfloat16().float()
    return meta, img1, img2


def main():
    precision = "bf16"
    if "--precision" in sys.argv:
        precision = sys.argv[sys.argv.index("--precision") + 1]
    do_emu = "--no-emu" not in sys.argv and precision == "bf16"
    torch.set_num_threads(usable_cpus())
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    sd = make_state_dict(0)
    kw = {} if precision == "bf16" else {"precision": precision}
    model = STA(**kw)
    model.load_state_dict(sd, strict=True)
    model.eval()
    dev = torch.device("cuda")
    model._ready(torch.empty(1, device=dev))
    orcbf = StaOracle(sd, emulate_bf16=True) if do_emu else None
    report = {"precision": precision, "cases": {}}
    for case in CASES:
        g = np.load(os.path.join(ROOT, "tests", "golden", case + ".npz"))
        meta, img1, img2 = golden_inputs(g)
        B, H, W = meta["B"], meta["H"], meta["W"]
        runs = {"as_is": (img1, img2)}
        if case == "pair_384x512":
            # pair 0 of a 16-pair bf16 batch = the golden pair; the other 15 pairs are fresh random images
            o1, o2 = make_images(15, H, W, 99)
            runs["in_batch16"] = (torch.cat([img1, o1]).bfloat16(), torch.cat([img2, o2]).bfloat16())
        t0 = time.time()
        emu = None
        if orcbf is not None:
            with torch.no_grad():
                emu = orcbf.forward_pair(img1, img2)
        rec = {"oracle_emu_s": time.time() - t0}
        for rname, (a, b) in runs.items():
            m, s = model.forward_pairs(a.to(dev), b.to(dev))
            torch.cuda.synchronize()
            for res, pre, ei in ((m, "main_", 0), (s, "support_", 1)):
                for k, gk in KEYS:
                    gold = torch.from_numpy(g[pre + gk])
                    got = res[k][:B]
                    r = {"cuda_vs_fp32": err(got, gold)}
                    if emu is not None:
                        r["cuda_vs_emu"] = err(got, emu[ei][k])
                        r["emu_vs_fp32"] = err(emu[ei][k], gold)
                    rec["%s/%s%s" % (rname, pre, gk)] = r
        # trunk features through the reference-shaped sub-entry points
        ts = torch.tensor([[H, W]] * B)
        f1, p1 = model._encode_image(img1.to(dev), ts, normalize=False)
        f2, p2 = model._encode_image(img2.to(dev), ts, normalize=False)
        d1, d2 = model._decode_stereo(f1, f2, p1, p2, layers=(12,))
        rec["enc_feat1"] = {"cuda_vs_fp32": err(f1, torch.from_numpy(g["enc_feat1"]))}
        rec["dec1_12"] = {"cuda_vs_fp32": err(d1[12], torch.from_numpy(g["dec1_12"]))}
        report["cases"][case] = rec
        print("== %s (%s) ==" % (case, precision))
        for k, v in rec.items():
            if isinstance(v, dict):
                print("  %-34s %s" % (k, "  ".join("%s max %.2e med %.2e" % (n, e["maxn"], e["medn"]) for n, e in v.items())),
                      flush=True)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    out = os.path.join(ROOT, "gpurun_out", "parity_report_%s.json" % precision)
    json.dump(report, open(out, "w"), indent=1)
    print("wrote", out)


if __name__ == "__main__":
    main()
