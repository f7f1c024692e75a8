"""A/B timing of two builds of the library on the same GPU, alternating, in one process tree.

    python tools/ab_bench.py BASE_LIB [--rounds N] [--steps S] [--out DIR]

BASE_LIB is a libsta_b200.so built from another commit (for example the parent: `git worktree add` it elsewhere, run
`python -m vista_slam_b200.build` there and copy the .so into a git-ignored path of this tree).  Each round runs
`bench.py --steps S --no-cpu-baseline` once with STA_B200_LIB=BASE_LIB and once with this tree's build, and prints
per side the pairs/s value, ms per step, the per-family kernel times of the profile, the launch count and the clocks.
Then both sides run once with --dump-outputs and the dumped arrays are compared bit for bit.  The card's name, power
limit and maximum SM clock are printed first: every number below belongs to them.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_LIB = os.path.join(ROOT, "vista_slam_b200", "csrc", "libsta_b200.so")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % r.stderr.strip())
    return r.stdout.strip()


def bench(lib, steps, extra=()):
    env = dict(os.environ, STA_B200_LIB=lib)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--no-cpu-baseline"]
    r = subprocess.run(cmd + list(extra), env=env, capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError("bench.py failed with %s:\n%s\n%s" % (lib, r.stdout[-4000:], r.stderr[-4000:]))
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    return json.loads(lines[-1])


def summary(side, res):
    fam = res["roofline"]["family_ms_per_step"]
    return "%-4s value %.2f pairs/s  ms/step %.3f  families %s  gpu_launches %d  clocks %s" % (
        side, res["value"], res["ms_per_step"], json.dumps({k: round(v, 3) for k, v in fam.items()}),
        res["gpu_launches"], json.dumps(res.get("clocks")))


def compare_dumps(dir_a, dir_b):
    names = sorted(f for f in os.listdir(dir_a) if f.endswith(".npy"))
    if not names or names != sorted(f for f in os.listdir(dir_b) if f.endswith(".npy")):
        raise RuntimeError("the two dumps hold different files: %s vs %s" % (names, sorted(os.listdir(dir_b))))
    same = True
    for n in names:
        a, b = np.load(os.path.join(dir_a, n)), np.load(os.path.join(dir_b, n))
        eq = a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()
        diff = "" if eq else " max|diff| %.3g" % float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())
        print("dump %-24s %s%s" % (n, "bit-identical" if eq else "DIFFERS", diff), flush=True)
        same = same and eq
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("base_lib")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None, help="directory for the dumped outputs (default: a temporary directory)")
    args = ap.parse_args()
    base = os.path.abspath(args.base_lib)
    for lib in (base, NEW_LIB):
        if not os.path.exists(lib):
            raise SystemExit("no library at %s" % lib)
    print("card:", card(), flush=True)
    rows = {"base": [], "new": []}
    for rnd in range(args.rounds):
        for side, lib in (("base", base), ("new", NEW_LIB)):
            res = bench(lib, args.steps)
            rows[side].append(res)
            print("round %d %s" % (rnd, summary(side, res)), flush=True)
    for side in ("base", "new"):
        v = [r["value"] for r in rows[side]]
        lin = [r["roofline"]["family_ms_per_step"]["gemm_linear"] for r in rows[side]]
        print("%-4s value min %.2f max %.2f | gemm_linear ms min %.3f max %.3f" % (side, min(v), max(v), min(lin), max(lin)))
    out = args.out or tempfile.mkdtemp(prefix="ab_bench_")
    dirs = {}
    for side, lib in (("base", base), ("new", NEW_LIB)):
        dirs[side] = os.path.join(out, side)
        os.makedirs(dirs[side], exist_ok=True)
        res = bench(lib, 2, ["--warmup", "1", "--dump-outputs", dirs[side]])
        print("dump %s gpu_launches %d" % (side, res["gpu_launches"]), flush=True)
    same = compare_dumps(dirs["base"], dirs["new"])
    print("outputs", "bit-identical" if same else "DIFFER", flush=True)
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
