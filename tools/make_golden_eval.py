"""Golden record of the UNMODIFIED reference evaluation (vista_slam/eval/eval_traj.py::full_traj_eval and
eval_recon.py::eval_recon_from_saved_data) on the seeded synthetic scene of oracle/eval_oracle.py::make_scene ->
tests/golden/eval.npz.

Runs only where the reference tree is present.  The reference code is imported unchanged; evo, open3d, pykdtree, munch
and matplotlib are the in-memory stand-ins of oracle/eval_stubs.py (backed by the oracle), colorama is stubbed as in
tools/make_golden_slam.py.  The scene (24 views at 48 x 64, written in save_data_all's format) is regenerated from the
seed by the tests; only the outputs are stored."""
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from oracle import eval_oracle as eo  # noqa: E402
from oracle import eval_stubs  # noqa: E402


def main(out_path=os.path.join(ROOT, "tests", "golden", "eval.npz")):
    eval_stubs.install()
    sys.modules["colorama"] = types.SimpleNamespace(Fore=types.SimpleNamespace(
        CYAN="c", BLUE="b", YELLOW="y", GREEN="g", RED="r", MAGENTA="m"), Style=types.SimpleNamespace(RESET_ALL=""))
    from tools.ref_import import REFERENCE_ROOT
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    from vista_slam.eval.eval_recon import eval_recon_from_saved_data
    from vista_slam.eval.eval_traj import full_traj_eval

    scene = eo.make_scene()
    out = {}
    with tempfile.TemporaryDirectory() as d:
        eo.write_scene(scene, d)
        # as evaluation_*.py call them: host fp32 poses for the trajectory, then the recon with its rel_est_gt
        est_poses = list(np.load(os.path.join(d, "trajectory.npy")))
        gt_poses = list(np.load(os.path.join(d, "gt_poses.npy")))
        _, _, r_a, t_a, s, ape = full_traj_eval(est_poses, gt_poses, os.path.join(d, "plots"), "traj")
        out.update(r_a=np.asarray(r_a, np.float64), t_a=np.asarray(t_a, np.float64), s=np.float64(s))
        for k in ("rmse", "mean", "median", "std", "min", "max", "sse"):
            out["ape_" + k] = np.float64(ape[k])
        # eval_recon_from_saved_data aligns the torch fp32 poses itself when rel_est_gt is None
        for tag, rel in (("", [r_a, t_a, s]), ("self_", None)):
            eval_stubs.ICP_CALLS.clear()
            acc, comp, ch, gt_pts, est_pts = eval_recon_from_saved_data(d, rel_est_gt=rel)
            icp = eval_stubs.ICP_CALLS[0]
            out.update({tag + "rmse_acc": np.float64(acc), tag + "rmse_comp": np.float64(comp), tag + "chamfer": np.float64(ch),
                        tag + "n_gt": np.int64(len(gt_pts)), tag + "n_est": np.int64(len(est_pts)),
                        tag + "icp_iterations": np.int64(icp["iterations"]), tag + "icp_fitness": np.float64(icp["fitness"]),
                        tag + "icp_transformation": icp["transformation"]})
    np.savez(out_path, **out)
    print("wrote", out_path, {k: (v.shape, v.dtype) for k, v in out.items()})
    return out


if __name__ == "__main__":
    torch.set_num_threads(1)
    main(*sys.argv[1:])
