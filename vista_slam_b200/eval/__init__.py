"""Drop-in replacements for vista_slam/eval: trajectory APE (eval_traj, host float64) and reconstruction accuracy,
completeness and Chamfer distance (eval_recon, on the GPU)."""
