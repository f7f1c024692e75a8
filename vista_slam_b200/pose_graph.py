"""Sim(3) pose-graph optimisation on the GPU (SURVEY.md section 8(f) rank 4).

Mirror of the optimisation OnlineSLAM.pose_graph_optimize runs through PyPose (vista_slam/slam.py:108-140 over
vista_slam/pose_graph.py:70-154): Levenberg-Marquardt with a trust-region damping on the nodes listed in
`to_optimize_idxs`, all other nodes fixed, edge weights diag(conf_e).  Each iteration is ONE C call
(sta_pose_graph_lm_step: residuals, Jacobians, normal equations, damped dense Cholesky solve, update and both losses, all on
the device) followed by one 32-byte read-back for the accept / reject decision -- the same host round trip pp.optim.LM makes.
Tensors use PyPose's Sim3 layout (tx ty tz | qx qy qz qw | s), fp32, CUDA only (no CPU path).

Two routes solve the damped normal equations, chosen in the constructor from the number of optimised nodes:
  * dense (num_opt <= _lib.PG_DENSE_MAX_OPT = 3657): sta_pose_graph_lm_step, a dense fp64 Cholesky of order 7 num_opt;
  * block-sparse (above): sta_pose_graph_lm_step_sparse, a block Cholesky (7x7 blocks) over a plan -- ordering,
    elimination tree, block pattern and update lists -- built on the host from the edge list and the optimised set.
Both compute the same residuals, Jacobians, normal equations, damping, update and losses.
"""
import ctypes

import torch

from . import _lib


class _SparsePlan:
    """Owner of one StaPgPlan (host analysis + device arrays + scratch) for one edge table and optimised set."""

    def __init__(self, edges, num_nodes, idxs_opt):
        L = _lib.lib()
        e = edges.detach().to(torch.int64).contiguous().cpu()  # the one device-to-host copy of the edge table
        o = idxs_opt.cpu()
        h = ctypes.c_void_p()
        _lib.check(L.sta_pg_plan_create(_lib.ptr(e), e.shape[0], num_nodes, _lib.ptr(o), o.shape[0], ctypes.byref(h)),
                   "sta_pg_plan_create")
        self.h = h
        self._destroy = L.sta_pg_plan_destroy

    def info(self):
        """{"l_blocks", "levels", "device_bytes", "updates"} of the plan."""
        out = (ctypes.c_int64 * 4)()
        _lib.check(_lib.lib().sta_pg_plan_info(self.h, out), "sta_pg_plan_info")
        return dict(zip(("l_blocks", "levels", "device_bytes", "updates"), map(int, out)))

    def __del__(self):
        if getattr(self, "h", None):
            self._destroy(self.h)
            self.h = None


class PoseGraphOpt:
    def __init__(self, nodes, to_optimize_idxs="all"):
        if not nodes.is_cuda:
            raise RuntimeError("vista_slam_b200.pose_graph runs only on CUDA tensors")
        self.nodes = nodes.detach().to(torch.float32).contiguous().clone()
        n = self.nodes.shape[0]
        if isinstance(to_optimize_idxs, str):
            to_optimize_idxs = torch.arange(n, device=nodes.device)
        self.idxs_opt = torch.as_tensor(to_optimize_idxs, device=nodes.device).long().contiguous()
        self._scratch = None
        self._info = torch.zeros(4, dtype=torch.float64, device=nodes.device)
        self.sparse = self.idxs_opt.shape[0] > _lib.PG_DENSE_MAX_OPT
        self._plan, self._plan_key = None, None

    def get_nodes(self):  # pose_graph.py:94-98
        return self.nodes.clone()

    def get_related_edge_idxs(self, edges):  # pose_graph.py:150-154
        m = torch.isin(edges, self.idxs_opt)
        return m[:, 0] | m[:, 1]

    def plan(self, edges):
        """The block-sparse route's plan for `edges`: built on the first call and reused while the same edges tensor
        (same storage pointer, length and version counter) comes back, as it does across the iterations of optimize().
        Building it costs one device-to-host copy of the edge table and a host analysis, once per optimize() call."""
        key = (edges.data_ptr(), edges.shape[0], edges._version, edges.dtype)
        if self._plan is None or self._plan_key != key:
            self._plan = None
            with torch.cuda.device(self.nodes.device):
                self._plan = _SparsePlan(edges, self.nodes.shape[0], self.idxs_opt)
            self._plan_key = key
        return self._plan

    @torch.no_grad()
    def lm_step(self, edges, poses, weight, damping, dmin=1e-6, dmax=1e32):
        """One damped Gauss-Newton solve; returns (candidate nodes, loss_before, loss_after, |delta|, cholesky_ok).
        Above PG_DENSE_MAX_OPT optimised nodes it runs on the block-sparse route (see plan())."""
        L = _lib.lib()
        if self.sparse:
            if poses.shape[0] != edges.shape[0] or weight.shape[0] != edges.shape[0]:
                raise ValueError("edges, poses and weight must have one row per edge")
            plan = self.plan(edges)
            poses = poses.to(torch.float32).contiguous()
            weight = weight.to(torch.float32).contiguous()
            out = torch.empty_like(self.nodes)
            with torch.cuda.device(self.nodes.device):
                _lib.check(L.sta_pose_graph_lm_step_sparse(plan.h, _lib.ptr(self.nodes), _lib.ptr(poses), _lib.ptr(weight),
                                                           float(damping), float(dmin), float(dmax), _lib.ptr(out),
                                                           _lib.ptr(self._info), _lib.cur_stream()),
                           "sta_pose_graph_lm_step_sparse")
            info = self._info.cpu()  # the one host synchronisation of the iteration
            return out, float(info[0]), float(info[1]), float(info[2]), bool(info[3] > 0.5)
        edges = edges.to(torch.int64).contiguous()
        poses = poses.to(torch.float32).contiguous()
        weight = weight.to(torch.float32).contiguous()
        E, Nn, No = edges.shape[0], self.nodes.shape[0], self.idxs_opt.shape[0]
        need = int(L.sta_pose_graph_scratch_bytes(Nn, E, No))
        if self._scratch is None or self._scratch.numel() * 8 < need:
            self._scratch = torch.empty((need + 7) // 8, dtype=torch.float64, device=self.nodes.device)
        out = torch.empty_like(self.nodes)
        with torch.cuda.device(self.nodes.device):
            _lib.check(L.sta_pose_graph_lm_step(_lib.ptr(self.nodes), Nn, _lib.ptr(edges), _lib.ptr(poses), _lib.ptr(weight), E,
                                                _lib.ptr(self.idxs_opt), No, float(damping), float(dmin), float(dmax),
                                                _lib.ptr(out), _lib.ptr(self._info), _lib.ptr(self._scratch), _lib.cur_stream()),
                       "sta_pose_graph_lm_step")
        info = self._info.cpu()  # the one host synchronisation of the iteration
        return out, float(info[0]), float(info[1]), float(info[2]), bool(info[3] > 0.5)

    @torch.no_grad()
    def optimize(self, edges, poses, weight, steps=20, patience=3, decreasing=1e-4, radius=1e4):
        """slam.py:121-134: LM(TrustRegion(radius=1e4), min=1e-6) driven by StopOnPlateau(steps=20, patience=3,
        decreasing=1e-4).  `weight` is [E, 7] (the diagonal of the reference's diag_embed).  Returns the loss history."""
        losses, stall = [], 0
        for _ in range(steps):
            cand, l0, l1, _, ok = self.lm_step(edges, poses, weight, 1.0 / radius)
            if ok and l1 <= l0:
                self.nodes = cand
                radius = min(radius * 2.0, 1e32)
            else:  # rejected step: keep the nodes, shrink the trust region
                radius = max(radius * 0.5, 1e-32)
                l1 = l0
            losses.append(l1)
            stall = stall + 1 if (l0 - l1) < decreasing else 0
            if stall >= patience:
                break
        return losses
