"""ORACLE -- test infrastructure, not product code.

In-memory stand-in for the part of `pypose` that vista_slam/slam.py and vista_slam/pose_graph.py use, so that the
unmodified reference OnlineSLAM can run where PyPose is not installed (tools/make_golden_slam.py).  Group arithmetic is
oracle/pose_graph_oracle.py in float64 on the stored values; results are stored back in the dtype of the operands
(float32 in the reference).  Only Sim(3) LieTensors occur in OnlineSLAM (SE(3) values are taken with `.data` at once).
`pp.optim.LM` + `StopOnPlateau.optimize` are routed to pose_graph_oracle.optimize; the reference's weight rows
(diag_embed(confs)[related_mask], one per related edge in edge order) are handed to it per edge in that order.

`install()` puts the modules into sys.modules; `LM_CALLS` records every optimisation (inputs and result)."""
import sys
import types

import numpy as np
import torch

from oracle import pose_graph_oracle as pg

LM_CALLS = []


def _f64(t):
    return torch.Tensor.as_subclass(t, torch.Tensor).detach().cpu().numpy().astype(np.float64)


class LieTensor(torch.Tensor):
    """A Sim(3) LieTensor [..., 8] (tx ty tz | qx qy qz qw | s)."""

    @staticmethod
    def wrap(t):
        return torch.Tensor.as_subclass(t, LieTensor)

    def tensor(self):
        return torch.Tensor.as_subclass(self, torch.Tensor)

    def __matmul__(self, other):
        a, b = _f64(self), _f64(other)
        shape = np.broadcast_shapes(a.shape[:-1], b.shape[:-1])
        a, b = np.broadcast_to(a, shape + (8,)).reshape(-1, 8), np.broadcast_to(b, shape + (8,)).reshape(-1, 8)
        out = np.stack([pg.sim3_mul(x, y) for x, y in zip(a, b)]).reshape(shape + (8,))
        return LieTensor.wrap(torch.from_numpy(out).to(self.dtype))

    def rotation(self):
        return _SO3(self.tensor()[..., 3:7])

    def translation(self):
        return self.tensor()[..., :3].clone()

    def scale(self):
        return self.tensor()[..., 7:8].clone()


class _SO3:
    def __init__(self, q):
        self.q = q

    def matrix(self):
        q = _f64(self.q).reshape(-1, 4)
        R = np.stack([pg.quat_to_rot(x) for x in q]).reshape(tuple(self.q.shape[:-1]) + (3, 3))
        return torch.from_numpy(R).to(self.q.dtype)


def Sim3(data):
    return LieTensor.wrap(torch.as_tensor(data))


def identity_Sim3(*n):
    t = torch.zeros(*n, 8)
    t[..., 6] = 1.0
    t[..., 7] = 1.0
    return LieTensor.wrap(t)


class _Data:
    def __init__(self, t):
        self.data = t


def identity_SE3(*n):
    t = torch.zeros(*n, 7)
    t[..., 6] = 1.0
    return _Data(t)


def mat2SE3(mat, check=True, atol=1e-3, rtol=1e-5):
    """4x4 -> SE(3) [tx ty tz | qx qy qz qw], quaternion with w >= 0; raises ValueError for a rotation that is not
    orthonormal with det +1 to atol."""
    M = _f64(mat).reshape(-1, 4, 4)
    out = []
    for m in M:
        R = m[:3, :3]
        if check and (np.abs(R @ R.T - np.eye(3)).max() > atol or abs(np.linalg.det(R) - 1.0) > atol):
            raise ValueError("Input rotation matrices are not all orthogonal matrix")
        out.append(np.concatenate([m[:3, 3], pg.rot_to_quat(R)]))
    return _Data(torch.from_numpy(np.stack(out).reshape(tuple(mat.shape[:-2]) + (7,))).to(mat.dtype))


def Parameter(t):
    return t


class _Cholesky:
    pass


class _TrustRegion:
    def __init__(self, radius=1e6, **kw):
        self.radius = radius


class _LM:
    def __init__(self, model, solver=None, strategy=None, min=1e-6, max=1e32, vectorize=True, **kw):
        self.model, self.radius, self.min, self.max = model, strategy.radius, min, max


class _StopOnPlateau:
    def __init__(self, optimizer, steps, patience=5, decreasing=1e-3, verbose=False):
        self.opt, self.steps, self.patience, self.decreasing = optimizer, steps, patience, decreasing

    def optimize(self, input, weight=None):
        """Runs pose_graph_oracle.optimize over the reference PoseGraphOpt's node split and writes the result into its
        optimised nodes."""
        graph = self.opt.model
        edges, poses = input
        edges_np = edges.cpu().numpy().astype(np.int64)
        nodes = _f64(graph.get_nodes())
        opt_idx = graph.idxs_opt.cpu().numpy().astype(np.int64)
        related = pg.related_edges(edges_np, opt_idx)
        w = np.ones((len(edges_np), 7))
        w[related] = np.diagonal(_f64(weight), axis1=-2, axis2=-1)  # row r of weight -> r-th related edge
        w32 = w.astype(np.float32).astype(np.float64)
        meas = _f64(poses)
        out, losses = pg.optimize(nodes, edges_np, meas, w32, opt_idx, steps=self.steps, patience=self.patience,
                                  decreasing=self.decreasing, radius=self.opt.radius)
        res = torch.from_numpy(out[opt_idx]).to(graph.nodes_opt.dtype)
        graph.nodes_opt = LieTensor.wrap(res)
        LM_CALLS.append({"nodes": nodes.astype(np.float32), "opt_idx": opt_idx, "related": related,
                         "num_edges": len(edges_np), "weight": w32.astype(np.float32),
                         "result": _f64(graph.get_nodes()).astype(np.float32), "losses": np.array(losses)})


def install():
    pp = types.ModuleType("pypose")
    for name in ("LieTensor", "Sim3", "identity_Sim3", "identity_SE3", "mat2SE3", "Parameter"):
        setattr(pp, name, globals()[name])
    optim = types.ModuleType("pypose.optim")
    solver = types.ModuleType("pypose.optim.solver")
    strategy = types.ModuleType("pypose.optim.strategy")
    scheduler = types.ModuleType("pypose.optim.scheduler")
    solver.Cholesky = _Cholesky
    strategy.TrustRegion = _TrustRegion
    scheduler.StopOnPlateau = _StopOnPlateau
    optim.LM = _LM
    optim.solver, optim.strategy, optim.scheduler = solver, strategy, scheduler
    pp.optim = optim
    sys.modules.update({"pypose": pp, "pypose.optim": optim, "pypose.optim.solver": solver,
                        "pypose.optim.strategy": strategy, "pypose.optim.scheduler": scheduler})
    return pp
