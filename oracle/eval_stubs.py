"""In-memory stand-ins for the libraries vista_slam/eval/eval_traj.py and eval_recon.py import (evo, open3d, pykdtree,
munch, matplotlib), backed by oracle/eval_oracle.py, so that the unmodified reference functions run on a host without
them.  `install()` puts them into sys.modules; ICP_CALLS records every registration_icp call (its iterations and result).

Only what the two modules call is provided:
  open3d      geometry.PointCloud (points, paint_uniform_color, get_center, voxel_down_sample, transform),
              utility.Vector3dVector, pipelines.registration.registration_icp / TransformationEstimationPointToPoint;
  pykdtree    kdtree.KDTree(data).query(x) -> (distances, indices);
  evo         core.trajectory.PoseTrajectory3D (align with scale), core.sync.associate_trajectories, core.metrics.APE /
              PoseRelation, tools.plot (no-op);
  munch       Munch;  matplotlib.pyplot.figure (no-op)."""
import sys
import types

import numpy as np

from oracle import eval_oracle as eo

ICP_CALLS = []


def Vector3dVector(a):
    return np.array(a, dtype=np.float64).reshape(-1, 3)


class PointCloud:
    def __init__(self, points=None):
        self.points = Vector3dVector(np.zeros((0, 3)) if points is None else points)

    def paint_uniform_color(self, c):
        self.colors = np.tile(np.asarray(c, np.float64), (len(self.points), 1))
        return self

    def get_center(self):
        return self.points.mean(axis=0) if len(self.points) else np.zeros(3)

    def voxel_down_sample(self, voxel_size):
        return PointCloud(eo.voxel_down(self.points, voxel_size))

    def transform(self, T):
        self.points = eo.transform(self.points, np.asarray(T, np.float64))
        return self


class TransformationEstimationPointToPoint:
    def __init__(self, with_scaling=False):
        assert not with_scaling


def registration_icp(source, target, max_correspondence_distance, init, estimation_method):
    assert np.array_equal(np.asarray(init), np.eye(4)) and isinstance(estimation_method, TransformationEstimationPointToPoint)
    r = eo.icp(source.points, target.points, max_correspondence_distance)
    ICP_CALLS.append(r)
    return types.SimpleNamespace(transformation=r["transformation"], fitness=r["fitness"], inlier_rmse=r["inlier_rmse"])


class KDTree:
    def __init__(self, data):
        self.data = np.asarray(data, np.float64)

    def query(self, x):
        return eo.nearest(self.data, x)


class PoseTrajectory3D:
    def __init__(self, poses_se3=None, timestamps=None):
        self.poses_se3 = [np.asarray(p, np.float64) for p in poses_se3]
        self.timestamps = np.asarray(timestamps, np.float64)

    @property
    def positions_xyz(self):
        return np.array([p[:3, 3] for p in self.poses_se3])

    def align(self, traj_ref, correct_scale=False):
        r, t, s = eo.umeyama(self.positions_xyz.T, traj_ref.positions_xyz.T, correct_scale)
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = r, t
        if correct_scale:
            self.poses_se3 = [np.vstack((np.hstack((p[:3, :3], s * p[:3, 3:4])), [0, 0, 0, 1])) for p in self.poses_se3]
        self.poses_se3 = [T.dot(p) for p in self.poses_se3]
        return r, t, s


def associate_trajectories(traj_1, traj_2):
    assert np.array_equal(traj_1.timestamps, traj_2.timestamps)
    return traj_1, traj_2


class APE:
    def __init__(self, relation):
        self.relation = relation

    def process_data(self, data):
        ref, est = data
        self.stats = eo.ape_statistics(np.stack(est.poses_se3), np.stack(ref.poses_se3))
        self.error = np.linalg.norm(ref.positions_xyz - est.positions_xyz, axis=1)

    def get_all_statistics(self):
        return dict(self.stats)


class _NoOp:
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _NoOp()

    def __getattr__(self, k):
        return _NoOp()


class Munch(dict):
    __getattr__ = dict.__getitem__


def install():
    m = types.ModuleType
    o3d = m("open3d")
    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud)
    o3d.utility = types.SimpleNamespace(Vector3dVector=Vector3dVector)
    o3d.pipelines = types.SimpleNamespace(registration=types.SimpleNamespace(
        registration_icp=registration_icp, TransformationEstimationPointToPoint=TransformationEstimationPointToPoint))
    pk = m("pykdtree")
    pk.kdtree = types.SimpleNamespace(KDTree=KDTree)
    evo, core, tools = m("evo"), m("evo.core"), m("evo.tools")
    core.trajectory = types.SimpleNamespace(PoseTrajectory3D=PoseTrajectory3D)
    core.sync = types.SimpleNamespace(associate_trajectories=associate_trajectories)
    core.metrics = types.SimpleNamespace(APE=APE, PoseRelation=types.SimpleNamespace(translation_part="translation_part"))
    tools.plot = _NoOp()
    evo.core, evo.tools = core, tools
    mpl, plt = m("matplotlib"), m("matplotlib.pyplot")
    plt.figure = _NoOp()
    mpl.pyplot = plt
    sys.modules.update({"open3d": o3d, "pykdtree": pk, "pykdtree.kdtree": pk.kdtree, "evo": evo, "evo.core": core,
                        "evo.core.trajectory": core.trajectory, "evo.core.sync": core.sync, "evo.core.metrics": core.metrics,
                        "evo.tools": tools, "evo.tools.plot": tools.plot, "munch": types.SimpleNamespace(Munch=Munch),
                        "matplotlib": mpl, "matplotlib.pyplot": plt})
