"""Drop-in `OnlineSLAM` (vista_slam/slam.py) that keeps the pose graph and the map on the device.

Same constructor (arguments and defaults) and the surface run.py, run_live.py and the evaluation scripts use: `device`,
`verbose`, `view_num`, `imgs`, `flow_tracker`, `lc_detector`, `frontend`, `time_dict`, `load_frontend`, `step`, `reset`,
`pose_graph_optimize`, `get_view`, `get_view_graph`, `save_data_all`, `get_pointmap_vis`, `save_pointmap`,
`get_time_dict`.  It is built from this package's stages:

  * KeyframeFrontend.regress_keyframes_gated: one decoder pass over all candidate edges of a keyframe, one read-back of
    their pose confidences (the gate), DPT heads and pointmap consumers for the kept edges only;
  * LoopDetector and FlowTracker on the device;
  * the device pose graph (csrc/slam_graph.cu, `sta_graph_*`): node / edge tables, the depth / confidence / intrinsics
    store and the per-view best node live in fixed-capacity device arrays sized from the reference's formulas
    (slam.py:33-36).  The map store takes 8 H W max_nodes bytes: 1.44 GB at the defaults (3600 nodes) and 224 x 224.
    Keyframes go in with two launches and no host synchronisation for up to 32 of them (sta_graph_add_keyframes):
    `step` inserts its keyframe at once; `step_many` and SLAMSessions.step queue the insertions of an edge chunk and
    launch them together at the chunk's end, and before anything reads the tables (a PGO, the fold of a background
    one, an export) or a capacity IndexError is raised.  save_data_all / get_view gather on the device, and the world
    point cloud is built and compacted there (count, exclusive scan, scatter);
  * PoseGraphOpt, working on slices of the node and edge tables.

A step synchronises with the host twice, as the GPU stages need: the loop-candidate read (detect_loop runs first: it
does not depend on the neighbour edges) and the gate read.  PGO iterations read back their accept / reject decision.
A rotation that is not orthonormal (pp.mat2SE3(atol=1e-3) would raise) raises a device flag, which is read at the next
of those read-backs and raises ValueError there.

`step_many(values)` steps through many keyframes of one size in one call, with the graph, the PGO calls and the host
bookkeeping of calling `step` on each in order.  The frontend work does not depend on the pose graph, so it runs across
keyframes at real batch sizes: the encoder over up to 41 views per call at 224 x 224, loop detection over all frames of
the call with one read-back, and the gated edge regression in chunks of up to 16 edges with one read-back each.  Its
keyframe loop is step_keyframes, which SLAMSessions.step runs over several sessions; `step` keeps its own
one-keyframe path, the reference step_many is tested against.

`pgo_background = True` (default False) runs each due PGO on a side stream while step goes on (PoseGraphOpt.start):
step and step_many poll it at every keyframe without waiting, and fold it when it is done -- its poses written, the
nodes inserted since its launch re-derived from them (sta_graph_replay_nodes) -- which leaves the graph bit-identical
to the synchronous path.  Until the fold, get_view shows the poses from before the PGO; the next due PGO,
pose_graph_optimize, save_data_all, reset and wait_pgo wait for a pending run (INTEGRATION.md §5).  In
SLAMSessions.step the PGOs that fall due in one call start together as one run (PoseGraphOpt.start_group), and
SLAMSessions.optimize(ks, background=True) starts one for the named sessions; each session folds its share as above.

`track(values, kf)` gives frames that are not keyframes a pose against a keyframe view without changing the session:
one transient encode, the keyframe path's regression launches for the pairs (frame, kf) with no gate, and
sta_graph_track_frames, which composes each pose from the first node of kf as a keyframe with that one edge would get
it.  frame_trajectory() recomposes every tracked frame on the current graph, so tracked frames follow their keyframes
through PGOs (track_frames; DESIGN.md §5).

Importing this module does not import pypose, munch, colorama or open3d.  `get_view` returns a `View` (attribute and key
access, as munch.Munch).  The PLY of save_data_all is written here: binary little-endian, float x y z and uchar
red green blue (colours rounded from [0, 1]); whether that is byte-identical to open3d's writer is not checked."""
import ctypes
import operator
import os
import time

import numpy as np
import torch
from tqdm import tqdm

from . import _lib
from .flow_tracker import FlowTracker
from .keyframe import KeyframeFrontend, add_views_group, encode_views, regress_frames
from .loop_detector import LoopDetector
from .pose_graph import PoseGraphOpt

def _min_consistent_views(k):
    """min_consistent_views of render, extract_mesh, save_mesh and save_data_all: None or an integer in [0, 8] (the
    most neighbours view_consistency counts); ValueError otherwise."""
    if k is None:
        return 0
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 0 <= k <= 8:
        raise ValueError("min_consistent_views must be None or an integer in [0, 8], got %r" % (k,))
    return int(k)


def _msg(prefix, text):
    """print_msg (utils/slam_utils.py:448-450) without colours."""
    tqdm.write(prefix + text)


class View(dict):
    """A dict with attribute access (what munch.Munch gives get_view's callers)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None

    def __setattr__(self, k, v):
        self[k] = v


class _DeviceImages(list):
    """The input images, kept on the device; reading one copies it to the host, as the reference's list holds
    image.squeeze(0).cpu() (slam.py:148)."""

    def __getitem__(self, v):
        x = list.__getitem__(self, v)
        return [t.cpu() for t in x] if isinstance(v, slice) else x.cpu()

    def __iter__(self):
        return (t.cpu() for t in list.__iter__(self))

    def device_stack(self):
        return torch.stack(list(list.__iter__(self)))


class _DevArray:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": tuple(shape), "typestr": typestr, "version": 3,
                                         "strides": None}


class _Graph:
    """Owner of one sta_graph handle and torch views of its tables."""

    def __init__(self, max_nodes, max_edges, max_views, H, W, device):
        self.H, self.W, self.device = H, W, device
        self.max_nodes, self.max_edges, self.max_views = max_nodes, max_edges, max_views
        L = _lib.lib()
        h = ctypes.c_void_p()
        with torch.cuda.device(device):
            _lib.check(L.sta_graph_create(max_nodes, max_edges, max_views, H, W, ctypes.byref(h)), "sta_graph_create")
        self.h = h
        p = (ctypes.c_void_p * 12)()
        _lib.check(L.sta_graph_tables(h, p), "sta_graph_tables")
        f4, i8 = "<f4", "<i8"
        spec = [("pose", (max_nodes, 8), f4), ("depth", (max_nodes, H, W), f4), ("conf", (max_nodes, H, W), f4),
                ("intri", (max_nodes, 3, 3), f4), ("cmean", (max_nodes,), f4), ("node_to_view", (max_nodes,), i8),
                ("node_to_connected_view", (max_nodes,), i8), ("best_node", (max_views,), i8),
                ("best_mean", (max_views,), f4), ("edges", (max_edges, 2), i8), ("meas", (max_edges, 8), f4),
                ("weight", (max_edges, 7), f4)]
        for k, (name, shape, ts) in enumerate(spec):
            setattr(self, name, torch.as_tensor(_DevArray(p[k], shape, ts), device=device))

    def __del__(self):
        if getattr(self, "h", None) and _lib._lib is not None:
            _lib.lib().sta_graph_destroy(self.h)
            self.h = None

    def flags(self):
        f = ctypes.c_int()
        _lib.check(_lib.lib().sta_graph_flags(self.h, ctypes.byref(f)), "sta_graph_flags")
        return f.value


class OnlineSLAM:
    def __init__(self, ckpt_path: str, vocab_path: str,
                 verbose: bool = False, max_view_num: int = 400,
                 neighbor_edge_num: int = 3, loop_edge_num: int = 3,
                 loop_dist_min: int = 40, loop_nms: int = 40,
                 loop_cand_thresh_neighbor: int = 5,
                 conf_thres: float = 4.2, rel_pose_thres: float = 0.75,
                 flow_thres: float = 5.0, pgo_every: int = 500, live_mode: bool = False):
        self.device = torch.device("cuda")
        self.verbose = verbose
        self.max_view_num = max_view_num
        self.neighbor_edge_num = neighbor_edge_num
        self.loop_edge_num = loop_edge_num
        # slam.py:33-36
        self.max_nodes = max_view_num * (neighbor_edge_num * 2 + loop_edge_num)
        scale_edges_num = neighbor_edge_num * 2 + loop_edge_num - 1
        pose_edges_num = (neighbor_edge_num * 2 + loop_edge_num) // 2 + 1
        self.max_edges = max_view_num * (scale_edges_num + pose_edges_num)
        self.conf_thres = conf_thres
        self.rel_pose_thres = rel_pose_thres

        self.frontend = self.load_frontend(ckpt_path)
        total_params = sum(p.numel() for p in self.frontend.parameters())
        if self.verbose:
            _msg("[INFO] ", f"Total parameters: {total_params}")
        self.kf = KeyframeFrontend(self.frontend)
        self.img_shapes = []
        self.imgs = _DeviceImages()
        self.view_names = []

        self.lc_detector = LoopDetector(vocab_path, loop_dist_min, loop_nms, loop_cand_thresh_neighbor)
        self.image_resolution = (224, 224)
        self.view_num = 0
        self.pgo_every = pgo_every
        self.flow_tracker = FlowTracker(flow_thres)
        self.time_dict = self._zero_times()
        self.live_mode = live_mode
        self.loop_related_views = set()
        self.pgo_window_size = 2 * pgo_every
        self.pgo_route = None  # PoseGraphOpt's route: None (by size), "sparse" or "dense"
        self.pgo_background = False  # run due PGOs on a side stream while step goes on (see the module docstring)
        self.consistency_thres = 0.05  # view_consistency's depth agreement threshold, in world units of the map
        self._pgo_run = None  # a background PGO not yet folded: (PoseGraphRun, its problem, nodes to replay)
        self._graph = None  # created at the first keyframe, when the map size is known
        self._kf_queue = []  # keyframe insertions not yet launched (_add_keyframe, insert_keyframes)
        self._tracked = []  # one record per track call and session (_track_store), in tracking order
        self._reset_host_graph()

    @staticmethod
    def _zero_times():
        return {"prepare_data": 0.0, "encoder": 0.0, "decoder": 0.0, "lc": 0.0, "pgo": 0.0, "graph_construction": 0.0}

    def _reset_host_graph(self):
        # integer mirror of PoseGraphNodes' lists (pose_graph.py:48-54): all of them follow from the keep decisions
        self.view_to_node = {}
        self.node_to_connected_view = []
        self.num_nodes = 0
        self.num_edges = 0

    def reset(self):
        """slam.py:76-93: the loop detector and loop_related_views are not reset."""
        self.kf = KeyframeFrontend(self.frontend)
        self.img_shapes = []
        self.imgs = _DeviceImages()
        self.view_names = []
        self.view_num = 0
        if self._pgo_run is not None:  # discarded, once its queued work has finished with the tables
            self._pgo_run[0].wait()
            self._pgo_run = None
        self._kf_queue = []
        self._tracked = []
        if self._graph is not None:
            with torch.cuda.device(self._graph.device):
                _lib.check(_lib.lib().sta_graph_reset(self._graph.h, _lib.cur_stream()), "sta_graph_reset")
        self._reset_host_graph()
        self.flow_tracker.reset()
        self.time_dict = self._zero_times()

    def load_frontend(self, ckpt_path: str):
        """The STA of the checkpoint at ckpt_path; an already-built STA passed in place of the path is used as it is
        (SLAMSessions: sessions sharing one model)."""
        if isinstance(ckpt_path, torch.nn.Module):
            return ckpt_path
        from .sta_model.sta_model import SymmetricTwoViewAssociation as STA
        frontend = STA()
        checkpoint = torch.load(ckpt_path, map_location="cpu", weights_only=False)
        frontend.load_state_dict(checkpoint["model"], strict=True)
        del checkpoint
        frontend.to(self.device)
        frontend.eval()
        return frontend

    # ------------------------------------------------------------------------------------------------ graph
    def _ensure_graph(self, image):
        H, W = int(image.shape[-2]), int(image.shape[-1])
        if self._graph is None:
            self._graph = _Graph(self.max_nodes, self.max_edges, self.max_nodes, H, W, self.device)
            self._identity = torch.zeros(8, dtype=torch.float32, device=self.device)
            self._identity[6:] = 1.0

    def _check_flags(self):
        """Called right after a read-back, so every earlier graph launch has completed."""
        if self._graph is not None and self._graph.flags() & _lib.GRAPH_FLAG_NOT_SO3:
            raise ValueError("a relative pose's rotation is not orthonormal (pp.mat2SE3(atol=1e-3) refuses it)")

    def _regress_keyframe(self, i, js):
        """The frontend's part of a keyframe: (the K pose confidences on the host, indices of the kept candidates, the
        device batch {pose [K,4,4], pose_conf [K], conf / depths [2,n,H,W], intri [n,3,3], conf_mean [2,n]})."""
        res, = self.kf.regress_keyframes_gated([(i, js)], self.rel_pose_thres)
        return res

    def _regress_keyframes(self, items):
        """The frontend's part of many keyframes items = [(i, js), ...]: per item, in order, what _regress_keyframe
        returns, or None when js is empty (KeyframeFrontend.regress_keyframes_gated; may be a generator)."""
        return self.kf.regress_keyframes_gated(items, self.rel_pose_thres)

    def _add_keyframe(self, i, js, keep, batch):
        """connect_view_i_j (slam.py:191-241) for the kept edges, in order: the host integers now, the launch queued
        (_kf_queue) for the next insert_keyframes; a capacity IndexError launches the queue first."""
        g = self._graph
        n = len(keep)
        kept_js = [js[k] for k in keep]
        if n > _lib.GRAPH_MAX_KEYFRAME_EDGES:
            self._insert_queued()
            raise ValueError("at most %d kept edges per keyframe" % _lib.GRAPH_MAX_KEYFRAME_EDGES)
        v2n = {v: list(self.view_to_node.get(v, [])) for v in set(kept_js) | {i}}
        first_j, n_scale = [], n - 1
        for k, j in enumerate(kept_js):
            v2n[i].append(self.num_nodes + 2 * k)
            first_j.append(v2n[j][0] if v2n[j] else -1)
            n_scale += first_j[-1] >= 0
            v2n[j].append(self.num_nodes + 2 * k + 1)
        if self.num_nodes + 2 * n > g.max_nodes or i >= g.max_views:
            self._insert_queued()
            raise IndexError("pose graph node capacity (%d) exceeded" % g.max_nodes)
        if self.num_edges + n_scale + n > g.max_edges:
            self._insert_queued()
            raise IndexError("pose graph edge capacity (%d) exceeded" % g.max_edges)
        H, W = batch["conf"].shape[-2:]
        args = ((ctypes.c_int64 * n)(*kept_js), (ctypes.c_int * n)(*keep), (ctypes.c_int * n)(*first_j))
        kf = _lib.StaGraphKeyframe(g.h, i, n, self.num_nodes, self.num_edges, H, W, *args,
                                   *[batch[k].data_ptr() for k in ("pose", "pose_conf", "conf", "depths", "intri",
                                                                   "conf_mean")])
        if not _lib.lib().sta_graph_add_keyframes_scratch_bytes(ctypes.byref(kf), 1):  # refused: nothing changes
            _lib.check(1, "sta_graph_add_keyframes")
        self._kf_queue.append((kf, args, batch))  # the host arrays and the device inputs live until the launch
        if self._pgo_run is not None:  # the nodes a pending background PGO's fold re-derives, in link order
            rec, e = self._pgo_run[2], self.num_edges
            for k in range(n):
                ni = self.num_nodes + 2 * k
                if k > 0:
                    rec.append((ni, self.num_nodes, e))
                    e += 1
                if first_j[k] >= 0:
                    rec.append((ni + 1, first_j[k], e))
                    e += 1
                if k == 0:
                    rec.append((ni, ni + 1, e))
                e += 1
        self.view_to_node.update(v2n)
        for j in kept_js:
            self.node_to_connected_view += [j, i]
        self.num_nodes += 2 * n
        self.num_edges += n_scale + n

    def _insert_queued(self):
        """Launch this session's queued keyframe insertions (insert_keyframes); called before anything reads the
        tables."""
        insert_keyframes([self])

    def _insert_keyframe(self, i, js, conf_host, keep, batch):
        """connect_view_i_j (slam.py:191-241) after the gate, for a registered view i: the reject and loop-closure
        messages, loop_related_views, and the kept edges into the graph (_add_keyframe)."""
        kept = set(keep)
        for k, j in enumerate(js):
            names = f"(view {i} [{self.view_names[i]}] -- view {j} [{self.view_names[j]}])"
            if k not in kept:
                if self.verbose:
                    _msg("[EdgeReject] ", f"Rejecting edge {names} with conf {conf_host[k]:.3f}")
            elif i - j > self.neighbor_edge_num and self.verbose:  # slam.py:199-203
                _msg("[LoopClosure] ", f"Adding loop closure edge {names} with conf {conf_host[k]:.3f}")
                self.loop_related_views.add(i)
                self.loop_related_views.add(j)
        if keep:
            self._add_keyframe(i, js, keep, batch)

    def _pgo_if_due(self, force_pgo, log_intermediate_results, output_folder, group=None):
        """slam.py:282-297: PGO every pgo_every views or when forced, after logging the trajectory if asked.  Returns
        whether it ran.  A background PGO is captured into `group` (SLAMSessions.step) when one is given."""
        if not (self.view_num % self.pgo_every == 0 or force_pgo):
            return False
        self.wait_pgo()
        if log_intermediate_results:
            self.save_data_all(f"{output_folder}", save_view_graph=False, traj_name_postfix=f"{self.view_num - 1}",
                               save_poses=True, save_images=False, save_scales=True, save_depths=False,
                               save_intrinsics=False, save_confs=False, save_ply=False)
        opt_start = time.time()
        if self.pgo_background:
            self._pgo_launch(group)
            self.time_dict["pgo"] += time.time() - opt_start
            return True
        self.pose_graph_optimize()
        self.time_dict["pgo"] += time.time() - opt_start
        torch.cuda.empty_cache()
        return True

    def _pgo_launch(self, group=None):
        """The background form of pose_graph_optimize: its opening messages and optimised set now, loop_related_views
        cleared now (keyframes inserted before the fold add to the next PGO's set, as after a synchronous PGO), and
        the optimisation started on a side stream (PoseGraphOpt.start), or captured into `group`, which starts it with
        the other PGOs it holds (group.add returns the run's handle: poll(), wait(), stream)."""
        problem = self._pgo_begin()
        self.loop_related_views = set()
        if problem is None:
            _msg("[PoseGraphOpt] ", "Pose graph optimization done.")
            return
        graph, args = problem
        self._pgo_run = (graph.start(*args) if group is None else group.add(graph, args), problem, [])

    @property
    def pgo_pending(self):
        """Whether a background PGO has started and not yet been folded into the graph."""
        return self._pgo_run is not None

    def wait_pgo(self):
        """Fold a pending background PGO into the graph, waiting for it to finish if it is still running."""
        self._pgo_fold(wait=True)

    def _pgo_poll(self):
        """Fold a pending background PGO if it has finished, or enqueue its next iteration; never waits."""
        self._pgo_fold(wait=False)

    def _pgo_fold(self, wait):
        """A finished background PGO into the graph: its poses over the nodes it optimised, the nodes inserted since its
        launch re-derived from them (sta_graph_replay_nodes), which leaves the graph as a synchronous PGO followed by
        those insertions would, bit for bit; then the closing message, the flag check and empty_cache."""
        if self._pgo_run is None:
            return
        run, problem, replay = self._pgo_run
        start = time.time()
        if wait:
            run.wait()
        elif not run.poll():
            return
        self._pgo_run = None
        self._pgo_write(problem, replay)
        _msg("[PoseGraphOpt] ", "Pose graph optimization done.")
        torch.cuda.empty_cache()
        self.time_dict["pgo"] += time.time() - start

    # ------------------------------------------------------------------------------------------------ step
    def add_view(self, image, image_shape, view_name):
        self.kf.add_view(image, image_shape)
        self.img_shapes.append(image_shape)
        self.imgs.append(image.squeeze(0).detach())
        self.view_names.append(view_name)
        self.view_num += 1

    def step(self, value, force_pgo=False, log_intermediate_results=False, output_folder=None):
        """slam.py:244-297."""
        prepare_start = time.time()
        image, image_shape, img_gray, view_name = value["rgb"], value["shape"], value["gray"], value["view_name"]
        i = self.view_num
        self._ensure_graph(image)
        if i == 0:
            self._graph.pose[0].copy_(self._identity)  # slam.py:251-253
        self._pgo_poll()
        self.time_dict["prepare_data"] += time.time() - prepare_start

        enc_start = time.time()
        self.add_view(image, image_shape, view_name)
        self.time_dict["encoder"] += time.time() - enc_start

        farthest_neighbor = max(0, i - self.neighbor_edge_num)
        loop_start = time.time()
        loop_candi_list = self.lc_detector.detect_loop(img_gray, farthest_neighbor)  # read-back: candidates
        self.time_dict["lc"] += time.time() - loop_start
        self._check_flags()

        graph_start = time.time()
        js = list(range(farthest_neighbor, i)) + [j for j, _ in loop_candi_list[:self.loop_edge_num]]
        if js:
            dec_start = time.time()
            res = self._regress_keyframe(i, js)  # read-back: the gate
            self.time_dict["decoder"] += time.time() - dec_start
            self._check_flags()
            self._insert_keyframe(i, js, *res)
            self._insert_queued()  # a group of one
        self._pgo_poll()
        self.time_dict["graph_construction"] += time.time() - graph_start
        return self._pgo_if_due(force_pgo, log_intermediate_results, output_folder)

    def step_many(self, values, force_pgo=False, log_intermediate_results=False, output_folder=None):
        """[self.step(v, force_pgo=force_pgo and k == len(values) - 1, ...) for k, v in enumerate(values)]: the same
        graph, PGO calls, host bookkeeping, messages and time buckets, with the frontend batched across keyframes.
        Returns the is_optimized flags.  All values must have one image size (ValueError before any launch).

        Order: all views are encoded (KeyframeFrontend.add_views) and loop-detected (LoopDetector.detect_loops, one
        read-back) first; then edge chunk by edge chunk, the gate's read-back, the kept edges' heads, and the keyframes
        of the chunk registered and inserted in order, with PGO where step would run it (so view_num, imgs and
        view_names hold exactly the views inserted so far).  A capacity IndexError leaves the graph, view_num, imgs and
        view_names as step would at that keyframe; the encoder cache and the loop database may then already hold later
        views of the call.  A non-orthonormal rotation raises ValueError by the end of the call.

        Host synchronisations: one for the loop candidates, one per edge chunk, one per PGO iteration, and one at the
        end of the call unless a PGO ran last (reading the rotation flag).  This is step_keyframes over this session
        alone; a background PGO that falls due starts at its keyframe."""
        return step_keyframes([(self, list(values))], [force_pgo], log_intermediate_results, [output_folder],
                              detect=lambda sessions, grays, fars: [self.lc_detector.detect_loops(grays[0], fars[0])],
                              regress=lambda items: self._regress_keyframes([(i, js) for _, i, js in items]),
                              group=None, polled=[self])[0]

    def _register_keyframe(self, v, i, js, res):
        """Keyframe i of step_many after its gate: the view's host lists, then its kept edges (_insert_keyframe)."""
        self.img_shapes.append(v["shape"])
        self.imgs.append(v["rgb"].squeeze(0).detach())
        self.view_names.append(v["view_name"])
        self.view_num += 1
        if js:
            self._insert_keyframe(i, js, *res)

    def pose_graph_optimize(self):
        """slam.py:108-140 through PoseGraphOpt on the device tables (per-edge weights: DESIGN.md §4).  Runs now, after
        folding a pending background PGO (wait_pgo), whatever pgo_background says."""
        self.wait_pgo()
        problem = self._pgo_begin()
        if problem is not None:
            graph, args = problem
            graph.optimize(*args)
        self._pgo_end(problem)

    def _pgo_begin(self):
        """The first half of a PGO (slam.py:108-120): its messages, then (PoseGraphOpt over the node table with the
        optimised node set, (edges, measurements, weights)), or None for a graph without nodes or edges.  The optimised
        set is the nodes of the last pgo_window_size views and the loop-related views (view ids, used as node ids)."""
        _msg("[PoseGraphOpt] ", f"Pose graph optimization (at keyframe {self.view_num}) ...")
        if self.live_mode:
            _msg("[PoseGraphOpt] ", "This may cause latency in live mode, please hold the camera steady if possible.")
        N, E = self.num_nodes, self.num_edges
        opt = set()
        for v in range(max(0, self.view_num - self.pgo_window_size), self.view_num):
            opt.update(self.view_to_node.get(v, []))
        opt.update(self.loop_related_views)  # view ids, used as node ids (slam.py:120)
        if not (N > 0 and E > 0):
            return None
        self._insert_queued()
        g = self._graph
        idx = torch.tensor(sorted(opt), dtype=torch.int64).to(self.device)
        graph = PoseGraphOpt(g.pose[:N], to_optimize_idxs=idx, route=self.pgo_route)
        return graph, (g.edges[:E], g.meas[:E], g.weight[:E])

    def _pgo_end(self, problem):
        """The second half of a PGO, after the optimisation of _pgo_begin's problem: the poses written back, the
        message, loop_related_views cleared."""
        if problem is not None:
            self._pgo_write(problem)
        _msg("[PoseGraphOpt] ", "Pose graph optimization done.")
        self.loop_related_views = set()

    def _pgo_write(self, problem, replay=()):
        """The optimised poses of _pgo_begin's problem into the node table, then the (node, parent, edge) triples of
        `replay` re-derived in order."""
        self._insert_queued()  # the replayed nodes' insertions come first
        g = self._graph
        nodes = problem[0].get_nodes()
        g.pose[:nodes.shape[0]] = nodes
        if replay:
            flat = (ctypes.c_int * (3 * len(replay)))(*[x for t in replay for x in t])
            with torch.cuda.device(g.device):
                _lib.check(_lib.lib().sta_graph_replay_nodes(g.h, len(replay), flat, _lib.cur_stream()),
                           "sta_graph_replay_nodes")
        self._check_flags()

    # ------------------------------------------------------------------------------------------------ export
    def _export(self, view0, num_views, cloud):
        """Device gather through the best nodes (and the world point cloud); no host synchronisation."""
        for v in range(view0, view0 + num_views):
            if not self.view_to_node.get(v):
                raise IndexError("view %d has no node in the pose graph" % v)
        self._insert_queued()
        g = self._graph
        dev = g.device
        H, W = g.H, g.W

        def f32(*s):
            return torch.empty(*s, dtype=torch.float32, device=dev)

        out = {"pose": f32(num_views, 4, 4), "scale": f32(num_views, 1), "depth": f32(num_views, H, W),
               "conf": f32(num_views, H, W), "intri": f32(num_views, 3, 3)}
        imgs = pts = cols = cnt = scratch = None
        if cloud:
            imgs = self.imgs.device_stack()[view0:view0 + num_views].to(torch.float32).contiguous()
            pts, cols = f32(num_views * H * W, 3), f32(num_views * H * W, 3)
            cnt = torch.zeros(1, dtype=torch.int64, device=dev)
            nbytes = int(_lib.lib().sta_graph_export_scratch_bytes(num_views, H))
            scratch = torch.empty((nbytes + 7) // 8, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().sta_graph_export(
                g.h, view0, num_views, float(self.conf_thres), _lib.ptr(imgs), _lib.ptr(out["pose"]), _lib.ptr(out["scale"]),
                _lib.ptr(out["depth"]), _lib.ptr(out["conf"]), _lib.ptr(out["intri"]), _lib.ptr(pts), _lib.ptr(cols),
                _lib.ptr(cnt), _lib.ptr(scratch), _lib.cur_stream()), "sta_graph_export")
        if cloud:
            out.update(points=pts, colors=cols, count=cnt, images=imgs)
        return out

    def get_view(self, v, filter_outlier=True, return_pose=True, return_depth=True, return_intri=True):
        """slam.py:299-326.  A background PGO is folded first if it has finished; while it runs, the view shows the
        poses from before it."""
        self._pgo_poll()
        ex = self._export(v, 1, cloud=False)
        view = View()
        if return_pose:
            view["pose"] = ex["pose"][0].cpu()
        self._check_flags()
        if return_depth:
            depth = (ex["depth"][0] * ex["scale"][0]).cpu()
            if filter_outlier:
                depth[ex["conf"][0].cpu() < self.conf_thres] = 0.0
            view["depth"] = depth
        if return_intri:
            view["intri"] = ex["intri"][0].cpu()
        return view

    def render(self, poses, K, size, point_radius=0, views=None, lines=None, background=(1.0, 1.0, 1.0),
               min_consistent_views=None):
        """Images of the map of `views` (a range; default: every view with a node) from cameras poses [C,4,4]
        (camera-to-world) with intrinsics K, drawn on the device by render.render_views: the confident points of
        save_data_all's PLY, z-buffered, and `lines` (render.camera_frusta, render.graph_segments) depth-tested with
        them.  Returns {rgb, depth, index} device tensors without a host synchronisation.  A background PGO is folded
        first if it has finished, never waited for (as get_view).  IndexError for a view without a node; nothing in
        the session changes.  min_consistent_views=k in [0, 8] keeps only the pixels whose view_consistency count
        over `views` is at least k (None or 0: every confident pixel)."""
        from .render import render_views
        k = _min_consistent_views(min_consistent_views)
        maps = self._consistent_maps(self._view_maps(views), k)
        return render_views(maps, self.conf_thres, poses, K, size, point_radius=point_radius, lines=lines,
                            background=background)

    def view_consistency(self, views=None):
        """Multi-view depth consistency of the map of `views` (a range; default: every view with a node): int32
        [len(views),H,W], per pixel the number of views of the range within 4 indices whose depth agrees with the
        pixel's reprojection within consistency_thres -- utils.slam_utils.view_consistency_check of get_view's
        depth (scaled, zero where conf < conf_thres), intri and pose of those views, bit for bit.  The window is
        clipped at the range's ends.  No host synchronisation; a background PGO is folded first if it has finished,
        never waited for (as render).  IndexError for a view without a node; nothing in the session changes."""
        return self._consistency(self._view_maps(views, images=False))

    def _consistency(self, maps):
        """view_consistency of an exported `maps` dict; depth * scale is get_view's single float32 multiply."""
        from .utils.slam_utils import view_consistency_check
        depth = (maps["depth"] * maps["scale"][:, :, None]).masked_fill(maps["conf"] < self.conf_thres, 0.0)
        return view_consistency_check(depth, maps["intri"], maps["pose"], self.consistency_thres)

    def _consistent_maps(self, maps, k):
        """maps with conf set to -inf where the view_consistency count is below k (maps unchanged for k = 0)."""
        if k:
            maps["conf"] = maps["conf"].masked_fill(self._consistency(maps) < k, float("-inf"))
        return maps

    def _view_maps(self, views, images=True):
        """The `maps` dict of render_views and fuse_views for `views` (a range; default: every view with a node), after
        folding a background PGO that has finished (never waiting for one).  IndexError for a view without a node.
        images=False leaves the images out."""
        self._pgo_poll()
        if views is None:
            n = 0
            while self.view_to_node.get(n):
                n += 1
            views = range(n)
        if not isinstance(views, range) or views.step != 1:
            raise ValueError("views must be a range with step 1")
        if len(views) == 0:
            dev = self.device if self._graph is None else self._graph.device
            return {k: torch.empty(s, dtype=torch.float32, device=dev)
                    for k, s in (("pose", (0, 4, 4)), ("scale", (0, 1)), ("depth", (0, 1, 1)), ("conf", (0, 1, 1)),
                                 ("intri", (0, 3, 3)), ("images", (0, 3, 1, 1)))}
        maps = self._export(views.start, len(views), cloud=False)
        if images:
            maps["images"] = torch.stack(list(list.__iter__(self.imgs))[views.start:views.stop]).to(torch.float32)
        return maps

    def extract_mesh(self, voxel_size, trunc=None, min_weight=1, views=None, min_consistent_views=None):
        """The map of `views` (a range; default: every view with a node) fused into a TSDF volume and meshed on the
        device by fusion.fuse_views: {bricks, tsdf, weight, color, vertices, vertex_colors, faces} device tensors.
        voxel_size in world units; trunc in (0, 4 voxel_size], default 4 voxel_size; min_weight: the views every
        corner of a meshed cube needs.  The volume is rebuilt from the current poses on every call, so it follows each
        PGO.  A background PGO is folded first if it has finished, never waited for (as render).  IndexError for a
        view without a node; nothing in the session changes.  min_consistent_views as in render."""
        from .fusion import fuse_views
        k = _min_consistent_views(min_consistent_views)
        maps = self._consistent_maps(self._view_maps(views), k)
        return fuse_views(maps, self.conf_thres, voxel_size, trunc=trunc, min_weight=min_weight)

    def render_surface(self, poses, K, size, voxel_size, trunc=None, min_weight=1, views=None, min_consistent_views=None,
                       background=(1.0, 1.0, 1.0)):
        """Images of the fused surface of `views` (a range; default: every view with a node) from cameras poses
        [C,4,4] (camera-to-world) with intrinsics K ([3,3] or [C,3,3]) at size (Ho, Wo): the map fused as
        extract_mesh fuses it (fusion.fuse_volume) and ray-cast on the device (fusion.raycast), without meshing.
        Returns {rgb, color [C,Ho,Wo,3], depth [C,Ho,Wo], normal [C,Ho,Wo,3]} device tensors.  The only host
        synchronisations are fusion's two counts.  voxel_size, trunc, min_weight and min_consistent_views as in
        extract_mesh; a background PGO is folded first if it has finished, never waited for (as render).  IndexError
        for a view without a node; nothing in the session changes.  Arguments are checked before any work
        (ValueError)."""
        from .fusion import _check_cameras, _fuse, _min_weight, _raycast, _voxel_args
        k = _min_consistent_views(min_consistent_views)
        _voxel_args(voxel_size, trunc)
        mw = _min_weight(min_weight)
        dev = self.device if self._graph is None else self._graph.device
        cams = _check_cameras(poses, K, size, 1e-3, background, dev)
        maps = self._consistent_maps(self._view_maps(views), k)
        vol, keys, vox = _fuse(maps, self.conf_thres, voxel_size, trunc, 2 ** 20, mw)
        return _raycast(keys, vol["tsdf"], vol["weight"], vol["color"], vox, mw, *cams)

    def save_mesh(self, output_folder, voxel_size, trunc=None, min_weight=1, views=None, min_consistent_views=None):
        """extract_mesh written to output_folder/mesh.ply (write_mesh_ply).  A pending background PGO is folded first
        (wait_pgo), as save_data_all does.  Returns the mesh's path."""
        _min_consistent_views(min_consistent_views)
        self.wait_pgo()
        mesh = self.extract_mesh(voxel_size, trunc=trunc, min_weight=min_weight, views=views,
                                 min_consistent_views=min_consistent_views)
        os.makedirs(output_folder, exist_ok=True)
        path = os.path.join(output_folder, "mesh.ply")
        write_mesh_ply(path, mesh["vertices"].cpu().numpy(), mesh["vertex_colors"].cpu().numpy(),
                       mesh["faces"].cpu().numpy())
        return path

    def get_view_graph(self):
        """slam.py:328-336."""
        return {v: [self.node_to_connected_view[u] for u in self.view_to_node.get(v, [])] for v in range(self.view_num)}

    def save_data_all(self, output_folder,
                      save_view_graph=True, traj_name_postfix=None,
                      save_poses=True, save_images=True, save_scales=True,
                      save_depths=True, save_intrinsics=True,
                      save_confs=True, save_ply=True,
                      gt_poses=None, gt_depths=None, gt_intrinsics=None, min_consistent_views=None):
        """slam.py:338-421: the same files, keys, shapes and dtypes.  A pending background PGO is folded first (wait_pgo).
        min_consistent_views=k in [0, 8] keeps in pointcloud.ply only the points whose view_consistency count over all
        views is at least k, in the same order (None or 0: every point); the other files do not change."""
        k = _min_consistent_views(min_consistent_views)
        self.wait_pgo()
        if not os.path.exists(output_folder):
            os.makedirs(output_folder)
        if save_view_graph:
            np.savez(f"{output_folder}/view_graph.npz", view_graph=self.get_view_graph(),
                     loop_min_dist=self.lc_detector.loop_dist_min, view_names=self.view_names)
        ex = self._export(0, self.view_num, cloud=save_ply)
        poses = ex["pose"].cpu()
        self._check_flags()
        traj_postfix = f"_{traj_name_postfix}" if traj_name_postfix is not None else ""
        if save_poses:
            np.save(f"{output_folder}/trajectory{traj_postfix}.npy", poses.numpy())
        if save_scales:
            np.save(f"{output_folder}/scales{traj_postfix}.npy", ex["scale"].cpu().numpy())
        if save_images:
            images = (self.imgs.device_stack().float().permute(0, 2, 3, 1) + 1.0) / 2.0
            np.save(f"{output_folder}/images.npy", images.cpu().numpy())
        if save_depths:
            np.save(f"{output_folder}/depths.npy", ex["depth"].cpu().numpy())
        if save_confs:
            np.savez(f"{output_folder}/confs.npz", confs=ex["conf"].cpu().numpy(), thres=self.conf_thres)
        if save_intrinsics:
            np.save(f"{output_folder}/intrinsics.npy", ex["intri"].cpu().numpy())
        if save_ply:
            n = int(ex["count"].cpu())
            points, colors = ex["points"][:n], ex["colors"][:n]
            if k:  # the cloud is the conf > conf_thres pixels in (view, row, column) order
                keep = self._consistency(ex)[ex["conf"] > self.conf_thres] >= k
                points, colors = points[keep], colors[keep]
            write_ply(f"{output_folder}/pointcloud.ply", points.cpu().numpy(), colors.cpu().numpy())
        if gt_poses is not None:
            np.save(f"{output_folder}/gt_poses.npy", np.array(gt_poses).astype(np.float32))
        if gt_depths is not None:
            np.save(f"{output_folder}/gt_depths.npy", np.array(gt_depths).astype(np.float32))
        if gt_intrinsics is not None:
            np.save(f"{output_folder}/gt_intrinsics.npy", gt_intrinsics)

    def get_pointmap_vis(self, v):
        """slam.py:423-432: the view's local point map (host) and an 8-bit rendering of it."""
        view = self.get_view(v, filter_outlier=False, return_pose=False, return_depth=True, return_intri=True)
        depth, intri = view.depth.numpy().astype(np.float64), view.intri.numpy().astype(np.float64)
        H, W = depth.shape
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        pix = np.stack([xx, yy, np.ones_like(xx)], -1).astype(np.float64)
        pcl = (pix @ np.linalg.inv(intri).T * depth[..., None]).astype(np.float32)
        min_vals = pcl.min(axis=(0, 1), keepdims=True)
        max_vals = pcl.max(axis=(0, 1), keepdims=True)
        normalized = (pcl - min_vals) / (max_vals - min_vals + 1e-8)
        return (normalized * 255).astype(np.uint8), pcl

    def save_pointmap(self, v, output_folder):
        import cv2
        if not os.path.exists(output_folder):
            os.makedirs(output_folder)
        img, pcl = self.get_pointmap_vis(v)
        np.save(f"{output_folder}/pointmap_cam_{v}.npy", pcl)
        cv2.imwrite(f"{output_folder}/pointmap_cam_{v}.png", cv2.cvtColor(img, cv2.COLOR_RGB2BGR))

    def get_time_dict(self):
        time_dict = self.time_dict.copy()
        time_dict["graph_construction"] = time_dict["graph_construction"] - time_dict["decoder"]
        time_dict["total"] = sum(time_dict.values())
        return time_dict

    # ------------------------------------------------------------------------------------------------ tracked frames
    def track(self, values, kf=None):
        """Poses for frames that are not keyframes: each frame of values (step-style dicts: rgb, shape, view_name; gray
        is ignored), all of the views' size, is tracked against keyframe view kf (default: the last stepped view),
        which must have a node.  Returns device tensors {pose [F,4,4] (scale dropped, as get_view), scale [F],
        pose_conf [F], valid [F] uint8}; no host synchronisation.  See track_frames for the semantics; ValueError,
        before any launch and with nothing changed, for a frame of another size or a kf out of range or without a
        node."""
        return track_frames([(self, list(values), kf)])[0]

    def _track_check(self, values, kf):
        """The refusals of track for this session; returns the keyframe view."""
        if self.view_num == 0 or self._graph is None:
            raise ValueError("nothing to track against: no view has been stepped")
        kf = self.view_num - 1 if kf is None else operator.index(kf)
        if not 0 <= kf < self.view_num:
            raise ValueError("keyframe view %d out of range (%d views)" % (kf, self.view_num))
        if not self.view_to_node.get(kf):
            raise ValueError("view %d has no node in the pose graph yet" % kf)
        size = tuple(self.kf.img_shapes[0])
        if any(tuple(v["rgb"].shape[-2:]) != size for v in values):
            raise ValueError("tracked frames must have the size of the session's views %s" % (size,))
        return kf

    def _track_store(self, kf, names, pose, pconf, depth, conf):
        """sta_graph_track_frames over this session's frames of a track call (regressed against view kf), recorded for
        frame_trajectory; returns track's result."""
        g = self._graph
        F = len(names)
        anchor = self.view_to_node[kf][0]
        dev = g.device

        def f32(*shape):
            return torch.empty(*shape, dtype=torch.float32, device=dev)

        meas, s_edge, pose_out, scale = f32(F, 8), f32(F), f32(F, 4, 4), f32(F)
        valid = torch.empty(F, dtype=torch.uint8, device=dev)
        L, M = _lib.lib(), _lib.GRAPH_MAX_TRACK_FRAMES
        with torch.cuda.device(dev):
            for a in range(0, F, M):
                b = min(F, a + M)
                need = int(L.sta_graph_track_frames_scratch_bytes(b - a))
                scratch = torch.empty((need + 7) // 8, dtype=torch.float64, device=dev)
                _lib.check(L.sta_graph_track_frames(
                    g.h, b - a, (ctypes.c_int * (b - a))(*[anchor] * (b - a)), _lib.ptr(pose[a:b]), _lib.ptr(depth[a:b]),
                    _lib.ptr(conf[a:b]), _lib.ptr(meas[a:b]), _lib.ptr(s_edge[a:b]), _lib.ptr(valid[a:b]),
                    _lib.ptr(pose_out[a:b]), _lib.ptr(scale[a:b]), _lib.ptr(scratch), need, _lib.cur_stream()),
                    "sta_graph_track_frames")
        self._tracked.append({"names": list(names), "kf": [kf] * F, "anchor": [anchor] * F, "meas": meas,
                              "scale_edge": s_edge, "pose_conf": pconf, "valid": valid})
        return {"pose": pose_out, "scale": scale, "pose_conf": pconf, "valid": valid}

    def frame_trajectory(self):
        """Every tracked frame, in tracking order, recomposed on the current graph with one sta_graph_frame_poses per
        GRAPH_MAX_TRACK_FRAMES frames: {names, kf (host lists), pose [F,4,4] (scale dropped), scale [F], pose_conf [F],
        valid [F]} and the stored values it is composed from: anchor (host list), meas [F,8] (T_fk as [t | q | s]),
        scale_edge [F].  A background PGO is folded first if it has finished (as get_view); no host synchronisation."""
        self._pgo_poll()
        self._insert_queued()
        recs = self._tracked
        out = {k: [x for r in recs for x in r[k]] for k in ("names", "kf", "anchor")}
        dev = self.device if self._graph is None else self._graph.device
        F = len(out["names"])
        for k, shape, dt in (("meas", (0, 8), torch.float32), ("scale_edge", (0,), torch.float32),
                             ("pose_conf", (0,), torch.float32), ("valid", (0,), torch.uint8)):
            out[k] = torch.cat([r[k] for r in recs]) if recs else torch.empty(shape, dtype=dt, device=dev)
        out["pose"] = torch.empty(F, 4, 4, dtype=torch.float32, device=dev)
        out["scale"] = torch.empty(F, dtype=torch.float32, device=dev)
        L, M = _lib.lib(), _lib.GRAPH_MAX_TRACK_FRAMES
        with torch.cuda.device(dev):
            for a in range(0, F, M):
                b = min(F, a + M)
                _lib.check(L.sta_graph_frame_poses(
                    self._graph.h, b - a, (ctypes.c_int * (b - a))(*out["anchor"][a:b]), _lib.ptr(out["meas"][a:b]),
                    _lib.ptr(out["scale_edge"][a:b]), _lib.ptr(out["pose"][a:b]), _lib.ptr(out["scale"][a:b]),
                    _lib.cur_stream()), "sta_graph_frame_poses")
        return out

    def save_frame_trajectory(self, output_folder, traj_name_postfix=None):
        """frame_trajectory() into output_folder, in save_data_all's style: frame_trajectory{_postfix}.npy [F,4,4],
        frame_scales{_postfix}.npy [F] and frame_info{_postfix}.npz (names, kf, pose_conf, valid).  A pending
        background PGO is folded first (wait_pgo), as save_data_all does."""
        self.wait_pgo()
        if not os.path.exists(output_folder):
            os.makedirs(output_folder)
        t = self.frame_trajectory()
        postfix = f"_{traj_name_postfix}" if traj_name_postfix is not None else ""
        np.save(f"{output_folder}/frame_trajectory{postfix}.npy", t["pose"].cpu().numpy())
        np.save(f"{output_folder}/frame_scales{postfix}.npy", t["scale"].cpu().numpy())
        np.savez(f"{output_folder}/frame_info{postfix}.npz", names=np.array(t["names"]),
                 kf=np.array(t["kf"], dtype=np.int64), pose_conf=t["pose_conf"].cpu().numpy(),
                 valid=t["valid"].cpu().numpy())


def insert_keyframes(sessions):
    """Launch the keyframe insertions the sessions have queued (OnlineSLAM._add_keyframe), every session's in its
    order: one sta_graph_add_keyframes (two launches, no host synchronisation) per GRAPH_MAX_GROUP_KEYFRAMES
    keyframes, whichever sessions they belong to.  Nothing is launched when no keyframe is queued."""
    owners = [s for s in sessions if s._kf_queue]
    if not owners:
        return
    queued = [q for s in owners for q in s._kf_queue]
    for s in owners:
        s._kf_queue = []
    L, M = _lib.lib(), _lib.GRAPH_MAX_GROUP_KEYFRAMES
    device = owners[0]._graph.device
    with torch.cuda.device(device):
        for c0 in range(0, len(queued), M):
            part = queued[c0:c0 + M]
            tab = (_lib.StaGraphKeyframe * len(part))(*[kf for kf, _, _ in part])
            need = int(L.sta_graph_add_keyframes_scratch_bytes(tab, len(part)))
            scratch = torch.empty((need + 7) // 8, dtype=torch.float64, device=device)
            _lib.check(L.sta_graph_add_keyframes(tab, len(part), _lib.ptr(scratch), need, _lib.cur_stream()),
                       "sta_graph_add_keyframes")


def _share(sessions, key, seconds):
    for s in sessions:
        s.time_dict[key] += seconds / len(sessions)


def step_keyframes(calls, force, log_intermediate_results, output_folders, *, detect, regress, group, polled):
    """The keyframe loop of OnlineSLAM.step_many and SLAMSessions.step, over distinct sessions that share one STA:
    calls = [(session, [value, ...]), ...], force[c] whether call c's last keyframe forces a PGO, output_folders[c] its
    folder for log_intermediate_results.  Returns each call's is_optimized flags ([] for a call without keyframes).

    The callers differ only in these arguments: detect(sessions, grays, fars) gives each session's loop candidates with
    one read-back; regress([(session, i, js), ...]) yields, per keyframe, what OnlineSLAM._regress_keyframe returns or
    None; a due background PGO is captured into `group`, which starts it with the others at the end of the call, or is
    started at its keyframe when group is None; `polled` are the sessions polled after every keyframe (each session of
    the call is also polled before its first).  Order, refusals, host synchronisations and time buckets: see
    SLAMSessions.step and the sessions module."""
    flags = [[] for _ in calls]
    live = [(s, vs, f, d, out) for (s, vs), f, d, out in zip(calls, force, output_folders, flags) if vs]
    if not live:
        return flags
    sess, vals, force, folders, out = zip(*live)
    size = tuple(vals[0][0]["rgb"].shape[-2:])
    for s, vs in zip(sess, vals):
        if any(tuple(v["rgb"].shape[-2:]) != size for v in vs):
            raise ValueError("all keyframes of a call must have the same image size")
        if s.kf.img_shapes and tuple(s.kf.img_shapes[0]) != size:
            raise ValueError("the keyframes of a session must have the size of its views %s" % (s.kf.img_shapes[0],))
    i0 = [s.view_num for s in sess]
    for s, vs in zip(sess, vals):
        t = time.time()
        s._ensure_graph(vs[0]["rgb"])
        if s.view_num == 0:
            s._graph.pose[0].copy_(s._identity)  # slam.py:251-253
        s._pgo_poll()
        s.time_dict["prepare_data"] += time.time() - t

    t = time.time()
    add_views_group([s.kf for s in sess], [[v["rgb"] for v in vs] for vs in vals],
                    [[v["shape"] for v in vs] for vs in vals])
    _share(sess, "encoder", time.time() - t)

    fars = [[max(0, i + m - s.neighbor_edge_num) for m in range(len(vs))] for s, i, vs in zip(sess, i0, vals)]
    t = time.time()
    loops = detect(sess, [[v["gray"] for v in vs] for vs in vals], fars)  # read-back: candidates
    _share(sess, "lc", time.time() - t)
    for s in sess:
        s._check_flags()

    items, owner = [], []
    for c, (s, i, vs) in enumerate(zip(sess, i0, vals)):
        for m in range(len(vs)):
            items.append((s, i + m, list(range(fars[c][m], i + m)) + [j for j, _ in loops[c][m][:s.loop_edge_num]]))
            owner.append(c)
    chunks = KeyframeFrontend.edge_chunks([(i, js) for _, i, js in items])
    part = [[sess[c]] for c in owner]  # the sessions of each item's edge chunk, which share the chunk's regression time
    for chunk in chunks:
        members = [sess[c] for c in sorted({owner[t] for t in chunk})]
        for t in chunk:
            part[t] = members
    chunk_ends = {chunk[-1] for chunk in chunks}
    checked = [True] * len(sess)
    results = iter(regress(items))
    try:
        for t, (s, i, js) in enumerate(items):
            c = owner[t]
            m = i - i0[c]
            dec_start = time.time()
            res = next(results)  # the first keyframe of an edge chunk runs the chunk: read-back of its gate
            dt = time.time() - dec_start
            _share(part[t], "decoder", dt)
            _share(part[t], "graph_construction", dt)
            graph_start = time.time()
            s._check_flags()
            s._register_keyframe(vals[c][m], i, js, res)
            if js:
                checked[c] = checked[c] and not res[1]
            if t in chunk_ends:  # the chunk's keyframes, of every session, go in with one sta_graph_add_keyframes
                insert_keyframes(sess)
            for p in polled:
                p._pgo_poll()
            s.time_dict["graph_construction"] += time.time() - graph_start
            last = m == len(vals[c]) - 1
            out[c].append(s._pgo_if_due(force[c] and last, log_intermediate_results, folders[c], group))
            if out[c][-1] and not s.pgo_background:  # a synchronous PGO's read-backs waited for the graph launches
                checked[c] = s.num_nodes > 0 and s.num_edges > 0
    finally:  # an exception mid-chunk still leaves every graph as its host bookkeeping says
        insert_keyframes(sess)
        if group is not None:
            group.start()  # the background PGOs that fell due in the call, as one run
    if not all(checked):
        torch.cuda.current_stream().synchronize()
        for s, ok in zip(sess, checked):
            if not ok:
                s._check_flags()
    return flags


def track_frames(calls):
    """Track frames in several sessions that share one STA: calls = [(session, [value, ...], kf or None), ...].
    Every refusal comes first (OnlineSLAM._track_check; all frames of the call must have one size), then each session's
    queued keyframe insertions are launched (the anchors' maps must be in the store), then one transient encode of all
    frames (encode_views: nothing is cached), one regression of the pairs (frame, kf) in edge chunks that mix sessions
    (regress_frames: the launches of the keyframe path, no gate, no read-back), and one sta_graph_track_frames per
    session.  Returns each call's track result, in order.

    Frame f tracked against view k, a = the first node of k: s is the scale edge a new node of k would get from a
    (estimate_scale_with_depth_and_confidence(depth_k, depth_a, conf_k, conf_a) over the pair's k-side maps), and
    pose_f = pose[a] * Sim3(0, id, s) * Sim3(T_fk), the pose node i of a keyframe whose first kept edge is (i, k) gets,
    bit for bit.  No gate: valid = 0 only where T_fk's rotation is not orthonormal (no graph flag is raised).  Nothing
    of the session changes but its record of tracked frames: not the graph, its host mirror, the views, the encoder
    cache, the loop detector, the flow tracker or time_dict, and a background PGO is neither polled nor waited for."""
    calls = [(s, list(vs), kf) for s, vs, kf in calls]
    kfs = [s._track_check(vs, kf) for s, vs, kf in calls]
    images = [v["rgb"] for _, vs, _ in calls for v in vs]
    if any(tuple(x.shape[-2:]) != tuple(images[0].shape[-2:]) for x in images):
        raise ValueError("all frames of a track call must have the same image size")
    if any(s.frontend is not calls[0][0].frontend for s, _, _ in calls):
        raise ValueError("the sessions of a track call must share one STA")
    for s, _, _ in calls:
        s._insert_queued()
    out = []
    if images:
        H, W = int(images[0].shape[-2]), int(images[0].shape[-1])
        feats = encode_views(calls[0][0].frontend, images, [v["shape"] for _, vs, _ in calls for v in vs])
        pairs = [(f, None) for f in feats]
        t = 0
        for (s, vs, _), kf in zip(calls, kfs):
            for m in range(len(vs)):
                pairs[t + m] = (feats[t + m], s.kf.enc_features[kf])
            t += len(vs)
        pose, pconf, depth, conf = regress_frames(calls[0][0].frontend, pairs, H, W)
    t = 0
    for (s, vs, _), kf in zip(calls, kfs):
        F = len(vs)
        if F:
            out.append(s._track_store(kf, [v["view_name"] for v in vs], pose[t:t + F], pconf[t:t + F],
                                      depth[t:t + F], conf[t:t + F]))
        else:
            dev = s._graph.device
            out.append({"pose": torch.empty(0, 4, 4, device=dev), "scale": torch.empty(0, device=dev),
                        "pose_conf": torch.empty(0, device=dev), "valid": torch.empty(0, dtype=torch.uint8, device=dev)})
        t += F
    return out


def write_ply(path, points, colors):
    """Binary little-endian PLY: float x y z, uchar red green blue (colours in [0, 1], rounded to 8 bits)."""
    n = len(points)
    rec = np.empty(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1")])
    for k, name in enumerate("xyz"):
        rec[name] = points[:, k]
    rgb = np.rint(np.clip(np.asarray(colors, np.float64), 0.0, 1.0) * 255.0).astype(np.uint8)
    for k, name in enumerate("rgb"):
        rec[name] = rgb[:, k]
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n" % n)
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(rec.tobytes())


def write_mesh_ply(path, vertices, colors, faces):
    """Binary little-endian PLY of a triangle mesh: float x y z and uchar red green blue per vertex (colours in [0, 1],
    rounded to 8 bits, as write_ply), then per face `property list uchar int vertex_indices` of 3."""
    vertices, faces = np.asarray(vertices), np.asarray(faces)
    n, m = len(vertices), len(faces)
    rec = np.empty(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1")])
    for k, name in enumerate("xyz"):
        rec[name] = vertices[:, k]
    rgb = np.rint(np.clip(np.asarray(colors, np.float64), 0.0, 1.0) * 255.0).astype(np.uint8)
    for k, name in enumerate("rgb"):
        rec[name] = rgb[:, k]
    frec = np.empty(m, dtype=[("n", "u1"), ("v", "<i4", (3,))])
    frec["n"] = 3
    frec["v"] = faces.reshape(m, 3)
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
              "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\n"
              "property list uchar int vertex_indices\nend_header\n" % (n, m))
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(rec.tobytes())
        f.write(frec.tobytes())


def read_mesh_ply(path):
    """(vertices [N,3] fp32, colours [N,3] uint8, faces [M,3] int32) of a file write_mesh_ply wrote."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode().splitlines()
    n = int([ln for ln in head if ln.startswith("element vertex")][0].split()[-1])
    m = int([ln for ln in head if ln.startswith("element face")][0].split()[-1])
    vdt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1")])
    rec = np.frombuffer(data, dtype=vdt, count=n, offset=end)
    frec = np.frombuffer(data, dtype=[("n", "u1"), ("v", "<i4", (3,))], count=m, offset=end + n * vdt.itemsize)
    if m and not (frec["n"] == 3).all():
        raise ValueError("%s: not a triangle mesh" % path)
    return (np.stack([rec["x"], rec["y"], rec["z"]], -1), np.stack([rec["r"], rec["g"], rec["b"]], -1),
            frec["v"].astype(np.int32).reshape(m, 3))


def read_ply(path):
    """(points [N,3] fp32, colours [N,3] uint8) of a file write_ply wrote."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    n = int([ln for ln in data[:end].decode().splitlines() if ln.startswith("element vertex")][0].split()[-1])
    rec = np.frombuffer(data[end:], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1")],
                        count=n)
    return np.stack([rec["x"], rec["y"], rec["z"]], -1), np.stack([rec["r"], rec["g"], rec["b"]], -1)
