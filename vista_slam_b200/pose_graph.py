"""Sim(3) pose-graph optimisation on the GPU (SURVEY.md section 8(f) rank 4).

Mirror of the optimisation OnlineSLAM.pose_graph_optimize runs through PyPose (vista_slam/slam.py:108-140 over
vista_slam/pose_graph.py:70-154): Levenberg-Marquardt with a trust-region damping on the nodes listed in
`to_optimize_idxs`, all other nodes fixed, edge weights diag(conf_e).  Each iteration is ONE C call
(sta_pose_graph_lm_step, or its group form sta_pose_graph_lm_step_group, which optimize() uses with one graph: residuals,
Jacobians, normal equations, damped dense Cholesky solve, update and both losses, all on the device) followed by one
32-byte read-back for the accept / reject decision -- the same host round trip pp.optim.LM makes.
Tensors use PyPose's Sim3 layout (tx ty tz | qx qy qz qw | s), fp32, CUDA only (no CPU path).

Two routes solve the damped normal equations, chosen in the constructor (route=None) from the number of optimised nodes:
  * dense (num_opt <= _lib.PG_DENSE_MAX_OPT = 3657): sta_pose_graph_lm_step, a dense fp64 Cholesky of order 7 num_opt;
  * block-sparse (above): sta_pose_graph_lm_step_sparse, a block Cholesky (7x7 blocks) over a plan -- ordering,
    elimination tree, block pattern and update lists -- built on the host from the edge list and the optimised set.
Both compute the same residuals, Jacobians, normal equations, damping, update and losses; route="sparse" takes the
block-sparse route at any size (much faster from a few hundred optimised nodes on), route="dense" insists on the dense one.

Groups: optimize_group(graphs, edges, poses, weights) optimises several independent graphs together and leaves each one
exactly as its own optimize() would.  Each LM iteration steps every dense-route graph still running with ONE
sta_pose_graph_lm_step_group launch sequence (the kernels take a graph index, so one launch covers every graph's
Cholesky panel, triangular solve and so on), every block-sparse-route graph still running with ONE
sta_pose_graph_lm_step_sparse_group launch sequence (one launch per elimination-tree level covers every graph), and
reads all their info rows back with ONE copy; each graph keeps its own trust radius and plateau count and leaves the
group when its plateau rule stops it.  optimize() is a group of one.
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


def _read_info(info):
    """The host copy of a step's info rows (device fp64 [..., 4]): the one host synchronisation of an LM iteration."""
    return info.cpu()


class _LMState:
    """slam.py:121-134 for each of n graphs as a state machine: LM(TrustRegion(radius), min=1e-6) driven by
    StopOnPlateau(steps, patience, decreasing).  dampings() gives the active graphs' dampings for the next step;
    advance(graphs, results) takes that step's results, per active graph (candidate nodes, loss before, loss after,
    Cholesky ok), accepts or rejects each candidate, and drops the graphs whose plateau rule stops them.  done once no
    graph is active or `steps` steps have run.  _lm_iterations drives it in a loop, PoseGraphRun one poll at a time."""

    def __init__(self, n, steps, patience, decreasing, radius):
        self.steps, self.patience, self.decreasing = steps, patience, decreasing
        self.radii, self.stall, self.losses = [radius] * n, [0] * n, [[] for _ in range(n)]
        self.active = list(range(n))
        self.iterations = 0

    @property
    def done(self):
        return not self.active or self.iterations >= self.steps

    def dampings(self):
        return [1.0 / self.radii[k] for k in self.active]

    def advance(self, graphs, results):
        still = []
        for k, (cand, l0, l1, ok) in zip(self.active, results):
            if ok and l1 <= l0:
                graphs[k].nodes = cand
                self.radii[k] = min(self.radii[k] * 2.0, 1e32)
            else:  # rejected step: keep the nodes, shrink the trust region
                self.radii[k] = max(self.radii[k] * 0.5, 1e-32)
                l1 = l0
            self.losses[k].append(l1)
            self.stall[k] = self.stall[k] + 1 if (l0 - l1) < self.decreasing else 0
            if self.stall[k] < self.patience:
                still.append(k)
        self.active = still
        self.iterations += 1


def _lm_iterations(graphs, step, steps, patience, decreasing, radius):
    """slam.py:121-134 for each of `graphs` (_LMState).  step(active graph indices, their dampings) -> per active graph
    (candidate nodes, loss before, loss after, Cholesky ok).  Returns the loss histories."""
    state = _LMState(len(graphs), steps, patience, decreasing, radius)
    while not state.done:
        state.advance(graphs, step(state.active, state.dampings()))
    return state.losses


def _check_group(graphs, edges, poses, weights):
    if not len(graphs) == len(edges) == len(poses) == len(weights):
        raise ValueError("graphs, edges, poses and weights must have one entry per graph")
    if len({id(g) for g in graphs}) != len(graphs):
        raise ValueError("a PoseGraphOpt is named twice in the group")
    if graphs and len({g.nodes.device for g in graphs}) != 1:
        raise ValueError("every graph of a group must be on one device")
    for e, p, w in zip(edges, poses, weights):
        if p.shape[0] != e.shape[0] or w.shape[0] != e.shape[0]:
            raise ValueError("edges, poses and weight must have one row per edge")


class PoseGraphOpt:
    def __init__(self, nodes, to_optimize_idxs="all", route=None):
        """route: None picks the block-sparse route above _lib.PG_DENSE_MAX_OPT optimised nodes and the dense one
        otherwise; "sparse" always takes the block-sparse route; "dense" always takes the dense one and raises
        ValueError above its limit.  The routes' results agree to rounding, not bit for bit (different orderings)."""
        if route not in (None, "dense", "sparse"):
            raise ValueError("route must be None, 'dense' or 'sparse', not %r" % (route,))
        if not nodes.is_cuda:
            raise RuntimeError("vista_slam_b200.pose_graph runs only on CUDA tensors")
        self.nodes = nodes.detach().to(torch.float32).contiguous().clone()
        n = self.nodes.shape[0]
        if isinstance(to_optimize_idxs, str):
            to_optimize_idxs = torch.arange(n, device=nodes.device)
        self.idxs_opt = torch.as_tensor(to_optimize_idxs, device=nodes.device).long().contiguous()
        self._scratch = None
        self._info = torch.zeros(4, dtype=torch.float64, device=nodes.device)
        num_opt = self.idxs_opt.shape[0]
        if route == "dense" and num_opt > _lib.PG_DENSE_MAX_OPT:
            raise ValueError("route='dense' takes at most %d optimised nodes, not %d" % (_lib.PG_DENSE_MAX_OPT, num_opt))
        self.sparse = num_opt > _lib.PG_DENSE_MAX_OPT if route is None else route == "sparse"
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
            info = _read_info(self._info)  # the one host synchronisation of the iteration
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
        info = _read_info(self._info)  # the one host synchronisation of the iteration
        return out, float(info[0]), float(info[1]), float(info[2]), bool(info[3] > 0.5)

    @torch.no_grad()
    def optimize(self, edges, poses, weight, steps=20, patience=3, decreasing=1e-4, radius=1e4):
        """slam.py:121-134: LM(TrustRegion(radius=1e4), min=1e-6) driven by StopOnPlateau(steps=20, patience=3,
        decreasing=1e-4).  `weight` is [E, 7] (the diagonal of the reference's diag_embed).  Returns the loss history."""
        return PoseGraphOpt.optimize_group([self], [edges], [poses], [weight], steps=steps, patience=patience,
                                           decreasing=decreasing, radius=radius)[0]

    @staticmethod
    @torch.no_grad()
    def optimize_group(graphs, edges, poses, weights, steps=20, patience=3, decreasing=1e-4, radius=1e4):
        """optimize() on several graphs at once: graphs[k] with edges[k], poses[k], weights[k].  Leaves every graph
        exactly as its own optimize() would and returns each graph's loss history.  Per iteration, the dense-route
        graphs still running take one sta_pose_graph_lm_step_group launch sequence, the block-sparse-route ones one
        sta_pose_graph_lm_step_sparse_group launch sequence (per PG_GROUP_MAX graphs), and all their info rows come
        back with one read-back.  Refused with ValueError before any launch: lists of different lengths, graphs on
        different devices, one PoseGraphOpt named twice, and edges, poses and weights whose row counts disagree."""
        graphs = list(graphs)
        edges, poses, weights = list(edges), list(poses), list(weights)
        _check_group(graphs, edges, poses, weights)
        if not graphs:
            return []
        group = _Group(graphs, edges, poses, weights)

        def step(active, dampings):
            outs, info, at = group.launch(active, dampings)
            return _Group.results(_read_info(info), outs, at)  # the one host synchronisation of the iteration

        losses = [None] * len(graphs)
        for k, h in zip(group.order, _lm_iterations([graphs[k] for k in group.order], step, steps=steps,
                                                    patience=patience, decreasing=decreasing, radius=radius)):
            losses[k] = h
        return losses

    @torch.no_grad()
    def start(self, edges, poses, weight, steps=20, patience=3, decreasing=1e-4, radius=1e4):
        """optimize() without waiting for it: returns a PoseGraphRun that steps this graph on a side stream, one LM
        iteration per poll().  Same kernels, dampings and accept / plateau decisions as optimize(), so the nodes and the
        loss history it ends with are optimize()'s, bit for bit.  The row-count refusal of optimize_group applies.
        A group of one (start_group)."""
        return PoseGraphRun([self], [edges], [poses], [weight], steps, patience, decreasing, radius, single=True)

    @staticmethod
    @torch.no_grad()
    def start_group(graphs, edges, poses, weights, steps=20, patience=3, decreasing=1e-4, radius=1e4):
        """optimize_group() without waiting for it: returns a PoseGraphRun that steps every graph on one side stream,
        one LM iteration of the group per poll(), with one _Group launch and one pinned copy of the info rows per
        iteration.  Each graph ends with optimize_group's nodes and loss history, bit for bit, dense, block-sparse or
        mixed.  The run's losses are the per-graph histories; graph_losses(k) and graph_done(k) report graph k while it
        runs.  optimize_group's refusals apply, before any launch."""
        return PoseGraphRun(graphs, edges, poses, weights, steps, patience, decreasing, radius)


class _Group:
    """optimize_group's LM step over a fixed list of graphs, dense-route graphs first (`order`): one info table (the
    dense group's rows first, compact over its active graphs, then one row per sparse graph).  launch(active, dampings)
    enqueues one step of the active positions in `order` and returns (their candidate nodes, the info rows to read
    back, the row of each); results() turns the host copy of those rows into the step's results."""

    def __init__(self, graphs, edges, poses, weights):
        dense = [k for k, g in enumerate(graphs) if not g.sparse]
        sparse = [k for k, g in enumerate(graphs) if g.sparse]
        self.nd = len(dense)
        self.order = dense + sparse
        self.info = torch.empty(len(graphs), 4, dtype=torch.float64, device=graphs[0].nodes.device)
        pick = lambda ks, a: [a[k] for k in ks]
        self.dg = _DenseGroup(pick(dense, graphs), pick(dense, edges), pick(dense, poses), pick(dense, weights),
                              info=self.info[:self.nd]) if dense else None
        self.sg = _SparseGroup(pick(sparse, graphs), pick(sparse, edges), pick(sparse, poses), pick(sparse, weights),
                               info=self.info[self.nd:]) if sparse else None

    def launch(self, active, dampings):  # positions in dense + sparse, ascending: the dense ones come first
        nd = self.nd
        da = [(t, d) for t, d in zip(active, dampings) if t < nd]
        sa = [(t - nd, d) for t, d in zip(active, dampings) if t >= nd]
        outs = self.dg.launch([t for t, _ in da], [d for _, d in da]) if da else []
        outs += self.sg.launch([m for m, _ in sa], [d for _, d in sa]) if sa else []
        at = list(range(len(da))) + [nd + m for m, _ in sa]
        return outs, (self.info if sa else self.info[:len(da)]), at

    @staticmethod
    def results(rows, outs, at):
        return [(out, float(rows[r][0]), float(rows[r][1]), bool(rows[r][3] > 0.5)) for out, r in zip(outs, at)]


class PoseGraphRun:
    """PoseGraphOpt.optimize() (start) or optimize_group() (start_group) in the background: each LM iteration of the
    group is enqueued on a non-blocking side stream, its info rows copied into pinned host memory and an event recorded.
    poll() never waits: when the event has completed it takes the iteration's accept / reject decisions and enqueues
    the next one.  wait() waits on that event until the run is done.

    Streams: the side stream starts after the work already queued on the stream that was current at start() (the
    "main" stream, which holds the PoseGraphOpts' snapshots of the nodes); the main-stream tensors the run reads are
    recorded on the side stream.  Once done, the main stream is ordered after the run, so every graph's nodes can be
    read there.  Block-sparse plans are built at the start, on the main stream.  Nothing here synchronises the
    device."""

    def __init__(self, graphs, edges, poses, weights, steps, patience, decreasing, radius, single=False):
        graphs, edges, poses, weights = list(graphs), list(edges), list(poses), list(weights)
        _check_group(graphs, edges, poses, weights)
        if not graphs:
            raise ValueError("a background run needs at least one graph")
        dev = graphs[0].nodes.device
        self.graphs, self._single = graphs, single
        self.main = torch.cuda.current_stream(dev)
        for g, e in zip(graphs, edges):
            if g.sparse:
                g.plan(e)  # its one edge-table copy waits only on the main stream's queued work
        self.stream = torch.cuda.Stream(dev)
        self.stream.wait_stream(self.main)
        for g, e, p, w in zip(graphs, edges, poses, weights):
            for t in (g.nodes, g.idxs_opt, e, p, w):
                t.record_stream(self.stream)  # no-op for memory the caching allocator does not own (the SLAM tables)
        self.state = _LMState(len(graphs), steps, patience, decreasing, radius)
        self.pinned = torch.empty(len(graphs), 4, dtype=torch.float64, pin_memory=True)
        self.event = torch.cuda.Event()
        with torch.cuda.stream(self.stream):
            self.group = _Group(graphs, edges, poses, weights)
        self.order = self.group.order  # the state machine runs over the graphs in this order, as optimize_group's
        self._at = {k: t for t, k in enumerate(self.order)}
        self._ordered = [graphs[k] for k in self.order]
        self._launch()

    @property
    def done(self):
        return self.state.done

    @property
    def losses(self):
        """The loss histories so far: once done, optimize()'s return value for a run of start(), optimize_group()'s
        for a run of start_group()."""
        if self._single:
            return self.state.losses[0]
        return [self.graph_losses(k) for k in range(len(self.graphs))]

    def graph_losses(self, k):
        """Graph k's loss history so far."""
        return self.state.losses[self._at[k]]

    def graph_done(self, k):
        """Whether graph k has left the group (its nodes are final once the run is done)."""
        return self.state.done or self._at[k] not in self.state.active

    def _launch(self):
        if self.state.done:
            self.main.wait_stream(self.stream)
            for g in self.graphs:
                g.nodes.record_stream(self.main)
            self.group = self._pending = None
            return
        with torch.cuda.stream(self.stream):
            outs, info, at = self.group.launch(self.state.active, self.state.dampings())
            self.pinned[:info.shape[0]].copy_(info, non_blocking=True)
            self.event.record(self.stream)
        self._pending = (outs, info.shape[0], at)

    @torch.no_grad()
    def poll(self):
        """Take the iteration in flight if it has finished, and enqueue the next; never waits.  Returns done."""
        if self.state.done:
            return True
        if not self.event.query():
            return False
        outs, rows, at = self._pending
        self.state.advance(self._ordered, _Group.results(self.pinned[:rows], outs, at))
        self._launch()
        return self.state.done

    def wait(self):
        """Run to the end, waiting on each iteration's event.  Returns the loss histories (losses)."""
        while not self.poll():
            self.event.synchronize()
        return self.losses


class _DenseGroup:
    """The dense-route LM step over a fixed list of graphs, of which any subset steps together: one scratch buffer and
    one info table for the whole group, inputs converted once."""

    def __init__(self, graphs, edges, poses, weights, dmin=1e-6, dmax=1e32, info=None):
        self.graphs = graphs
        self.edges = [e.to(torch.int64).contiguous() for e in edges]
        self.poses = [p.to(torch.float32).contiguous() for p in poses]
        self.weights = [w.to(torch.float32).contiguous() for w in weights]
        self.dmin, self.dmax = dmin, dmax
        self.device = graphs[0].nodes.device
        self.info = torch.empty(len(graphs), 4, dtype=torch.float64, device=self.device) if info is None else info
        self.scratch = None
        self.L = _lib.lib()

    def _table(self, members, dampings, outs):
        tab = (_lib.StaPgGraph * len(members))()
        for t, (k, damping, out) in enumerate(zip(members, dampings, outs)):
            g = self.graphs[k]
            tab[t] = _lib.StaPgGraph(g.nodes.data_ptr(), self.edges[k].data_ptr(), self.poses[k].data_ptr(),
                                     self.weights[k].data_ptr(), g.idxs_opt.data_ptr(), out.data_ptr(), g.nodes.shape[0],
                                     self.edges[k].shape[0], g.idxs_opt.shape[0], float(damping))
        return tab

    def step(self, members, dampings):
        """One LM step of graphs[members] (at most PG_GROUP_MAX per launch sequence) -> per member (candidate nodes,
        loss before, loss after, Cholesky ok); one info read-back in all."""
        outs = self.launch(members, dampings)
        info = _read_info(self.info[:len(members)])  # the one host synchronisation of the iteration
        return [(out, float(r[0]), float(r[1]), bool(r[3] > 0.5)) for out, r in zip(outs, info)]

    def launch(self, members, dampings):
        """Enqueue one LM step of graphs[members] -> their candidate nodes; info rows at self.info[:len(members)]."""
        outs = [torch.empty_like(self.graphs[k].nodes) for k in members]
        rows = len(members)
        with torch.cuda.device(self.device):
            for c0 in range(0, rows, _lib.PG_GROUP_MAX):
                c1 = min(rows, c0 + _lib.PG_GROUP_MAX)
                tab = self._table(members[c0:c1], dampings[c0:c1], outs[c0:c1])
                need = int(self.L.sta_pose_graph_group_scratch_bytes(tab, c1 - c0))  # 0: the step refuses the table
                if need and (self.scratch is None or self.scratch.numel() * 8 < need):
                    self.scratch = torch.empty((need + 7) // 8, dtype=torch.float64, device=self.device)
                _lib.check(self.L.sta_pose_graph_lm_step_group(tab, c1 - c0, self.dmin, self.dmax,
                                                               _lib.ptr(self.info[c0:c1]), _lib.ptr(self.scratch), need,
                                                               _lib.cur_stream()), "sta_pose_graph_lm_step_group")
        return outs


class _SparseGroup:
    """The block-sparse-route LM step over a fixed list of graphs, of which any subset steps together: each graph's
    plan (PoseGraphOpt.plan), one group plan over them per PG_GROUP_MAX graphs, and one info row per graph.  A single
    graph takes sta_pose_graph_lm_step_sparse, as PoseGraphOpt.lm_step does."""

    def __init__(self, graphs, edges, poses, weights, dmin=1e-6, dmax=1e32, info=None):
        self.graphs = graphs
        self.plans = [g.plan(e) for g, e in zip(graphs, edges)]  # held here: the group plans borrow them
        self.poses = [p.to(torch.float32).contiguous() for p in poses]
        self.weights = [w.to(torch.float32).contiguous() for w in weights]
        self.dmin, self.dmax = dmin, dmax
        self.device = graphs[0].nodes.device
        self.info = torch.empty(len(graphs), 4, dtype=torch.float64, device=self.device) if info is None else info
        self.L = _lib.lib()
        self._destroy = self.L.sta_pg_group_plan_destroy
        self.chunks = []  # (first graph, end, group plan)
        if len(graphs) > 1:
            with torch.cuda.device(self.device):
                for c0 in range(0, len(graphs), _lib.PG_GROUP_MAX):
                    c1 = min(len(graphs), c0 + _lib.PG_GROUP_MAX)
                    h = ctypes.c_void_p()
                    tab = (ctypes.c_void_p * (c1 - c0))(*[p.h for p in self.plans[c0:c1]])
                    _lib.check(self.L.sta_pg_group_plan_create(tab, c1 - c0, ctypes.byref(h)), "sta_pg_group_plan_create")
                    self.chunks.append((c0, c1, h))

    def plan_info(self):
        """{"G", "levels", "launches", "device_bytes"} of each group plan."""
        out = []
        for _, _, h in self.chunks:
            v = (ctypes.c_int64 * 4)()
            _lib.check(self.L.sta_pg_group_plan_info(h, v), "sta_pg_group_plan_info")
            out.append(dict(zip(("G", "levels", "launches", "device_bytes"), map(int, v))))
        return out

    def launch(self, members, dampings):
        """Enqueue one LM step of graphs[members] -> their candidate nodes; graph k's info row at self.info[k]."""
        outs = [torch.empty_like(self.graphs[k].nodes) for k in members]
        damp = dict(zip(members, dampings))
        out_of = dict(zip(members, outs))
        with torch.cuda.device(self.device):
            if not self.chunks:  # one graph
                g = self.graphs[0]
                _lib.check(self.L.sta_pose_graph_lm_step_sparse(self.plans[0].h, _lib.ptr(g.nodes), _lib.ptr(self.poses[0]),
                                                                _lib.ptr(self.weights[0]), float(damp[0]), self.dmin,
                                                                self.dmax, _lib.ptr(outs[0]), _lib.ptr(self.info[0]),
                                                                _lib.cur_stream()), "sta_pose_graph_lm_step_sparse")
                return outs
            for c0, c1, h in self.chunks:
                if not any(c0 <= k < c1 for k in members):
                    continue
                steps = (_lib.StaPgSparseStep * (c1 - c0))()
                for k in range(c0, c1):
                    if k in damp:
                        steps[k - c0] = _lib.StaPgSparseStep(self.graphs[k].nodes.data_ptr(), self.poses[k].data_ptr(),
                                                             self.weights[k].data_ptr(), out_of[k].data_ptr(),
                                                             float(damp[k]), 1)
                _lib.check(self.L.sta_pose_graph_lm_step_sparse_group(h, steps, self.dmin, self.dmax,
                                                                      _lib.ptr(self.info[c0:c1]), _lib.cur_stream()),
                           "sta_pose_graph_lm_step_sparse_group")
        return outs

    def step(self, members, dampings):
        """One LM step of graphs[members] -> per member (candidate nodes, loss before, loss after, Cholesky ok); one
        info read-back in all."""
        outs = self.launch(members, dampings)
        info = _read_info(self.info)  # the one host synchronisation of the iteration
        return [(out, float(info[k][0]), float(info[k][1]), bool(info[k][3] > 0.5)) for k, out in zip(members, outs)]

    def __del__(self):
        for _, _, h in getattr(self, "chunks", []):
            self._destroy(h)
        self.chunks = []
