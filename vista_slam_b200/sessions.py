"""Several OnlineSLAM sessions stepped together on one GPU, sharing one STA frontend and one loop-closure vocabulary.

An evaluation that runs a list of scenes, or a server that runs SLAM for several cameras, holds one session per
sequence.  On its own, each OnlineSLAM loads its own copy of the checkpoint and of the vocabulary, and a keyframe at a
time leaves most of the GPU idle.  `SLAMSessions` loads both once, and `step({k: [value, ...], ...})` runs the new
keyframes of every named session through one batched frontend pass:

  * one sequence of encoder calls over all new views (keyframe.add_views_group);
  * one loop-detection pass over all their frames with one read-back (loop_detector.detect_loops_group);
  * the gated edge regression in chunks of at most 16 edges that mix sessions, one read-back per chunk
    (keyframe.regress_keyframes_gated_group).

Graph insertion runs once per edge chunk for all sessions (one sta_graph_add_keyframes), and step's PGOs per session,
in the order step_many would run them.  The keyframe loop is slam.step_keyframes, which OnlineSLAM.step_many runs over
one session; this class adds the group hooks (detection and regression across sessions, due background PGOs started
together at the end of the call).  `optimize(ks)` runs the PGO of the named sessions now, together: one
PoseGraphOpt.optimize_group, whose LM iterations step every session's graph with one launch sequence and one
read-back; `optimize(ks, background=True)` starts the same group on a side stream and returns (INTEGRATION.md §5).
`track({k: [value, ...]})` gives frames that are not keyframes a pose against
a keyframe of their session, all sessions' frames through one encode and one regression pass (OnlineSLAM.track).
With pgo_every beyond the sequence length, an evaluation over a scene list ends with one
`optimize(range(len(scenes)))`, and a live server runs `optimize` on the sessions that are due.  A call leaves every
session as `for k in sorted(values): sessions[k].step_many(values[k], force_pgo=k in force_pgo, ...)` would: the
graph tables, host bookkeeping, loop candidates, gate decisions, PGO calls, written files and returned flags.  Frontend floats may
differ from that loop within rounding, as step_many's differ from step's, because batch sizes change the GEMMs' split-K.

Timing: each session's time_dict gets its share of the batched phases.  The wall time of the encoder calls and of the
loop detection is split evenly across the sessions that have keyframes in the call; the time of an edge chunk's
regression is split evenly across the sessions with keyframes in that chunk (added to their "decoder" and
"graph_construction" buckets, as step_many counts the decoder inside graph construction).  Preparation, graph insertion
and step's PGO are timed per session; the wall time of an optimize call is split evenly across its sessions ("pgo").

All sessions run on the current CUDA device and stream.  The class is not thread-safe."""
import operator
import time

import torch

from .keyframe import regress_keyframes_gated_group
from .loop_detector import Vocabulary, detect_loops_group
from .pose_graph import PoseGraphOpt
from .slam import OnlineSLAM, _share, step_keyframes, track_frames


class _Batch:
    """PGO problems (PoseGraphOpt, (edges, measurements, weights)) of several sessions, started together as one
    PoseGraphOpt.start_group run."""

    def __init__(self):
        self.problems, self.run = [], None

    def start(self):
        if self.run is None:
            graphs, args = [g for g, _ in self.problems], [a for _, a in self.problems]
            self.run = PoseGraphOpt.start_group(graphs, *[[a[i] for a in args] for i in range(3)])
        return self.run


class _SessionRun:
    """A session's handle on a shared background run (OnlineSLAM._pgo_run[0]): poll() is True once the whole run is
    done and never waits or starts it; wait() starts the run if it has not started, then waits for it."""

    def __init__(self, batch):
        self.batch = batch

    @property
    def stream(self):
        return self.batch.start().stream

    def poll(self):
        return self.batch.run is not None and self.batch.run.poll()

    def wait(self):
        self.batch.start().wait()


class _CallGroup:
    """The background PGOs that fall due during one SLAMSessions.step call: captured at their keyframes (add), then
    started as one run at the end of the call (start).  Waiting on a captured run starts the group at that point;
    PGOs captured after that go into a new group."""

    def __init__(self):
        self.batches = [_Batch()]

    def add(self, graph, args):
        if self.batches[-1].run is not None:
            self.batches.append(_Batch())
        self.batches[-1].problems.append((graph, args))
        return _SessionRun(self.batches[-1])

    def start(self):
        for b in self.batches:
            if b.problems:
                b.start()


class SLAMSessions:
    def __init__(self, ckpt_path, vocab_path, num_sessions, frontend=None, **online_slam_kwargs):
        """num_sessions OnlineSLAM sessions built with online_slam_kwargs.  The checkpoint at ckpt_path is loaded once,
        or `frontend`, an already-built STA (e.g. STA(precision="fp8") with its weights loaded), is used instead.  The
        vocabulary at vocab_path (or a loaded Vocabulary) is parsed and uploaded once; every session's LoopDetector
        uses it."""
        n = operator.index(num_sessions)
        if n < 1:
            raise ValueError("num_sessions must be at least 1")
        self.vocab = vocab_path if isinstance(vocab_path, Vocabulary) else Vocabulary(vocab_path)
        self.sessions = []
        for _ in range(n):
            model = frontend if frontend is not None else (self.sessions[0].frontend if self.sessions else ckpt_path)
            self.sessions.append(self._new_session(model, online_slam_kwargs))
        self.frontend = self.sessions[0].frontend

    def _new_session(self, frontend, kwargs):
        """One session on the shared frontend (a model or, for the first session, the checkpoint path)."""
        return OnlineSLAM(frontend, self.vocab, **kwargs)

    def __len__(self):
        return len(self.sessions)

    def __getitem__(self, k):
        return self.sessions[k]

    def _index(self, k):
        try:
            k = operator.index(k)
        except TypeError:
            raise ValueError("unknown session index %r" % (k,)) from None
        if not 0 <= k < len(self.sessions):
            raise ValueError("unknown session index %d (there are %d sessions)" % (k, len(self.sessions)))
        return k

    def _calls(self, values):
        """[(k, [value, ...]), ...] sorted by session from a mapping or a sequence of (k, values) pairs."""
        pairs = list(values.items()) if hasattr(values, "items") else [tuple(p) for p in values]
        calls, seen = [], set()
        for k, vs in pairs:
            k = self._index(k)
            if k in seen:
                raise ValueError("session %d is named twice" % k)
            seen.add(k)
            calls.append((k, list(vs)))
        return sorted(calls, key=lambda c: c[0])

    def _detect_loops(self, sessions, grays, fars):
        """Loop candidates of the sessions' new frames, per session: one detect_loops_group (one read-back)."""
        return detect_loops_group([s.lc_detector for s in sessions], grays, fars)

    def _regress_keyframes(self, items):
        """The gated regression of items = [(session, i, js), ...] in edge chunks that mix sessions: per item in order,
        what OnlineSLAM._regress_keyframes yields."""
        return regress_keyframes_gated_group([(s.kf, i, js) for s, i, js in items], self.sessions[0].rel_pose_thres)

    def step(self, values, force_pgo=(), log_intermediate_results=False, output_folders=None):
        """Step sessions through new keyframes: values = {k: [value, ...], ...} (or (k, [value, ...]) pairs) names any
        subset of the sessions; force_pgo holds the sessions whose last keyframe of the call forces a PGO;
        output_folders = {k: folder} for log_intermediate_results.  Returns {k: [is_optimized, ...]}.

        Refused with ValueError before any launch, with no session changed: an unknown or repeated session index,
        keyframes of different sizes within the call, or a size other than a session's existing views.  A capacity
        IndexError in one session propagates; every session is then left as a prefix of its own step_many would leave
        it (the encoder caches and loop databases may hold later views of the call).  A non-orthonormal rotation
        raises ValueError by the end of the call.

        Host synchronisations: one for the loop candidates of all sessions, one per edge chunk, one per PGO iteration,
        and one at the end of the call unless every session's flag has been read since its last graph launch.  The
        kept edges of each edge chunk, of every session, go into the graphs with one sta_graph_add_keyframes.  The
        PGOs of sessions with pgo_background that fall due during the call are captured at their keyframes and started
        as one PoseGraphOpt.start_group run at the end of the call (a session due again within the call waits for its
        run, which starts the group then).  Each session of the call is polled before its first keyframe, and every
        session with a pending PGO after each keyframe (slam.step_keyframes, the loop step_many runs)."""
        calls = self._calls(values)
        force = {self._index(k) for k in force_pgo}
        folders = [output_folders.get(k) if output_folders else None for k, _ in calls]
        flags = step_keyframes([(self.sessions[k], vs) for k, vs in calls], [k in force for k, _ in calls],
                               log_intermediate_results, folders, detect=self._detect_loops,
                               regress=self._regress_keyframes, group=_CallGroup(), polled=self.sessions)
        return {k: f for (k, _), f in zip(calls, flags)}

    def optimize(self, ks, background=False):
        """Optimise the pose graphs of sessions ks now, together.  Leaves each session as sessions[k].pose_graph_optimize()
        would: the same optimised node set (the window and the loop-related views), the same poses bit for bit,
        loop_related_views cleared and the same messages (every session's opening messages, then the optimisation,
        then every session's closing message); a session without nodes or edges only prints them.  An unknown or
        repeated index raises ValueError before anything runs.  Host synchronisations: one per LM iteration of the
        group, whichever route each session's graph takes (OnlineSLAM.pgo_route).  A pending background PGO of a named
        session is folded first (OnlineSLAM.wait_pgo).

        background=True does the same up to the optimisation -- folds, opening messages, optimised sets,
        loop_related_views cleared -- then starts one PoseGraphOpt.start_group run over the named sessions' graphs on
        a side stream and returns.  Each of those sessions then has a pending PGO (OnlineSLAM.pgo_pending), which its
        polls fold as they fold its own background PGOs (INTEGRATION.md §5): afterwards it equals optimize(ks) bit
        for bit.  A session without nodes or edges prints its closing message now."""
        order, seen = [], set()
        for k in ks:
            k = self._index(k)
            if k in seen:
                raise ValueError("session %d is named twice" % k)
            seen.add(k)
            order.append(k)
        if not order:
            return
        sess = [self.sessions[k] for k in order]
        for s in sess:
            s.wait_pgo()
        t = time.time()
        problems = [s._pgo_begin() for s in sess]
        if background:
            batch = _Batch()
            for s, p in zip(sess, problems):
                s.loop_related_views = set()
                if p is None:
                    s._pgo_end(None)
                else:
                    batch.problems.append(p)
                    s._pgo_run = (_SessionRun(batch), p, [])
            if batch.problems:
                batch.start()
            _share(sess, "pgo", time.time() - t)
            return
        run = [p for p in problems if p is not None]
        if run:
            PoseGraphOpt.optimize_group([g for g, _ in run], *[[a[i] for _, a in run] for i in range(3)])
        for s, p in zip(sess, problems):
            s._pgo_end(p)
        _share(sess, "pgo", time.time() - t)
        torch.cuda.empty_cache()

    def track(self, values, kfs=None):
        """Track frames in several sessions at once: values = {k: [value, ...], ...} (or (k, [value, ...]) pairs) names
        any subset of the sessions, kfs = {k: keyframe view} (default: each session's last stepped view).  One
        transient encode of all frames, one regression whose edge chunks mix sessions, one sta_graph_track_frames per
        session (slam.track_frames).  Returns {k: result of OnlineSLAM.track}.  Refused with ValueError before any
        launch, with no session changed: an unknown or repeated session, a kfs entry for a session not in values,
        frames of different sizes within the call, and every refusal of OnlineSLAM.track."""
        calls = self._calls(values)
        kfs = {} if kfs is None else {self._index(k): kf for k, kf in (kfs.items() if hasattr(kfs, "items") else kfs)}
        if set(kfs) - {k for k, _ in calls}:
            raise ValueError("kfs names sessions that track no frames: %s" % sorted(set(kfs) - {k for k, _ in calls}))
        res = track_frames([(self.sessions[k], vs, kfs.get(k)) for k, vs in calls])
        return {k: r for (k, _), r in zip(calls, res)}
