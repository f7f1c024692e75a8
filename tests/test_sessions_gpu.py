"""GPU: SLAMSessions (vista_slam_b200/sessions.py) and the group loop detection under it.

  * detect_loops_group over three detectors on one vocabulary is bit-identical to each detector's own detect_loop:
    candidates, similarities, stored vectors and None vectors, whatever frames each detector brings to a call;
  * with the frontend and loops replayed from oracle streams, a group call leaves every session exactly as
    `for k in sorted(values): sessions[k].step_many(values[k], ...)` on an independent OnlineSLAM would: graph tables,
    host bookkeeping, PGO calls, flags and written files, bit for bit;
  * with the real frontend the batch sizes change the GEMMs' split-K, so frontend outputs are held to the bounds of
    test_slam_batch_gpu.py's real-frontend test (pose 1e-2, pose confidence 4e-3, maps 4e-2, max-normalised), gate
    decisions at thresholds more than 4e-3 from every confidence;
  * one session at one keyframe per call launches what OnlineSLAM.step launches: every device table bit for bit."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import loop_detector_oracle as O
from oracle import slam_oracle as so
from test_slam_batch_gpu import _LoopsMany, _assert_same_state, _files, _real_slam, _state, maxn
from test_slam_gpu import CFG, VOCAB, _batch, _Frontend, _value

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ group loop detection
def _loop_frames():
    g = np.load(os.path.join(GOLDEN_DIR, "loop.npz"))
    seed, n, H, W = json.loads(str(g["meta"]))["sequences"][0]
    frames = O.make_sequence(seed, n, H, W)
    flat = np.full((H, W), 77, np.uint8)  # no keypoint: a None vector
    # each list comes back to earlier views (the sequence revisits its start after 44 frames)
    return [frames, frames[30:] + [flat] + frames[:12], frames[::2]]


LOOP_ARGS = [(40, 40, 5), (6, 2, 3), (10, 4, 5)]
# frames per detector per call: 0, 1 or several, until every detector has run out
SCHEDULE = [(1, 0, 3), (5, 1, 0), (0, 0, 1), (1, 1, 1), (7, 9, 2), (0, 4, 0), (2, 0, 6)]


def test_group_loop_detection_equals_per_detector():
    from vista_slam_b200.loop_detector import LoopDetector, Vocabulary, detect_loops_group
    frames = _loop_frames()
    vocab = Vocabulary(VOCAB)
    seq = [LoopDetector(VOCAB, *a) for a in LOOP_ARGS]
    want = [[s.detect_loop(f, max(0, t - 3)) for t, f in enumerate(fr)] for s, fr in zip(seq, frames)]
    grp = [LoopDetector(vocab, *a) for a in LOOP_ARGS]
    got = [[] for _ in grp]
    at, c = [0, 0, 0], 0
    while any(a < len(fr) for a, fr in zip(at, frames)):
        counts = SCHEDULE[c % len(SCHEDULE)]
        c += 1
        ims = [fr[a:a + m] for fr, a, m in zip(frames, at, counts)]
        fars = [[max(0, a + t - 3) for t in range(len(x))] for a, x in zip(at, ims)]
        for k, r in enumerate(detect_loops_group(grp, ims, fars)):
            assert len(r) == len(ims[k])
            got[k] += r
        at = [a + len(x) for a, x in zip(at, ims)]
    assert c > len(SCHEDULE)
    assert sum(len(x) for w in want for x in w) > 5  # the comparison sees candidates
    for k in range(3):
        assert got[k] == want[k], k
        assert len(grp[k].bow_feats) == len(frames[k])
        for t in range(len(frames[k])):
            assert (grp[k].bow_feats[t] is None) == (seq[k].bow_feats[t] is None), (k, t)
            for a, b in zip(grp[k]._view_vector(t), seq[k]._view_vector(t)):
                np.testing.assert_array_equal(a, b)
    assert grp[1].bow_feats[24] is None
    # a detector's own calls after group calls continue its database exactly
    extra = frames[0][:3]
    for t, f in enumerate(extra):
        i = len(frames[0]) + t
        assert grp[0].detect_loop(f, i - 3) == seq[0].detect_loop(f, i - 3)
        np.testing.assert_array_equal(grp[0].similarities(), seq[0].similarities())


def test_group_loop_refusals():
    from vista_slam_b200 import _lib
    from vista_slam_b200.loop_detector import LoopDetector, Vocabulary, detect_loops_group
    frames = _loop_frames()[0]
    vocab = Vocabulary(VOCAB)
    a, b = LoopDetector(vocab, 4, 3, 5), LoopDetector(vocab, 4, 3, 5)
    detect_loops_group([a, b], [frames[:3], frames[3:5]], [[0, 0, 0], [0, 0]])
    L = _lib.lib()

    def views():
        return [(L.sta_loop_views(d._h), len(d.bow_feats), [d._view_vector(t)[0].tolist() for t in range(len(d.bow_feats))])
                for d in (a, b)]

    before = views()
    other = LoopDetector(VOCAB, 4, 3, 5)
    with pytest.raises(ValueError, match="one Vocabulary"):
        detect_loops_group([a, other], [frames[:1], frames[:1]], [[0], [0]])
    small = torch.from_numpy(np.ascontiguousarray(frames[0][:64, :96])).cuda()
    with pytest.raises(ValueError, match="same size"):
        detect_loops_group([a, b], [frames[:1], [small]], [[0], [0]])
    with pytest.raises(ValueError, match="farthest"):
        detect_loops_group([a, b], [frames[:1], frames[:1]], [[0], [3]])
    with pytest.raises(ValueError, match="twice"):
        detect_loops_group([a, a], [frames[:1], frames[:1]], [[0], [0]])
    assert views() == before and L.sta_loop_views(other._h) == 0
    # the C entry points refuse before any launch too
    f = torch.from_numpy(np.stack(frames[:2])).cuda()
    st = _lib.cur_stream()

    def dets(*ds):
        return (ctypes.c_void_p * len(ds))(*[d._h.value for d in ds])

    assert L.sta_loop_add_frames_group(dets(a, other), 2, _lib.ptr(f), 0, *f.shape[1:], st) != 0
    assert b"vocabulary" in L.sta_last_error()
    f3 = torch.from_numpy(np.stack(frames[:3])).cuda()
    assert L.sta_loop_add_frames_group(dets(a, b, a), 3, _lib.ptr(f3), 0, *f3.shape[1:], st) != 0
    assert b"consecutive" in L.sta_last_error()
    assert views() == before
    # a detect with an out-of-range farthest neighbour, or other detectors than the last group add's, is refused
    assert L.sta_loop_add_frames_group(dets(a, b), 2, _lib.ptr(f), 0, *f.shape[1:], st) == 0
    n = (ctypes.c_int * 4)()
    assert L.sta_loop_detect_group(dets(a, b), 2, (ctypes.c_int * 2)(0, 7), n, None, None, 0, st) != 0
    assert b"farthest" in L.sta_last_error()
    assert L.sta_loop_detect_group(dets(b, a), 2, (ctypes.c_int * 2)(0, 0), n, None, None, 0, st) != 0
    assert L.sta_loop_detect_group(dets(a, b), 2, (ctypes.c_int * 2)(0, 0), n, None, None, 0, st) == 0
    a.bow_feats.append(None)
    b.bow_feats.append(None)
    # similarities after a group detect: refused until the detector's own next detect
    with pytest.raises(RuntimeError, match="group detect"):
        a.similarities()
    a.detect_loop(frames[7], 0)
    assert len(a.similarities()) == 4


# ------------------------------------------------------------------------------------------------ replayed frontend
def _replay_session(stream, frontend, vocab, kwargs):
    from vista_slam_b200.slam import OnlineSLAM

    class ReplaySLAM(OnlineSLAM):
        def _regress_keyframe(self, i, js):
            return _batch(stream, i, js, self.rel_pose_thres)

        def _regress_keyframes(self, items):
            return [_batch(stream, i, js, self.rel_pose_thres) if js else None for i, js in items]

    slam = ReplaySLAM(frontend, vocab, **kwargs)
    slam.lc_detector = _LoopsMany(stream["loops"], kwargs["loop_dist_min"])
    slam.stream = stream
    return slam


def _replay_sessions(streams, **over):
    from vista_slam_b200.sessions import SLAMSessions

    class ReplaySessions(SLAMSessions):
        def _new_session(self, frontend, kwargs):
            return _replay_session(streams[len(self.sessions)], frontend, self.vocab, kwargs)

        def _detect_loops(self, sessions, grays, fars):
            return [s.lc_detector.detect_loops(g, f) for s, g, f in zip(sessions, grays, fars)]

        def _regress_keyframes(self, items):
            return [_batch(s.stream, i, js, s.rel_pose_thres) if js else None for s, i, js in items]

    c = dict(CFG, verbose=True)
    c.update(over)
    return ReplaySessions("unused", VOCAB, len(streams), frontend=_Frontend(), **c)


def _record_pgo(monkeypatch):
    """PGO calls as (session tag, [node set, input poses, result poses])."""
    import vista_slam_b200.slam as S
    calls, cur = [], [None]

    class RecordingPGO(S.PoseGraphOpt):
        def optimize(self, edges, poses, weight, **kw):
            rec = [self.idxs_opt.cpu().numpy(), self.nodes.cpu().numpy()]
            out = super().optimize(edges, poses, weight, **kw)
            calls.append((cur[0], rec + [self.nodes.cpu().numpy()]))
            return out

    orig = S.OnlineSLAM.pose_graph_optimize

    def pgo(self):
        cur[0] = getattr(self, "tag", None)
        return orig(self)

    monkeypatch.setattr(S, "PoseGraphOpt", RecordingPGO)
    monkeypatch.setattr(S.OnlineSLAM, "pose_graph_optimize", pgo)
    return calls


def _streams():
    return [so.make_stream(seed=3, n_views=20), so.make_stream(seed=8, n_views=14), so.make_stream(seed=21, n_views=23)]


def _plan(shape, lengths):
    """Per call {k: number of keyframes} until every session has run out."""
    if shape == "all":
        return [{k: n for k, n in enumerate(lengths)}]
    pattern = {"ones": [(1, 1, 1)], "uneven": [(3, 0, 5), (0, 2, 1), (7, 7, 0), (1, 0, 0), (0, 1, 9)]}[shape]
    plan, at, c = [], [0] * len(lengths), 0
    while any(a < n for a, n in zip(at, lengths)):
        counts = pattern[c % len(pattern)]
        c += 1
        call = {k: min(m, n - a) for k, (m, a, n) in enumerate(zip(counts, at, lengths)) if m and a < n}
        if shape == "uneven" and c % 3 == 0:
            call[1] = call.get(1, 0)  # an idle session named with an empty list
        plan.append(call)
        at = [a + call.get(k, 0) for k, a in enumerate(at)]
    return plan


@pytest.mark.parametrize("shape", ["ones", "uneven", "all"])
def test_sessions_replay_equals_independent_step_many(shape, tmp_path, monkeypatch):
    streams = _streams()
    images = [so.stream_images(s) for s in streams]
    lengths = [s["n_views"] for s in streams]
    plan = _plan(shape, lengths)
    pgo = _record_pgo(monkeypatch)
    ses = _replay_sessions(streams)
    seq = [_replay_session(s, _Frontend(), VOCAB, dict(CFG, verbose=True)) for s in streams]
    for k in range(3):
        ses[k].tag, seq[k].tag = ("ses", k), ("seq", k)
    at = [0, 0, 0]
    flags_ses, flags_seq = [[] for _ in streams], [[] for _ in streams]
    for call in plan:
        values = {k: [_value(images[k], i, streams[k]) for i in range(at[k], at[k] + m)] for k, m in call.items()}
        force = {k for k, m in call.items() if m and at[k] + m == lengths[k]}
        out = ses.step(values, force_pgo=force, log_intermediate_results=True,
                       output_folders={k: str(tmp_path / "ses" / str(k)) for k in range(3)})
        assert sorted(out) == sorted(call)
        for k in sorted(values):
            flags_ses[k] += out[k]
            flags_seq[k] += seq[k].step_many(values[k], force_pgo=k in force, log_intermediate_results=True,
                                             output_folder=str(tmp_path / "seq" / str(k)))
            at[k] += call[k]
    assert at == lengths and flags_ses == flags_seq and all(any(f) for f in flags_ses)
    for k in range(3):
        _assert_same_state(_state(ses[k]), _state(seq[k]))
        mine = [r for t, r in pgo if t == ("ses", k)]
        ref = [r for t, r in pgo if t == ("seq", k)]
        assert len(mine) == len(ref) > 0
        for a, b in zip(mine, ref):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
        assert _files(tmp_path / "ses" / str(k)) == _files(tmp_path / "seq" / str(k))
        assert ses[k].lc_detector.calls == lengths[k]
        t = ses[k].get_time_dict()
        assert set(t) == set(seq[k].get_time_dict())


def test_sessions_refusals_and_overflow():
    streams = _streams()
    images = [so.stream_images(s) for s in streams]

    def vals(k, i0, n):
        return [_value(images[k], i, streams[k]) for i in range(i0, i0 + n)]

    def untouched(ses):
        return all(s.view_num == 0 and s.kf.view_num == 0 and s.lc_detector.calls == 0 and s._graph is None for s in ses)

    ses = _replay_sessions(streams)
    assert len(ses) == 3 and ses.step({}) == {} and ses.step({1: []}) == {1: []}
    for bad in ({3: vals(0, 0, 1)}, {-1: vals(0, 0, 1)}, {"0": vals(0, 0, 1)}, [(0, vals(0, 0, 1)), (0, vals(0, 1, 1))]):
        with pytest.raises(ValueError, match="session"):
            ses.step(bad)
    with pytest.raises(ValueError, match="session"):
        ses.step({0: vals(0, 0, 1)}, force_pgo={5})
    wide = dict(vals(1, 0, 1)[0], rgb=torch.zeros(1, 3, streams[1]["H"], streams[1]["W"] + 16, device="cuda"))
    with pytest.raises(ValueError, match="same image size"):
        ses.step({0: vals(0, 0, 2), 1: [wide]})
    assert untouched(ses)
    ses.step({0: vals(0, 0, 2)})
    with pytest.raises(ValueError, match="size of its views"):
        ses.step({1: [wide], 0: [dict(vals(0, 2, 1)[0], rgb=wide["rgb"])]})
    assert ses[0].view_num == 2 and ses[0].kf.view_num == 2 and untouched([ses[1], ses[2]])
    ses[0].reset()
    assert ses[0].view_num == 0 and ses[1].kf.frontend is ses[0].kf.frontend

    # capacity (max_view_num = 1: 9 nodes) overflows in session 1 only; every session is left as a prefix of its own
    # step_many would leave it
    ses = _replay_sessions(streams, max_view_num=1)
    counts = {0: 3, 1: 6, 2: 2}
    with pytest.raises(IndexError):
        ses.step({k: vals(k, 0, m) for k, m in counts.items()})
    ref0 = _replay_session(streams[0], _Frontend(), VOCAB, dict(CFG, verbose=True, max_view_num=1))
    ref0.step_many(vals(0, 0, 3))
    _assert_same_state(_state(ses[0]), _state(ref0))
    ref1 = _replay_session(streams[1], _Frontend(), VOCAB, dict(CFG, verbose=True, max_view_num=1))
    with pytest.raises(IndexError):
        ref1.step_many(vals(1, 0, 6))
    _assert_same_state(_state(ses[1]), _state(ref1))
    s2 = ses[2]
    assert (s2.view_num, s2.num_nodes, s2.num_edges, s2.view_names, s2.view_to_node) == (0, 0, 0, [], {})
    assert (s2._graph.node_to_view == -1).all()


# ------------------------------------------------------------------------------------------------ real frontend
def _frames(n, seed):
    g = torch.Generator().manual_seed(seed)
    H = W = 224
    base = torch.rand(1, 3, H // 8, W // 8, generator=g)
    out = []
    for i in range(n):
        img = torch.nn.functional.interpolate(base.roll(i, dims=3), size=(H, W), mode="bilinear") * 2 - 1
        img = (img + 0.05 * torch.rand(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        out.append({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                    "view_name": "%d" % i})
    return out


def _real_sessions(model, n, recorded, **kw):
    from vista_slam_b200.sessions import SLAMSessions

    class Run(SLAMSessions):
        def _regress_keyframes(self, items):
            for (s, i, js), r in zip(items, super()._regress_keyframes(items)):
                if r is not None:
                    recorded[(self.sessions.index(s), i)] = (list(js), r[0], r[1],
                                                             {k: v.cpu().numpy().copy() for k, v in r[2].items()})
                yield r

    c = dict(verbose=False, loop_dist_min=4, pgo_every=5)
    c.update(kw)
    return Run("unused", VOCAB, n, frontend=model, **c)


def test_sessions_real_frontend(cuda_model):
    lengths = [10, 7, 12]
    streams = [_frames(n, 11 + k) for k, n in enumerate(lengths)]
    confs = []
    for st in streams:
        probe = {}
        s = _real_slam(cuda_model, 0.5, probe)
        for v in st:
            s.step(v)
        confs += [c for i in probe for c in probe[i][1]]
    confs = np.array(confs)
    for thres in (float(confs.min()) - 0.05, float(confs.max()) + 0.05):
        rec = {}
        ses = _real_sessions(cuda_model, 3, rec, rel_pose_thres=thres)
        for i in range(5):  # the live case: one keyframe per session per call, session 2 idle
            ses.step({k: [st[i]] for k, st in enumerate(streams) if k < 2})
        ses.step({k: st[5 if k < 2 else 0:] for k, st in enumerate(streams)}, force_pgo={0, 1, 2})
        for k, st in enumerate(streams):
            rs = {}
            seq = _real_slam(cuda_model, thres, rs)
            for i, v in enumerate(st):
                seq.step(v, force_pgo=(i == len(st) - 1))
            rb = {i: r for (kk, i), r in rec.items() if kk == k}
            assert sorted(rb) == sorted(rs)
            for i in rs:
                js, cs, ks, bs = rs[i]
                jb, cb, kb, bb = rb[i]
                assert js == jb and ks == kb
                assert all(abs(c - thres) > 4e-3 for c in cs + cb)
                assert maxn(bb["pose"], bs["pose"]) < 1e-2 and maxn(bb["pose_conf"], bs["pose_conf"]) < 4e-3
                if ks:
                    for key in ("conf", "depths", "intri"):
                        assert maxn(bb[key], bs[key]) < 4e-2, (k, i, key)
            a, b = _state(seq), _state(ses[k])
            assert a["host"] == b["host"]
            for key in ("node_to_view", "node_to_connected_view", "edges"):
                np.testing.assert_array_equal(a[key], b[key])


def _tables(slam):
    """Every device table over its rows in use (nodes, edges, views)."""
    G = slam._graph
    rows = {"pose": slam.num_nodes, "depth": slam.num_nodes, "conf": slam.num_nodes, "intri": slam.num_nodes,
            "cmean": slam.num_nodes, "node_to_view": None, "node_to_connected_view": None, "best_node": None,
            "best_mean": slam.view_num, "edges": None, "meas": slam.num_edges, "weight": slam.num_edges}
    return {k: getattr(G, k)[:n].cpu().numpy() for k, n in rows.items()}


def test_one_session_equals_step(cuda_model):
    frames = _frames(9, 5)
    ses = _real_sessions(cuda_model, 1, {})
    ref = _real_slam(cuda_model, 0.75, {})
    out = []
    for i, v in enumerate(frames):
        out += ses.step({0: [v]}, force_pgo={0} if i == len(frames) - 1 else ())[0]
    want = [ref.step(v, force_pgo=(i == len(frames) - 1)) for i, v in enumerate(frames)]
    assert out == want and any(out)
    _assert_same_state(_state(ses[0]), _state(ref))
    a, b = _tables(ses[0]), _tables(ref)
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_sessions_share_one_model_and_vocabulary(state_dict, monkeypatch):
    from vista_slam_b200 import _lib
    from vista_slam_b200.sessions import SLAMSessions
    counts = {"load": 0, "vocab": 0}

    def load(*a, **kw):
        counts["load"] += 1
        return {"model": state_dict}

    L = _lib.lib()
    orig = L.sta_vocab_load

    def vocab_load(*a):
        counts["vocab"] += 1
        return orig(*a)

    monkeypatch.setattr(torch, "load", load)
    monkeypatch.setattr(L, "sta_vocab_load", vocab_load)
    ses = SLAMSessions("ckpt.pth", VOCAB, 3)
    assert counts == {"load": 1, "vocab": 1}
    assert all(s.frontend is ses.frontend and s.kf.frontend is ses.frontend for s in ses.sessions)
    assert all(s.lc_detector.vocab is ses.vocab for s in ses.sessions)
    v = _frames(2, 1)
    assert ses.step({0: v, 2: v[:1]}) == {0: [False, False], 2: [False]}
    ses[1].reset()
    assert ses[1].kf.frontend is ses.frontend
    del ses


def test_sessions_read_backs(cuda_model, monkeypatch):
    """Per call: ONE loop-candidate read-back for all sessions, ONE gate read-back per edge chunk, and at most one
    stream synchronisation (the end-of-call flag check)."""
    import vista_slam_b200.sessions as S
    from vista_slam_b200.keyframe import KeyframeFrontend
    counts = {"loops": 0, "gate": 0, "chunks": 0, "sync": 0}
    ses = _real_sessions(cuda_model, 3, {}, pgo_every=1000)
    orig_loops, orig_read, orig_chunk = S.detect_loops_group, KeyframeFrontend._read_confs, KeyframeFrontend._regress_chunk
    orig_sync = torch.cuda.Stream.synchronize

    def loops(*a):
        counts["loops"] += 1
        return orig_loops(*a)

    def read(self, t):
        counts["gate"] += 1
        return orig_read(self, t)

    def chunk(self, *a):
        counts["chunks"] += 1
        return orig_chunk(self, *a)

    def sync(self):
        counts["sync"] += 1
        return orig_sync(self)

    monkeypatch.setattr(S, "detect_loops_group", loops)
    monkeypatch.setattr(KeyframeFrontend, "_read_confs", read)
    monkeypatch.setattr(KeyframeFrontend, "_regress_chunk", chunk)
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", sync)
    streams = [_frames(6, 20 + k) for k in range(3)]
    for i in range(6):
        before = dict(counts)
        ses.step({k: [st[i]] for k, st in enumerate(streams)})
        d = {k: counts[k] - before[k] for k in counts}
        assert d["loops"] == 1 and d["gate"] == d["chunks"] and (d["chunks"] == 0) == (i == 0) and d["sync"] <= 1
        # three keyframes of up to 3 neighbour and 3 loop edges each: chunks of at most 16 edges
        assert d["chunks"] <= 2
    before = dict(counts)
    ses.step({k: st[:0] for k, st in enumerate(streams)})
    assert counts == before
    assert all(s.num_edges > 0 for s in ses.sessions)
