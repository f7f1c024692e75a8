"""GPU: OnlineSLAM.step_many and the frame-batched loop detector against the per-keyframe path.

  * loop detection over frame batches of one detector (detect_loops, through sta_loop_add_frames_group /
    sta_loop_detect_group) is bit-identical to detect_loop on each frame in order, and batched ORB to sta_op_orb per
    frame;
  * with the frontend and loops replayed from the golden stream (as in test_slam_gpu.py), step_many in any chunking
    gives the graph tables, host mirrors, PGO calls and written files of sequential step, bit for bit;
  * with the real frontend at 224 x 224 the batch sizes change the GEMMs' split-K.  test_keyframe_gpu.py bounds one
    batched stage against per-edge calls (pose 5e-3, pose confidence 2e-3, maps 2e-2, max-normalised); step_many
    batches two stages, the encoder and the decoder with its heads, so the bounds here are twice those (pose 1e-2,
    pose confidence 4e-3, maps 4e-2), and gate decisions are compared at thresholds more than 4e-3 away from every
    confidence."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle import loop_detector_oracle as O
from oracle import slam_oracle as so
from test_slam_gpu import CFG, POSE_TOL, SCALE_TOL, VOCAB, _assert_points, _batch, _Frontend, _Loops, _value

pytestmark = pytest.mark.gpu
VOCABS = [os.path.join(GOLDEN_DIR, f) for f in ("loop_vocab.txt", "loop_vocab.bin", "loop_vocab.dbow3")]


def maxn(a, b):
    a, b = torch.as_tensor(a).float().cpu(), torch.as_tensor(b).float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------ loop detection
@pytest.fixture(scope="module")
def loop_golden():
    import json
    g = np.load(os.path.join(GOLDEN_DIR, "loop.npz"))
    return g, json.loads(str(g["meta"]))


def _frames(meta, s):
    seed, n, H, W = meta["sequences"][s]
    return O.make_sequence(seed, n, H, W)


@pytest.mark.parametrize("path", VOCABS)
@pytest.mark.parametrize("chunk", [1, 5, None])
def test_detect_loops_equals_detect_loop(loop_golden, path, chunk):
    from vista_slam_b200.loop_detector import LoopDetector
    g, meta = loop_golden
    args = meta["loop_args"]
    for s in (0, 1):
        frames = _frames(meta, s)
        n = len(frames)
        seq = LoopDetector(path, **args)
        want, rows = [], []
        for t, f in enumerate(frames):
            want.append(seq.detect_loop(f, max(0, t - 3)))
            rows.append(seq.similarities())
        bat = LoopDetector(path, **args)
        c = n if chunk is None else chunk
        got = []
        for t0 in range(0, n, c):
            part = frames[t0:t0 + c]
            got += bat.detect_loops(part, [max(0, t - 3) for t in range(t0, t0 + len(part))])
            t_last = t0 + len(part) - 1
            row = bat.similarities()
            assert np.array_equal(row, rows[t_last], equal_nan=True), t_last
        assert got == want
        for t in range(n):
            ref = g["s%d_k%d_cand" % (s, t)]
            assert [j for j, _ in got[t]] == [int(j) for j in ref[:, 0]]
            np.testing.assert_array_equal(np.array([x for _, x in got[t]], np.float64), ref[:, 1])
        assert len(bat.bow_feats) == n
        for t in range(n):
            assert (bat.bow_feats[t] is None) == (seq.bow_feats[t] is None), t
            if seq.bow_feats[t] is not None:
                for a, b in zip(bat.bow_feats[t].to_numpy(), seq.bow_feats[t].to_numpy()):
                    np.testing.assert_array_equal(a, b)


def _orb_many(frames_u8):
    from vista_slam_b200 import _lib
    F, H, W = frames_u8.shape
    M = _lib.ORB_MAX_KEYPOINTS
    L = _lib.lib()
    nbytes = int(L.sta_orb_scratch_bytes(H, W))
    dev = frames_u8.device
    scratch = torch.empty(F * nbytes, dtype=torch.uint8, device=dev)
    out = {"xy": torch.empty(F, M, 2, dtype=torch.int32, device=dev), "level": torch.empty(F, M, dtype=torch.int32, device=dev),
           "pts": torch.empty(F, M, 2, dtype=torch.float32, device=dev), "angle": torch.empty(F, M, device=dev),
           "response": torch.empty(F, M, device=dev), "desc": torch.empty(F, M, 32, dtype=torch.uint8, device=dev)}
    cnt = torch.empty(F, dtype=torch.int32, device=dev)
    _lib.check(L.sta_op_orb_many(_lib.ptr(frames_u8), 0, F, H, W, *[_lib.ptr(out[k]) for k in ("xy", "level", "pts", "angle",
                                                                                            "response", "desc")],
                                 _lib.ptr(cnt), _lib.ptr(scratch), _lib.cur_stream()), "sta_op_orb_many")
    return out, cnt.cpu(), scratch.view(F, nbytes)


@pytest.mark.parametrize("hw", [(224, 224), (480, 640), (70, 90)])
def test_batched_orb_equals_per_frame(hw):
    from vista_slam_b200.loop_detector import orb_detect_and_compute
    H, W = hw
    rng = np.random.default_rng(H)
    frames = [O._texture(rng, H, W) for _ in range(3)] + [np.full((H, W), 77, np.uint8)]  # a flat frame: no keypoint
    out, cnt, scratch = _orb_many(torch.from_numpy(np.stack(frames)).cuda())
    assert int(cnt[3]) == 0
    for f, fr in enumerate(frames):
        r = orb_detect_and_compute(torch.from_numpy(fr).cuda())
        n = int(cnt[f])
        assert n == len(r["desc"])
        for k in ("xy", "level", "pts", "angle", "response", "desc"):
            assert torch.equal(out[k][f, :n], r[k]), (f, k)
        lay = r["layout"]
        pix = lay[12 + 4 * 7] + lay[10 + 4 * 7] * lay[11 + 4 * 7]
        for o in lay[1:4]:  # pyramid, blurred levels and FAST scores of the frame's scratch slice
            np.testing.assert_array_equal(scratch[f, o:o + pix].cpu().numpy(), r["scratch"][o:o + pix].cpu().numpy())


def test_loop_group_of_one_detector_refusals():
    from vista_slam_b200 import _lib
    from vista_slam_b200.loop_detector import LoopDetector
    det = LoopDetector(VOCAB, 40, 40, 5)
    a = torch.zeros(64, 64, dtype=torch.uint8, device="cuda")
    b = torch.zeros(64, 96, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="same size"):
        det.detect_loops([a, b], [0, 0])
    with pytest.raises(ValueError, match="farthest"):
        det.detect_loops([a, a], [0, 2])
    assert det.detect_loops([], []) == [] and len(det.bow_feats) == 0
    L = _lib.lib()
    assert L.sta_loop_views(det._h) == 0

    def dets(k):
        return (ctypes.c_void_p * k)(*[det._h.value] * k)

    assert L.sta_loop_add_frames_group(dets(1), 0, _lib.ptr(a), 0, 64, 64, _lib.cur_stream()) != 0
    assert b"frame count" in L.sta_last_error()
    # the C entry point refuses an out-of-range farthest neighbour, or another row count than the last add's, before
    # any launch
    assert det.detect_loops([a, a], [0, 1]) == [[], []]
    n = (ctypes.c_int * 6)()
    rc = L.sta_loop_detect_group(dets(2), 2, (ctypes.c_int * 2)(0, 5), n, None, None, 0, _lib.cur_stream())
    assert rc != 0 and b"farthest" in L.sta_last_error()
    rc = L.sta_loop_detect_group(dets(3), 3, (ctypes.c_int * 3)(0, 0, 0), n, None, None, 0, _lib.cur_stream())
    assert rc != 0


# ------------------------------------------------------------------------------------------------ replayed frontend
class _LoopsMany(_Loops):
    def detect_loops(self, images, farthest_neighbors):
        torch.cuda.synchronize()  # the real detector reads its candidates back here, once per call
        out = [list(self.loops[self.calls + k]) for k in range(len(images))]
        self.calls += len(images)
        return out


def _replay_slam(stream, **over):
    from vista_slam_b200.slam import OnlineSLAM

    class ReplaySLAM(OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return _Frontend()

        def _regress_keyframe(self, i, js):
            return _batch(stream, i, js, self.rel_pose_thres)

        def _regress_keyframes(self, items):
            return [_batch(stream, i, js, self.rel_pose_thres) if js else None for i, js in items]

    c = dict(CFG)
    c.update(over)
    slam = ReplaySLAM("unused", VOCAB, verbose=True, **c)
    slam.lc_detector = _LoopsMany(stream["loops"], c["loop_dist_min"])
    return slam


def _state(slam):
    G = slam._graph
    N, E, V = slam.num_nodes, slam.num_edges, slam.view_num
    return {"node_to_view": G.node_to_view.cpu().numpy(), "node_to_connected_view": G.node_to_connected_view.cpu().numpy(),
            "edges": G.edges.cpu().numpy(), "best_node": G.best_node.cpu().numpy(), "meas": G.meas[:E].cpu().numpy(),
            "weight": G.weight[:E].cpu().numpy(), "pose": G.pose[:N].cpu().numpy(),
            "host": (N, E, V, dict(slam.view_to_node), list(slam.node_to_connected_view), set(slam.loop_related_views),
                     list(slam.view_names), len(slam.imgs), len(slam.img_shapes))}


def _assert_same_state(a, b):
    assert a["host"] == b["host"]
    for k in a:
        if k != "host":
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def _record_pgo(monkeypatch):
    import vista_slam_b200.slam as S
    calls = []
    base = S.PoseGraphOpt

    class RecordingPGO(base):
        def optimize(self, edges, poses, weight, **kw):
            rec = [self.idxs_opt.cpu().numpy(), self.nodes.cpu().numpy()]
            out = super().optimize(edges, poses, weight, **kw)
            calls.append(rec + [self.nodes.cpu().numpy()])
            return out

    monkeypatch.setattr(S, "PoseGraphOpt", RecordingPGO)
    return calls


def _files(folder):
    return {f: open(os.path.join(folder, f), "rb").read() for f in sorted(os.listdir(folder))}


@pytest.mark.parametrize("chunking", ["ones", "five_rest", "all"])
def test_step_many_replay_equals_step(chunking, tmp_path, monkeypatch):
    stream = so.make_stream()
    images = so.stream_images(stream)
    n = stream["n_views"]
    pgo = _record_pgo(monkeypatch)
    seq = _replay_slam(stream)
    flags_seq = [seq.step(_value(images, i, stream), force_pgo=(i == n - 1), log_intermediate_results=True,
                          output_folder=str(tmp_path / "seq")) for i in range(n)]
    pgo_seq = list(pgo)
    pgo.clear()
    bat = _replay_slam(stream)
    sizes = {"ones": [1] * n, "five_rest": [5, n - 5], "all": [n]}[chunking]
    flags, t0 = [], 0
    for m in sizes:
        flags += bat.step_many([_value(images, i, stream) for i in range(t0, t0 + m)], force_pgo=(t0 + m == n),
                               log_intermediate_results=True, output_folder=str(tmp_path / "bat"))
        t0 += m
    assert flags == flags_seq and any(flags)
    _assert_same_state(_state(bat), _state(seq))
    assert len(pgo) == len(pgo_seq)
    for a, b in zip(pgo, pgo_seq):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x, y)
    assert _files(tmp_path / "bat") == _files(tmp_path / "seq")
    assert bat.lc_detector.calls == n and set(bat.get_time_dict()) == set(seq.get_time_dict())


def test_step_many_refusals(tmp_path):
    stream = so.make_stream()
    images = so.stream_images(stream)
    assert _replay_slam(stream).step_many([]) == []
    # capacity: the same keyframe, the same state as step at the failure
    seq = _replay_slam(stream, max_view_num=1)
    with pytest.raises(IndexError):
        for i in range(6):
            seq.step(_value(images, i, stream))
    bat = _replay_slam(stream, max_view_num=1)
    with pytest.raises(IndexError):
        bat.step_many([_value(images, i, stream) for i in range(6)])
    _assert_same_state(_state(bat), _state(seq))
    # mixed sizes: refused before anything runs
    fresh = _replay_slam(stream)
    other = dict(_value(images, 1, stream), rgb=torch.zeros(1, 3, stream["H"], stream["W"] + 16, device="cuda"))
    with pytest.raises(ValueError, match="same image size"):
        fresh.step_many([_value(images, 0, stream), other])
    assert fresh.view_num == 0 and fresh.kf.view_num == 0 and fresh.lc_detector.calls == 0
    # a non-orthonormal relative rotation: ValueError by the end of the call
    s2 = so.make_stream()
    s2["edges"][(3, 2)]["pose"] = s2["edges"][(3, 2)]["pose"].copy()
    s2["edges"][(3, 2)]["pose"][:3, :3] *= np.float32(1.01)
    bad = _replay_slam(s2)
    with pytest.raises(ValueError, match="orthonormal"):
        bad.step_many([_value(so.stream_images(s2), i, s2) for i in range(4)])


# ------------------------------------------------------------------------------------------------ real frontend
def _frames_224(n):
    g = torch.Generator().manual_seed(3)
    H = W = 224
    base = torch.rand(1, 3, H // 8, W // 8, generator=g)
    out = []
    for i in range(n):
        img = torch.nn.functional.interpolate(base.roll(i, dims=3), size=(H, W), mode="bilinear") * 2 - 1
        img = (img + 0.05 * torch.rand(1, 3, H, W, generator=g)).clamp(-1, 1).cuda()
        out.append({"rgb": img, "shape": torch.tensor([[H, W]]), "gray": ((img[0].mean(0) + 1) / 2).contiguous(),
                    "view_name": "%d" % i})
    return out


def _real_slam(model, thres, recorded):
    import vista_slam_b200.slam as S

    class Run(S.OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return model

        def _regress_keyframe(self, i, js):
            r = super()._regress_keyframe(i, js)
            recorded[i] = (list(js), r[0], r[1], {k: v.cpu().numpy().copy() for k, v in r[2].items()})
            return r

        def _regress_keyframes(self, items):
            for (i, js), r in zip(items, super()._regress_keyframes(items)):
                if r is not None:
                    recorded[i] = (list(js), r[0], r[1], {k: v.cpu().numpy().copy() for k, v in r[2].items()})
                yield r

    return Run("unused", VOCAB, verbose=False, loop_dist_min=4, pgo_every=5, rel_pose_thres=thres)


def test_step_many_real_frontend(cuda_model, monkeypatch):
    from vista_slam_b200 import _lib
    from vista_slam_b200.keyframe import KeyframeFrontend
    n = 24
    values = _frames_224(n)
    probe = {}
    s = _real_slam(cuda_model, 0.5, probe)
    for i, v in enumerate(values):
        s.step(v, force_pgo=(i == n - 1))
    confs = np.array([c for i in probe for c in probe[i][1]])
    for thres in (float(confs.min()) - 0.05, float(confs.max()) + 0.05):
        rec_s, rec_b = {}, {}
        seq = _real_slam(cuda_model, thres, rec_s)
        for i, v in enumerate(values):
            seq.step(v, force_pgo=(i == n - 1))
        bat = _real_slam(cuda_model, thres, rec_b)
        assert bat.step_many(values[:10]) == [False] * 4 + [True] + [False] * 4 + [True]
        bat.step_many(values[10:], force_pgo=True)
        assert sorted(rec_b) == sorted(rec_s)
        for i in rec_s:
            js, cs, ks, bs = rec_s[i]
            jb, cb, kb, bb = rec_b[i]
            assert js == jb and ks == kb
            assert all(abs(c - thres) > 4e-3 for c in cs + cb)  # the gate is decided far from the threshold
            assert maxn(bb["pose"], bs["pose"]) < 1e-2 and maxn(bb["pose_conf"], bs["pose_conf"]) < 4e-3
            if ks:
                for k in ("conf", "depths", "intri"):
                    assert maxn(bb[k], bs[k]) < 4e-2, (i, k)
        a, b = _state(seq), _state(bat)
        assert a["host"] == b["host"]
        # best_node is chosen by a strict comparison of confidence means, so a near-tie may part under the rounding
        # above; it is checked exactly against the oracle on this run's own outputs below
        for k in ("node_to_view", "node_to_connected_view", "edges"):
            np.testing.assert_array_equal(a[k], b[k])
        # the batched graph against the oracle replayed on the batched run's own frontend outputs
        stream = {"n_views": n, "H": 224, "W": 224, "loops": [], "edges": {}, "seed": 0}
        cmeans = {}
        for i in range(n):
            js, conf_host, keep, bt = rec_b.get(i, ([], [], [], {}))
            nb = max(0, i - 3)
            stream["loops"].append([(j, 0.0) for j in js[i - nb:]])
            for k, j in enumerate(js):
                e = {"pose": bt["pose"][k], "conf": np.float32(conf_host[k])}
                if k in keep:
                    p = keep.index(k)
                    e.update(confs=bt["conf"][:, p], depths=bt["depths"][:, p], intri=bt["intri"][p])
                    cmeans[(i, j)] = bt["conf_mean"][:, p]
                stream["edges"][(i, j)] = e
        graph, _, _ = so.run(stream, rel_pose_thres=thres, pgo_every=5, cmeans=cmeans)
        N, E = bat.num_nodes, bat.num_edges
        assert (N, E) == (graph.num_nodes, graph.num_edges) and N > 0
        G = bat._graph
        np.testing.assert_array_equal(G.edges[:E].cpu().numpy(), graph.edges[:E])
        np.testing.assert_array_equal(G.best_node[:n].cpu().numpy(), graph.best_node[:n])
        np.testing.assert_allclose(G.weight[:E].cpu().numpy(), graph.weight[:E], atol=SCALE_TOL, rtol=1e-5)
        np.testing.assert_allclose(G.meas[:E].cpu().numpy(), graph.meas[:E], atol=POSE_TOL, rtol=1e-5)
        # q and -q are the same rotation: random-init poses include rotations near the conversion's sign branch
        got, want = G.pose[:N].cpu().numpy(), graph.pose[:N].copy()
        flip = (got[:, 3:7] * want[:, 3:7]).sum(1) < 0
        want[flip, 3:7] *= -1
        np.testing.assert_allclose(got, want, atol=POSE_TOL, rtol=1e-4)
        ex = so.export(graph, n, bat.conf_thres, bat.imgs.device_stack().cpu().numpy())
        out = bat._export(0, n, cloud=True)
        m = int(out["count"])
        assert m == len(ex["points"])
        _assert_points(out["points"][:m].cpu().numpy(), ex["points"])

    # host read-backs of one call: one for the loop candidates, one per edge chunk (PGO reads back on its own)
    counts = {"loops": 0, "gate": 0}
    again = _real_slam(cuda_model, 0.5, {})
    det = again.lc_detector
    orig_loops, orig_read = det.detect_loops, KeyframeFrontend._read_confs

    def loops(*a):
        counts["loops"] += 1
        return orig_loops(*a)

    def read(self, t):
        counts["gate"] += 1
        return orig_read(self, t)

    orig_chunk = KeyframeFrontend._regress_chunk

    def chunk(self, *a):
        counts["chunks"] = counts.get("chunks", 0) + 1
        return orig_chunk(self, *a)

    det.detect_loops = loops
    monkeypatch.setattr(KeyframeFrontend, "_read_confs", read)
    monkeypatch.setattr(KeyframeFrontend, "_regress_chunk", chunk)
    again.step_many(values)
    assert counts["loops"] == 1 and counts["gate"] == counts["chunks"] >= 4

    # the CUDA-graph cache: a repeated identical run replays every graphed call
    L = _lib.lib()
    calls = {"n": 0}
    for name in ("sta_encode", "sta_regress_pairs_begin", "sta_regress_pairs_finish"):
        f = getattr(L, name)

        def wrap(*a, _f=f, _name=name):
            if _name != "sta_regress_pairs_finish" or a[2] > 0:
                calls["n"] += 1
            return _f(*a)

        monkeypatch.setattr(L, name, wrap)
    _real_slam(cuda_model, 0.5, {}).step_many(values)  # sees again every key a cache flush may have dropped
    final = _real_slam(cuda_model, 0.5, {})
    calls["n"] = 0
    r0 = int(L.sta_graph_replays(cuda_model._handle))
    final.step_many(values)
    assert int(L.sta_graph_replays(cuda_model._handle)) - r0 == calls["n"] > 0
    _assert_same_state(_state(final), _state(again))


def test_step_read_backs_real_frontend(cuda_model, monkeypatch):
    """step with no PGO due: per keyframe ONE detect_loop, ONE gate read-back when the keyframe has candidates, and no
    stream synchronisation (the rotation flag is read at the next read-back)."""
    from vista_slam_b200.keyframe import KeyframeFrontend
    counts = {"loops": 0, "gate": 0, "sync": 0}
    slam = _real_slam(cuda_model, 0.5, {})
    slam.pgo_every = 1000
    det = slam.lc_detector
    orig_loop, orig_read, orig_sync = det.detect_loop, KeyframeFrontend._read_confs, torch.cuda.Stream.synchronize

    def loop(*a):
        counts["loops"] += 1
        return orig_loop(*a)

    def read(self, t):
        counts["gate"] += 1
        return orig_read(self, t)

    def sync(self):
        counts["sync"] += 1
        return orig_sync(self)

    det.detect_loop = loop
    monkeypatch.setattr(KeyframeFrontend, "_read_confs", read)
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", sync)
    for i, v in enumerate(_frames_224(6)):
        before = dict(counts)
        assert slam.step(v) is False
        assert counts["loops"] - before["loops"] == 1
        assert counts["gate"] - before["gate"] == (1 if i > 0 else 0)
        assert counts["sync"] == 0
    assert slam.num_edges > 0
