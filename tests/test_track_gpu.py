"""GPU: tracked frames (OnlineSLAM.track, SLAMSessions.track, sta_graph_track_frames / sta_graph_frame_poses).

  1. A frame tracked against view n gets, bit for bit, the measurements and the pose its first node gets when a twin
     session steps it as keyframe n + 1 with one neighbour edge.
  2. Each frame's scale edge, stored quaternion and pose against float64 built from the device's own inputs (the
     helpers and bounds of tests/test_slam_graph_fp64_cpu.py, tests/test_track_cpu.py), through the C ABI at 224 x 224
     and 384 x 512, with the clamp planted and rotations at every rot_to_quat branch; non-orthonormal rotations give
     valid = 0 and leave the graph flag clear.
  3. After a synchronous PGO and after a folded background PGO, frame_trajectory() follows the new anchor poses.
  4. A session that tracks between its steps, also while a background PGO is pending, ends with the graph, host
     mirror, loop candidates and save_data_all files of one that does not, and track leaves time_dict as it was.
  5. Batched calls (F = 1, 15, 16, 17, 40, and three sessions at once) against one-frame calls within the bounds of
     tests/test_slam_batch_gpu.py: pose 1e-2, pose confidence 4e-3, maps (the scale edge) 4e-2, max-normalised.
  6. track makes no host synchronisation.
  7. Refusals come before any launch and change nothing."""
import ctypes

import numpy as np
import pytest
import torch

from test_slam_batch_gpu import _files, _frames_224, _state, maxn
from test_slam_graph_fp64_cpu import ROT_CASES, Q_ABS, rot_to_quat, scale_errs, scale_maps, scale_stats_ref, sim3
from test_slam_gpu import VOCAB
from test_track_cpu import track_err

pytestmark = pytest.mark.gpu


def _slam(model, **kw):
    from vista_slam_b200.slam import OnlineSLAM

    class Run(OnlineSLAM):
        def load_frontend(self, ckpt_path):
            return model

    c = dict(verbose=False, neighbor_edge_num=1, loop_edge_num=0, loop_dist_min=4, pgo_every=1000)
    c.update(kw)
    return Run("unused", VOCAB, **c)


def _record_regressions(monkeypatch):
    """The regression outputs each track call composes from: [(pose, pose_conf, depth_k, conf_k)] per call."""
    import vista_slam_b200.slam as S
    calls = []
    base = S.regress_frames

    def rec(sta, pairs, H, W):
        out = base(sta, pairs, H, W)
        calls.append(out)
        return out

    monkeypatch.setattr(S, "regress_frames", rec)
    return calls


def _recomposition_err(slam, traj):
    """max err / bound of frame_trajectory() against the float64 recomposition of its stored values on the anchors'
    current poses."""
    poses = slam._graph.pose.cpu().numpy()
    meas, se = traj["meas"].cpu().numpy(), traj["scale_edge"].cpu().numpy()
    P, sc = traj["pose"].cpu().numpy(), traj["scale"].cpu().numpy()
    return max(track_err(P[f], sc[f], poses[a], se[f], meas[f]) for f, a in enumerate(traj["anchor"]))


# ------------------------------------------------------------------------------------------------ (1)
def test_tracked_frame_equals_its_keyframe_bit_for_bit(cuda_model):
    n = 5
    vals = _frames_224(n + 2)
    a, b = _slam(cuda_model), _slam(cuda_model)
    for v in vals[:n + 1]:
        a.step(v)
        b.step(v)
    r = a.track([vals[n + 1]])
    b.step(vals[n + 1])
    t = a.frame_trajectory()
    E = b.num_edges
    node0 = b.view_to_node[n + 1][0]
    assert t["kf"] == [n] and t["anchor"] == [b.view_to_node[n][0]] and int(r["valid"][0]) == 1
    meas = b._graph.meas[:E].cpu()
    assert torch.equal(t["meas"][0].cpu(), meas[E - 1])  # the pose edge (n + 1, n)
    assert torch.equal(t["scale_edge"][0].cpu(), meas[E - 2][7])  # the scale edge of view n's new node
    view = b.get_view(n + 1)
    assert torch.equal(r["pose"][0].cpu(), view["pose"])
    assert torch.equal(r["scale"][0].cpu(), b._graph.pose[node0][7].cpu())
    assert torch.equal(t["pose"][0], r["pose"][0]) and torch.equal(t["scale"][0], r["scale"][0])


# ------------------------------------------------------------------------------------------------ (2)
def _abi_graph(H, W):
    from vista_slam_b200.slam import _Graph
    return _Graph(8, 8, 8, H, W, torch.device("cuda"))


def _abi_track(g, anchors, M, depth, conf):
    from vista_slam_b200 import _lib
    L = _lib.lib()
    F = len(anchors)
    dev = torch.device("cuda")
    out = {"meas": torch.empty(F, 8, device=dev), "s": torch.empty(F, device=dev),
           "valid": torch.empty(F, dtype=torch.uint8, device=dev), "pose": torch.empty(F, 4, 4, device=dev),
           "scale": torch.empty(F, device=dev)}
    need = int(L.sta_graph_track_frames_scratch_bytes(F))
    scratch = torch.empty(need // 8, dtype=torch.float64, device=dev)
    _lib.check(L.sta_graph_track_frames(g.h, F, (ctypes.c_int * F)(*anchors), _lib.ptr(M), _lib.ptr(depth), _lib.ptr(conf),
                                        _lib.ptr(out["meas"]), _lib.ptr(out["s"]), _lib.ptr(out["valid"]),
                                        _lib.ptr(out["pose"]), _lib.ptr(out["scale"]), _lib.ptr(scratch), need,
                                        _lib.cur_stream()), "sta_graph_track_frames")
    return out


@pytest.mark.parametrize("H,W", [(224, 224), (384, 512)])
def test_track_frames_against_fp64(H, W):
    from vista_slam_b200 import _lib
    g = _abi_graph(H, W)
    F = len(ROT_CASES)
    anchors = [k % 3 for k in range(F)]
    nodes = [sim3([0.4, -1.2, 2.0], [1, 2, 3], 0.7, 1.3), sim3([1e2, -3e1, 5e1], [0, 0, 1], 3.0, 1e-1),
             sim3([-2.0, 0.5, 0.1], [-1, 0.2, 0.4], 2.9, 8.0)]
    for k, p in enumerate(nodes):
        g.pose[k] = torch.from_numpy(p).cuda()
    maps = [scale_maps(H * W, 100 + k) for k in range(3 + F)]  # planted: the clamp binds, sums partly cancel
    for k in range(3):
        g.depth[k] = torch.from_numpy(maps[k][0].reshape(H, W)).cuda()
        g.conf[k] = torch.from_numpy(maps[k][2].reshape(H, W)).cuda()
    depth = torch.from_numpy(np.stack([maps[3 + f][1] for f in range(F)]).reshape(F, H, W)).cuda()
    conf = torch.from_numpy(np.stack([maps[3 + f][3] for f in range(F)]).reshape(F, H, W)).cuda()
    M = torch.from_numpy(np.stack([c[1] for c in ROT_CASES])).cuda()
    before = {k: getattr(g, k).clone() for k in ("pose", "depth", "conf", "meas", "edges")}
    out = _abi_track(g, anchors, M, depth, conf)
    torch.cuda.synchronize()
    assert g.flags() == 0  # planted non-orthonormal rotations raise no graph flag
    for k, v in before.items():
        assert torch.equal(getattr(g, k), v), k
    o = {k: v.cpu().numpy() for k, v in out.items()}
    gd, gc = g.depth.cpu().numpy().reshape(8, -1), g.conf.cpu().numpy().reshape(8, -1)
    worst = {"scale": 0.0, "pose": 0.0}
    for f, (name, Mf, (_, _, ok)) in enumerate(ROT_CASES):
        a = anchors[f]
        assert o["valid"][f] == int(ok), name
        # the scale edge (depth_k, depth_a, conf_k, conf_a)
        stats = scale_stats_ref(maps[3 + f][1], gd[a], maps[3 + f][3], gc[a])
        worst["scale"] = max(worst["scale"], scale_errs(o["s"][f], stats[2] / stats[6], stats)[0])
        q, _, _, _ = rot_to_quat(Mf)
        assert (np.abs(o["meas"][f][3:7] - q) <= 2.0 ** -23 * np.abs(q) + Q_ABS).all(), name
        np.testing.assert_array_equal(o["meas"][f][[0, 1, 2, 7]], [Mf[0, 3], Mf[1, 3], Mf[2, 3], 1.0])
        worst["pose"] = max(worst["pose"], track_err(o["pose"][f], o["scale"][f], nodes[a], o["s"][f], o["meas"][f]))
    print("track err / bound at %dx%d:" % (H, W), worst)
    assert worst["scale"] <= 1.0 and worst["pose"] <= 1.0, worst
    # sta_graph_frame_poses on unchanged anchors gives the same bits; on moved anchors, the fp64 recomposition
    L = _lib.lib()
    for moved in (False, True):
        if moved:
            g.pose[:3] = torch.from_numpy(np.stack([sim3([3.0, 1.0, -1.0], [0, 1, 1], 1.1, 2.5), nodes[2], nodes[0]])).cuda()
        P, S = torch.empty(F, 4, 4, device="cuda"), torch.empty(F, device="cuda")
        _lib.check(L.sta_graph_frame_poses(g.h, F, (ctypes.c_int * F)(*anchors), _lib.ptr(out["meas"]), _lib.ptr(out["s"]),
                                           _lib.ptr(P), _lib.ptr(S), _lib.cur_stream()), "sta_graph_frame_poses")
        if not moved:
            assert torch.equal(P, out["pose"]) and torch.equal(S, out["scale"])
        else:
            poses = g.pose.cpu().numpy()
            Pn, Sn = P.cpu().numpy(), S.cpu().numpy()
            assert max(track_err(Pn[f], Sn[f], poses[a], o["s"][f], o["meas"][f]) for f, a in enumerate(anchors)) <= 1.0


def test_track_frames_refusals_leave_the_graph():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    g = _abi_graph(32, 32)
    M = torch.eye(4, device="cuda").expand(2, 4, 4).contiguous()
    d = torch.ones(2, 32, 32, device="cuda")
    outs = [torch.empty(2, 8, device="cuda"), torch.empty(2, device="cuda"), torch.empty(2, dtype=torch.uint8, device="cuda"),
            torch.empty(2, 4, 4, device="cuda"), torch.empty(2, device="cuda")]
    scratch = torch.empty(int(L.sta_graph_track_frames_scratch_bytes(2)) // 8, dtype=torch.float64, device="cuda")
    need = scratch.numel() * 8
    before = g.pose.clone()

    def call(anchors, M=M, scratch_bytes=need, host=False):
        ins = [M.cpu() if host else M, d, d]
        return L.sta_graph_track_frames(g.h, 2, (ctypes.c_int * 2)(*anchors), *[_lib.ptr(x) for x in ins],
                                        *[_lib.ptr(x) for x in outs], _lib.ptr(scratch), scratch_bytes, _lib.cur_stream())

    assert call([0, 8]) != 0 and b"anchor" in L.sta_last_error()
    assert call([-1, 0]) != 0 and b"anchor" in L.sta_last_error()
    assert call([0, 1], scratch_bytes=need - 1) != 0 and b"scratch" in L.sta_last_error()
    assert call([0, 1], host=True) != 0 and b"device memory" in L.sta_last_error()
    assert L.sta_graph_frame_poses(g.h, 2, (ctypes.c_int * 2)(0, 8), _lib.ptr(outs[0]), _lib.ptr(outs[1]),
                                   _lib.ptr(outs[3]), _lib.ptr(outs[4]), _lib.cur_stream()) != 0
    torch.cuda.synchronize()
    assert torch.equal(g.pose, before)
    assert call([0, 1]) == 0


# ------------------------------------------------------------------------------------------------ (3)
def test_frame_trajectory_follows_pgo(cuda_model):
    vals = _frames_224(30)
    s = _slam(cuda_model, neighbor_edge_num=2, loop_edge_num=1)
    for k in range(12):
        s.step(vals[2 * k])
        if k >= 1:
            s.track([vals[2 * k + 1]])
    before = s.frame_trajectory()
    assert _recomposition_err(s, before) <= 1.0
    s.pose_graph_optimize()
    after = s.frame_trajectory()
    assert _recomposition_err(s, after) <= 1.0
    assert not torch.equal(before["pose"], after["pose"])  # the frames moved with their keyframes
    # background: started at a step, tracked while pending, folded by wait_pgo
    s.pgo_background = True
    s.step(vals[24], force_pgo=True)
    assert s.pgo_pending
    s.track([vals[25], vals[27]])
    s.wait_pgo()
    t = s.frame_trajectory()
    assert len(t["names"]) == 13 and _recomposition_err(s, t) <= 1.0


# ------------------------------------------------------------------------------------------------ (4)
def test_tracking_changes_nothing_of_the_session(cuda_model, tmp_path):
    vals = _frames_224(40)
    kw = dict(neighbor_edge_num=2, loop_edge_num=2, loop_dist_min=4, pgo_every=4)
    a, b = _slam(cuda_model, **kw), _slam(cuda_model, **kw)
    a.pgo_background = b.pgo_background = True
    pending_seen = False
    for k in range(14):
        v = vals[2 * k]
        a.step(v)
        b.step(v)
        if k >= 1:
            pending_seen = pending_seen or a.pgo_pending
            times, pending = dict(a.time_dict), a.pgo_pending
            a.track([vals[2 * k + 1]] + ([vals[2 * k + 3]] if k % 3 == 0 else []))
            assert a.time_dict == times and a.pgo_pending == pending  # no poll, no fold, no time
    assert pending_seen
    a.wait_pgo()
    b.wait_pgo()
    sa, sb = _state(a), _state(b)
    assert sa["host"] == sb["host"]
    for k in sa:
        if k != "host":
            np.testing.assert_array_equal(sa[k], sb[k], err_msg=k)
    for k in ("depth", "conf", "intri", "cmean", "best_mean"):
        assert torch.equal(getattr(a._graph, k)[:a.num_nodes if k != "best_mean" else a.view_num],
                           getattr(b._graph, k)[:b.num_nodes if k != "best_mean" else b.view_num]), k
    assert len(a.kf.enc_features) == len(b.kf.enc_features) == a.view_num
    assert all(torch.equal(x, y) for x, y in zip(a.kf.enc_features, b.kf.enc_features))
    assert set(a.time_dict) == set(b.time_dict) and a.loop_related_views == b.loop_related_views
    assert vars(a.flow_tracker).keys() == vars(b.flow_tracker).keys()
    probe = vals[39]["gray"]
    assert a.lc_detector.detect_loop(probe, a.view_num - 1) == b.lc_detector.detect_loop(probe, b.view_num - 1)
    a.save_data_all(str(tmp_path / "a"))
    b.save_data_all(str(tmp_path / "b"))
    assert _files(tmp_path / "a") == _files(tmp_path / "b")
    a.save_frame_trajectory(str(tmp_path / "ft"), traj_name_postfix="x")
    got = np.load(tmp_path / "ft" / "frame_trajectory_x.npy")
    info = np.load(tmp_path / "ft" / "frame_info_x.npz")
    t = a.frame_trajectory()
    assert got.shape == (len(t["names"]), 4, 4) and list(info["names"]) == t["names"]
    np.testing.assert_array_equal(got, t["pose"].cpu().numpy())
    np.testing.assert_array_equal(np.load(tmp_path / "ft" / "frame_scales_x.npy"), t["scale"].cpu().numpy())


# ------------------------------------------------------------------------------------------------ (5)
def _compare_batched(s1, rec1, sb, recb, F):
    t1, tb = s1.frame_trajectory(), sb.frame_trajectory()
    assert t1["kf"] == tb["kf"] and t1["anchor"] == tb["anchor"] and t1["names"] == tb["names"]
    assert torch.equal(t1["valid"], tb["valid"])
    p1 = torch.cat([r[0] for r in rec1])[-F:]
    pb = torch.cat([r[0] for r in recb])[-F:]
    assert maxn(pb, p1) < 1e-2 and maxn(tb["pose_conf"][-F:], t1["pose_conf"][-F:]) < 4e-3
    assert maxn(tb["scale_edge"][-F:], t1["scale_edge"][-F:]) < 4e-2
    assert _recomposition_err(s1, t1) <= 1.0 and _recomposition_err(sb, tb) <= 1.0


def test_batched_track_against_one_frame_calls(cuda_model, monkeypatch):
    rec = _record_regressions(monkeypatch)
    vals = _frames_224(48)
    s1, sb = _slam(cuda_model, neighbor_edge_num=2), _slam(cuda_model, neighbor_edge_num=2)
    for v in vals[:4]:
        s1.step(v)
        sb.step(v)
    frames = vals[4:]
    for F in (1, 15, 16, 17, 40):
        rec.clear()
        for f in frames[:F]:
            s1.track([f], kf=2)
        rec1 = list(rec)
        rec.clear()
        r = sb.track(frames[:F], kf=2)
        assert len(rec) == 1 and r["pose"].shape == (F, 4, 4) and r["valid"].dtype == torch.uint8
        _compare_batched(s1, rec1, sb, list(rec), F)


def test_sessions_track_against_per_session_track(cuda_model, monkeypatch):
    from vista_slam_b200.sessions import SLAMSessions
    rec = _record_regressions(monkeypatch)
    vals = _frames_224(30)
    kw = dict(verbose=False, neighbor_edge_num=1, loop_edge_num=0, pgo_every=1000)
    group = SLAMSessions("unused", VOCAB, 3, frontend=cuda_model, **kw)
    solo = [_slam(cuda_model, **kw) for _ in range(3)]
    for k in range(3):
        for v in vals[k:k + 3 + k]:
            group[k].step(v)
            solo[k].step(v)
    calls = {0: vals[10:15], 1: vals[15:16], 2: vals[16:28]}
    rec.clear()
    res = group.track(calls, kfs={1: 1})
    assert len(rec) == 1 and sorted(res) == [0, 1, 2]
    total = torch.cat([r[0] for r in rec])
    t0 = 0
    for k in range(3):
        rec.clear()
        solo[k].track(calls[k], kf=1 if k == 1 else None)
        F = len(calls[k])
        t1, tb = solo[k].frame_trajectory(), group[k].frame_trajectory()
        assert t1["kf"] == tb["kf"] and t1["anchor"] == tb["anchor"] and torch.equal(t1["valid"], tb["valid"])
        assert maxn(total[t0:t0 + F], rec[0][0]) < 1e-2 and maxn(tb["pose_conf"], t1["pose_conf"]) < 4e-3
        assert maxn(tb["scale_edge"], t1["scale_edge"]) < 4e-2
        assert _recomposition_err(group[k], tb) <= 1.0
        assert torch.equal(res[k]["pose"], tb["pose"])
        t0 += F


# ------------------------------------------------------------------------------------------------ (6)
def test_track_does_not_synchronise(cuda_model):
    vals = _frames_224(40)
    s = _slam(cuda_model)
    for v in vals[:3]:
        s.step(v)
    s.track(vals[3:4])
    s.track(vals[4:24])  # warm-up of every shape the checked calls use
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        s.track(vals[24:25])
        s.track(vals[20:40])
        s.frame_trajectory()
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ------------------------------------------------------------------------------------------------ (7)
def test_track_refusals_change_nothing(cuda_model, monkeypatch):
    import vista_slam_b200.slam as S
    from vista_slam_b200.sessions import SLAMSessions
    vals = _frames_224(6)
    s = _slam(cuda_model)
    with pytest.raises(ValueError):
        s.track(vals[:1])  # nothing stepped
    s.step(vals[0])
    with pytest.raises(ValueError, match="no node"):
        s.track(vals[1:2])  # view 0 has no node until view 1 is stepped
    s.step(vals[1])
    s.step(vals[2])

    def no_launch(*a, **k):
        raise AssertionError("launched")

    monkeypatch.setattr(S, "encode_views", no_launch)
    monkeypatch.setattr(S, "regress_frames", no_launch)
    before = _state(s)
    other = dict(vals[3], rgb=torch.zeros(1, 3, 224, 240, device="cuda"))
    for args, kw in (([other], {}), (vals[3:4], {"kf": 3}), (vals[3:4], {"kf": -1}), ([vals[3], other], {})):
        with pytest.raises(ValueError):
            s.track(args, **kw)
    group = SLAMSessions("unused", VOCAB, 2, frontend=cuda_model, verbose=False, neighbor_edge_num=1, loop_edge_num=0)
    group[0].step(vals[0])
    group[0].step(vals[1])
    for bad in ({3: vals[2:3]}, [(0, vals[2:3]), (0, vals[3:4])], {1: vals[2:3]}, {0: [other]}):
        with pytest.raises(ValueError):
            group.track(bad)
    with pytest.raises(ValueError):
        group.track({0: vals[2:3]}, kfs={1: 0})
    monkeypatch.undo()
    after = _state(s)
    assert before["host"] == after["host"] and s._tracked == [] and group[0]._tracked == []
    for k in before:
        if k != "host":
            np.testing.assert_array_equal(before[k], after[k], err_msg=k)
    # reset clears the tracked frames
    s.track(vals[3:5])
    assert len(s.frame_trajectory()["names"]) == 2
    s.reset()
    assert s._tracked == []
