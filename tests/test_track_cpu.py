"""CPU companion of tests/test_track_gpu.py: the float64 oracle of a tracked frame's pose (OnlineSLAM.track,
sta_graph_track_frames / sta_graph_frame_poses) on closed-form cases, its bounds shown to accept the fp32 mirror of the
device algebra, the C refusals that need no device, and the public surface.

A tracked frame's pose is pose[a] * Sim3(0, id, s) * Sim3(T), two sim3_mul products, then the export's quaternion ->
4x4.  Bounds (u = 2^-24, helpers of tests/test_slam_graph_fp64_cpu.py):
  * translation, quaternion and scale of the product: 2 C_SIM3 u S_c per component, S_c the magnitude of the chain
    (the first product's error enters the second with at most its magnitude);
  * the 4x4 rotation: C_ROT u of the export's magnitude plus 8 |q| max dq, the quaternion error carried through the
    degree-2 formula.
"""
import ctypes

import numpy as np
import pytest

from test_slam_graph_fp64_cpu import (C_ROT, C_SIM3, CLAMP, F32, _ratio, pose44, quat_to_rot_export, rot, rot_to_quat,
                                      scale_errs, scale_maps, scale_stats_f32, scale_stats_ref, sim3, sim3_mul64,
                                      sim3_mul_f32)


def track_ref(pose_a, s, T):
    """fp64 pose of a tracked frame from the device's stored values: the anchor's pose [8], the scale edge s and T_fk
    as [t | q | s] [8].  Returns (P [4,4] with the scale dropped, scale, bound [4,4], scale bound)."""
    S = np.array([0, 0, 0, 0, 0, 0, 1, np.float32(s)], np.float32)
    j, Sj, _ = sim3_mul64(pose_a, S)
    p, _, _ = sim3_mul64(j, T)
    _, Sc, _ = sim3_mul64(Sj, np.abs(np.asarray(T, np.float64)))  # the chain's magnitude
    b = 2 * C_SIM3 * F32 * np.asarray(Sc)
    R, M = quat_to_rot_export(p[3:7], np.float64)
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = R, p[:3]
    B = np.zeros((4, 4))
    B[:3, :3] = C_ROT * F32 * M + 8 * np.abs(p[3:7]).max() * b[3:7].max()
    B[:3, 3] = b[:3]
    return P, p[7], B, b[7]


def track_f32(pose_a, s, T):
    """The device's product in fp32 operation by operation (no FMA contraction), then the export's 4x4."""
    S = np.array([0, 0, 0, 0, 0, 0, 1, s], np.float32)
    p = sim3_mul_f32(sim3_mul_f32(pose_a, S), T)
    R, _ = quat_to_rot_export(p[3:7], np.float32)
    P = np.eye(4, dtype=np.float32)
    P[:3, :3], P[:3, 3] = R, p[:3]
    return P, p[7]


def track_err(P_got, scale_got, pose_a, s, T):
    """max over the 4x4 and the scale of |got - ref| / bound."""
    P, sc, B, bs = track_ref(pose_a, s, T)
    return max(_ratio(np.abs(np.asarray(P_got, np.float64) - P), B), _ratio(abs(float(scale_got) - sc), bs))


def measurement(M):
    """T_fk as the device stores it: [t | rot_to_quat(R) | 1] (fp32) and whether R passed the SO(3) check."""
    q, ok, _, _ = rot_to_quat(M)
    M = np.asarray(M, np.float32)
    return np.concatenate([[M[0, 3], M[1, 3], M[2, 3]], q.astype(np.float32), [1.0]]).astype(np.float32), ok


IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1, 1], np.float32)


def test_identity_anchor_and_unit_scale_give_T():
    M = pose44(rot([1, 2, 3], 0.7), t=(0.3, -0.2, 0.5))
    T, ok = measurement(M)
    P, sc, B, _ = track_ref(IDENTITY, 1.0, T)
    assert ok and sc == 1.0
    np.testing.assert_allclose(P, M.astype(np.float64), atol=1e-6)
    assert (B >= 0).all()


def test_pure_scale_multiplies_translation_and_scale():
    pose_a = sim3([1.0, -2.0, 0.5], [0, 0, 1], 0.0, 2.0)
    T, _ = measurement(pose44(np.eye(3), t=(1.0, 2.0, 3.0)))
    P, sc, _, _ = track_ref(pose_a, 0.5, T)
    np.testing.assert_allclose(P[:3, 3], [1.0 + 1.0, -2.0 + 2.0, 0.5 + 3.0], atol=1e-12)  # t_a + s_a s t_T
    np.testing.assert_allclose(P[:3, :3], np.eye(3), atol=1e-12)
    assert abs(sc - 1.0) < 1e-12


def test_known_rotation_composes():
    pose_a = sim3([0.0, 0.0, 0.0], [0, 0, 1], np.pi / 2, 1.0)
    T, _ = measurement(pose44(rot([0, 0, 1], np.pi / 2), t=(1.0, 0.0, 0.0)))
    P, sc, _, _ = track_ref(pose_a, 3.0, T)
    np.testing.assert_allclose(P[:3, :3], rot([0, 0, 1], np.pi), atol=1e-6)
    np.testing.assert_allclose(P[:3, 3], [0.0, 3.0, 0.0], atol=1e-6)  # R_a (s t_T)
    assert abs(sc - 3.0) < 1e-6


def test_clamp_of_the_scale_reduction():
    """A frame whose confidences all sit under the clamp: w = 1e-6f everywhere, so s = sum Di Dj / sum Di^2."""
    r = np.random.default_rng(4)
    Di, Dj = r.uniform(0.5, 2, 5000).astype(np.float32), r.uniform(0.5, 2, 5000).astype(np.float32)
    ci = cj = np.full(5000, 1e-4, np.float32)
    stats = scale_stats_ref(Di, Dj, ci, cj)
    want = float((Di.astype(np.float64) * Dj).sum() / (Di.astype(np.float64) ** 2).sum())
    assert abs(stats[0] / stats[1] - want) <= 1e-6 * want  # the clamp weight cancels
    assert float(np.float32(ci[0]) * np.float32(cj[0])) < CLAMP
    s, c = scale_stats_f32(Di, Dj, ci, cj)
    assert max(scale_errs(s, c, stats)) <= 1.0


@pytest.mark.parametrize("seed", range(6))
def test_bound_accepts_the_fp32_chain(seed):
    r = np.random.default_rng(seed)
    worst = 0.0
    for _ in range(300):
        q = r.standard_normal(4)
        q /= np.linalg.norm(q)
        pose_a = np.concatenate([r.uniform(-50, 50, 3), q, [10 ** r.uniform(-1, 1)]]).astype(np.float32)
        axis = r.standard_normal(3)
        T, _ = measurement(pose44(rot(axis, r.uniform(0, np.pi)), t=r.uniform(-2, 2, 3)))
        s = np.float32(10 ** r.uniform(-1, 1))
        P, sc = track_f32(pose_a, s, T)
        worst = max(worst, track_err(P, sc, pose_a, s, T))
    assert worst <= 0.5, worst


def test_bound_rejects_a_wrong_order():
    """T * Sim3(s) instead of Sim3(s) * T: the scale no longer multiplies T's translation."""
    pose_a = sim3([1.0, 2.0, 3.0], [1, 2, 3], 0.7, 1.3)
    T, _ = measurement(pose44(rot([0, 1, 0], 0.4), t=(0.5, -0.3, 0.2)))
    S = np.array([0, 0, 0, 0, 0, 0, 1, 0.8], np.float32)
    p = sim3_mul_f32(sim3_mul_f32(pose_a, T), S)
    R, _ = quat_to_rot_export(p[3:7], np.float32)
    P = np.eye(4, dtype=np.float32)
    P[:3, :3], P[:3, 3] = R, p[:3]
    assert track_err(P, p[7], pose_a, 0.8, T) > 1.0


def test_c_refusals_without_a_device():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    one = (ctypes.c_int * 1)(0)
    assert L.sta_graph_track_frames_scratch_bytes(0) == 0
    assert L.sta_graph_track_frames_scratch_bytes(_lib.GRAPH_MAX_TRACK_FRAMES + 1) == 0
    assert L.sta_graph_track_frames_scratch_bytes(3) == 3 * 64 * 8 * 8
    for F in (0, -1, _lib.GRAPH_MAX_TRACK_FRAMES + 1):
        assert L.sta_graph_track_frames(None, F, one, *[None] * 8, None, 0, None) != 0
        assert b"frames per call" in L.sta_last_error()
        assert L.sta_graph_frame_poses(None, F, one, None, None, None, None, None) != 0
        assert b"frames per call" in L.sta_last_error()
    assert L.sta_graph_track_frames(None, 1, one, *[None] * 8, None, 0, None) != 0
    assert b"null argument" in L.sta_last_error()
    assert L.sta_graph_frame_poses(None, 1, None, None, None, None, None, None) != 0
    assert b"null argument" in L.sta_last_error()


def test_track_surface():
    from vista_slam_b200.sessions import SLAMSessions
    from vista_slam_b200.slam import OnlineSLAM, track_frames
    for name in ("track", "frame_trajectory", "save_frame_trajectory"):
        assert callable(getattr(OnlineSLAM, name))
    assert callable(SLAMSessions.track) and callable(track_frames)
