"""ctypes binding of libsta_b200.so (C ABI: include/sta_b200.h).

PyTorch is used only as the owner of device memory and streams: every call passes raw
device pointers (`tensor.data_ptr()`) and the current CUDA stream handle.  There is no
CPU fallback: if the shared library is missing this module raises at import of `lib()`.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("STA_B200_LIB") or os.path.join(_HERE, "csrc", "libsta_b200.so")  # env override: A/B timing of builds

EPI_BF16, EPI_GELU, EPI_F32, EPI_ROPE, EPI_PIXSHUF, EPI_HEAD, EPI_GELU_FP8 = range(7)
PRECISION_BF16, PRECISION_X3, PRECISION_FP8 = 0, 1, 2


class StaGemmDesc(Structure):
    _fields_ = [
        ("conv3x3", c_int), ("epi", c_int),
        ("A", c_void_p), ("lda", c_int64),
        ("W", c_void_p), ("ldw", c_int64),
        ("M", c_int), ("N", c_int), ("K", c_int),
        ("nimg", c_int), ("H", c_int), ("Wd", c_int), ("Cin", c_int),
        ("bias", c_void_p),
        ("out", c_void_p), ("ldo", c_int64),
        ("out2", c_void_p), ("resid", c_void_p), ("resid2", c_void_p),
        ("relu_main", c_int), ("rowmap_n", c_int),
        ("pos", c_void_p), ("rope_cols", c_int),
        ("ps_k", c_int), ("ps_cout", c_int), ("ps_h", c_int), ("ps_w", c_int),
        ("head_w", c_void_p), ("head_b", c_void_p), ("pts3d", c_void_p), ("conf", c_void_p),
        ("splitk_ws", c_void_p), ("splitk_ws_bytes", c_int64),
        ("split_precision", c_int),
        ("tile_n", c_int),
    ]


class StaGemmFp8Desc(Structure):
    _fields_ = [
        ("epi", c_int),
        ("A", c_void_p), ("lda", c_int64), ("a_scale", c_void_p),
        ("W", c_void_p), ("ldw", c_int64), ("w_scale", c_void_p),
        ("M", c_int), ("N", c_int), ("K", c_int),
        ("bias", c_void_p),
        ("out", c_void_p), ("ldo", c_int64),
        ("resid", c_void_p), ("out_scale", c_void_p),
        ("pos", c_void_p), ("rope_cols", c_int),
        ("splitk_ws", c_void_p), ("splitk_ws_bytes", c_int64),
    ]


FLOW_MAX_CORNERS = 1000
GRAPH_MAX_KEYFRAME_EDGES = 32
GRAPH_MAX_GROUP_KEYFRAMES = 32  # STA_GRAPH_MAX_GROUP_KEYFRAMES: keyframes per sta_graph_add_keyframes call
GRAPH_FLAG_NOT_SO3 = 1
GRAPH_MAX_TRACK_FRAMES = 4096  # STA_GRAPH_MAX_TRACK_FRAMES: frames per sta_graph_track_frames / _frame_poses call
ORB_MAX_KEYPOINTS = 4096
PG_DENSE_MAX_OPT = 3657  # STA_PG_DENSE_MAX_OPT: above it PoseGraphOpt takes the block-sparse route
PG_GROUP_MAX = 16  # STA_PG_GROUP_MAX: graphs per sta_pose_graph_lm_step_group call or sta_pg_group_plan
RENDER_MAX_RADIUS = 4  # STA_RENDER_MAX_RADIUS: largest point radius of sta_render
RENDER_MAX_SIDE = 8192  # cameras per sta_render call and output rows / columns
FUSION_BRICK = 8  # STA_FUSION_BRICK: samples per brick side
FUSION_BRICK_BITS = 21  # STA_FUSION_BRICK_BITS: bits per brick coordinate in a key
FUSION_MAX_BRICKS = 1 << 20  # STA_FUSION_MAX_BRICKS: bricks per sta_fusion_integrate / sta_fusion_mesh call
FUSION_MAX_SIDE = 65535  # views, rows and columns per sta_fusion_bricks / sta_fusion_integrate call


class StaPgGraph(Structure):
    _fields_ = [
        ("nodes", c_void_p), ("edges", c_void_p), ("meas", c_void_p), ("weights", c_void_p), ("opt_idx", c_void_p),
        ("nodes_out", c_void_p),
        ("num_nodes", c_int), ("num_edges", c_int), ("num_opt", c_int),
        ("damping", ctypes.c_double),
    ]


class StaPgSparseStep(Structure):
    _fields_ = [
        ("nodes", c_void_p), ("meas", c_void_p), ("weights", c_void_p), ("nodes_out", c_void_p),
        ("damping", ctypes.c_double), ("active", c_int),
    ]


class StaGraphKeyframe(Structure):
    _fields_ = [
        ("graph", c_void_p), ("view", c_int), ("n", c_int), ("node0", c_int), ("edge0", c_int), ("H", c_int),
        ("W", c_int), ("js", POINTER(c_int64)), ("cand", POINTER(c_int)), ("first_j", POINTER(c_int)),
        ("pose", c_void_p), ("pose_conf", c_void_p), ("confs", c_void_p), ("depths", c_void_p), ("intri", c_void_p),
        ("conf_mean", c_void_p),
    ]


class StaTap(Structure):
    _fields_ = [("name", c_char_p), ("dst", c_void_p), ("capacity", c_int64), ("written", c_int64), ("fired", c_int32)]


class StaFlowStats(Structure):
    _fields_ = [("n_corners", c_int32), ("n_tracked", c_int32), ("abs_sum", ctypes.c_double),
                ("mean_disparity", ctypes.c_double)]


_lib = None


def lib():
    """Load the shared library once; raise loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libsta_b200.so is missing (%s). Build it with `python -m vista_slam_b200.build`; "
            "the STA path has no CPU/PyTorch fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp, i, i64 = c_void_p, c_int, c_int64
    L.sta_last_error.restype = c_char_p
    L.sta_last_error.argtypes = []
    L.sta_version.restype = i
    L.sta_device_synchronize.restype = i
    L.sta_create.argtypes = [POINTER(vp)]
    L.sta_create_ex.argtypes = [POINTER(vp), i]
    L.sta_destroy.argtypes = [vp]
    L.sta_destroy.restype = None
    L.sta_load_tensor.argtypes = [vp, c_char_p, vp, POINTER(c_int64), i, i]
    L.sta_missing_tensors.argtypes = [vp]
    L.sta_weight_arena.argtypes = [vp, POINTER(vp), POINTER(c_int64)]
    L.sta_mark_all_loaded.argtypes = [vp]
    L.sta_weight_slot.argtypes = [vp, c_char_p, POINTER(vp), POINTER(c_int64), POINTER(vp)]
    L.sta_encode.argtypes = [vp, vp, i, i, i, i, vp, vp, vp]
    L.sta_decode.argtypes = [vp, vp, vp, vp, vp, i, i, POINTER(vp), POINTER(vp), vp]
    L.sta_head_pose.argtypes = [vp, vp, i, vp, vp, vp]
    L.sta_head_pts.argtypes = [vp, vp, vp, vp, vp, i, i, i, vp, vp, vp]
    L.sta_graph_replays.argtypes = [vp]
    L.sta_graph_replays.restype = i64
    L.sta_regress_pairs.argtypes = [vp, vp, vp, i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.sta_regress_pairs_begin.argtypes = [vp, vp, vp, i, i, i, vp, vp, vp]
    L.sta_regress_pairs_finish.argtypes = [vp, POINTER(c_int), i, vp, vp, vp, vp, vp, vp, vp]
    L.sta_forward_pairs.argtypes = [vp, vp, vp, i, i, i, i, vp, vp, vp, vp, vp]
    L.sta_forward_pairs_host.argtypes = [vp, vp, vp, i, i, i, i, vp, vp, vp, vp, vp]
    L.sta_launch_count.argtypes = [vp]
    L.sta_launch_count.restype = i64
    L.sta_device_bytes.argtypes = [vp]
    L.sta_device_bytes.restype = i64
    L.sta_profile.argtypes = [vp, i]
    L.sta_profile_read.argtypes = [vp, POINTER(ctypes.c_double), POINTER(c_int64), POINTER(ctypes.c_double)]
    L.sta_set_taps.argtypes = [vp, POINTER(StaTap), i]
    L.sta_op_gemm.argtypes = [POINTER(StaGemmDesc), vp]
    L.sta_op_gemm_fp8.argtypes = [POINTER(StaGemmFp8Desc), vp]
    L.sta_op_layernorm_fp8.argtypes = [vp, i, i, c_float, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.sta_op_quant_fp8.argtypes = [vp, i64, i, vp, vp, vp]
    L.sta_op_attention.argtypes = [vp, i64, i, vp, i64, i, vp, i64, i, vp, i64, i, i, i, i, i, c_float, vp]
    L.sta_op_attention_split.argtypes = L.sta_op_attention.argtypes
    L.sta_op_layernorm.argtypes = [vp, i, i, c_float, vp, vp, vp, vp, vp, vp, i, vp]
    L.sta_op_patch_im2col.argtypes = [vp, i, i, i, i, vp, vp]
    L.sta_op_upsample2x.argtypes = [vp, vp, i, i, i, i, vp]
    L.sta_op_im2col_3x3_s2.argtypes = [vp, vp, i, i, i, i, vp]
    L.sta_op_cast_f32_bf16.argtypes = [vp, vp, i64, i, i, vp]
    L.sta_preprocess_shape.argtypes = [i, i, i, i, i, i, POINTER(c_int)]
    L.sta_preprocess_geometry.argtypes = [i, i, i, i, i, i, POINTER(c_int)]
    L.sta_preprocess_coeffs.argtypes = [i, i, POINTER(c_int), POINTER(c_int), POINTER(c_int), i64]
    L.sta_preprocess_rgb8.argtypes = [vp, i, i, i, i, i, i, vp, vp, vp, vp]
    L.sta_preprocess_rgb8_many.argtypes = [vp, i, i, i, i, i, i, i, vp, vp, vp, vp]
    L.sta_pointmap_scratch_bytes.argtypes = [i]
    L.sta_pointmap_scratch_bytes.restype = ctypes.c_size_t
    L.sta_pointmap_consumers.argtypes = [vp, vp, i, i, i, i, vp, vp, vp, vp, vp]
    L.sta_depth_scale.argtypes = [vp, vp, vp, vp, i64, vp, vp, vp]
    L.sta_pose_graph_scratch_bytes.argtypes = [i, i, i]
    L.sta_pose_graph_scratch_bytes.restype = ctypes.c_size_t
    L.sta_pose_graph_lm_step.argtypes = [vp, i, vp, vp, vp, i, vp, i, ctypes.c_double, ctypes.c_double, ctypes.c_double, vp, vp,
                                         vp, vp]
    L.sta_pose_graph_group_scratch_bytes.argtypes = [POINTER(StaPgGraph), i]
    L.sta_pose_graph_group_scratch_bytes.restype = ctypes.c_size_t
    L.sta_pose_graph_lm_step_group.argtypes = [POINTER(StaPgGraph), i, ctypes.c_double, ctypes.c_double, vp, vp,
                                               ctypes.c_size_t, vp]
    L.sta_pg_plan_create.argtypes = [vp, i, i, vp, i, POINTER(vp)]
    L.sta_pg_plan_destroy.argtypes = [vp]
    L.sta_pg_plan_destroy.restype = None
    L.sta_pg_plan_info.argtypes = [vp, POINTER(c_int64)]
    L.sta_pg_plan_analyze.argtypes = [vp, i, i, vp, i, POINTER(c_int64), vp, vp, vp, vp, vp, vp]
    L.sta_pg_plan_last_delta.argtypes = [vp, vp, vp]
    L.sta_pose_graph_lm_step_sparse.argtypes = [vp, vp, vp, vp, ctypes.c_double, ctypes.c_double, ctypes.c_double, vp, vp,
                                                vp]
    L.sta_pg_group_plan_create.argtypes = [POINTER(vp), i, POINTER(vp)]
    L.sta_pg_group_plan_destroy.argtypes = [vp]
    L.sta_pg_group_plan_destroy.restype = None
    L.sta_pg_group_plan_info.argtypes = [vp, POINTER(c_int64)]
    L.sta_pose_graph_lm_step_sparse_group.argtypes = [vp, POINTER(StaPgSparseStep), ctypes.c_double, ctypes.c_double, vp,
                                                      vp]
    L.sta_flow_create.argtypes = [i, i, POINTER(vp)]
    L.sta_flow_destroy.argtypes = [vp]
    L.sta_flow_destroy.restype = None
    L.sta_flow_set_keyframe_group.argtypes = [POINTER(vp), i, vp, i, vp]
    L.sta_flow_track_group.argtypes = [POINTER(vp), i, POINTER(c_int), vp, i, POINTER(StaFlowStats), vp]
    L.sta_flow_promote_group.argtypes = [POINTER(vp), i, POINTER(c_int), vp]
    L.sta_flow_keyframe_points.argtypes = [vp, vp, vp, vp]
    L.sta_flow_keyframe_level0.argtypes = [vp, vp, vp, vp]
    L.sta_flow_scratch_bytes.argtypes = [i, i]
    L.sta_flow_scratch_bytes.restype = ctypes.c_size_t
    L.sta_op_good_features.argtypes = [vp, i, i, vp, vp, vp, vp]
    L.sta_op_lk_track.argtypes = [vp, vp, i, i, vp, i, vp, vp, vp, vp]
    L.sta_vocab_load.argtypes = [c_char_p, POINTER(vp)]
    L.sta_vocab_info.argtypes = [vp, POINTER(c_int64)]
    L.sta_vocab_destroy.argtypes = [vp]
    L.sta_vocab_destroy.restype = None
    L.sta_loop_create.argtypes = [vp, i, i, i, POINTER(vp)]
    L.sta_loop_destroy.argtypes = [vp]
    L.sta_loop_destroy.restype = None
    L.sta_loop_views.argtypes = [vp]
    L.sta_loop_add_frames_group.argtypes = [POINTER(vp), i, vp, i, i, i, vp]
    L.sta_loop_detect_group.argtypes = [POINTER(vp), i, POINTER(c_int), POINTER(c_int), POINTER(c_int64),
                                        POINTER(ctypes.c_double), i, vp]
    L.sta_loop_view.argtypes = [vp, i, POINTER(c_int32), POINTER(ctypes.c_double), i, POINTER(c_int), vp]
    L.sta_loop_similarities.argtypes = [vp, POINTER(ctypes.c_double), i, vp]
    L.sta_orb_scratch_bytes.argtypes = [i, i]
    L.sta_orb_scratch_bytes.restype = ctypes.c_size_t
    L.sta_orb_layout.argtypes = [i, i, POINTER(c_int64)]
    L.sta_op_orb.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.sta_op_orb_many.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.sta_op_bow_transform.argtypes = [vp, vp, i, vp, vp, vp]
    L.sta_op_bow_vector.argtypes = [vp, vp, vp, i, vp, vp, vp, vp]
    L.sta_op_bow_score.argtypes = [vp, vp, vp, vp, vp, vp, vp, i, vp, vp]
    L.sta_graph_create.argtypes = [i, i, i, i, i, POINTER(vp)]
    L.sta_graph_destroy.argtypes = [vp]
    L.sta_graph_destroy.restype = None
    L.sta_graph_tables.argtypes = [vp, POINTER(vp)]
    L.sta_graph_reset.argtypes = [vp, vp]
    L.sta_graph_flags.argtypes = [vp, POINTER(c_int)]
    L.sta_graph_add_keyframe.argtypes = [vp, i, i, POINTER(c_int64), POINTER(c_int), POINTER(c_int), i, i, i, i, vp, vp, vp, vp,
                                         vp, vp, vp]
    L.sta_graph_add_keyframes_scratch_bytes.argtypes = [POINTER(StaGraphKeyframe), i]
    L.sta_graph_add_keyframes_scratch_bytes.restype = ctypes.c_size_t
    L.sta_graph_add_keyframes.argtypes = [POINTER(StaGraphKeyframe), i, vp, ctypes.c_size_t, vp]
    L.sta_graph_replay_nodes.argtypes = [vp, i, POINTER(c_int), vp]
    L.sta_graph_track_frames_scratch_bytes.argtypes = [i]
    L.sta_graph_track_frames_scratch_bytes.restype = ctypes.c_size_t
    L.sta_graph_track_frames.argtypes = [vp, i, POINTER(c_int), vp, vp, vp, vp, vp, vp, vp, vp, vp, ctypes.c_size_t, vp]
    L.sta_graph_frame_poses.argtypes = [vp, i, POINTER(c_int), vp, vp, vp, vp, vp]
    L.sta_graph_export_scratch_bytes.argtypes = [i, i]
    L.sta_graph_export_scratch_bytes.restype = ctypes.c_size_t
    L.sta_graph_export.argtypes = [vp, i, i, c_float, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    f64, sz = ctypes.c_double, ctypes.c_size_t
    L.sta_render_scratch_bytes.argtypes = [i, i, i]
    L.sta_render_scratch_bytes.restype = sz
    L.sta_render.argtypes = [vp, vp, vp, vp, vp, vp, i, i, i, c_float, vp, vp, i, i, i, i, c_float, vp, vp, i,
                             POINTER(c_float), vp, sz, vp, vp, vp, vp]
    L.sta_fusion_bricks_scratch_bytes.argtypes = [i, i, i, i64]
    L.sta_fusion_bricks_scratch_bytes.restype = sz
    L.sta_fusion_bricks.argtypes = [vp, vp, vp, vp, vp, i, i, i, c_float, c_float, c_float, i64, vp, sz, vp, vp, vp]
    L.sta_fusion_integrate_scratch_bytes.argtypes = [i64, i]
    L.sta_fusion_integrate_scratch_bytes.restype = sz
    L.sta_fusion_integrate.argtypes = [vp, vp, vp, vp, vp, vp, i, i, i, c_float, vp, i64, c_float, c_float, vp, sz, vp,
                                       vp, vp, vp]
    L.sta_fusion_mesh_scratch_bytes.argtypes = [i64]
    L.sta_fusion_mesh_scratch_bytes.restype = sz
    L.sta_fusion_mesh.argtypes = [vp, i64, vp, vp, vp, c_float, c_float, i64, i64, vp, sz, vp, vp, vp, vp, vp]
    L.sta_raycast_scratch_bytes.argtypes = [i64]
    L.sta_raycast_scratch_bytes.restype = sz
    L.sta_raycast.argtypes = [vp, i64, vp, vp, vp, c_float, c_float, vp, vp, i, i, i, c_float, POINTER(c_float), vp, sz,
                              vp, vp, vp, vp, vp]
    L.sta_view_consistency.argtypes = [vp, vp, vp, i, i, i, c_float, vp, vp]
    L.sta_sort_scratch_bytes.argtypes = [i64]
    L.sta_sort_scratch_bytes.restype = sz
    L.sta_op_radix_sort.argtypes = [vp, vp, i64, i, vp, vp, vp, vp]
    L.sta_eval_clouds_scratch_bytes.argtypes = [i, i]
    L.sta_eval_clouds_scratch_bytes.restype = sz
    L.sta_eval_clouds.argtypes = [i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, c_float, vp, vp, vp, vp, vp]
    L.sta_voxel_scratch_bytes.argtypes = [i64]
    L.sta_voxel_scratch_bytes.restype = sz
    L.sta_voxel_down.argtypes = [vp, i64, f64, vp, POINTER(c_int64), vp, vp]
    L.sta_nn_create.argtypes = [vp, i64, POINTER(vp), vp]
    L.sta_nn_destroy.argtypes = [vp]
    L.sta_nn_destroy.restype = None
    L.sta_nn_query_scratch_bytes.argtypes = [i64]
    L.sta_nn_query_scratch_bytes.restype = sz
    L.sta_nn_query.argtypes = [vp, vp, i64, f64, vp, vp, vp, vp]
    L.sta_reduce_scratch_bytes.argtypes = []
    L.sta_reduce_scratch_bytes.restype = sz
    L.sta_op_moments.argtypes = [vp, vp, vp, i64, vp, vp, vp]
    L.sta_icp_scratch_bytes.argtypes = [i64]
    L.sta_icp_scratch_bytes.restype = sz
    L.sta_icp_moments.argtypes = [vp, vp, vp, i64, f64, vp, vp, vp]
    L.sta_transform_points.argtypes = [vp, i64, POINTER(f64), vp]
    L.sta_sum_sq_clipped.argtypes = [vp, i64, f64, vp, vp, vp]
    _lib = L
    return L


def check(rc, what="sta call"):
    if rc != 0:
        msg = lib().sta_last_error()
        raise RuntimeError("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))


def ptr(t):
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return None if t is None else c_void_p(t.data_ptr())


def cur_stream():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)
