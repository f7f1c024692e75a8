"""Keyframe selection by sparse optical flow on the device, with the surface of vista_slam/flow_tracker.py::FlowTracker.

`compute_disparity(image)` decides whether a frame becomes a keyframe exactly as the reference does with
cv2.goodFeaturesToTrack + cv2.calcOpticalFlowPyrLK on the host, but runs Shi-Tomasi corners and pyramidal Lucas-Kanade
as CUDA kernels (csrc/flow.cu) and reads back only a few bytes of statistics: one host synchronisation per call, which
the caller's `if` needs anyway.  The frame may stay on the device from SLAM_image_only.process_image.  There is no CPU
path."""
import ctypes

import numpy as np
import torch

from . import _lib

MAX_CORNERS = _lib.FLOW_MAX_CORNERS
MIN_TRACKED = 10  # flow_tracker.py:28,45


def _as_device_frame(image, device=None):
    """-> (contiguous CUDA tensor (H, W), is_f32).  Accepts a numpy uint8 (H, W) (uploaded), a CUDA uint8 (H, W), or the
    CUDA fp32 gray (1, H, W) / (H, W) in [0, 1] of SLAM_image_only.process_image."""
    if isinstance(image, np.ndarray):
        if image.dtype != np.uint8 or image.ndim != 2:
            raise ValueError("expected an (H, W) uint8 frame")
        if not torch.cuda.is_available():
            raise RuntimeError("the flow tracker runs on CUDA only; no CUDA device is available")
        image = torch.from_numpy(np.ascontiguousarray(image)).to(device or "cuda", non_blocking=True)
    if not isinstance(image, torch.Tensor):
        raise TypeError("expected a numpy array or a torch tensor")
    if not image.is_cuda:
        raise RuntimeError("the flow tracker runs on CUDA only: pass a CUDA tensor or a numpy array")
    if image.dtype == torch.float32:
        if image.dim() == 3 and image.shape[0] == 1:
            image = image[0]
        is_f32 = 1
    elif image.dtype == torch.uint8:
        is_f32 = 0
    else:
        raise ValueError("expected a uint8 frame or an fp32 gray in [0, 1]")
    if image.dim() != 2:
        raise ValueError("expected an (H, W) frame")
    return image.contiguous(), is_f32


class _Tracker:
    """Owner of one C tracker handle (one frame size, one device)."""

    def __init__(self, H, W, device):
        self.H, self.W, self.device = H, W, device
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().sta_flow_create(H, W, ctypes.byref(h)), "sta_flow_create")
        self.h = h
        self.stats = _lib.StaFlowStats()

    def __del__(self):
        if getattr(self, "h", None) and _lib._lib is not None:
            _lib.lib().sta_flow_destroy(self.h)
            self.h = None


class FlowTracker:
    def __init__(self, min_disparity):
        self.min_disparity = min_disparity  # minimum mean disparity (pixels) that makes a new keyframe
        self._tracker = None
        self.reset()

    def reset(self):
        self.last_kf = None
        self.kf_gray = None
        self.last_mean_disparity = None
        self._kf_pts = None  # cached read-back of the keyframe corners

    @property
    def kf_pts(self):
        """Keyframe corners, (N, 1, 2) fp32 CUDA in selection order, or None when the keyframe has none (as
        cv2.goodFeaturesToTrack returns).  Reading it synchronises the stream."""
        if self.last_kf is None:
            return None
        if self._kf_pts is None:
            t = self._tracker
            pts = torch.empty(MAX_CORNERS, 2, dtype=torch.float32, device=t.device)
            cnt = torch.empty(1, dtype=torch.int32, device=t.device)
            with torch.cuda.device(t.device):
                _lib.check(_lib.lib().sta_flow_keyframe_points(t.h, _lib.ptr(pts), _lib.ptr(cnt), _lib.cur_stream()),
                           "sta_flow_keyframe_points")
            n = int(cnt.item())
            self._kf_pts = (pts[:n].reshape(n, 1, 2),) if n else (None,)
        return self._kf_pts[0]

    def _tracker_for(self, frame):
        H, W = frame.shape
        t = self._tracker
        if t is None or (t.H, t.W) != (H, W) or t.device != frame.device:
            t = self._tracker = _Tracker(H, W, frame.device)
        return t

    def initialize_keyframe(self, image):
        frame, is_f32 = _as_device_frame(image)
        t = self._tracker_for(frame)
        with torch.cuda.device(frame.device):
            _lib.check(_lib.lib().sta_flow_set_keyframe(t.h, _lib.ptr(frame), is_f32, _lib.cur_stream()),
                       "sta_flow_set_keyframe")
        self._set_keyframe(image, t)

    def _set_keyframe(self, image, t):
        self.last_kf = image
        self._kf_pts = None
        gray = torch.empty(t.H, t.W, dtype=torch.uint8, device=t.device)
        with torch.cuda.device(t.device):
            _lib.check(_lib.lib().sta_flow_keyframe_level0(t.h, _lib.ptr(gray), None, _lib.cur_stream()),
                       "sta_flow_keyframe_level0")
        self.kf_gray = gray

    def compute_disparity(self, image, visualize=False):
        """flow_tracker.py:26-66.  True when `image` becomes the new keyframe:
          1. no keyframe yet, or the keyframe has fewer than 10 corners;
          2. fewer than 10 keyframe corners were tracked into `image`;
          3. the mean disparity exceeds min_disparity.
        Cases 1-3 re-initialise the keyframe from `image`.

        The mean disparity is the reference's quantity as written: its points are (N, 1, 2), so
        np.linalg.norm(good_next - good_kf, axis=1) runs over the axis of size 1 and returns |dx| and |dy| separately.
        It is therefore the mean of the 2M absolute components |dx|, |dy| of the M tracked points, not their mean
        Euclidean displacement (a 3-pixel shift in x gives about 1.5, not 3).  It is kept in last_mean_disparity
        (None when the call did not track).

        One host synchronisation: the statistics read that this `if` needs."""
        if visualize:
            raise NotImplementedError("visualize=True draws with cv2.imshow; the device tracker has no UI")
        self.last_mean_disparity = None
        if self.last_kf is None:
            self.initialize_keyframe(image)
            return True
        frame, is_f32 = _as_device_frame(image, self._tracker.device)
        t = self._tracker
        if tuple(frame.shape) != (t.H, t.W):
            raise ValueError("frame size %s differs from the keyframe's %s" % (tuple(frame.shape), (t.H, t.W)))
        with torch.cuda.device(frame.device):
            _lib.check(_lib.lib().sta_flow_track(t.h, _lib.ptr(frame), is_f32, ctypes.byref(t.stats), _lib.cur_stream()),
                       "sta_flow_track")
        s = t.stats
        if s.n_corners < MIN_TRACKED or s.n_tracked < MIN_TRACKED:
            self._promote(image, t)
            return True
        self.last_mean_disparity = float(s.mean_disparity)
        if self.last_mean_disparity > self.min_disparity:
            self._promote(image, t)
            return True
        return False

    def _promote(self, image, t):
        with torch.cuda.device(t.device):
            _lib.check(_lib.lib().sta_flow_promote(t.h, _lib.cur_stream()), "sta_flow_promote")
        self._set_keyframe(image, t)


def _scratch(H, W, device):
    n = _lib.lib().sta_flow_scratch_bytes(H, W)
    if n == 0:
        raise ValueError("frame sides must be in [32, 2048], got %dx%d" % (H, W))
    return torch.empty(n, dtype=torch.uint8, device=device)


def good_features_to_track(gray):
    """cv2.goodFeaturesToTrack(gray, maxCorners=1000, qualityLevel=0.01, minDistance=8, blockSize=7) on the device:
    (N, 1, 2) fp32 CUDA, or None when there is no corner (synchronises to read N)."""
    frame, is_f32 = _as_device_frame(gray)
    if is_f32:
        raise ValueError("expected a uint8 frame")
    H, W = frame.shape
    scratch = _scratch(H, W, frame.device)
    pts = torch.empty(MAX_CORNERS, 2, dtype=torch.float32, device=frame.device)
    cnt = torch.empty(1, dtype=torch.int32, device=frame.device)
    with torch.cuda.device(frame.device):
        _lib.check(_lib.lib().sta_op_good_features(_lib.ptr(frame), H, W, _lib.ptr(pts), _lib.ptr(cnt), _lib.ptr(scratch),
                                                   _lib.cur_stream()), "sta_op_good_features")
    n = int(cnt.item())
    return pts[:n].reshape(n, 1, 2) if n else None


def calc_optical_flow_pyr_lk(prev, nxt, pts):
    """cv2.calcOpticalFlowPyrLK(prev, nxt, pts, None, winSize=(21, 21), maxLevel=3,
    criteria=(EPS|COUNT, 30, 0.01)) on the device -> (next_pts (N, 1, 2) fp32, status (N, 1) uint8), CUDA tensors."""
    a, fa = _as_device_frame(prev)
    b, fb = _as_device_frame(nxt, a.device)
    if fa or fb:
        raise ValueError("expected uint8 frames")
    if a.shape != b.shape:
        raise ValueError("the two frames differ in size")
    H, W = a.shape
    p = torch.as_tensor(pts, dtype=torch.float32).to(a.device).reshape(-1, 2).contiguous()
    n = p.shape[0]
    scratch = _scratch(H, W, a.device)
    out = torch.empty(n, 2, dtype=torch.float32, device=a.device)
    st = torch.empty(n, dtype=torch.uint8, device=a.device)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().sta_op_lk_track(_lib.ptr(a), _lib.ptr(b), H, W, _lib.ptr(p), n, _lib.ptr(out), _lib.ptr(st),
                                              _lib.ptr(scratch), _lib.cur_stream()), "sta_op_lk_track")
    return out.reshape(n, 1, 2), st.reshape(n, 1)
