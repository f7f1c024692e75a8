"""Keyframe selection by sparse optical flow on the device, with the surface of vista_slam/flow_tracker.py::FlowTracker.

`compute_disparity(image)` decides whether a frame becomes a keyframe exactly as the reference does with
cv2.goodFeaturesToTrack + cv2.calcOpticalFlowPyrLK on the host, but runs Shi-Tomasi corners and pyramidal Lucas-Kanade
as CUDA kernels (csrc/flow.cu) and reads back only a few bytes of statistics: one host synchronisation per call, which
the caller's `if` needs anyway.  The frame may stay on the device from SLAM_image_only.process_image.  There is no CPU
path.

`compute_disparities(frames)` and `compute_disparities_group(trackers, frames_per_tracker)` make the same decisions
for many frames and many trackers in rounds: every pending frame (at most ROUND per tracker) is tracked against its
tracker's current keyframe in one launch per stage and one host synchronisation.  The frames after a keyframe depend
on each other only through that keyframe, so the first frame of a round that meets a promotion condition is the frame
the one-frame loop would promote; the frames after it are tracked again, against the new keyframe, in the next
round, reusing their pyramids."""
import ctypes

import numpy as np
import torch

from . import _lib

MAX_CORNERS = _lib.FLOW_MAX_CORNERS
MIN_TRACKED = 10  # flow_tracker.py:28,45
# frames per tracker per round of compute_disparities: a promotion wastes the rest of its round, and a round costs
# about one launch sequence whatever its length (tools/flow_batch_stream.py's sweep, DESIGN.md section 5)
ROUND = 16


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
    """Owner of one C tracker handle (one frame size, one device), with the one-element tables of its one-frame group
    calls."""

    def __init__(self, H, W, device):
        self.H, self.W, self.device = H, W, device
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().sta_flow_create(H, W, ctypes.byref(h)), "sta_flow_create")
        self.h = h
        self.group = (ctypes.c_void_p * 1)(h.value)
        self.frame0 = (ctypes.c_int * 1)(0)
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
        return self._tracker_of_size(*frame.shape, frame.device)

    def _tracker_of_size(self, H, W, device):
        t = self._tracker
        if t is None or (t.H, t.W) != (H, W) or t.device != device:
            t = self._tracker = _Tracker(H, W, device)
        return t

    def initialize_keyframe(self, image):
        frame, is_f32 = _as_device_frame(image)
        t = self._tracker_for(frame)
        with torch.cuda.device(frame.device):
            _lib.check(_lib.lib().sta_flow_set_keyframe_group(t.group, 1, _lib.ptr(frame), is_f32, _lib.cur_stream()),
                       "sta_flow_set_keyframe_group")
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
            _lib.check(_lib.lib().sta_flow_track_group(t.group, 1, None, _lib.ptr(frame), is_f32, ctypes.byref(t.stats),
                                                       _lib.cur_stream()), "sta_flow_track_group")
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
            _lib.check(_lib.lib().sta_flow_promote_group(t.group, 1, t.frame0, _lib.cur_stream()), "sta_flow_promote_group")
        self._set_keyframe(image, t)

    def compute_disparities(self, frames):
        """compute_disparity over `frames` in order -> list of bools, leaving the tracker exactly as
        [self.compute_disparity(f) for f in frames] would (last_kf, kf_gray, kf_pts, last_mean_disparity, and the
        keyframe on the device), so calls chain and mix with compute_disparity.  `frames` is a list of frames of one
        size and type in any form compute_disparity accepts, or a stacked (F, H, W) uint8 / (F, 1, H, W) fp32 CUDA
        tensor.  One host synchronisation per round (see compute_disparities_group); kf_gray is copied out only for
        the last keyframe."""
        return compute_disparities_group([self], [frames])[0]


class _Frames:
    """One tracker's frames of a group call: their size and type (read without touching the device), frame i as the
    caller passed it (what last_kf keeps), and all of them as one contiguous (F, H, W) CUDA tensor."""

    def __init__(self, frames):
        self.stacked = isinstance(frames, torch.Tensor)
        if self.stacked:
            if frames.dtype == torch.uint8 and frames.dim() == 3:
                self.is_f32 = 0
            elif frames.dtype == torch.float32 and frames.dim() == 4 and frames.shape[1] == 1:
                self.is_f32 = 1
            else:
                raise ValueError("expected stacked frames (F, H, W) uint8 or (F, 1, H, W) fp32")
            self.items = frames
            self.n = frames.shape[0]
            self.H, self.W = frames.shape[-2:]
            return
        self.items = list(frames)
        self.n = len(self.items)
        info = {_frame_info(x) for x in self.items}
        if len(info) > 1:
            raise ValueError("all frames of a call must have the same size and type")
        self.H, self.W, self.is_f32 = info.pop() if info else (0, 0, 0)

    def device(self):
        """The CUDA device the frames are on, None for host frames."""
        x = self.items if self.stacked else next((x for x in self.items if isinstance(x, torch.Tensor)), None)
        return x.device if x is not None and x.is_cuda else None

    def on_device(self, device):
        if self.stacked:
            if not self.items.is_cuda:
                raise RuntimeError("the flow tracker runs on CUDA only: pass a CUDA tensor or numpy arrays")
            return (self.items[:, 0] if self.is_f32 else self.items).contiguous()
        if all(isinstance(x, np.ndarray) for x in self.items):  # one upload
            return torch.from_numpy(np.stack(self.items)).to(device, non_blocking=True)
        return torch.stack([_as_device_frame(x, device)[0] for x in self.items])


def _frame_info(image):
    """(H, W, is_f32) of a frame compute_disparity accepts, read without touching the device."""
    if isinstance(image, np.ndarray):
        if image.dtype != np.uint8 or image.ndim != 2:
            raise ValueError("expected an (H, W) uint8 frame")
        return image.shape[0], image.shape[1], 0
    if not isinstance(image, torch.Tensor):
        raise TypeError("expected a numpy array or a torch tensor")
    shape = tuple(image.shape)
    if image.dtype == torch.float32:
        shape = shape[1:] if len(shape) == 3 and shape[0] == 1 else shape
    elif image.dtype != torch.uint8:
        raise ValueError("expected a uint8 frame or an fp32 gray in [0, 1]")
    if len(shape) != 2:
        raise ValueError("expected an (H, W) frame")
    return shape[0], shape[1], int(image.dtype == torch.float32)


def compute_disparities_group(trackers, frames_per_tracker):
    """compute_disparities on each tracker with its own frames -> one list of bools per tracker; each tracker ends as
    its own compute_disparities(frames) would leave it.  Trackers that have never seen a frame take their first frame
    as the keyframe, together, in one launch sequence.  Then, in rounds, the next frames of every tracker (at most
    ROUND each; the frames after a promotion come first again) are tracked against their keyframes in one launch per
    stage with one read-back for all of them; a tracker's round ends at its first promotion, and the promotions of a
    round are enqueued together without a synchronisation.

    The trackers must be distinct, and all frames of one size and type, stacked or listed as compute_disparities takes
    them.  A repeated tracker, frames of different sizes or types, or a size other than a tracker's keyframe raises
    ValueError before anything runs, and no tracker changes."""
    trackers = list(trackers)
    frames = [_Frames(x) for x in frames_per_tracker]
    if len(frames) != len(trackers):
        raise ValueError("one frame list per tracker")
    if len({id(t) for t in trackers}) != len(trackers):
        raise ValueError("a tracker appears twice in the group")
    busy = [k for k, fr in enumerate(frames) if fr.n]
    out = [[] for _ in trackers]
    if not busy:
        return out
    if len({(frames[k].H, frames[k].W) for k in busy}) > 1:
        raise ValueError("all frames of a group must have the same size")
    if len({frames[k].is_f32 for k in busy}) > 1:
        raise ValueError("all frames of a group must have the same type")
    H, W, is_f32 = frames[busy[0]].H, frames[busy[0]].W, frames[busy[0]].is_f32
    for k in busy:
        t = trackers[k]._tracker
        if trackers[k].last_kf is not None and (t.H, t.W) != (H, W):
            raise ValueError("frame size %s differs from the keyframe's %s (tracker %d)" % ((H, W), (t.H, t.W), k))
    devices = {trackers[k]._tracker.device for k in busy if trackers[k].last_kf is not None}
    devices |= {d for d in (frames[k].device() for k in busy) if d is not None}
    if len(devices) > 1:
        raise ValueError("the trackers and frames of a group must be on one device")
    if not torch.cuda.is_available():
        raise RuntimeError("the flow tracker runs on CUDA only; no CUDA device is available")
    device = devices.pop() if devices else torch.device("cuda", torch.cuda.current_device())

    L = _lib.lib()
    dev = {k: frames[k].on_device(device) for k in busy}
    pos = {k: 0 for k in busy}       # the tracker's next undecided frame
    held = {k: 0 for k in busy}      # frames from pos on whose pyramids the tracker holds
    mean = {k: None for k in busy}   # last_mean_disparity after the tracker's newest decided frame
    kf_at = {k: None for k in busy}  # the tracker's newest keyframe in this call
    with torch.cuda.device(device):
        stream = _lib.cur_stream()
        fresh = [k for k in busy if trackers[k].last_kf is None]
        if fresh:
            hs = [trackers[k]._tracker_of_size(H, W, device).h.value for k in fresh]
            first = torch.stack([dev[k][0] for k in fresh]) if len(fresh) > 1 else dev[fresh[0]][:1]
            _lib.check(L.sta_flow_set_keyframe_group((ctypes.c_void_p * len(hs))(*hs), len(hs), _lib.ptr(first), is_f32,
                                                     stream), "sta_flow_set_keyframe_group")
            for k in fresh:
                out[k].append(True)
                pos[k], kf_at[k] = 1, 0
        while True:
            active = [k for k in busy if pos[k] < frames[k].n]
            if not active:
                break
            hs, flags, new, counts = [], [], [], []
            for k in active:
                m, h = min(ROUND, frames[k].n - pos[k]), held[k]
                hs += [trackers[k]._tracker.h.value] * m
                flags += [1] * h + [0] * (m - h)
                if h < m:
                    new.append(dev[k][pos[k] + h:pos[k] + m])
                counts.append(m)
            F = len(hs)
            new = None if not new else new[0] if len(new) == 1 else torch.cat(new)
            stats = (_lib.StaFlowStats * F)()
            _lib.check(L.sta_flow_track_group((ctypes.c_void_p * F)(*hs), F, (ctypes.c_int * F)(*flags), _lib.ptr(new),
                                              is_f32, stats, stream), "sta_flow_track_group")
            promoted, f = [], 0
            for k, m in zip(active, counts):
                for j in range(m):
                    s = stats[f + j]
                    if s.n_corners < MIN_TRACKED or s.n_tracked < MIN_TRACKED:
                        mean[k], promote = None, True
                    else:
                        mean[k] = float(s.mean_disparity)
                        promote = mean[k] > trackers[k].min_disparity
                    out[k].append(promote)
                    if promote:
                        break
                f += m
                if promote:
                    promoted.append((trackers[k]._tracker.h.value, j))
                    kf_at[k], held[k] = pos[k] + j, m - j - 1
                    pos[k] += j + 1
                else:
                    held[k] = 0
                    pos[k] += m
            if promoted:
                n = len(promoted)
                _lib.check(L.sta_flow_promote_group((ctypes.c_void_p * n)(*[h for h, _ in promoted]), n,
                                                    (ctypes.c_int * n)(*[j for _, j in promoted]), stream),
                           "sta_flow_promote_group")
    for k in busy:
        tr = trackers[k]
        tr.last_mean_disparity = mean[k]
        if kf_at[k] is not None:
            tr._set_keyframe(frames[k].items[kf_at[k]], tr._tracker)
    return out


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
