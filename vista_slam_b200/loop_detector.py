"""Loop-closure candidates on the device, with the surface of vista_slam/loop_detector.py::LoopDetector.

`detect_loop(image, farthest_neighbor)` returns the reference's [(j, similarity), ...] -- cv2.ORB_create() features,
the DBoW3 vocabulary transform and L1 scores against the earlier keyframes -- but runs ORB (csrc/orb.cu) and the
bag-of-words transform, database and scoring (csrc/bow.cu) as CUDA kernels, with one host synchronisation per call: the
read-back of the candidate list.  `detect_loops_group(detectors, ...)` does the same for many frames of one size and of
several detectors that share one `Vocabulary` (SLAM sessions stepped together) with one host synchronisation for all of
them, and `detect_loops(images, farthest_neighbors)` for many frames of one detector.  All three run one path, a group
of frames (csrc/bow.cu's sta_loop_add_frames_group / sta_loop_detect_group).  The frame may stay on the device from
SLAM_image_only.process_image.  There is no CPU path.

The vocabulary is a DBoW3 text file (what the shipped configs name, e.g. pretrains/ORBvoc.txt) or a DBoW3 binary file,
plain or QuickLZ-compressed, with binary descriptors and L1 scoring."""
import ctypes

import numpy as np
import torch

from . import _lib
from .flow_tracker import _as_device_frame

MAX_KEYPOINTS = _lib.ORB_MAX_KEYPOINTS


class Vocabulary:
    """A DBoW3 vocabulary parsed on the host and uploaded to the current CUDA device once."""

    def __init__(self, path):
        if not torch.cuda.is_available():
            raise RuntimeError("the loop detector runs on CUDA only; no CUDA device is available")
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().sta_vocab_load(str(path).encode(), ctypes.byref(h)), "sta_vocab_load")
        self.h = h
        info = (ctypes.c_int64 * 6)()
        _lib.check(_lib.lib().sta_vocab_info(h, info), "sta_vocab_info")
        self.k, self.L, self.scoring, self.weighting, self.n_nodes, self.n_words = (int(v) for v in info)

    def __del__(self):
        if getattr(self, "h", None) and _lib._lib is not None:
            _lib.lib().sta_vocab_destroy(self.h)
            self.h = None


class BowVector:
    """A view's normalised bag-of-words vector as stored in the device database (read back on demand)."""

    def __init__(self, detector, view):
        self._det, self.view = detector, view

    def to_numpy(self):
        """(word ids int32 ascending, values fp64)."""
        return self._det._view_vector(self.view)

    def __len__(self):
        return len(self.to_numpy()[0])


class LoopDetector:
    def __init__(self, vocab_path, loop_dist_min, loop_nms, loop_cand_thresh_neighbor):
        """vocab_path: a vocabulary file, or a loaded Vocabulary that several detectors share."""
        self.vocab = vocab_path if isinstance(vocab_path, Vocabulary) else Vocabulary(vocab_path)
        self.bow_feats = []
        self.loop_dist_min = loop_dist_min            # if node i has a loop edge to node j, then |i-j| > loop_dist_min
        self.loop_nms = loop_nms                      # non-maximum suppression for loop closure
        self.loop_cand_thresh_neighbor = loop_cand_thresh_neighbor  # candidates must beat the last x neighbours
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().sta_loop_create(self.vocab.h, loop_dist_min, loop_nms, loop_cand_thresh_neighbor,
                                               ctypes.byref(h)), "sta_loop_create")
        self._h = h
        self._group = (ctypes.c_void_p * 1)(h.value)  # the detector table of its own calls: a group of one
        self._device = torch.device("cuda", torch.cuda.current_device())

    def __del__(self):
        if getattr(self, "_h", None) and _lib._lib is not None:
            _lib.lib().sta_loop_destroy(self._h)
            self._h = None

    def compute_bow_feat(self, image):
        """loop_detector.py:13-21: ORB on `image`, its vector appended to the database and to bow_feats.  Returns a
        BowVector, or None when ORB finds no keypoint.  Deciding None synchronises the stream."""
        view = self._add(image)
        self.bow_feats.append(BowVector(self, view))
        if self._view_len(view) < 0:
            self.bow_feats[view] = None
        return self.bow_feats[view]

    def _add(self, image):
        frame, is_f32 = _as_device_frame(image, self._device)
        H, W = frame.shape
        with torch.cuda.device(frame.device):
            _lib.check(_lib.lib().sta_loop_add_frames_group(self._group, 1, _lib.ptr(frame), is_f32, H, W,
                                                            _lib.cur_stream()), "sta_loop_add_frames_group")
        return len(self.bow_feats)

    def detect_loop(self, image, farthest_neighbor):
        """loop_detector.py:23-50: [(j, similarity), ...] sorted by descending similarity (ties in descending j).
        One host synchronisation: the candidate list, which also tells whether this view's vector is None."""
        i = len(self.bow_feats)
        if not 0 <= farthest_neighbor <= i:
            raise ValueError("farthest_neighbor must be in [0, %d]" % i)
        self._add(image)
        # the view is in the device database from here on, so bow_feats gets its entry even if the detection fails
        self.bow_feats.append(BowVector(self, i))
        n = (ctypes.c_int * 2)()
        cap = max(i, 1)
        js = (ctypes.c_int64 * cap)()
        sims = (ctypes.c_double * cap)()
        with torch.cuda.device(self._device):
            _lib.check(_lib.lib().sta_loop_detect_group(self._group, 1, ctypes.byref(ctypes.c_int(farthest_neighbor)), n,
                                                        js, sims, cap, _lib.cur_stream()), "sta_loop_detect_group")
        if n[1] < 0:
            self.bow_feats[i] = None
        return [(int(js[k]), float(sims[k])) for k in range(n[0])]

    def detect_loops(self, images, farthest_neighbors):
        """detect_loop on each image in order, with its farthest neighbour, as one batch: ORB, the transform and the
        database append over all frames, one score and one detect launch over their rows and ONE host synchronisation.
        Returns the list of candidate lists.  The frames must share one size and type; a refusal comes before any
        launch."""
        return detect_loops_group([self], [images], [farthest_neighbors])[0]

    def similarities(self):
        """fp64 scores of the newest view against every earlier one from the last detect_loop (NaN where either
        vector is None).  Refused after a detect_loops_group with other detectors, until this detector's own next
        detection."""
        i = len(self.bow_feats) - 1
        out = np.zeros(max(i, 0), np.float64)
        if i > 0:
            with torch.cuda.device(self._device):
                _lib.check(_lib.lib().sta_loop_similarities(self._h, out.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                            i, _lib.cur_stream()), "sta_loop_similarities")
        return out

    def _view_len(self, view):
        n = ctypes.c_int()
        with torch.cuda.device(self._device):
            _lib.check(_lib.lib().sta_loop_view(self._h, view, None, None, 0, ctypes.byref(n), _lib.cur_stream()),
                       "sta_loop_view")
        return n.value

    def _view_vector(self, view):
        n = self._view_len(view)
        words = np.zeros(max(n, 0), np.int32)
        vals = np.zeros(max(n, 0), np.float64)
        ln = ctypes.c_int()
        with torch.cuda.device(self._device):
            _lib.check(_lib.lib().sta_loop_view(self._h, view, words.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                                vals.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), max(n, 0),
                                                ctypes.byref(ln), _lib.cur_stream()), "sta_loop_view")
        return words, vals


def detect_loops_group(detectors, images_per_detector, farthest_per_detector):
    """detect_loop on each detector's images in order, with their farthest neighbours, as one batch over all of them: ORB,
    the transform and the appends over every frame, one score and one detect launch over all rows and ONE host
    synchronisation.  The detectors must be distinct and share one Vocabulary, and all frames one size and type; a
    detector may have no frame.  Refusals come before any launch.  Returns, per detector, its list of candidate lists."""
    detectors = list(detectors)
    images = [list(x) for x in images_per_detector]
    far = [[int(f) for f in x] for x in farthest_per_detector]
    if not (len(images) == len(far) == len(detectors)):
        raise ValueError("one image list and one farthest_neighbor list per detector")
    if len({id(d) for d in detectors}) != len(detectors):
        raise ValueError("a detector appears twice in the group")
    if any(d.vocab is not detectors[0].vocab for d in detectors):
        raise ValueError("all detectors of a group must share one Vocabulary")
    owners = []
    for k, (det, ims, fs) in enumerate(zip(detectors, images, far)):
        if len(ims) != len(fs):
            raise ValueError("one farthest_neighbor per image (detector %d)" % k)
        i0 = len(det.bow_feats)
        for f, x in enumerate(fs):
            if not 0 <= x <= i0 + f:
                raise ValueError("farthest_neighbor of frame %d of detector %d must be in [0, %d]" % (f, k, i0 + f))
        owners += [k] * len(ims)
    out = [[] for _ in detectors]
    F = len(owners)
    if F == 0:
        return out
    device = detectors[owners[0]]._device
    frames = [_as_device_frame(im, device) for ims in images for im in ims]
    if any(t.shape != frames[0][0].shape or k != frames[0][1] for t, k in frames):
        raise ValueError("all frames of a batch must have the same size and type")
    batch = torch.stack([t for t, _ in frames]).contiguous() if F > 1 else frames[0][0]
    H, W = frames[0][0].shape
    dets = (ctypes.c_void_p * F)(*[detectors[k]._h.value for k in owners])
    L = _lib.lib()
    with torch.cuda.device(batch.device):
        _lib.check(L.sta_loop_add_frames_group(dets, F, _lib.ptr(batch), frames[0][1], H, W, _lib.cur_stream()),
                   "sta_loop_add_frames_group")
    # the views are in the device databases from here on, so bow_feats gets their entries even if detection fails
    first = {}
    for k in sorted(set(owners)):
        first[k] = len(detectors[k].bow_feats)
        detectors[k].bow_feats.extend(BowVector(detectors[k], first[k] + f) for f in range(len(images[k])))
    n = (ctypes.c_int * (2 * F))()
    cap = max(max(len(detectors[k].bow_feats) for k in owners) - 1, 1)
    js = (ctypes.c_int64 * (F * cap))()
    sims = (ctypes.c_double * (F * cap))()
    fars = [x for fs in far for x in fs]
    with torch.cuda.device(device):
        _lib.check(L.sta_loop_detect_group(dets, F, (ctypes.c_int * F)(*fars), n, js, sims, cap, _lib.cur_stream()),
                   "sta_loop_detect_group")
    for f, k in enumerate(owners):
        det = detectors[k]
        view = first[k] + len(out[k])
        if n[2 * f + 1] < 0:
            det.bow_feats[view] = None
        out[k].append([(int(js[f * cap + c]), float(sims[f * cap + c])) for c in range(n[2 * f])])
    return out


def orb_detect_and_compute(gray):
    """cv2.ORB_create().detectAndCompute(gray, None) on the device, in (level, y, x) order: dict of CUDA tensors
    xy (N, 2) int32 level pixels, level (N,), pts (N, 2) fp32 level-0 pixels, angle (N,) degrees, response (N,) Harris,
    desc (N, 32) uint8; plus 'scratch' and 'layout' for reading the intermediate stages (synchronises to read N)."""
    frame, is_f32 = _as_device_frame(gray)
    H, W = frame.shape
    nbytes = _lib.lib().sta_orb_scratch_bytes(H, W)
    if nbytes == 0:
        raise ValueError("frame sides must be in [32, 4096], got %dx%d" % (H, W))
    dev = frame.device
    M = MAX_KEYPOINTS
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    xy = torch.empty(M, 2, dtype=torch.int32, device=dev)
    level = torch.empty(M, dtype=torch.int32, device=dev)
    pts = torch.empty(M, 2, dtype=torch.float32, device=dev)
    angle = torch.empty(M, dtype=torch.float32, device=dev)
    resp = torch.empty(M, dtype=torch.float32, device=dev)
    desc = torch.empty(M, 32, dtype=torch.uint8, device=dev)
    cnt = torch.empty(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().sta_op_orb(_lib.ptr(frame), is_f32, H, W, _lib.ptr(xy), _lib.ptr(level), _lib.ptr(pts),
                                         _lib.ptr(angle), _lib.ptr(resp), _lib.ptr(desc), _lib.ptr(cnt), _lib.ptr(scratch),
                                         _lib.cur_stream()), "sta_op_orb")
    lay = (ctypes.c_int64 * 42)()
    _lib.check(_lib.lib().sta_orb_layout(H, W, lay), "sta_orb_layout")
    n = int(cnt.item())
    ctr = scratch[lay[6]:lay[6] + 16].view(torch.int32).cpu()
    if int(ctr[3]):
        raise RuntimeError("the frame has more ORB candidates or keypoints than the kernels hold")
    return {"xy": xy[:n], "level": level[:n], "pts": pts[:n], "angle": angle[:n], "response": resp[:n], "desc": desc[:n],
            "scratch": scratch, "layout": list(lay)}


def bow_transform(vocab, desc):
    """Per descriptor (N, 32) uint8 (CUDA or numpy): (word ids int32, weights fp64) CUDA tensors."""
    d = torch.as_tensor(np.asarray(desc) if isinstance(desc, np.ndarray) else desc)
    if d.dtype != torch.uint8 or d.dim() != 2 or d.shape[1] != 32:
        raise ValueError("expected (N, 32) uint8 binary descriptors")
    d = d.to("cuda").contiguous()
    n = d.shape[0]
    words = torch.empty(n, dtype=torch.int32, device=d.device)
    weights = torch.empty(n, dtype=torch.float64, device=d.device)
    with torch.cuda.device(d.device):
        _lib.check(_lib.lib().sta_op_bow_transform(vocab.h, _lib.ptr(d), n, _lib.ptr(words), _lib.ptr(weights),
                                                   _lib.cur_stream()), "sta_op_bow_transform")
    return words, weights


def bow_vector(vocab, words, weights):
    """The normalised BowVector of per-descriptor (word, weight) pairs: (word ids ascending, values) CUDA tensors."""
    n = words.shape[0]
    if n > MAX_KEYPOINTS:
        raise ValueError("at most %d descriptors" % MAX_KEYPOINTS)
    w_out = torch.empty(max(n, 1), dtype=torch.int32, device=words.device)
    v_out = torch.empty(max(n, 1), dtype=torch.float64, device=words.device)
    ln = torch.empty(1, dtype=torch.int32, device=words.device)
    with torch.cuda.device(words.device):
        _lib.check(_lib.lib().sta_op_bow_vector(vocab.h, _lib.ptr(words.contiguous()), _lib.ptr(weights.contiguous()), n,
                                                _lib.ptr(w_out), _lib.ptr(v_out), _lib.ptr(ln), _lib.cur_stream()),
                   "sta_op_bow_vector")
    m = int(ln.item())
    return w_out[:max(m, 0)], v_out[:max(m, 0)]


def bow_score(query, database):
    """L1 scores of query = (words, values) or None against a list of such vectors (None allowed): fp64 CUDA tensor,
    NaN where either side is None."""
    dev = torch.device("cuda", torch.cuda.current_device())
    nv = len(database)

    def cat(vs, idx, dtype):
        parts = [torch.as_tensor(v[idx]).to(dev, dtype) for v in vs if v is not None]
        return torch.cat(parts) if parts else torch.empty(1, dtype=dtype, device=dev)

    lens = [len(v[0]) if v is not None else -1 for v in database]
    starts = np.concatenate([[0], np.cumsum([max(x, 0) for x in lens])])[:-1] if nv else np.zeros(0)
    dbw, dbv = cat(database, 0, torch.int32), cat(database, 1, torch.float64)
    qw = cat([query], 0, torch.int32)
    qv = cat([query], 1, torch.float64)
    qlen = torch.tensor([len(query[0]) if query is not None else -1], dtype=torch.int32, device=dev)
    db_start = torch.as_tensor(np.asarray(starts, np.int64)).to(dev)
    db_len = torch.tensor(lens, dtype=torch.int32, device=dev)
    out = torch.empty(max(nv, 1), dtype=torch.float64, device=dev)
    _lib.check(_lib.lib().sta_op_bow_score(_lib.ptr(qw), _lib.ptr(qv), _lib.ptr(qlen), _lib.ptr(dbw), _lib.ptr(dbv),
                                           _lib.ptr(db_start), _lib.ptr(db_len), nv, _lib.ptr(out), _lib.cur_stream()),
               "sta_op_bow_score")
    return out[:nv]
