"""Keyframe step of the SLAM frontend (SURVEY.md section 8(f) rank 1).

`OnlineSLAM` (vista_slam/slam.py) calls the STA model once per keyframe for the encoder (add_view, :142-151) and once
per candidate edge for decoder + heads (regress_two_views, :153-189), each edge with its own host synchronisation
(`rel_pose_conf_ij < thres`, :169).  `KeyframeFrontend` keeps the same per-view cache (encoder features on the GPU)
but regresses ALL edges of a keyframe in one batched call (sta_regress_pairs): one decoder pass over K feature pairs,
both pose heads, both DPT heads and the pointmap consumers (per-edge shared intrinsics, depth maps, confidence means),
with no host synchronisation inside -- the caller reads `pose_conf` once per keyframe.

Results are numerically the per-edge results of the reference sequence (the decoder has no cross-sample op), so
`regress_two_views(i, j)` is also offered as the K = 1 special case with the reference's return convention.

Across keyframes (OnlineSLAM.step_many): `add_views` encodes many views per sta_encode call, and
`regress_keyframes_gated` runs the gated step over the candidate edges of many keyframes in chunks of up to 16 edges,
one pose-confidence read-back per chunk.  Batch sizes change the GEMMs' split-K, so these outputs equal the per-keyframe
ones within rounding, not bit for bit.

Across caches (SLAMSessions): `add_views_group` encodes the new views of several caches that share one STA in the same
calls, and `regress_keyframes_gated_group` runs the gated step over keyframes of several caches, a chunk's edges mixing
caches.  One cache through them launches exactly what add_views / regress_keyframes_gated launch.

Tracked frames (OnlineSLAM.track): `encode_views` encodes frames without caching them and `regress_frames` regresses
each (frame, keyframe) pair through `regress_pairs`, the chunk regression the keyframe path runs, with no gate."""
import ctypes

import torch

from . import _lib
from .utils.slam_utils import _scratch_for

GRAPH_MAX_TOKENS = 8192  # runtime.cu kGraphMaxTokens: larger calls run without CUDA-graph replay
MAX_EDGES = 16           # edges per sta_regress_pairs_begin call (check_edges)


class KeyframeFrontend:
    def __init__(self, sta):
        self.frontend = sta
        self.enc_features = []   # like OnlineSLAM.enc_features (slam.py:145)
        self.img_shapes = []

    @property
    def view_num(self):
        return len(self.enc_features)

    def add_view(self, image, image_shape=None):
        """slam.py:142-151: encode one view (B = 1) and cache its features; returns the view index."""
        return self.add_views([image], [image_shape])[0]

    def add_views(self, images, image_shapes=None):
        """add_view for each image (1, 3, H, W) in order, all of one size, encoded B at a time with B N <= GRAPH_MAX_TOKENS
        (N = H W / 256 tokens; 41 views at 224 x 224), so every call is replayed as a CUDA graph.  Returns the view
        indices."""
        images = list(images)
        shapes = [None] * len(images) if image_shapes is None else list(image_shapes)
        return add_views_group([self], [images], [shapes])[0]

    @staticmethod
    def edge_chunks(items):
        """Keyframe-major chunks of the edges of items = [(i, js), ...]: lists of item indices whose edges add up to at
        most MAX_EDGES; a keyframe's edges are never split.  Keyframes without candidates belong to no chunk."""
        chunks, cur, n = [], [], 0
        for k, (_, js) in enumerate(items):
            m = len(js)
            if m == 0:
                continue
            if m > MAX_EDGES:
                raise ValueError("a keyframe has more than %d candidate edges" % MAX_EDGES)
            if n + m > MAX_EDGES:
                chunks.append(cur)
                cur, n = [], 0
            cur.append(k)
            n += m
        if cur:
            chunks.append(cur)
        return chunks

    def _read_confs(self, pconf):
        """The gate's read-back: the candidates' pose confidences on the host."""
        return [float(c) for c in pconf.cpu()]

    def regress_keyframes_gated(self, items, rel_pose_thres):
        """regress_views_gated over the keyframes items = [(i, js), ...], chunk by chunk (edge_chunks): per chunk ONE
        sta_regress_pairs_begin over its edges, ONE read-back of their confidences, and one _finish for the survivors
        (`conf >= thres or i - j == 1`).  When the call has more than one chunk, every chunk is padded to MAX_EDGES with
        copies of its last edge (ignored), so that the CUDA-graph keys stay few.

        A generator: it yields, per item in order, (the K confidences on the host, indices of the kept candidates, the
        keyframe's device batch {pose [K,4,4], pose_conf [K], conf / depths [2,n,H,W], intri [n,3,3], conf_mean [2,n]})
        -- what OnlineSLAM._add_keyframe takes -- or None for an item without candidates.  A chunk runs when its first
        keyframe is asked for."""
        return regress_keyframes_gated_group([(self, i, js) for i, js in items], rel_pose_thres)

    @torch.no_grad()
    def _regress_chunk(self, items, rel_pose_thres, pad):
        """One edge chunk of items = [(cache, i, js), ...], the caches sharing self's STA."""
        edges = [(c, i, j) for c, i, js in items for j in js]
        K = MAX_EDGES if pad else len(edges)
        run = edges + [edges[-1]] * (K - len(edges))
        H, W = edges[0][0].img_shapes[edges[0][1]]
        if any(c.img_shapes[v] != (H, W) for c, i, j in edges for v in (i, j)):
            raise ValueError("all views of a batch must have the same size")
        fi = torch.cat([c.enc_features[i] for c, i, _ in run], dim=0)
        fj = torch.cat([c.enc_features[j] for c, _, j in run], dim=0)

        def gate(conf_host):
            return [e for e, (_, i, j) in enumerate(edges) if not (conf_host[e] < rel_pose_thres and i - j != 1)]

        pose, pconf, conf_host, keep, maps = regress_pairs(self.frontend, fi, fj, H, W, len(edges), gate,
                                                           self._read_confs)
        e0 = p0 = 0
        for _, i, js in items:
            e1 = e0 + len(js)
            kf_keep = [e - e0 for e in keep if e0 <= e < e1]
            p1 = p0 + len(kf_keep)
            batch = {"pose": pose[0, e0:e1], "pose_conf": pconf[0, e0:e1]}
            if kf_keep:
                conf, depth, intri, cmean = maps
                batch.update(conf=conf[:, p0:p1].contiguous(), depths=depth[:, p0:p1].contiguous(), intri=intri[p0:p1],
                             conf_mean=cmean[:, p0:p1].contiguous())
            yield conf_host[e0:e1], kf_keep, batch
            e0, p0 = e1, p1

    def _edge_batch(self, i, js):
        """The inputs of a batched step over the K = len(js) edges (i, j): the library, the feature pairs fi / fj, the
        image size, a float32 allocator on their device and the pose outputs [2, K, 4, 4] / [2, K] of both directions."""
        K = len(js)
        H, W = self.img_shapes[i]
        if any(self.img_shapes[j] != (H, W) for j in js):
            raise ValueError("all views of a batch must have the same size")
        fi = self.enc_features[i].expand(K, -1, -1).contiguous() if K > 1 else self.enc_features[i]
        fj = torch.cat([self.enc_features[j] for j in js], dim=0) if K > 1 else self.enc_features[js[0]]
        L = self.frontend._ready(fi)

        def f32(*shape):
            return torch.empty(*shape, device=fi.device, dtype=torch.float32)

        return L, fi, fj, H, W, f32, f32(2, K, 4, 4), f32(2, K)

    @torch.no_grad()
    def regress_views(self, i, js):
        """All edges (i, j) for j in js in one batch.  Returns a dict of CUDA tensors, edge-major:
        pose [K,4,4] and pose_conf [K] of the i -> j direction (slam.py:164-167), pts3d [2,K,H,W,3], conf [2,K,H,W]
        ([0] = ij, [1] = ji as in the torch.cat of slam.py:181-182), intri [K,3,3], depths [2,K,H,W], conf_mean [2,K]."""
        js = list(js)
        K = len(js)
        if K == 0:
            raise ValueError("no edges")
        L, fi, fj, H, W, f32, pose, pconf = self._edge_batch(i, js)
        pts = f32(2, K, H, W, 3)
        conf = f32(2, K, H, W)
        intri = f32(K, 3, 3)
        depth = f32(2, K, H, W)
        cmean = f32(2, K)
        dev = fi.device
        m = self.frontend
        with torch.cuda.device(dev):
            _lib.check(L.sta_regress_pairs(m._handle, _lib.ptr(fi), _lib.ptr(fj), K, H, W, _lib.ptr(pose), _lib.ptr(pconf),
                                           _lib.ptr(pts), _lib.ptr(conf), _lib.ptr(intri), _lib.ptr(depth), _lib.ptr(cmean),
                                           _lib.ptr(_scratch_for(dev, 2 * K)), _lib.cur_stream()), "sta_regress_pairs")
        return {"pose": pose[0], "pose_conf": pconf[0], "pose_ji": pose[1], "pose_conf_ji": pconf[1], "pts3d": pts,
                "conf": conf, "intri": intri, "depths": depth, "conf_mean": cmean}

    @torch.no_grad()
    def regress_views_gated(self, i, js, rel_pose_thres):
        """The keyframe step with the reference's early-out (slam.py:169-170) kept: ONE decoder + pose-head pass over all
        candidate edges (i, j), ONE device-to-host copy of the K pose confidences, then the DPT heads and the pointmap
        consumers only for the edges the reference would keep (`conf >= thres or i - j == 1`).  The one-keyframe,
        unpadded case of regress_keyframes_gated.

        Returns a list with one entry per candidate, in the return convention of OnlineSLAM.regress_two_views
        (slam.py:153-189) minus the pypose conversion, which stays with the caller:
            (pose_ij [1,4,4], rel_pose_conf_ij [1], confs [2,H,W] | None, intri [3,3] | None, depths [2,H,W] | None)
        -- the last three are None for rejected edges, exactly where the reference returns None."""
        js = list(js)
        if not js:
            return []
        (_, keep, b), = self._regress_chunk([(self, i, js)], rel_pose_thres, pad=False)
        out = [(b["pose"][k:k + 1], b["pose_conf"][k:k + 1], None, None, None) for k in range(len(js))]
        for p, k in enumerate(keep):
            out[k] = out[k][:2] + (b["conf"][:, p], b["intri"][p], b["depths"][:, p])
        return out

    @torch.no_grad()
    def regress_two_views(self, i, j):
        """K = 1 with the return convention of slam.py:153-189 minus the pypose conversion:
        (pose_ij [1,4,4], rel_pose_conf_ij [1], confs [2,H,W], intri [3,3], depths [2,H,W])."""
        r = self.regress_views(i, [j])
        return r["pose"], r["pose_conf"], r["conf"][:, 0], r["intri"][0], r["depths"][:, 0]


@torch.no_grad()
def encode_views(sta, images, shapes):
    """The encoder features (1, N, 1024) of images (1, 3, H, W) of one size, in order, from B at a time with
    B N <= GRAPH_MAX_TOKENS (N = H W / 256 tokens; 41 views at 224 x 224), so every call is replayed as a CUDA graph."""
    if not images:
        return []
    H, W = int(images[0].shape[-2]), int(images[0].shape[-1])
    if any(tuple(im.shape[-2:]) != (H, W) for im in images):
        raise ValueError("all views of a batch must have the same size")
    B = max(1, GRAPH_MAX_TOKENS // ((H // 16) * (W // 16)))
    feats = []
    for c0 in range(0, len(images), B):
        chunk = images[c0:c0 + B]
        x = torch.cat([im.reshape(1, *im.shape[-3:]) for im in chunk]) if len(chunk) > 1 else chunk[0]
        feat, _ = sta._encode_image(x, shapes[c0], normalize=False)
        feats += [feat[b:b + 1] for b in range(len(chunk))]
    return feats


@torch.no_grad()
def add_views_group(caches, images_per_cache, shapes_per_cache=None):
    """KeyframeFrontend.add_views for several caches that share one STA, as one sequence of encoder calls: the new views
    of all caches in order (cache by cache), all of one size, B at a time as add_views chunks them (encode_views), each
    feature appended to its own cache.  Returns each cache's new view indices."""
    caches = list(caches)
    images = [list(x) for x in images_per_cache]
    shapes = [[None] * len(x) for x in images] if shapes_per_cache is None else [list(x) for x in shapes_per_cache]
    if any(c.frontend is not caches[0].frontend for c in caches):
        raise ValueError("the caches of a group must share one STA")
    flat = [(c, im, sh) for c, ims, shs in zip(caches, images, shapes) for im, sh in zip(ims, shs)]
    firsts = [c.view_num for c in caches]
    if flat:
        feats = encode_views(caches[0].frontend, [im for _, im, _ in flat], [sh for _, _, sh in flat])
        H, W = int(flat[0][1].shape[-2]), int(flat[0][1].shape[-1])
        for (c, _, _), feat in zip(flat, feats):
            c.enc_features.append(feat)
            c.img_shapes.append((H, W))
    return [list(range(f, c.view_num)) for f, c in zip(firsts, caches)]


@torch.no_grad()
def regress_pairs(sta, fi, fj, H, W, n, gate=None, read_confs=None):
    """The edge regression of one chunk, shared by keyframes and tracked frames: the feature pairs fi / fj [K, N, 1024]
    (edges 0 .. n - 1 real, the rest padding) through ONE sta_regress_pairs_begin, then ONE sta_regress_pairs_finish
    over the kept edges.  With a gate, the kept edges are gate(conf_host), conf_host being the n pose confidences read
    back once (read_confs); without one, all n edges are kept and nothing is read back.

    Returns (pose [2,K,4,4], pose_conf [2,K], conf_host or None, keep, maps), maps = (conf, depths [2,n',H,W],
    intri [n',3,3], conf_mean [2,n']) over the n' kept edges ([0] = i side, [1] = j side), or None when none is kept."""
    K = fi.shape[0]
    L = sta._ready(fi)
    dev = fi.device

    def f32(*shape):
        return torch.empty(*shape, device=dev, dtype=torch.float32)

    pose, pconf = f32(2, K, 4, 4), f32(2, K)
    maps = conf_host = None
    with torch.cuda.device(dev):
        _lib.check(L.sta_regress_pairs_begin(sta._handle, _lib.ptr(fi), _lib.ptr(fj), K, H, W, _lib.ptr(pose),
                                             _lib.ptr(pconf), _lib.cur_stream()), "sta_regress_pairs_begin")
        if gate is None:
            keep = list(range(n))
        else:
            conf_host = read_confs(pconf[0, :n])  # the one host synchronisation of the chunk
            keep = gate(conf_host)
        m = len(keep)
        if m:
            conf, depth = f32(2, m, H, W), f32(2, m, H, W)
            pts, intri, cmean = f32(2, m, H, W, 3), f32(m, 3, 3), f32(2, m)
            idx = (ctypes.c_int * m)(*keep)
            _lib.check(L.sta_regress_pairs_finish(sta._handle, idx, m, _lib.ptr(pts), _lib.ptr(conf), _lib.ptr(intri),
                                                  _lib.ptr(depth), _lib.ptr(cmean), _lib.ptr(_scratch_for(dev, 2 * m)),
                                                  _lib.cur_stream()), "sta_regress_pairs_finish")
            maps = (conf, depth, intri, cmean)
    return pose, pconf, conf_host, keep, maps


def regress_frames(sta, pairs, H, W):
    """The ungated regression of tracked frames: pairs = [(frame feature, keyframe feature), ...] (each (1, N, 1024),
    one image size H x W) as the edges (i = frame, j = keyframe view), in chunks of at most MAX_EDGES with the padding
    rule of regress_keyframes_gated_group (every chunk padded to MAX_EDGES when there is more than one), each chunk
    through regress_pairs with no gate and no read-back.  Returns, over all pairs in order, (pose [F,4,4] of i -> j,
    pose_conf [F], depth [F,H,W] and conf [F,H,W] of the keyframe side)."""
    pad = len(pairs) > MAX_EDGES
    parts = []
    for c0 in range(0, len(pairs), MAX_EDGES):
        run = pairs[c0:c0 + MAX_EDGES]
        n = len(run)
        run = run + [run[-1]] * ((MAX_EDGES if pad else n) - n)
        fi = torch.cat([f for f, _ in run], dim=0)
        fj = torch.cat([k for _, k in run], dim=0)
        pose, pconf, _, _, (conf, depth, _, _) = regress_pairs(sta, fi, fj, H, W, n)
        parts.append((pose[0, :n], pconf[0, :n], depth[1], conf[1]))
    if len(parts) == 1:
        return parts[0]
    return tuple(torch.cat(x) for x in zip(*parts))


def regress_keyframes_gated_group(items, rel_pose_thres):
    """KeyframeFrontend.regress_keyframes_gated over keyframes items = [(cache, i, js), ...] of several caches that share
    one STA: the same chunks of at most MAX_EDGES edges (a keyframe never split, padded when there is more than one
    chunk), a chunk's edges mixing caches, one confidence read-back per chunk.  A generator with the same yields, per
    item in order."""
    items = [(c, i, list(js)) for c, i, js in items]
    if any(c.frontend is not items[0][0].frontend for c, _, _ in items):
        raise ValueError("the caches of a group must share one STA")
    chunks = KeyframeFrontend.edge_chunks([(i, js) for _, i, js in items])
    pad = len(chunks) > 1
    at = 0
    for chunk in chunks:
        # a keyframe without candidates may sit between two of a chunk's keyframes (another session's first view)
        members = set(chunk)
        results = items[chunk[0]][0]._regress_chunk([items[k] for k in chunk], rel_pose_thres, pad)
        for k in range(at, chunk[-1] + 1):
            yield next(results) if k in members else None
        at = chunk[-1] + 1
    for k in range(at, len(items)):
        yield None
