"""GPU: the ORB and bag-of-words kernels are bit-exact with oracle/loop_detector_oracle.py, and LoopDetector gives the
reference's candidate lists (tests/golden/loop.npz)."""
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import loop_detector_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VOCAB_TXT = os.path.join(GOLDEN, "loop_vocab.txt")
VOCAB_BIN = os.path.join(GOLDEN, "loop_vocab.bin")
VOCAB_QLZ = os.path.join(GOLDEN, "loop_vocab.dbow3")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLDEN, "loop.npz"))


@pytest.fixture(scope="module")
def meta(g):
    return json.loads(str(g["meta"]))


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from vista_slam_b200 import loop_detector
    return loop_detector


def frames_of(meta, s):
    seed, n, H, W = meta["sequences"][s]
    return O.make_sequence(seed, n, H, W)


def extra_frames():
    rng = np.random.default_rng(11)
    return [O._texture(rng, 480, 640), O._texture(rng, 181, 263), O._texture(rng, 70, 90)]


def check_orb(L, f):
    r = L.orb_detect_and_compute(torch.from_numpy(f).cuda())
    o = O.orb_detect_and_compute(f, with_stages=True)
    st = o["stages"]
    lay = r["layout"]
    scratch = r["scratch"].cpu().numpy()
    for l in range(O.NLEVELS):
        h, w, ofs = lay[10 + 4 * l], lay[11 + 4 * l], lay[12 + 4 * l]
        np.testing.assert_array_equal(scratch[lay[1] + ofs:lay[1] + ofs + h * w].reshape(h, w), st["pyramid"][l])
        np.testing.assert_array_equal(scratch[lay[2] + ofs:lay[2] + ofs + h * w].reshape(h, w), st["blurred"][l])
        np.testing.assert_array_equal(scratch[lay[3] + ofs:lay[3] + ofs + h * w].reshape(h, w), st["fast"][l])
    # FAST candidates past the border filter, with their Harris responses where retainBest(2n) kept them
    ncand = int(scratch[lay[6]:lay[6] + 4].view(np.uint32)[0])
    cand = scratch[lay[4]:lay[4] + 16 * ncand].view(np.int32).reshape(-1, 4)
    resp = scratch[lay[5]:lay[5] + 4 * ncand].view(np.float32)
    for l in range(O.NLEVELS):
        ys, xs, s, rr = st["cand"][l]
        m = cand[:, 0] == l
        got = {(int(x), int(y)): (int(sc), r_) for (_, x, y, sc), r_ in zip(cand[m], resp[m])}
        for y, x, sc, r_ in zip(ys, xs, s, rr):
            assert got[(int(x), int(y))][0] == sc
            assert got[(int(x), int(y))][1] == r_
    np.testing.assert_array_equal(r["level"].cpu().numpy(), o["level"])
    np.testing.assert_array_equal(r["xy"].cpu().numpy(), o["xy_level"])
    np.testing.assert_array_equal(r["pts"].cpu().numpy(), o["pts"])
    np.testing.assert_array_equal(r["angle"].cpu().numpy(), o["angle"])
    np.testing.assert_array_equal(r["response"].cpu().numpy(), o["response"])
    np.testing.assert_array_equal(r["desc"].cpu().numpy(), o["desc"])
    return r


def test_orb_equals_oracle_golden_frames(L, meta):
    for s in (0, 1):
        for f in frames_of(meta, s):
            check_orb(L, f)


def test_orb_equals_oracle_more_sizes(L):
    for f in extra_frames():
        check_orb(L, f)


def test_orb_equals_cv2_goldens(L, g, meta):
    for s in (0, 1):
        for t, f in enumerate(frames_of(meta, s)):
            r = L.orb_detect_and_compute(torch.from_numpy(f).cuda())
            np.testing.assert_array_equal(r["desc"].cpu().numpy(), g["s%d_f%d_desc" % (s, t)].reshape(-1, 32))
            np.testing.assert_array_equal(r["pts"].cpu().numpy(), g["s%d_f%d_pts" % (s, t)].reshape(-1, 2))


def test_f32_gray_equals_u8(L, meta):
    f = frames_of(meta, 0)[2]
    gray = torch.from_numpy(f).cuda().float() / 255.0
    u8 = (gray.cpu().numpy() * np.float32(255)).astype(np.uint8)
    a = L.orb_detect_and_compute(gray[None])
    b = L.orb_detect_and_compute(torch.from_numpy(u8).cuda())
    for k in ("xy", "angle", "response", "desc"):
        assert torch.equal(a[k], b[k])


def test_bow_transform_vector_score(L, meta):
    v = O.load_vocab_txt(VOCAB_TXT)
    voc = L.Vocabulary(VOCAB_TXT)
    assert (voc.k, voc.L, voc.n_nodes, voc.n_words) == (v.k, v.L, v.n_nodes, v.n_words)
    vecs = []
    for f in frames_of(meta, 0)[:20]:
        d = O.orb_detect_and_compute(f)["desc"]
        if len(d) == 0:
            vecs.append(None)
            continue
        w, x = L.bow_transform(voc, d)
        ow, ox = O.transform_words(v, d)
        np.testing.assert_array_equal(w.cpu().numpy(), ow)
        np.testing.assert_array_equal(x.cpu().numpy(), ox)
        bw, bv = L.bow_vector(voc, w, x)
        ref = O.bow_vector(v, d)
        np.testing.assert_array_equal(bw.cpu().numpy(), ref[0])
        np.testing.assert_array_equal(bv.cpu().numpy(), ref[1])
        vecs.append(ref)
    sims = L.bow_score(vecs[-1], vecs).cpu().numpy()
    for j, b in enumerate(vecs):
        if b is None or vecs[-1] is None:
            assert np.isnan(sims[j])
        else:
            assert sims[j] == O.l1_score(vecs[-1], b)


@pytest.mark.parametrize("path", [VOCAB_TXT, VOCAB_BIN, VOCAB_QLZ])
def test_loop_detector_equals_reference(L, g, meta, path):
    """detect_loop == the unmodified loop_detector.py on every keyframe; vectors and similarity rows == oracle."""
    v = O.load_vocab_txt(VOCAB_TXT)
    args = meta["loop_args"]
    for s in (0, 1):
        det = L.LoopDetector(path, **args)
        feats = []
        for t, f in enumerate(frames_of(meta, s)):
            c = det.detect_loop(f, max(0, t - 3))
            ref = g["s%d_k%d_cand" % (s, t)]
            assert [j for j, _ in c] == [int(j) for j in ref[:, 0]], "keyframe %d" % t
            np.testing.assert_array_equal(np.array([x for _, x in c], np.float64), ref[:, 1])
            d = O.orb_detect_and_compute(f)["desc"]
            feats.append(O.bow_vector(v, d) if len(d) else None)
            assert (det.bow_feats[t] is None) == (feats[t] is None)
            if t % 7 == 0 and feats[t] is not None:
                w, x = det.bow_feats[t].to_numpy()
                np.testing.assert_array_equal(w, feats[t][0])
                np.testing.assert_array_equal(x, feats[t][1])
            if t % 11 == 5:
                row = det.similarities()
                for j in range(t):
                    if feats[t] is None or feats[j] is None:
                        assert np.isnan(row[j])
                    else:
                        assert row[j] == O.l1_score(feats[t], feats[j])
        assert len(det.bow_feats) == len(frames_of(meta, s))


def test_vocabulary_files_load_to_the_same_tree(L):
    for path in (VOCAB_TXT, VOCAB_BIN, VOCAB_QLZ):
        voc = L.Vocabulary(path)
        assert (voc.k, voc.L, voc.scoring, voc.weighting, voc.n_nodes, voc.n_words) == (10, 3, 0, 0, 1098, 987)


def test_database_grows_past_its_first_reservation(L, meta):
    """650 compute_bow_feat calls without a detect_loop (the database's first reservation holds 64 views of the
    largest size): every stored vector still equals the oracle's."""
    v = O.load_vocab_txt(VOCAB_TXT)
    frames = frames_of(meta, 0)
    ref = []
    for f in frames:
        d = O.orb_detect_and_compute(f)["desc"]
        ref.append(O.bow_vector(v, d) if len(d) else None)
    det = L.LoopDetector(VOCAB_TXT, 40, 40, 5)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    n = 650
    for t in range(n):
        det.compute_bow_feat(dev[t % len(frames)])
    assert len(det.bow_feats) == n
    for t in range(0, n, 7):
        r = ref[t % len(frames)]
        if r is None:
            assert det.bow_feats[t] is None
            continue
        w, x = det.bow_feats[t].to_numpy()
        np.testing.assert_array_equal(w, r[0])
        np.testing.assert_array_equal(x, r[1])
    c = det.detect_loop(dev[0], n - 3)
    row = det.similarities()
    for j in range(0, n, 13):
        r0, rj = ref[0], ref[j % len(frames)]
        assert row[j] == O.l1_score(r0, rj) if rj is not None else np.isnan(row[j])
    assert all(0 <= j < n for j, _ in c)


def test_detect_loop_fp32_gray_and_repeat(L, meta):
    frames = frames_of(meta, 0)
    runs = []
    for mode in ("u8", "f32", "u8"):
        det = L.LoopDetector(VOCAB_TXT, 40, 40, 5)
        out = []
        for t, f in enumerate(frames):
            x = torch.from_numpy(f).cuda()
            if mode == "f32":
                # exactly representable: (f / 255) * 255 truncates back to f for every 8-bit value
                x = (x.float() / 255.0)[None]
                assert np.array_equal((x[0].cpu().numpy() * np.float32(255)).astype(np.uint8), f)
            out.append(det.detect_loop(x, max(0, t - 3)))
        runs.append(out)
    assert runs[0] == runs[1] == runs[2]


def _random_deep_vocab(path, seed=3):
    rng = np.random.default_rng(seed)
    parent, desc, weight, word = [-1], [np.zeros(32, np.uint8)], [0.0], [-1]
    children = [[]]
    frontier = [0]
    for level in range(6):
        nxt = []
        for n in frontier:
            k = 10 if level == 0 else int(rng.integers(0, 11)) if rng.random() < 0.25 else 0
            for _ in range(k):
                nid = len(parent)
                parent.append(n)
                desc.append(rng.integers(0, 256, 32).astype(np.uint8))
                weight.append(float(np.float32(rng.random() * 3)) if rng.random() > 0.05 else 0.0)
                word.append(-1)
                children.append([])
                children[n].append(nid)
                nxt.append(nid)
        frontier = nxt
    nw = 0
    for n in range(1, len(parent)):
        if not children[n]:
            word[n] = nw
            nw += 1
    v = O.Vocabulary(10, 6, 0, O.TF_IDF, parent, np.stack(desc), weight, word)
    v.children = children
    O.save_vocab_txt(v, path)
    return O.load_vocab_txt(path)


def test_random_deep_vocabulary(L, tmp_path):
    p = str(tmp_path / "deep.txt")
    v = _random_deep_vocab(p)
    voc = L.Vocabulary(p)
    rng = np.random.default_rng(4)
    d = rng.integers(0, 256, (3000, 32)).astype(np.uint8)
    w, x = L.bow_transform(voc, d)
    ow, ox = O.transform_words(v, d)
    np.testing.assert_array_equal(w.cpu().numpy(), ow)
    np.testing.assert_array_equal(x.cpu().numpy(), ox)
    bw, bv = L.bow_vector(voc, w, x)
    ref = O.bow_vector(v, d)
    np.testing.assert_array_equal(bw.cpu().numpy(), ref[0])
    np.testing.assert_array_equal(bv.cpu().numpy(), ref[1])


def test_refusals(L, tmp_path):
    p = tmp_path / "l2.txt"
    p.write_text("10 3 1 0\n0 1 " + " ".join(["0"] * 32) + " 1.0\n")
    with pytest.raises(RuntimeError, match="L1"):
        L.Vocabulary(str(p))
    p = tmp_path / "float.txt"
    p.write_text("10 3 0 0\n0 1 " + " ".join(["0.5"] * 64) + " 1.0\n")
    with pytest.raises(RuntimeError, match="binary"):
        L.Vocabulary(str(p))
    det = L.LoopDetector(VOCAB_TXT, 40, 40, 5)
    with pytest.raises(RuntimeError, match="CUDA"):
        det.detect_loop(torch.zeros(64, 64, dtype=torch.uint8), 0)
    with pytest.raises(ValueError, match="32"):
        L.orb_detect_and_compute(torch.zeros(16, 16, dtype=torch.uint8).cuda())
