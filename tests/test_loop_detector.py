"""CPU checks of oracle/loop_detector_oracle.py against cv2 4.13, the compiled unmodified DBoW3 and the unmodified
reference loop detector, through tests/golden/loop.npz and loop_vocab.* (written by tools/make_golden_loop.py; neither
cv2 nor DBoW3 is needed here)."""
import json
import os

import numpy as np
import pytest

from oracle import loop_detector_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLDEN, "loop.npz"))


@pytest.fixture(scope="module")
def meta(g):
    return json.loads(str(g["meta"]))


def frames_of(meta, s):
    seed, n, H, W = meta["sequences"][s]
    return O.make_sequence(seed, n, H, W)


def test_primitives_equal_cv2(g):
    src = g["prim_resize_src"]
    for (h, w) in ((81, 109), (40, 55), (97, 130)):
        np.testing.assert_array_equal(O.resize_linear_exact(src, h, w), g["prim_resize_%dx%d" % (h, w)])
    np.testing.assert_array_equal(O.gaussian_blur_orb(src), g["prim_blur"])
    y, x = g["prim_atan_yx"]
    np.testing.assert_array_equal(O.fast_atan2(y, x), g["prim_atan"])


def test_level_geometry():
    assert O.features_per_level() == [109, 90, 75, 63, 52, 44, 36, 31]
    assert O.level_sizes(224, 224)[7] == (63, 63)


@pytest.mark.parametrize("s", [0, 1])
def test_oracle_orb_equals_cv2(g, meta, s):
    """Same keypoint sets (pt, octave, angle, response) and descriptors as cv2 on every golden frame, exactly."""
    for t, f in enumerate(frames_of(meta, s)):
        r = O.orb_detect_and_compute(f)
        key = "s%d_f%d_" % (s, t)
        np.testing.assert_array_equal(r["level"], g[key + "octave"], err_msg="frame %d" % t)
        np.testing.assert_array_equal(r["pts"], g[key + "pts"].reshape(-1, 2), err_msg="frame %d" % t)
        np.testing.assert_array_equal(r["angle"], g[key + "angle"], err_msg="frame %d" % t)
        np.testing.assert_array_equal(r["response"], g[key + "response"], err_msg="frame %d" % t)
        np.testing.assert_array_equal(r["desc"], g[key + "desc"].reshape(-1, 32), err_msg="frame %d" % t)


def test_golden_sequences_cover_the_branches(meta):
    for s in (0, 1):
        assert meta["s%d_none" % s], "a frame without descriptors (the None branch)"
        assert meta["s%d_ncand" % s] > 0, "keyframes with loop candidates"


def _same_tree(a, b):
    assert (a.k, a.L, a.scoring, a.weighting) == (b.k, b.L, b.scoring, b.weighting)
    np.testing.assert_array_equal(a.parent, b.parent)
    np.testing.assert_array_equal(a.desc, b.desc)
    np.testing.assert_array_equal(a.weight, b.weight)
    np.testing.assert_array_equal(a.word_id, b.word_id)
    assert a.children == b.children


def test_vocabulary_formats_load_equal():
    """Text, DBoW3's binary stream and its QuickLZ-compressed stream (both saved by the compiled DBoW3) load to the
    same tree."""
    a = O.load_vocab_txt(os.path.join(GOLDEN, "loop_vocab.txt"))
    assert (a.k, a.L, a.scoring, a.weighting) == (10, 3, 0, O.TF_IDF)
    with open(os.path.join(GOLDEN, "loop_vocab.dbow3"), "rb") as f:
        assert f.read(9)[8] == 1, "the .dbow3 golden is compressed"
    _same_tree(a, O.load_vocab_bin(os.path.join(GOLDEN, "loop_vocab.bin")))
    _same_tree(a, O.load_vocab_bin(os.path.join(GOLDEN, "loop_vocab.dbow3")))


def test_oracle_bow_equals_reference_dbow3(g, meta):
    """Vectors (Vocabulary::transform) and L1 similarities of the compiled DBoW3, bit for bit."""
    v = O.load_vocab_txt(os.path.join(GOLDEN, "loop_vocab.txt"))
    n = meta["sequences"][0][1]
    vecs = []
    for t in range(n):
        d = g["s0_f%d_desc" % t].reshape(-1, 32)
        vecs.append(O.bow_vector(v, d) if len(d) else None)
        if vecs[-1] is None:
            assert "s0_f%d_bow_words" % t not in g
            continue
        np.testing.assert_array_equal(vecs[-1][0], g["s0_f%d_bow_words" % t])
        np.testing.assert_array_equal(vecs[-1][1], g["s0_f%d_bow_vals" % t])
    sims = g["s0_sims"]
    for i in range(n):
        for j in range(i):
            if vecs[i] is None or vecs[j] is None:
                assert np.isnan(sims[i, j])
            else:
                assert O.l1_score(vecs[i], vecs[j]) == sims[i, j], (i, j)


@pytest.mark.parametrize("s", [0, 1])
def test_oracle_candidates_equal_reference(g, meta, s):
    """oracle detect_loop == the unmodified loop_detector.py with the compiled DBoW3 on every keyframe (cv2 ORB
    descriptors from the goldens)."""
    v = O.load_vocab_txt(os.path.join(GOLDEN, "loop_vocab.txt"))
    args = meta["loop_args"]
    feats = []
    n = meta["sequences"][s][1]
    for t in range(n):
        d = g["s%d_f%d_desc" % (s, t)].reshape(-1, 32)
        feats.append(O.bow_vector(v, d) if len(d) else None)
        c = O.detect_loop(feats, t, max(0, t - 3), args["loop_dist_min"], args["loop_nms"],
                          args["loop_cand_thresh_neighbor"])
        ref = g["s%d_k%d_cand" % (s, t)]
        assert [j for j, _ in c] == [int(j) for j in ref[:, 0]], "keyframe %d" % t
        np.testing.assert_array_equal(np.array([x for _, x in c], np.float64), ref[:, 1])


def test_detect_loop_ties_keep_descending_j():
    ids = np.array([1, 2], np.int64)
    same = (ids, np.array([0.5, 0.5]))
    other = (np.array([3], np.int64), np.array([1.0]))
    feats = [same, same, other, other, same]
    # view 4 against 0 and 1 (equal similarity 1.0); no neighbour gate beyond the views in range
    c = O.detect_loop(feats, 4, 2, loop_dist_min=0, loop_nms=0, loop_cand_thresh_neighbor=1)
    assert c == [(1, 1.0), (0, 1.0)]


def test_refusals(tmp_path):
    p = tmp_path / "v.txt"
    p.write_text("10 3 1 0\n0 1 " + " ".join(["0"] * 32) + " 1.0\n")
    v = O.load_vocab_txt(str(p))
    with pytest.raises(ValueError, match="L1"):
        O.check_supported(v)
