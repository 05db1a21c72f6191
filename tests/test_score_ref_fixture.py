"""The numpy restatement of the score-CNN pre-training data path (tests/score_oracle.py) against what the reference's OWN
train_score.cpp computes (tests/golden/ref_score.npz, frozen by tests/golden/make_ref_score.py): getRandHyp sequences,
and two consecutive assembleData rounds for T = 1, 3 and 16 OpenMP threads -- frames and sampling grids exactly, labels
within 1e-9, reprojection-error images within 1e-3 px."""
import math
import os

import numpy as np
import pytest

import obj_oracle as OO
import score_oracle as SO
from conftest import GOLDEN

REF = np.load(os.path.join(GOLDEN, "ref_score.npz"))


def stub_coords(gt_jp, frame, pix, focal, cx, cy):
    """The coordinate stub of tests/golden/ref_score/ref_train_score.cpp: depth 1500 + (7x + 13y + 29f) mod 1000,
    back-projected into the jp camera frame, R^T (cam - t), floor(v + 0.5) -> int16 mm [1600][3]."""
    P = gt_jp[frame]
    out = np.zeros((len(pix), 3), np.int16)
    for k, (x, y) in enumerate(pix):
        d = 1500.0 + float((7 * int(x) + 13 * int(y) + 29 * int(frame)) % 1000)
        cam = ((float(x) - cx) * d / focal, -((float(y) - cy) * d / focal), -d)
        q = (cam[0] - P[9], cam[1] - P[10], cam[2] - P[11])
        for r in range(3):
            out[k, r] = math.floor(P[r] * q[0] + P[3 + r] * q[1] + P[6 + r] * q[2] + 0.5)
    return out


@pytest.mark.parametrize("seed", [1305, 7])
def test_rand_hyp_sequences_match_reference(seed):
    """getRandHyp's draws in the reference's own evaluation order, 64 calls of getRandHyp(2, 2) and then 64 of
    getRandHyp(10, 100) on one generator: the translations bit for bit, the rotation matrices of Hypothesis(v) within
    1e-12.  The reversed order (x drawn first) does not match."""
    bg = np.random.MT19937()
    bg._legacy_seeding(seed)
    words = lambda: int(bg.random_raw())   # noqa: E731
    for rot, trans in ((2.0, 2.0), (10.0, 100.0)):
        key = "randhyp/%d/%g_%g" % (seed, rot, trans)
        t_ref, R_ref = REF[key + "/trans"], REF[key + "/rot"]
        v = np.stack([SO.rand_hyp(words, rot, trans) for _ in range(len(t_ref))])
        assert np.array_equal(np.ascontiguousarray(v[:, 3:]).view(np.uint64), t_ref.view(np.uint64))
        for k in range(len(v)):
            assert np.abs(SO.hypothesis_rotation(v[k]).reshape(9) - R_ref[k]).max() <= 1e-12
        assert not np.array_equal(v[:, [5, 4, 3]], t_ref)


@pytest.mark.parametrize("name,T", [("small", 1), ("small", 3), ("small", 16), ("vga", 3)])
def test_assemble_rounds_match_reference(name, T):
    W, H, F = (int(v) for v in REF[name + "/size"])
    gt = REF[name + "/gt_jp"]
    n_images, hyps = int(REF["n_images"]), int(REF["hyps"])
    focal, cx, cy = float(REF["focal"]), float(W // 2), float(H // 2)
    st = OO.rng_init(int(REF["seed"]), T)
    unclamped = 0
    for rnd in range(2):
        key = "%s/T%d/round%d" % (name, T, rnd)
        img, pix, drift, noise = SO.draw(st, F, W, H, n_images, hyps)
        assert np.array_equal(img, REF[key + "/frames"])
        assert np.array_equal(pix, REF[key + "/grid"].astype(np.int32))
        maps, labels = REF[key + "/maps"], REF[key + "/labels"]
        for i in range(n_images):
            coords = stub_coords(gt, img[i], pix[i], focal, cx, cy)
            for h in range(hyps):
                k = i * hyps + h
                lab = SO.sample(gt[img[i]], noise[k])[0]
                assert abs(labels[k] - lab) <= 1e-9 * max(1.0, abs(lab))
                ref = SO.diff_map(gt[img[i]], noise[k], coords, pix[i], focal, cx, cy)
                assert np.abs(maps[k] - ref).max() <= 1e-3
                unclamped += int((maps[k] < 100).sum())
    assert unclamped > 0 and (drift == 0).any()
