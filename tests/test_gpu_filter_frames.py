"""The sampler's conservative filter inside the engine, on frames whose first candidate is an adversarial minimal set.

Each case writes one integer minimal set into the four cells of the first candidate that the sampler draws for seed
1305 (oracle.candidates), in an all-outlier synthetic frame (inlier ratio 0: few other candidates are accepted, so a
skipped candidate shows in the first hypotheses).  The reference accepts the planted set, so its first hypothesis is
candidate 0.  If the engine's filter (k1_filter / k1_fused / k_sample) called the set "certainly rejected",
the engine would skip it, and every sampled index after it would differ from the oracle's.  Sampled indices, candidate
indices and candidate counts must be bit-exact.

The sets: a triangle 10 .. 25 m away and a 4th point a few centimetres in front of the camera, its pixel 9.5 .. 10 px
from where the exact pose projects it (tests/adversarial_sets.py, near camera).  The fp32 4th-point stage of the filter
used to put such a pixel beyond thr + 0.25 px.
"""
import numpy as np
import pytest

import adversarial_sets as A

pytestmark = pytest.mark.gpu

CASES = [
    ("f525", 525.0) + A.NEAR_CAMERA_CASE,
    ("f1500", 1500.0,
     np.array([-13482, -8928, 9690, -16440, -8618, 7719, -10924, -7875, 6859, 2758, -210, 2520], np.float32),
     np.array([114, 172, 208, 376, 69, 321, 18, 412], np.float32)),
    ("f2500_a", 2500.0,
     np.array([1240, -16107, 12948, 4284, -14112, 14655, 1623, -12275, 9450, -845, -2322, 656], np.float32),
     np.array([561, 96, 44, 232, 467, 249, 498, 412], np.float32)),
    ("f2500_b", 2500.0,
     np.array([-3025, -16094, -12969, -1776, -17147, -14897, -252, -8920, -8116, 2036, -504, -270], np.float32),
     np.array([263, 83, 428, 215, 464, 125, 160, 72], np.float32)),
]


@pytest.mark.parametrize("name,f,obj,img", CASES, ids=[c[0] for c in CASES])
def test_engine_keeps_near_camera_candidate(engine_mod, oracle, name, f, obj, img):
    E, O = engine_mod, oracle
    coords, pix, gt_cv, gt_jp = E.synth_frames(1, rho=0.0, focal=f)
    cells, _ = O.candidates(1305, O.default_config(seed=1305).stream_skip, 1)
    idx = cells[0, :, 1] * 40 + cells[0, :, 0]
    coords[0, idx] = obj.reshape(4, 3).astype(np.int16)
    pix[0, idx] = img.reshape(4, 2).astype(np.int32)
    for H in (1, 3, 8):
        eng = E.Engine(max_frames=1, n_hyps=H, focal=f)
        res = eng.forward(coords, pix, gt_jp)
        eng.close()
        o = O.forward(O.default_config(seed=1305, n_hyps=H, f=f), coords[0], pix[0], gt_jp[0, :9], gt_jp[0, 9:])
        assert o.n_fragile == 0 and o.cand_idx[0] == 0, (name, "the reference must accept the set", o.cand_idx[:H])
        print("%s H=%d: oracle candidates %s, engine %s" % (name, H, o.cand_idx.tolist(), res.cand_idx[0].tolist()))
        assert np.array_equal(o.img_idx, res.img_idx[0]), (name, H)
        assert np.array_equal(o.cand_idx, res.cand_idx[0]), (name, H)
        assert o.n_candidates == res.n_candidates[0], (name, H)
