"""The rig oracle (tests/host_shim/rig_oracle.cpp) with one camera and a zero extrinsic is the oracle's forward: handed
orc_forward's own pool, it gives its scores, softmax, soft-argmax, refinement, inlier map and evaluation bit for bit.  With
several cameras the lift composed with each extrinsic returns the camera's hypothesis."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import rig_oracle as RO
from oracle import oracle as O


@pytest.fixture(scope="module")
def frames():
    from dsac_b200 import engine as E
    return E.synth_frames(3)


@pytest.mark.parametrize("H", [16, 40])
def test_one_camera_zero_extrinsic_is_orc_forward(frames, H):
    coords, pix, gt_cv, gt_jp = frames
    for f in range(3):
        cfg = O.default_config(seed=1305 + f, n_hyps=H)
        ofw = O.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], want_diffmaps=False)
        pool = np.concatenate([ofw.hyp_rvec, ofw.hyp_tvec], 1)
        r = RO.forward(cfg, coords[f:f + 1], pix[f:f + 1], [[cfg.f, cfg.cx, cfg.cy]], np.zeros((1, 6)), pool[None], gt_jp[f])
        assert np.array_equal(r["rig_hyp"], pool)
        for k, want in (("scores", ofw.scores), ("sf", ofw.sf), ("entropy", ofw.entropy), ("avg_pose", ofw.avg),
                        ("ref_pose", ofw.ref), ("inlier_map", ofw.inlier_map[None]), ("steps_done", ofw.ref_steps_done),
                        ("loss", ofw.loss), ("rot_err", ofw.rot_err), ("t_err", ofw.t_err), ("correct", ofw.correct)):
            assert np.array_equal(r[k], want), k
        assert ofw.correct == 1


def test_lift_composed_with_the_extrinsic_is_the_camera_pose(frames):
    coords, pix, gt_cv, gt_jp = frames
    rng = np.random.default_rng(5)
    C, H = 3, 8
    cfg = O.default_config(n_hyps=H)
    ext = np.concatenate([Rotation.random(C, random_state=rng).as_rotvec(), rng.normal(scale=100.0, size=(C, 3))], 1)
    hyp = np.concatenate([Rotation.random(C * H, random_state=rng).as_rotvec(), rng.normal(scale=500.0, size=(C * H, 3))], 1)
    r = RO.forward(cfg, coords, pix, np.tile([[525.0, 320.0, 240.0]], (C, 1)), ext, hyp.reshape(C, H, 6))
    for j in range(C * H):
        c = j // H
        Rc, Rr = Rotation.from_rotvec(ext[c, :3]), Rotation.from_rotvec(r["rig_hyp"][j, :3])
        assert ((Rc * Rr) * Rotation.from_rotvec(hyp[j, :3]).inv()).magnitude() < 1e-12
        assert np.allclose(Rc.apply(r["rig_hyp"][j, 3:]) + ext[c, 3:], hyp[j, 3:], atol=1e-9)
    assert abs(r["sf"].sum() - 1) < 1e-12
