"""Rig pose modes (dsac_rig_pose_modes_device) on the host: the numpy restatement of which slots of a rig's pool take part
(occupied_rig) and of the selection over the pool (select_rig, test_pose_modes_host.select on those slots), checked on
hand-built pools with known answers.  tests/test_gpu_rig_pose_modes.py checks the engine against the same restatement."""
import numpy as np

import test_pose_modes_host as MH

BAD_PRIOR, BAD_RIG = 128, 256


def occupied_rig(img_idx, status, prior_k):
    """Step 1 over rig r's pool of C H slots: slot c H + h is occupied when frame r C + c sampled h (img_idx [C][H][4]),
    or when the pass had k = prior_k rig priors and h >= H - k; a rig with DSAC_ST_BAD_RIG or DSAC_ST_BAD_PRIOR has none."""
    img_idx = np.asarray(img_idx).reshape(-1, np.asarray(img_idx).shape[-2], 4)
    C_, H = img_idx.shape[:2]
    if int(status) & (BAD_PRIOR | BAD_RIG):
        return np.zeros(C_ * H, bool)
    occ = img_idx[:, :, 0] >= 0
    if prior_k:
        occ[:, H - prior_k:] = True
    return occ.reshape(-1)


def select_rig(rig_hyp, img_idx, scores, sf, status, prior_k, M, rot, trans):
    """Steps 1-3 of one rig: (seed slots, their mass, their member counts, owner of every slot or -1), the walk of a
    frame's pool over the rig poses rig_hyp [C H][6] and the pool's scores and sf."""
    occ = occupied_rig(img_idx, status, prior_k)
    marks = np.full((len(occ), 4), -1, np.int32)
    marks[occ, 0] = 0
    return MH.select(rig_hyp, marks, scores, sf, 0, 0, M, rot, trans)


def _pool(C_, H, rng):
    img_idx = np.zeros((C_, H, 4), np.int32)
    poses = np.concatenate([rng.normal(scale=0.5, size=(C_ * H, 3)), rng.normal(scale=1000.0, size=(C_ * H, 3))], 1)
    return img_idx, poses


def test_occupancy_takes_every_cameras_samples_and_prior_slots():
    C_, H, k = 3, 8, 2
    img_idx = np.zeros((C_, H, 4), np.int32)
    img_idx[1, 2] = -1           # camera 1 sampled nothing in slot 2
    img_idx[2, H - 1] = -1       # a prior slot occupied because of the priors
    occ = occupied_rig(img_idx, 0, k)
    assert occ.shape == (C_ * H,)
    assert not occ[1 * H + 2] and occ[2 * H + H - 1]
    assert occ.sum() == C_ * H - 1
    assert not occupied_rig(img_idx, 0, 0)[2 * H + H - 1]
    for bad in (BAD_PRIOR, BAD_RIG, BAD_PRIOR | BAD_RIG | 2):
        assert not occupied_rig(img_idx, bad, k).any()
    # other status bits (a refinement abort, DSAC_ST_NO_DEPTH of one camera) leave the pool as it is
    assert np.array_equal(occupied_rig(img_idx, 2 | 64, k), occ)


def test_one_camera_is_a_frame():
    """C = 1 without a bad prior: the rig restatement is the frame's."""
    rng = np.random.default_rng(0)
    H, k = 16, 3
    img_idx, poses = _pool(1, H, rng)
    img_idx[0, [1, 4, H - 2]] = -1
    scores = rng.normal(size=H)
    scores[5] = np.nan
    sf = rng.uniform(size=H)
    for prior_k in (0, k):
        a = select_rig(poses, img_idx, scores, sf, 2, prior_k, 4, 0.4, 900.0)
        b = MH.select(poses, img_idx[0], scores, sf, 2, prior_k, 4, 0.4, 900.0)
        assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2] and np.array_equal(a[3], b[3])


def test_walk_over_two_cameras():
    """Two cameras whose hypotheses form two clusters across the cameras: a seed gathers members from both cameras, the
    mass is the members' sf in rank order, the ranking breaks ties to the lower slot, and empty slots join nothing."""
    C_, H = 2, 4
    A = np.array([0.1, 0.0, 0.0, 0.0, 0.0, 2000.0])
    B = np.array([0.1, 0.5, 0.0, 1000.0, 0.0, 2000.0])
    poses = np.array([A, B, A + [0, 0, 0, 5, 0, 0], B, B + [0.01, 0, 0, 0, 0, 0], A, A, B], np.float64)
    scores = np.array([3.0, 5.0, 1.0, 0.0, 5.0, 2.0, 9.0, 4.0])
    sf = np.array([0.1, 0.2, 0.05, 0.01, 0.2, 0.04, 0.3, 0.1])
    img_idx = np.zeros((C_, H, 4), np.int32)
    img_idx[1, 2] = -1           # slot 6, the best score, is empty
    seeds, mass, members, owner = select_rig(poses, img_idx, scores, sf, 0, 0, 4, 0.05, 50.0)
    # ranking: 1 (5.0), 4 (5.0, a tie: the lower slot first), 7, 0, 5, 2, 3
    assert seeds == [1, 0]
    assert members == [4, 3]
    assert mass == [0.2 + 0.2 + 0.1 + 0.01, 0.1 + 0.04 + 0.05]
    assert owner[6] == -1 and owner[4] == 0 and owner[5] == 1
    # M = 1: the second cluster joins nothing
    seeds, mass, members, owner = select_rig(poses, img_idx, scores, sf, 0, 0, 1, 0.05, 50.0)
    assert seeds == [1] and members == [4] and (owner[[0, 2, 5]] == -1).all()
    # a spoiled rig: no seeds
    assert select_rig(poses, img_idx, scores, sf, BAD_RIG, 0, 4, 0.05, 50.0)[0] == []
