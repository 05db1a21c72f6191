"""The oracle's seeded backward chains (orc_backward_seeded, orc_backward_dsac_seeded): seeded with what the loss round
uses, they reproduce the loss round's backward."""
import numpy as np
import pytest
import seeded_oracle as S


def _gt6(oracle, gt_jp):
    return np.concatenate([oracle.rodrigues_inv(gt_jp[:9]), gt_jp[9:]])   # poseGT.getRodVecAndTrans()


@pytest.mark.parametrize("fix_q4", [0, 1])
def test_seeded_softam_backward_with_dloss_max_equals_backward(oracle, engine_mod, fix_q4):
    """seed = dLossMax(jp6(refined), gt): dLoss/dObj and every factor bit for bit."""
    O = oracle
    nf = 3
    coords, pix, gt_cv, gt_jp = engine_mod.synth_frames(nf, frame0=4)
    for f in range(nf):
        cfg = O.default_config(seed=1305 + 4 + f, n_hyps=24, fix_q4=fix_q4)
        fw = O.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
        want = O.backward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], fw)
        seed = O.dloss_max(O.jp6(fw.ref[:3], fw.ref[3:]), _gt6(O, gt_jp[f]))
        assert np.array_equal(seed, want.dloss_dref)
        got = S.backward_seeded(O, cfg, coords[f], pix[f], fw, seed)
        assert np.array_equal(got.dloss_dobj, want.dloss_dobj)
        assert np.array_equal(got.score_grads, want.score_grads)
        assert np.array_equal(got.dref_dhyp, want.dref_dhyp)
        assert np.abs(got.dloss_dobj).max() > 0


def test_seeded_dsac_backward_with_expected_loss_seeds_equals_backward_dsac(oracle, engine_mod):
    """seed_h = sf_h dLossMax(jp6(refined_h), gt), grad_sf = losses: the same selection, jobs and score gradients; dLoss/dObj
    differs only by sf being multiplied in before the sum over the pose instead of after."""
    O = oracle
    nf, H = 2, 16
    coords, pix, gt_cv, gt_jp = engine_mod.synth_frames(nf, frame0=1)
    for f in range(nf):
        cfg = O.default_config(seed=1305 + 1 + f, n_hyps=H)
        fw = O.forward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], random_draw=False)
        want = O.backward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], fw)
        gt6 = _gt6(O, gt_jp[f])
        seed = np.stack([fw.sf[h] * O.dloss_max(O.jp6(fw.ref_pose[h, :3], fw.ref_pose[h, 3:]), gt6) for h in range(H)])
        got = S.backward_dsac_seeded(O, cfg, coords[f], pix[f], fw, seed, fw.losses)
        assert got.n_selected == want.n_selected and got.n_selected >= 1
        assert got.n_refine_jobs == want.n_refine_jobs
        assert np.array_equal(got.score_grads, want.score_grads)
        assert np.array_equal(got.path2, want.path2)
        assert np.abs(got.dloss_dobj - want.dloss_dobj).max() <= 1e-13 * np.abs(want.dloss_dobj).max()
        assert np.abs(want.path1).max() > 0


def test_seeded_dsac_backward_selection_and_null_seeds(oracle, engine_mod):
    """Zero seeds select nothing; a null grad_sf zeroes path II; only the seeded hypotheses are refined."""
    O = oracle
    H = 16
    coords, pix, gt_cv, gt_jp = engine_mod.synth_frames(1)
    cfg = O.default_config(n_hyps=H)
    fw = O.forward_dsac(cfg, coords[0], pix[0], gt_jp[0, :9], gt_jp[0, 9:], random_draw=False)
    none = S.backward_dsac_seeded(O, cfg, coords[0], pix[0], fw, np.zeros((H, 6)), None)
    assert none.n_selected == 0 and none.n_refine_jobs == 0
    assert not none.dloss_dobj.any() and not none.score_grads.any()
    pick = int(np.argmax(fw.sf))
    seed = np.zeros((H, 6))
    seed[pick] = [0.5, -0.25, 1.0, 0.01, 0.02, -0.03]
    one = S.backward_dsac_seeded(O, cfg, coords[0], pix[0], fw, seed, None)
    assert one.n_selected == int(fw.sf[pick] > 1e-4) == 1
    assert np.abs(one.path1).max() > 0 and not one.path2.any()
