"""The given-pool oracle (tests/host_shim/pool_oracle.cpp) reproduces the oracle bit for bit when it is handed the
sampler's own pool: the soft-argmax and DSAC-variant forwards and both backward passes.  With a pose prior in the pool it
treats the prior as a constant: no dPNP, no minimal-set jobs, refinement jobs from the prior's pose."""
import numpy as np
import pytest

import pool_oracle as P
from oracle import oracle as O


def _frames(n):
    from dsac_b200 import engine as E
    return E.synth_frames(n)


@pytest.fixture(scope="module")
def frames():
    return _frames(2)


@pytest.mark.parametrize("H,fix_q4", [(16, 0), (24, 1)])
def test_softam_pool_matches_oracle(frames, H, fix_q4):
    coords, pix, gt_cv, gt_jp = frames
    for f in range(2):
        cfg = O.default_config(seed=1305 + f, n_hyps=H, fix_q4=fix_q4)
        ofw = O.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], want_diffmaps=False)
        pool = np.concatenate([ofw.hyp_rvec, ofw.hyp_tvec], 1)
        pfw = P.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], pool, ofw.img_idx)
        for k in ("scores", "sf", "inlier_map", "pixel_idxs"):
            assert np.array_equal(getattr(pfw, k), getattr(ofw, k)), k
        for k in ("entropy", "avg", "ref", "ref_steps_done", "n_perm_steps", "loss", "rot_err", "t_err", "correct"):
            assert np.array_equal(getattr(pfw, k), getattr(ofw, k)), k
        obw = O.backward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw)
        pbw = P.backward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], pfw)
        for k in ("dloss_dobj", "dref_dobj", "score_grads", "dpnp", "dloss_dref", "dref_dhyp"):
            assert np.array_equal(getattr(pbw, k), getattr(obw, k)), k


def test_dsac_pool_matches_oracle(frames):
    coords, pix, gt_cv, gt_jp = frames
    H = 16
    for f in range(2):
        cfg = O.default_config(seed=1305 + f, n_hyps=H)
        ofw = O.forward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], random_draw=False)
        pool = np.concatenate([ofw.hyp_rvec, ofw.hyp_tvec], 1)
        pfw = P.forward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], pool, ofw.img_idx)
        for k in ("sf", "ref_pose", "losses", "inlier_maps", "steps_done"):
            assert np.array_equal(getattr(pfw, k), getattr(ofw, k)), k
        for k in ("entropy", "expected_loss", "hyp_idx", "rot_err", "t_err", "correct"):
            assert getattr(pfw, k) == getattr(ofw, k), k
        obw = O.backward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw)
        pbw = P.backward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], pfw, 0)
        for k in ("dloss_dobj", "path1", "path2", "score_grads"):
            assert np.array_equal(getattr(pbw, k), getattr(obw, k)), k
        assert (pbw.n_selected, pbw.n_refine_jobs) == (obw.n_selected, obw.n_refine_jobs)


def test_prior_is_a_constant(frames):
    """A ground-truth prior in the last slot: it wins the pool, has no dPNP, and in the DSAC variant contributes refinement
    jobs from its own pose but no minimal-set jobs."""
    coords, pix, gt_cv, gt_jp = frames
    H = 16
    cfg = O.default_config(seed=1305, n_hyps=H - 1)
    ofw = O.forward_dsac(cfg, coords[0], pix[0], gt_jp[0, :9], gt_jp[0, 9:], random_draw=False)
    pool = np.concatenate([np.concatenate([ofw.hyp_rvec, ofw.hyp_tvec], 1), gt_cv[:1]])
    idx = np.concatenate([ofw.img_idx, -np.ones((1, 4), np.int32)])
    cfg = O.default_config(seed=1305, n_hyps=H)
    pfw = P.forward_dsac(cfg, coords[0], pix[0], gt_jp[0, :9], gt_jp[0, 9:], pool, idx)
    assert pfw.hyp_idx == H - 1 and pfw.sf[H - 1] > 1e-4
    pbw = P.backward_dsac(cfg, coords[0], pix[0], gt_jp[0, :9], gt_jp[0, 9:], pfw, 1)
    assert np.isfinite(pbw.dloss_dobj).all() and np.abs(pbw.path1).max() > 0
    sel = (pfw.sf > 1e-4)
    assert pbw.n_selected == sel.sum()
    sfw = P.forward(cfg, coords[0], pix[0], gt_jp[0, :9], gt_jp[0, 9:], pool, idx)
    sbw = P.backward(cfg, coords[0], pix[0], gt_jp[0, :9], gt_jp[0, 9:], sfw)
    assert (sbw.dpnp[H - 1] == 0).all() and np.isfinite(sbw.dloss_dobj).all()
