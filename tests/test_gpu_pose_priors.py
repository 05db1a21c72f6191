"""Pose priors (dsac_set_pose_priors_device) on the GPU: the sampled slots of a k-prior pass are those of an engine with
n_hyps - k in every sampler path; the prior slots carry the given bits; a pool of priors equal to sampled hypotheses gives
the very pass that sampled them; the covariance gate keeps exactly the candidates numpy's gate keeps; bad priors empty
their frame only; the backward passes treat priors as constants; clearing, refusals and the autograd keyword."""
import os

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

pytestmark = pytest.mark.gpu
N = 1600
BAD_PRIOR = 128


def _priors(eng, poses, info=None, gate=0.0):
    """Set the priors from host arrays; returns the device tensors (kept alive by the caller)."""
    p = torch.from_numpy(np.ascontiguousarray(poses, np.float64)).cuda()
    i = torch.from_numpy(np.ascontiguousarray(info, np.float64)).cuda() if info is not None else None
    eng.set_pose_priors_device(p.shape[0], p.shape[1], p.data_ptr(), i.data_ptr() if i is not None else None, gate)
    torch.cuda.synchronize()
    return p, i


def _prior_poses(gt_cv, k, seed):
    rng = np.random.default_rng(seed)
    n = len(gt_cv)
    out = np.empty((n, k, 6))
    for f in range(n):
        for j in range(k):
            rv = (Rotation.from_rotvec(rng.normal(scale=0.05, size=3)) * Rotation.from_rotvec(gt_cv[f, :3])).as_rotvec()
            out[f, j] = np.concatenate([rv, gt_cv[f, 3:] + rng.normal(scale=30.0, size=3)])
    return out


def _engine(E, n, H, T, mono=False, **kw):
    if mono:
        os.environ["DSAC_K1_MODE"] = "mono"
    try:
        return E.Engine(max_frames=n, n_hyps=H, n_streams=T, **kw)
    finally:
        os.environ.pop("DSAC_K1_MODE", None)


def _setup(E, eng, n, mode, depth, keep):
    """Per-pass settings of a sampler mode on an engine (depth: _frames' for RGB-D); tensors go to `keep`."""
    if mode == "guided":
        lg = torch.from_numpy(np.random.default_rng(3).normal(size=(n, N)).astype(np.float32)).cuda()
        eng.set_sampling_logits_device(n, lg.data_ptr())
        keep.append(lg)
    if mode == "rgbd":
        d = torch.from_numpy(np.ascontiguousarray(depth, np.float32)).cuda()
        eng.set_cell_depth_device(n, d.data_ptr())
        keep.append(d)
    if mode == "cams":
        cams = np.tile([[525.0, 320.0, 240.0]], (n, 1))
        cams[1::2] = [580.0, 310.5, 250.25]
        eng.set_cameras(cams)
    torch.cuda.synchronize()


def _frames(E, mode, n, T, rho=None):
    if mode == "rgbd":
        import rgbd_oracle as R
        return R.synth(n, seed=5, holes=0.1, **({"rho": rho} if rho else {}))
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=T, **({"rho": rho} if rho else {}))
    return coords, pix, None, gt_cv, gt_jp


CASES = [
    # (frames, H, streams, sampler mode, k1 mono)
    (4, 64, 1, "uniform", False),
    (2, 512, 8, "uniform", False),      # speculative first round (quota >= 64)
    (1024, 64, 4, "uniform", False),    # two lanes
    (3, 64, 2, "uniform", True),        # k1_mode 0: the monolithic k_sample
    (4, 64, 2, "guided", False),
    (4, 64, 2, "rgbd", False),
    (4, 64, 2, "cams", False),
]


@pytest.mark.parametrize("n,H,T,mode,mono", CASES)
def test_sampled_slots_match_smaller_engine(engine_mod, n, H, T, mode, mono):
    E = engine_mod
    coords, pix, depth, gt_cv, gt_jp = _frames(E, mode, n, T)
    for k in (1, 7):
        keep = []
        eng = _engine(E, n, H, T, mono)
        _setup(E, eng, n, mode, depth, keep)
        pri = _prior_poses(gt_cv, k, seed=k)
        keep.append(_priors(eng, pri))
        res = eng.forward(coords, pix, gt_jp, frame0=3)
        # prior slots hold the given bits, with -1 indices
        assert np.array_equal(res.hyp_pose[:, H - k:].view(np.uint64), pri.view(np.uint64))
        assert (res.img_idx[:, H - k:] == -1).all() and (res.cand_idx[:, H - k:] == -1).all()
        assert not (res.status & BAD_PRIOR).any()
        assert np.isfinite(res.ref_pose).all()
        eng.close()
        small = _engine(E, n, H - k, min(T, H - k), mono)
        _setup(E, small, n, mode, depth, keep)
        ref = small.forward(coords, pix, gt_jp, frame0=3)
        small.close()
        if T > H - k:
            continue   # a smaller engine cannot have more streams than hypotheses
        assert np.array_equal(res.hyp_pose[:, :H - k].view(np.uint64), ref.hyp_pose.view(np.uint64)), (mode, k)
        assert np.array_equal(res.img_idx[:, :H - k], ref.img_idx)
        assert np.array_equal(res.cand_idx[:, :H - k], ref.cand_idx)
        assert np.array_equal(res.n_candidates, ref.n_candidates)
        assert np.array_equal(res.status, ref.status)


@pytest.mark.parametrize("mode", ["uniform", "guided", "rgbd"])
def test_all_slots_priors_samples_nothing(engine_mod, mode):
    """k == H: nothing is sampled; the pass scores and refines the priors."""
    E = engine_mod
    n, H = 3, 16
    coords, pix, depth, gt_cv, gt_jp = _frames(E, mode, n, 2)
    keep = []
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    _setup(E, eng, n, mode, depth, keep)
    pri = _prior_poses(gt_cv, H, seed=2)
    keep.append(_priors(eng, pri))
    res = eng.forward(coords, pix, gt_jp)
    assert np.array_equal(res.hyp_pose.view(np.uint64), pri.view(np.uint64))
    assert (res.img_idx == -1).all() and (res.n_candidates == 0).all() and (res.status == 0).all()
    assert np.isfinite(res.sf).all() and np.isfinite(res.ref_pose).all()
    d = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    assert np.isfinite(d.losses).all() and ((d.hyp_idx >= 0) & (d.hyp_idx < H)).all()
    eng.close()


@pytest.mark.parametrize("mode", ["uniform", "rgbd"])
def test_pool_of_sampled_poses_gives_the_same_pass(engine_mod, mode):
    """With one stream the first H - k hypotheses of an H engine are those of an H - k engine, so priors equal to the H
    engine's last k hypotheses rebuild its pool: every output after sampling must be the same bits."""
    E = engine_mod
    n, H, k = 4, 64, 5
    coords, pix, depth, gt_cv, gt_jp = _frames(E, mode, n, 1)
    keep = []
    base = E.Engine(max_frames=n, n_hyps=H, n_streams=1)
    _setup(E, base, n, mode, depth, keep)
    r0 = base.forward(coords, pix, gt_jp)
    d0 = base.forward_dsac(coords, pix, gt_jp, random_draw=False)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=1)
    _setup(E, eng, n, mode, depth, keep)
    keep.append(_priors(eng, r0.hyp_pose[:, H - k:]))
    r1 = eng.forward(coords, pix, gt_jp)
    d1 = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    assert np.array_equal(r1.hyp_pose, r0.hyp_pose)
    for name in ("scores", "sf", "entropy", "avg_pose", "ref_pose", "loss", "rot_err", "t_err", "correct", "inlier_map"):
        assert np.array_equal(getattr(r1, name), getattr(r0, name)), name
    for name in ("sf", "entropy", "ref_pose", "losses", "expected_loss", "hyp_idx"):
        assert np.array_equal(getattr(d1, name), getattr(d0, name)), name
    base.close()
    eng.close()


def _d2(poses_h, prior, info):
    rel = Rotation.from_rotvec(poses_h[:, :3]) * Rotation.from_rotvec(prior[:3]).inv()
    xi = np.concatenate([rel.as_rotvec(), poses_h[:, 3:] - prior[3:]], 1)
    return np.einsum("ni,ij,nj->n", xi, info, xi)


# every gated acceptance site: k1_solve_gate (uniform, guided rounds), k1_solve_cam_gate (cams), k1_kabsch_gate (rgbd),
# k_sample_gate (mono: k1_mode 0), and the tails that continue the rounds' streams (k_sample_gate / k1_gtail_gate resume)
@pytest.mark.parametrize("mode", ["uniform", "rgbd", "guided", "cams", "mono"])
def test_gate_keeps_numpy_survivors_in_order(engine_mod, mode):
    E = engine_mod
    n, H, k = 2, 64, 1
    mono = mode == "mono"
    smode = "uniform" if mono else mode
    coords, pix, depth, gt_cv, gt_jp = _frames(E, smode, n, 1, rho=0.8)   # enough survivors among 1024 accepted hypotheses
    keep = []
    # every accepted candidate of the stream, long enough to hold the gated pass's quota of survivors
    big = _engine(E, n, 1024, 1, mono, max_candidates=2000000)
    _setup(E, big, n, smode, depth, keep)
    ug = big.forward(coords, pix, gt_jp)
    big.close()
    prior = ug.ref_pose[:, None, :].copy()   # the refined pose: the hypotheses cluster around it in every mode
    info = np.tile(np.diag([1 / 0.05 ** 2] * 3 + [1 / 100.0 ** 2] * 3), (n, k, 1, 1))
    chi2 = 16.81
    eng = _engine(E, n, H, 1, mono, max_candidates=2000000)
    _setup(E, eng, n, smode, depth, keep)
    keep.append(_priors(eng, prior, info, chi2))
    res = eng.forward(coords, pix, gt_jp)
    for f in range(n):
        d2 = _d2(ug.hyp_pose[f], prior[f, 0], info[f, 0])
        surv = ug.cand_idx[f][d2 <= chi2]
        assert len(surv) >= H - k, "the ungated pass is too short for this frame"
        assert np.array_equal(res.cand_idx[f, :H - k], surv[:H - k]), f
        assert (_d2(res.hyp_pose[f, :H - k], prior[f, 0], info[f, 0]) <= chi2 * (1 + 1e-9)).all()
    eng.close()
    # a gate far from every candidate exhausts the streams at max_candidates
    tight = _engine(E, n, H, 2, mono, max_candidates=3000)
    _setup(E, tight, n, smode, depth, keep)
    far = prior.copy()
    far[:, :, 3:] += 5000.0
    keep.append(_priors(tight, far, np.tile(np.eye(6) * 1e6, (n, k, 1, 1)), chi2))
    rt = tight.forward(coords, pix, gt_jp)
    assert (rt.status & 1).all() and (rt.n_candidates == 2 * 3000).all()
    assert (rt.img_idx[:, :H - k] == -1).all()
    tight.close()


def test_bad_priors_empty_their_frame_only(engine_mod):
    E = engine_mod
    n, H, k = 4, 64, 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=2)
    pri = _prior_poses(gt_cv, k, seed=1)
    info = np.tile(np.eye(6), (n, k, 1, 1))
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    keep = [_priors(eng, pri, info, 1e9)]
    good = eng.forward(coords, pix, gt_jp)
    pri_bad, info_bad = pri.copy(), info.copy()
    pri_bad[1, 2, 4] = np.nan
    info_bad[2, 0] = np.diag([1, 1, 1, 1, 1, -1.0])                   # indefinite
    keep.append(_priors(eng, pri_bad, info_bad, 1e9))
    bad = eng.forward(coords, pix, gt_jp)
    for f in (1, 2):
        assert bad.status[f] & BAD_PRIOR and not bad.status[f] & 1      # (the refinement of an empty frame aborts: bit 2)
        assert (bad.img_idx[f] == -1).all() and (bad.hyp_pose[f] == 0).all() and bad.n_candidates[f] == 0
    for f in (0, 3):
        for name in ("hyp_pose", "img_idx", "cand_idx", "scores", "sf", "ref_pose", "status", "n_candidates"):
            assert np.array_equal(getattr(bad, name)[f], getattr(good, name)[f]), (f, name)
    eng.close()


@pytest.mark.parametrize("deriv", ["central", "implicit"])
@pytest.mark.parametrize("mode", ["uniform", "rgbd"])
def test_backward_treats_priors_as_constants(engine_mod, deriv, mode):
    E = engine_mod
    n, H, k = 3, 64, 1
    coords, pix, depth, gt_cv, gt_jp = _frames(E, mode, n, 1)
    keep = []
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=1)
    _setup(E, eng, n, mode, depth, keep)
    eng.set_coord_derivatives(deriv)
    keep.append(_priors(eng, gt_cv[:, None, :]))                      # the ground truth: it dominates sf
    fw = eng.forward(coords, pix, gt_jp)
    assert (fw.sf[:, H - 1] > 1e-4).all(), fw.sf[:, H - 1]            # the prior takes part in path I
    bw = eng.backward(coords, pix, gt_jp)
    assert np.isfinite(bw.dloss_dobj).all()
    assert (bw.dpnp[:, H - k:] == 0).all()                            # no minimal set: no dPNP
    d = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    bd = eng.backward_dsac(n)
    assert np.isfinite(bd.dloss_dobj).all()
    sel_prior = d.sf[:, H - 1] > 1e-4
    sel_sampled = (d.sf[:, :H - k] > 1e-4) & (d.img_idx[:, :H - k, 0] >= 0)
    assert np.array_equal(bd.n_selected, sel_prior + sel_sampled.sum(1))
    if deriv == "implicit":   # 9 minimal-set pairs (18 jobs) per sampled hypothesis, none for the prior
        assert np.array_equal(bd.n_refine_jobs, 18 * sel_sampled.sum(1))
    eng.close()


def _rel(a, b, floor=1e-300):
    return np.abs(a - b).max() / max(floor, np.abs(b).max())


@pytest.mark.parametrize("H,fix_q4", [(16, 0), (32, 1)])
def test_backward_matches_pool_oracle(engine_mod, oracle, H, fix_q4):
    """Central differences, RGB, a ground-truth prior that wins the pool, against the oracle restated for a given pool
    (tests/pool_oracle.py), at test_gpu_backward.py's tolerances; n_selected and n_refine_jobs exactly."""
    import pool_oracle as P
    E, O = engine_mod, oracle
    n, k = 2, 1
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    eng = E.Engine(max_frames=n, n_hyps=H, fix_q4=fix_q4)
    keep = [_priors(eng, gt_cv[:, None, :])]
    fwd = eng.forward(coords, pix, gt_jp)
    bw = eng.backward(coords, pix, gt_jp)
    for f in range(n):
        cfg = O.default_config(seed=1305 + f, n_hyps=H, fix_q4=fix_q4)
        pfw = P.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], fwd.hyp_pose[f], fwd.img_idx[f])
        assert pfw.sf[H - 1] > 0.5                                    # the prior dominates
        assert np.abs(pfw.sf - fwd.sf[f]).max() <= 1e-4 and np.abs(pfw.ref - fwd.ref_pose[f]).max() <= 1e-3
        pbw = P.backward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], pfw)
        assert _rel(bw.dloss_dref[f], pbw.dloss_dref) <= 1e-9
        assert _rel(bw.dref_dhyp[f], pbw.dref_dhyp, floor=1e-3) <= 1e-7
        assert _rel(bw.dref_dobj[f], pbw.dref_dobj, floor=1e-3) <= 1e-7
        assert _rel(bw.dpnp[f], pbw.dpnp) <= 1e-7 and (bw.dpnp[f, H - k:] == 0).all()
        assert _rel(bw.score_grads[f], pbw.score_grads, floor=1e-6) <= 1e-4
        assert _rel(bw.dloss_dobj[f], pbw.dloss_dobj, floor=1e-6) <= 1e-3
    d = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    bd = eng.backward_dsac(n)
    for f in range(n):
        cfg = O.default_config(seed=1305 + f, n_hyps=H)
        pfw = P.forward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], d.hyp_pose[f], d.img_idx[f])
        assert pfw.hyp_idx == d.hyp_idx[f] == H - 1
        assert np.abs(pfw.sf - d.sf[f]).max() <= 1e-4 and np.abs(pfw.ref_pose - d.ref_pose[f]).max() <= 1e-3
        ofw = O.ForwardDsac(cfg)   # the engine's forward state, as test_gpu_backward.py feeds the oracle
        ofw.hyp_rvec[:] = d.hyp_pose[f][:, :3]; ofw.hyp_tvec[:] = d.hyp_pose[f][:, 3:]
        ofw.img_idx[:] = d.img_idx[f]; ofw.sf[:] = d.sf[f]; ofw.ref_pose[:] = d.ref_pose[f]; ofw.losses[:] = d.losses[f]
        pbw = P.backward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw, k)
        assert pbw.n_selected == bd.n_selected[f] and d.sf[f, H - 1] > 1e-4
        assert pbw.n_refine_jobs == bd.n_refine_jobs[f]              # central mode: the prior has no minimal-set jobs
        assert _rel(bd.score_grads[f], pbw.score_grads, floor=1e-12) <= 1e-9
        assert np.abs(pbw.path1).max() > 0
        assert _rel(bd.path1[f], pbw.path1) <= 1e-5
        assert _rel(bd.path2[f], pbw.path2) <= 1e-6
        assert _rel(bd.dloss_dobj[f], pbw.dloss_dobj) <= 1e-5
    eng.close()


def test_lifecycle_and_refusals(engine_mod):
    E = engine_mod
    n, H = 3, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=2)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    r0 = eng.forward(coords, pix, gt_jp)
    keep = [_priors(eng, _prior_poses(gt_cv, 2, 0))]
    p = keep[0][0]
    with pytest.raises(RuntimeError):
        eng.set_pose_priors_device(n + 1, 2, p.data_ptr())            # n > max_frames
    with pytest.raises(RuntimeError):
        eng.set_pose_priors_device(n, 17, p.data_ptr())               # k > DSAC_MAX_PRIORS
    with pytest.raises(RuntimeError):
        eng.set_pose_priors_device(n, 2, p.data_ptr(), p.data_ptr(), float("nan"))   # a gate that is not finite
    with pytest.raises(RuntimeError):
        eng.set_pose_priors_device(n, 2, p.data_ptr(), p.data_ptr(), 0.0)
    r1 = eng.forward(coords, pix, gt_jp)                              # the refusals left the setting in force
    assert np.array_equal(r1.hyp_pose[:, H - 2:].view(np.uint64), keep[0][0].cpu().numpy().view(np.uint64))
    eng.set_pose_priors_device(n, 0, None)                            # clear: backward and queries refuse the pass before
    buf = torch.zeros(n * 6, dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError):
        eng.refined_jp6_device(n, buf.data_ptr())
    with pytest.raises(RuntimeError):
        eng.backward(coords, pix, gt_jp)
    r2 = eng.forward(coords, pix, gt_jp)
    for name in ("hyp_pose", "img_idx", "cand_idx", "sf", "ref_pose", "status", "n_candidates"):
        assert np.array_equal(getattr(r2, name), getattr(r0, name)), name
    keep.append(_priors(eng, _prior_poses(gt_cv, 2, 0)))
    with pytest.raises(RuntimeError):
        eng.forward(coords[:2], pix[:2], gt_jp[:2])                   # the setting has 3 frames
    ok = torch.zeros(n, dtype=torch.int32, device="cuda")
    eng.forward(coords, pix, gt_jp)
    eng.pose_uncertainty_device(n, ok=ok.data_ptr())                  # the pass of this setting: accepted
    keep.append(_priors(eng, _prior_poses(gt_cv, 3, 1)))              # set again: the queries refuse that pass
    with pytest.raises(RuntimeError):
        eng.pose_uncertainty_device(n, ok=ok.data_ptr())
    with pytest.raises(RuntimeError):
        eng.backward_device(n)
    # a submitted pass that has not been awaited: the setting cannot change
    h = eng.forward_submit(coords, pix, gt_jp)
    with pytest.raises(RuntimeError):
        eng.set_pose_priors_device(n, 2, p.data_ptr())
    with pytest.raises(RuntimeError):
        eng.set_pose_priors_device(n, 0, None)
    eng.forward_wait()
    r3 = eng.forward(coords, pix, gt_jp)                              # the 3-prior setting is still the one in force
    assert (r3.img_idx[:, H - 3:] == -1).all() and (r3.img_idx[:, :H - 3] >= 0).all()
    del h
    eng.close()


def test_sampling_log_prob_refuses_after_priors_change(engine_mod):
    E = engine_mod
    n, H = 2, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    eng = E.Engine(max_frames=n, n_hyps=H)
    keep = []
    _setup(E, eng, n, "guided", None, keep)
    keep.append(_priors(eng, _prior_poses(gt_cv, 1, 0)))
    eng.forward(coords, pix, gt_jp)
    logp = torch.zeros(n, dtype=torch.float64, device="cuda")
    gl = torch.ones(n, dtype=torch.float64, device="cuda")
    grad = torch.zeros((n, N), dtype=torch.float32, device="cuda")
    eng.sampling_log_prob_device(n, logp.data_ptr())                  # the pass of this setting: accepted
    eng.set_pose_priors_device(n, 0, None)
    with pytest.raises(RuntimeError):
        eng.sampling_log_prob_device(n, logp.data_ptr())
    with pytest.raises(RuntimeError):
        eng.sampling_log_prob_backward_device(n, gl.data_ptr(), grad.data_ptr())
    eng.close()


def test_autograd_keyword(engine_mod):
    E = engine_mod
    from dsac_b200 import autograd as A
    n, H, k = 3, 64, 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    eng = E.Engine(max_frames=n, n_hyps=H)
    pred = (torch.from_numpy(coords.astype(np.float32)) / 1000).cuda().requires_grad_(True)
    pix_t = torch.from_numpy(pix).cuda()
    gt = torch.from_numpy(gt_jp).cuda()
    poses = torch.from_numpy(_prior_poses(gt_cv, k, 4)).cuda()
    info = torch.eye(6, dtype=torch.float64, device="cuda").expand(n, k, 6, 6) * 1e-3
    pp = (poses, info, 1e6)
    for fn in (lambda: A.softam_loss(eng, pred, pix_t, gt, pose_priors=pp),
               lambda: A.dsac_expected_loss(eng, pred, pix_t, gt, pose_priors=pp),
               lambda: A.softam_pose(eng, pred, pix_t, pose_priors=pp).sum(1),
               lambda: A.dsac_hypotheses(eng, pred, pix_t, pose_priors=(poses, None, 0.0))[0][:, H - 1]):
        pred.grad = None
        fn().sum().backward()
        assert pred.grad is not None and torch.isfinite(pred.grad).all()
    with pytest.raises(ValueError):
        A.softam_loss(eng, pred, pix_t, gt, pose_priors=(poses.float(), None, 0.0))
    eng.close()
