"""Rig tracking on the GPU (dsac_set_rig_pose_priors_device, dsac_rig_pose_uncertainty_device): with one camera behind a zero
extrinsic the rig pass with rig priors, its covariance and its backward are the ordinary pass with per-frame priors bit for
bit; with C > 1 every frame samples as an ordinary engine given the composed priors, the pool holds the rig priors' bits
and the gate is the rig-frame gate; the covariance agrees with the host build over the cells the CPU rig oracle selects;
bad priors spoil only their rig; the refusals; ordering, the two-lane batch and a tracker over a two-cluster rig trajectory."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import rig_grad_oracle as RG
import rig_tracking_oracle as RT
from test_gpu_pose_uncertainty import support_errors
from test_gpu_rig import _bits, _compose, _dev, _jp, _setup, _two_cluster_rig
from test_gpu_rig_grad import Rig, _near, _scene

pytestmark = pytest.mark.gpu
N = 1600
BAD_PRIOR, BAD_RIG = 128, 256
CHI2 = 16.81
UNC = ("cov_jp6", "cov_xi", "sigma2", "n_fit", "support", "ok")


def _rig(eng, coords, pix, ext, C, gt_rig=None, frame0=0, fields=None, keep=None):
    """dsac_forward_rig_device on device copies of host arrays, which are appended to `keep` (the covariance and the
    backward read the pass's inputs); returns host copies of every output."""
    n = len(coords)
    R, P, H = n // C, C * eng.cfg.n_hyps, eng.cfg.n_hyps
    ins = [_dev(coords, np.int16), _dev(pix, np.int32), _dev(ext, np.float64)]
    gt = _dev(gt_rig, np.float64) if gt_rig is not None else None
    f64, i32 = dict(dtype=torch.float64, device="cuda"), dict(dtype=torch.int32, device="cuda")
    out = {"hyp_pose": torch.zeros((n, H, 6), **f64), "rig_hyp": torch.zeros((R, P, 6), **f64),
           "scores": torch.zeros((R, P), **f64), "sf": torch.zeros((R, P), **f64), "entropy": torch.zeros(R, **f64),
           "avg_pose": torch.zeros((R, 6), **f64), "ref_pose": torch.zeros((R, 6), **f64),
           "inlier_map": torch.zeros((n, N), **i32), "steps_done": torch.zeros(R, **i32), "status": torch.zeros(R, **i32),
           "loss": torch.zeros(R, **f64), "rot_err": torch.zeros(R, **f64), "t_err": torch.zeros(R, **f64),
           "correct": torch.zeros(R, **i32)}
    if fields is not None:
        out = {k: v for k, v in out.items() if k in fields}
    eng.forward_rig_device(n, C, ins[0].data_ptr(), ins[1].data_ptr(), ins[2].data_ptr(), 0,
                           gt.data_ptr() if gt is not None else None, frame0, **{k: v.data_ptr() for k, v in out.items()})
    torch.cuda.synchronize()
    if keep is not None:
        keep += ins + [gt]
    return {k: v.cpu().numpy() for k, v in out.items()}


def _ordinary(eng, coords, pix, gt_jp=None, frame0=0, keep=None):
    n = len(coords)
    dc, dp = _dev(coords, np.int16), _dev(pix, np.int32)
    dg = _dev(gt_jp, np.float64) if gt_jp is not None else None
    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr() if dg is not None else None, frame0)
    res = eng.fetch(n)
    torch.cuda.synchronize()
    if keep is not None:
        keep += [dc, dp, dg]
    return res


def _host(d):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in d.items()}


def _unc(E, eng, n):
    from dsac_b200 import autograd as A
    return _host(A.pose_uncertainty(eng, n))


def _rig_unc(eng, n, C, stream=None):
    from dsac_b200 import autograd as A
    return _host(A.rig_pose_uncertainty(eng, n, C))


def _priors(rng, poses, k, gated):
    """k priors per entry near the given cv poses [m][6], and their information (or None)."""
    m = len(poses)
    out = np.empty((m, k, 6))
    for i in range(m):
        for j in range(k):
            dR = Rotation.from_rotvec(rng.normal(scale=0.01, size=3))
            out[i, j, :3] = (dR * Rotation.from_rotvec(poses[i, :3])).as_rotvec()
            out[i, j, 3:] = poses[i, 3:] + rng.normal(scale=20.0, size=3)
    if not gated:
        return out, None
    info = np.zeros((m, k, 6, 6))
    info[:, :, range(3), range(3)] = 1.0 / 0.15 ** 2
    info[:, :, range(3, 6), range(3, 6)] = 1.0 / 150.0 ** 2
    return out, info


def _set_rig_priors(eng, n, C, poses, info, gate=CHI2):
    keep = [_dev(poses, np.float64)] + ([_dev(info, np.float64)] if info is not None else [])
    eng.set_rig_pose_priors_device(n, C, poses.shape[1], keep[0].data_ptr(), keep[1].data_ptr() if info is not None else None, gate)
    torch.cuda.synchronize()
    return keep


def _set_priors(eng, n, poses, info, gate=CHI2):
    keep = [_dev(poses, np.float64)] + ([_dev(info, np.float64)] if info is not None else [])
    eng.set_pose_priors_device(n, poses.shape[1], keep[0].data_ptr(), keep[1].data_ptr() if info is not None else None, gate)
    torch.cuda.synchronize()
    return keep


@pytest.mark.parametrize("mode", ["uniform", "guided", "cams"])
@pytest.mark.parametrize("gated", [False, True])
def test_one_camera_zero_extrinsic_is_the_ordinary_pass_with_priors(engine_mod, mode, gated):
    E = engine_mod
    n, H, k = 4, 64, 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=2)
    poses, info = _priors(np.random.default_rng(1), gt_cv, k, gated)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    eng.set_coord_derivatives("implicit")
    keep = []
    _setup(eng, n, mode, keep)
    # the ordinary pass with per-frame priors: outputs, covariance, implicit backward
    keep += _set_priors(eng, n, poses, info)
    ref = _ordinary(eng, coords, pix, gt_jp, frame0=3, keep=keep)
    ref_unc = _unc(E, eng, n)
    ref_bw = eng.backward(coords, pix, gt_jp)
    eng.set_pose_priors_device(n, 0, None)
    # the same through a rig of one camera
    keep += _set_rig_priors(eng, n, 1, poses, info)
    rig = _rig(eng, coords, pix, np.zeros((n, 6)), 1, gt_jp, frame0=3, keep=keep)
    got_unc = _rig_unc(eng, n, 1)
    r2 = Rig(eng, coords, pix, np.zeros((n, 6)), 1, gt_jp, frame0=3)
    got_bw = r2.backward()
    eng.close()
    assert np.array_equal(_bits(rig["hyp_pose"]), _bits(ref.hyp_pose))
    assert np.array_equal(_bits(rig["rig_hyp"]), _bits(ref.hyp_pose))
    for key in ("scores", "sf", "entropy", "avg_pose", "ref_pose", "inlier_map", "loss", "rot_err", "t_err", "correct", "status"):
        assert np.array_equal(_bits(rig[key]), _bits(getattr(ref, key).astype(rig[key].dtype))), (mode, key)
    assert np.array_equal(rig["steps_done"], ref.ref_steps_done)
    assert rig["correct"].sum() > 0
    for key in UNC:
        assert np.array_equal(_bits(got_unc[key]), _bits(ref_unc[key])), key
    assert ref_unc["ok"].all()
    for key in ("dloss_dref", "dref_dhyp", "score_grads", "dref_dobj"):
        assert np.array_equal(_bits(got_bw[key]), _bits(getattr(ref_bw, key))), key
    assert _near(got_bw["dobj"], ref_bw.dloss_dobj, 1e-12)
    assert np.abs(ref_bw.dloss_dobj).max() > 0


@pytest.mark.parametrize("C,mode", [(2, "uniform"), (3, "cams"), (4, "guided")])
def test_frames_sample_as_an_ordinary_engine_with_the_composed_priors(engine_mod, C, mode):
    """Ungated: each frame's sampled slots and its prior slots against an ordinary engine given the composed poses (taken
    from the rig pass's hyp_pose prior slots, which are checked against the host composition); the pool's prior slots hold
    the rig priors' bits."""
    E = engine_mod
    R, H, k = 3, 64, 2
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=C)
    rng = np.random.default_rng(C)
    rp, _ = _priors(rng, rng.normal(scale=[0.3, 0.3, 0.3, 300, 300, 300], size=(R, 6)) + [0, 0, 0, 0, 0, 1500.0], k, False)
    keep = []
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=4)
    _setup(eng, n, mode, keep)
    keep += _set_rig_priors(eng, n, C, rp, None)
    rig = _rig(eng, coords, pix, ext, C, frame0=2)
    comp = rig["hyp_pose"][:, H - k:]
    for f in range(n):
        for j in range(k):
            ok, want, _ = RT.compose(ext[f], rp[f // C, j])
            assert ok and np.allclose(comp[f, j], want, rtol=0, atol=1e-9)
    eng.set_rig_pose_priors_device(n, C, 0, None)
    keep += _set_priors(eng, n, comp, None)
    ref = _ordinary(eng, coords, pix, frame0=2)
    eng.close()
    assert np.array_equal(_bits(rig["hyp_pose"]), _bits(ref.hyp_pose))
    assert not (rig["status"] & (BAD_PRIOR | BAD_RIG)).any()
    for r in range(R):
        for c in range(C):
            assert np.array_equal(_bits(rig["rig_hyp"][r, c * H + H - k:(c + 1) * H]), _bits(rp[r]))


@pytest.mark.parametrize("C", [2, 4])
def test_gated_rig_samples_pass_the_rig_frame_gate(engine_mod, C):
    """Gated: every sampled hypothesis, lifted to the rig, passes the rig-frame gate on the host (a hypothesis within 1e-9
    of the bound may fall either way), and the pool's prior slots hold the rig priors' bits.
    The sampled slots against an ordinary engine given the composed priors, whose information is composed in numpy: equal
    unless a candidate's distance lies within 1e-9 of the bound."""
    E = engine_mod
    R, H, k = 2, 64, 1
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=10 + C)
    truth = np.stack([np.concatenate([Rotation.from_matrix(np.diag([1, -1, -1]) @ g[:9].reshape(3, 3)).as_rotvec(),
                                      g[9:] * [1, -1, -1]]) for g in gt])
    rp, info = _priors(np.random.default_rng(C), truth, k, True)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=4)
    keep = _set_rig_priors(eng, n, C, rp, info)
    rig = _rig(eng, coords, pix, ext, C, frame0=1)
    comp = rig["hyp_pose"][:, H - k:].copy()
    info_c = np.stack([RT.compose_np(ext[f], rp[f // C, 0], info[f // C, 0])[1] for f in range(n)])[:, None]
    eng.set_rig_pose_priors_device(n, C, 0, None)
    keep += _set_priors(eng, n, comp, info_c)
    ref = _ordinary(eng, coords, pix, frame0=1)
    eng.close()
    rejected = 0
    for f in range(n):
        r = f // C
        for h in range(H - k):
            hp = rig["hyp_pose"][f, h]
            if not hp.any():
                continue
            d2 = RT.prior_d2(RT.lift(ext[f], hp), rp[r, 0], info[r, 0])
            assert d2 <= CHI2 * (1 + 1e-9), (f, h, d2)
        if not np.array_equal(_bits(rig["hyp_pose"][f]), _bits(ref.hyp_pose[f])):
            # a flip of the gate between the two compositions: only at the bound
            d_rig = [RT.prior_d2(RT.lift(ext[f], hp), rp[r, 0], info[r, 0]) for hp in ref.hyp_pose[f, :H - k]]
            assert min(abs(d - CHI2) for d in d_rig) <= 1e-9 * CHI2, f
            rejected += 1
    assert rejected <= 1
    for r in range(R):
        for c in range(C):
            assert np.array_equal(_bits(rig["rig_hyp"][r, c * H + H - k:(c + 1) * H]), _bits(rp[r]))
    assert not (rig["status"] & (BAD_PRIOR | BAD_RIG)).any()


@pytest.mark.parametrize("C", [2, 3, 4])
def test_rig_covariance_matches_the_host_over_the_oracle_cells(engine_mod, C):
    from oracle import oracle as O
    E = engine_mod
    R, H = 2, 64
    coords, pix, ext, gt = _scene(E, C, R, seed=20 + C)
    eng = E.Engine(max_frames=R * C, n_hyps=H)
    keep = []
    rig = _rig(eng, coords, pix, ext, C, keep=keep)
    unc = _rig_unc(eng, R * C, C)
    eng.close()
    cfg = eng.cfg
    compared = 0
    for r in range(R):
        steps = int(rig["steps_done"][r])
        fr = slice(r * C, (r + 1) * C)
        intr = np.tile([[cfg.focal, cfg.cx, cfg.cy]], (C, 1))
        cam, cell, margin, run = RG.last_step_cells(O.default_config(n_hyps=H), coords[fr], pix[fr], intr, ext[fr],
                                                    rig["hyp_pose"][fr], rig["avg_pose"][r], steps)
        # support: the count of every camera at the composed pose, up to cells at the threshold (check_support's rule)
        sure = amb = 0
        for c in range(C):
            e64, e32 = support_errors(coords[r * C + c], pix[r * C + c], _compose(ext[r * C + c], rig["ref_pose"][r]), intr[c])
            a = (np.abs(e64 - cfg.thr2d) <= 1e-4) | (np.abs(e32 - cfg.thr2d) <= 1e-4) | ((e64 < cfg.thr2d) != (e32 < cfg.thr2d))
            sure += int(((e64 < cfg.thr2d) & ~a).sum())
            amb += int(a.sum())
        assert sure <= unc["support"][r] <= sure + amb
        if margin <= 1e-4:
            continue
        compared += 1
        assert unc["n_fit"][r] == len(cell)
        ok, cxi, cjp, s2 = RT.rig_cov(cam, coords[fr][cam, cell], pix[fr][cam, cell], ext[fr], intr, rig["ref_pose"][r])
        assert ok and unc["ok"][r] == 1
        for key, h in (("cov_xi", cxi), ("cov_jp6", cjp)):
            assert np.abs(unc[key][r] - h).max() <= 1e-9 * np.abs(h).max(), key
        assert abs(unc["sigma2"][r] - s2) <= 1e-9 * s2
    assert compared >= 1


def test_bad_priors_spoil_only_their_rig(engine_mod):
    """Rig 1: a non-finite rig prior; rig 2: a singular information; rig 3: a NaN extrinsic.  Rig 0 is bit-identical to
    the same pass without the others."""
    E = engine_mod
    C, R, H, k = 2, 4, 64, 1
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=3)
    truth = np.stack([np.concatenate([Rotation.from_matrix(np.diag([1, -1, -1]) @ g[:9].reshape(3, 3)).as_rotvec(),
                                      g[9:] * [1, -1, -1]]) for g in gt])
    rp, info = _priors(np.random.default_rng(0), truth, k, True)
    rp[1, 0, 4] = np.inf
    info[2, 0] = 0.0
    info[2, 0, 0, 0] = 1.0
    ext = ext.copy()
    ext[7, 2] = np.nan
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    keep = _set_rig_priors(eng, n, C, rp, info)
    rig = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    unc = _rig_unc(eng, n, C)
    r2 = Rig(eng, coords, pix, ext, C, gt)
    bw = r2.backward()
    keep += _set_rig_priors(eng, C, C, rp[:1], info[:1])
    alone = _rig(eng, coords[:C], pix[:C], ext[:C], C, gt[:1], keep=keep)
    alone_unc = _rig_unc(eng, C, C)
    eng.close()
    for r in (1, 2, 3):
        assert rig["status"][r] & BAD_PRIOR, r
        assert bool(rig["status"][r] & BAD_RIG) == (r == 3)
        for key in ("rig_hyp", "scores", "sf", "entropy", "avg_pose", "ref_pose", "steps_done", "loss", "correct"):
            assert not rig[key][r].any(), (r, key)
        assert not rig["inlier_map"][r * C:(r + 1) * C].any()
        assert not rig["hyp_pose"][r * C:(r + 1) * C].any()
        for key in UNC:
            assert not unc[key][r].any(), (r, key)
        assert not bw["dobj"][r * C:(r + 1) * C].any()
    assert not rig["status"][0] & (BAD_PRIOR | BAD_RIG) and rig["correct"][0] == 1
    for key in ("rig_hyp", "scores", "sf", "avg_pose", "ref_pose", "status", "loss"):
        assert np.array_equal(_bits(rig[key][:1]), _bits(alone[key])), key
    for key in UNC:
        assert np.array_equal(_bits(unc[key][:1]), _bits(alone_unc[key])), key
    assert unc["ok"][0] == 1


def test_refusals_leave_the_engine_usable(engine_mod):
    E = engine_mod
    C, R, H = 2, 2, 32
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=5)
    rp, info = _priors(np.random.default_rng(0), np.zeros((R, 6)) + [0, 0, 0, 0, 0, 1500.0], 1, True)
    dp, di = _dev(rp, np.float64), _dev(info, np.float64)
    eng = E.Engine(max_frames=n, n_hyps=H)
    dc, dpix = _dev(coords, np.int16), _dev(pix, np.int32)
    out = torch.zeros((R, 6, 6), dtype=torch.float64, device="cuda")

    def refused(fn, text):
        with pytest.raises(RuntimeError, match=text):
            fn()

    # the setter's validation
    refused(lambda: eng.set_rig_pose_priors_device(n - 1, C, 1, dp.data_ptr()), "multiple")
    refused(lambda: eng.set_rig_pose_priors_device(n, 9, 1, dp.data_ptr()), "n_cameras")
    refused(lambda: eng.set_rig_pose_priors_device(n, C, 0, dp.data_ptr()), "k 0 out of range")
    refused(lambda: eng.set_rig_pose_priors_device(n, C, 33, dp.data_ptr()), "k 33 out of range")
    refused(lambda: eng.set_rig_pose_priors_device(n, C, 1, dp.data_ptr(), di.data_ptr(), 0.0), "gate")
    refused(lambda: eng.set_rig_pose_priors_device(2 * n, C, 1, dp.data_ptr()), "out of range")
    # no rig pass yet
    refused(lambda: eng.rig_pose_uncertainty_device(n, C, cov_xi=out.data_ptr()), "must follow a dsac_forward_rig_device")
    _ordinary(eng, coords, pix)
    refused(lambda: eng.rig_pose_uncertainty_device(n, C, cov_xi=out.data_ptr()), "must follow a dsac_forward_rig_device")
    # while rig priors are set the ordinary passes refuse, naming the setter
    eng.set_rig_pose_priors_device(n, C, 1, dp.data_ptr(), di.data_ptr(), CHI2)
    refused(lambda: eng.forward_device(n, dc.data_ptr(), dpix.data_ptr()), "dsac_set_rig_pose_priors_device")
    refused(lambda: eng.forward(coords, pix), "dsac_set_rig_pose_priors_device")
    refused(lambda: eng.forward_dsac(coords, pix, None), "dsac_set_rig_pose_priors_device")
    refused(lambda: eng.forward_dsac_device(n, dc.data_ptr(), dpix.data_ptr()), "dsac_set_rig_pose_priors_device")
    refused(lambda: eng.forward_submit(coords, pix), "dsac_set_rig_pose_priors_device")
    # a rig pass of another shape
    refused(lambda: _rig(eng, coords[:C], pix[:C], ext[:C], C), "rig pose priors")
    refused(lambda: _rig(eng, coords, pix, ext, 1), "rig pose priors")
    # the existing refusal of per-frame priors keeps its text
    keep = _set_priors(eng, n, rp.repeat(C, 0), None)
    refused(lambda: _rig(eng, coords, pix, ext, C), "cell depth or pose priors are set; a rig pass takes neither")
    eng.set_pose_priors_device(n, 0, None)
    rig = Rig(eng, coords, pix, ext, C, gt)
    unc = _rig_unc(eng, n, C)
    refused(lambda: eng.rig_pose_uncertainty_device(n, 1, cov_xi=out.data_ptr()), "n_cameras 1 differs")
    # the consumers refuse after the rig priors changed, and accept again after a new pass
    eng.set_rig_pose_priors_device(n, C, 1, dp.data_ptr(), None)
    refused(lambda: eng.rig_pose_uncertainty_device(n, C, cov_xi=out.data_ptr()), "rig pose priors were changed")
    refused(lambda: rig.jp6(), "rig pose priors were changed")
    refused(lambda: rig.backward(), "rig pose priors were changed")
    eng.set_rig_pose_priors_device(n, C, 1, dp.data_ptr(), di.data_ptr(), CHI2)
    rig = Rig(eng, coords, pix, ext, C, gt)
    again = _rig_unc(eng, n, C)
    for key in UNC:
        assert np.array_equal(_bits(again[key]), _bits(unc[key])), key
    rig.backward()
    # clearing the setting lets the ordinary passes run again
    eng.set_rig_pose_priors_device(n, C, 0, None)
    _ordinary(eng, coords, pix)
    eng.close()
    del keep


def test_refusal_after_a_guided_rig_pass_for_the_log_probability(engine_mod):
    E = engine_mod
    C, R, H = 2, 2, 32
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=6)
    rp, _ = _priors(np.random.default_rng(0), np.zeros((R, 6)) + [0, 0, 0, 0, 0, 1500.0], 1, False)
    eng = E.Engine(max_frames=n, n_hyps=H)
    keep = []
    _setup(eng, n, "guided", keep)
    keep += _set_rig_priors(eng, n, C, rp, None)
    _rig(eng, coords, pix, ext, C)
    logp = torch.zeros(n, dtype=torch.float64, device="cuda")
    eng.sampling_log_prob_device(n, logp.data_ptr())
    torch.cuda.synchronize()
    assert np.isfinite(logp.cpu().numpy()).all()
    keep += _set_rig_priors(eng, n, C, rp + 1.0, None)
    with pytest.raises(RuntimeError, match="rig pose priors were changed"):
        eng.sampling_log_prob_device(n, logp.data_ptr())
    eng.close()


def test_covariance_on_another_stream_changes_no_backward(engine_mod):
    E = engine_mod
    C, R, H = 3, 2, 64
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=8)
    rp, info = _priors(np.random.default_rng(2), np.zeros((R, 6)) + [0, 0, 0, 0, 0, 1500.0], 2, True)
    eng = E.Engine(max_frames=n, n_hyps=H)
    keep = _set_rig_priors(eng, n, C, rp, info)
    rig = Rig(eng, coords, pix, ext, C, gt)
    first = rig.backward()
    side = torch.cuda.Stream()
    outs = {k: torch.zeros((R, 6, 6), dtype=torch.float64, device="cuda") for k in ("cov_xi", "cov_jp6")}
    eng.rig_pose_uncertainty_device(n, C, side.cuda_stream, **{k: v.data_ptr() for k, v in outs.items()})
    second = rig.backward()
    torch.cuda.synchronize()
    eng.close()
    for key in first:
        assert np.array_equal(_bits(first[key]), _bits(second[key])), key


def test_two_lane_batch_samples_as_the_ordinary_pass_with_the_composed_priors(engine_mod):
    """1024 frames (the sampler's two-lane path) of 256 rigs of 4 cameras with rig priors: every frame's hypotheses are the
    ordinary two-lane pass's under the composed per-frame priors, bit for bit, every rig's prior slots hold its rig prior,
    and the rig covariance repeats bit for bit.  (A frame's draw is compared within one batch size: at this size the
    ordinary sampler's schedule differs from that of four frames alone, with or without priors.)"""
    E = engine_mod
    C, H, k = 4, 64, 1
    n = 1024
    R = n // C
    coords, pix, ext, gt = _scene(E, C, 8, seed=9)
    reps = R // 8
    coords, pix, ext, gt = np.tile(coords, (reps, 1, 1)), np.tile(pix, (reps, 1, 1)), np.tile(ext, (reps, 1)), np.tile(gt, (reps, 1))
    truth = np.stack([np.concatenate([Rotation.from_matrix(np.diag([1, -1, -1]) @ g[:9].reshape(3, 3)).as_rotvec(),
                                      g[9:] * [1, -1, -1]]) for g in gt])
    rp, _ = _priors(np.random.default_rng(4), truth, k, False)
    eng = E.Engine(max_frames=n, n_hyps=H)
    keep = _set_rig_priors(eng, n, C, rp, None)
    big = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    unc = _rig_unc(eng, n, C)
    again = _rig_unc(eng, n, C)
    eng.set_rig_pose_priors_device(n, C, 0, None)
    keep += _set_priors(eng, n, big["hyp_pose"][:, H - k:].copy(), None)
    ref = _ordinary(eng, coords, pix)
    eng.close()
    assert np.array_equal(_bits(big["hyp_pose"]), _bits(ref.hyp_pose))
    for r in range(R):
        for c in range(C):
            assert np.array_equal(_bits(big["rig_hyp"][r, c * H + H - k:(c + 1) * H]), _bits(rp[r]))
    for key in UNC:
        assert np.array_equal(_bits(unc[key]), _bits(again[key])), key
    assert big["correct"].mean() > 0.8 and unc["ok"].mean() > 0.8


def _moved(coords, true, step):
    """The two-cluster rig's scene at step `step` of a trajectory: the scene moved by Y' = A Y + b (A 2 degrees per step
    about y, b 60 mm per step along x), so that the rig, whose cameras see the same points, has the pose T o (A, b)^-1;
    the wrong cluster moves with the scene."""
    A = Rotation.from_rotvec([0.0, np.radians(2.0 * step), 0.0])
    b = np.array([60.0 * step, 0.0, 0.0])
    moved = np.clip(np.round(A.apply(coords.reshape(-1, 3).astype(np.float64)) + b), -32767, 32767).astype(np.int16)
    R = Rotation.from_rotvec(true[:3]) * A.inv()
    return moved.reshape(coords.shape), np.concatenate([R.as_rotvec(), true[3:] - R.apply(b)])


def test_tracker_over_a_two_cluster_trajectory(engine_mod):
    """The rig version of the constant-position tracker: prior = the previous refined rig pose, information inv(cov_xi + Q)
    from rig_pose_uncertainty, chi^2 16.81.  Correct at every step; then a wrong prior under a tight gate exhausts the
    streams (status & 1) and keeps its prior slots."""
    from dsac_b200 import autograd as A
    E = engine_mod
    C, H = 4, 128
    coords, pix, ext, true, wrong = _two_cluster_rig(E, C)
    eng = E.Engine(max_frames=C, n_hyps=H, n_streams=2)
    Q = np.diag([1e-3] * 3 + [100.0 ** 2] * 3)   # the motion per step: 2 degrees, 60 mm
    pix_t = torch.tensor(pix, dtype=torch.int32, device="cuda")
    ext_t = torch.tensor(ext, dtype=torch.float64, device="cuda")
    prior = None
    for step in range(6):
        moved, pose = _moved(coords, true, step)
        pred = torch.tensor(moved.astype(np.float32) / 1000.0, device="cuda")
        gt_t = torch.tensor(_jp(pose)[None], dtype=torch.float64, device="cuda")
        out = A.rig_pose(eng, pred, pix_t, ext_t, C, frame0=100 * step, gt_jp=gt_t, rig_priors=prior)
        torch.cuda.synchronize()
        assert out["correct"][0].item() == 1, (step, out["rot_err"], out["t_err"])
        assert not out["status"][0].item() & (BAD_PRIOR | BAD_RIG)
        unc = A.rig_pose_uncertainty(eng, C, C)
        assert unc["ok"][0].item() == 1
        info = torch.linalg.inv(unc["cov_xi"] + torch.tensor(Q, device="cuda"))
        prior = (out["ref_pose"][:, None].clone(), info[:, None].contiguous(), CHI2)
    # a wrong prior under a tight gate: no sampled hypothesis passes, the streams run out, the prior slot stays
    eng2 = E.Engine(max_frames=C, n_hyps=H, n_streams=2, max_candidates=20000)
    pred = torch.tensor(coords.astype(np.float32) / 1000.0, device="cuda")
    far = torch.tensor(wrong[None, None], dtype=torch.float64, device="cuda")
    tight = torch.tensor(np.diag([1e8] * 3 + [1e4] * 3)[None, None], dtype=torch.float64, device="cuda")
    out = A.rig_pose(eng2, pred, pix_t, ext_t, C, rig_priors=(far, tight, CHI2))
    torch.cuda.synchronize()
    assert out["status"][0].item() & 1
    rig_hyp = out["rig_hyp"].cpu().numpy()
    for c in range(C):
        assert np.array_equal(_bits(rig_hyp[0, c * H + H - 1]), _bits(wrong))
    eng.close()
    eng2.close()
