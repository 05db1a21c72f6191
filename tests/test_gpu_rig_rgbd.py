"""RGB-D rigs (dsac_set_rig_cell_depth_device) on the GPU: one camera behind a zero extrinsic is the ordinary RGB-D pass
and its covariance bit for bit, and its implicit backward bit for bit but for the direct term, which agrees to rounding; with C > 1 every frame samples as an ordinary RGB-D pass, the
refinement agrees with the CPU restatement (tests/rig_rgbd_oracle.py) and the direct gradient term with the host IFT of
the rig Kabsch fit; holes, batch independence, rig priors with rig depth, a rig that resolves a camera a single frame
gets wrong, the refusals, and the autograd functions."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import rgbd_oracle as RD
import rig_rgbd_oracle as RR
from test_gpu_rig import _bits, _cams, _compose, _jp, _setup, _two_cluster_rig
from test_gpu_rig_grad import Rig, _near
from test_gpu_rig_tracking import UNC, _ordinary, _priors, _rig, _rig_unc, _set_priors, _set_rig_priors, _unc

pytestmark = pytest.mark.gpu
N = 1600
REFINE_ABORTED, NO_DEPTH, BAD_RIG = 2, 64, 256


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _set_depth(eng, depth, C=None):
    """The rig cell depth for n frames of C cameras (C None: the ordinary cell depth); the device copy, to keep."""
    d = _dev(depth, np.float32)
    if C is None:
        eng.set_cell_depth_device(len(depth), d.data_ptr())
    else:
        eng.set_rig_cell_depth_device(len(depth), C, d.data_ptr())
    torch.cuda.synchronize()
    return d


def _intr(n, mode):
    return _cams(n) if mode == "cams" else np.tile([[525.0, 320.0, 240.0]], (n, 1))


@pytest.mark.parametrize("mode", ["uniform", "guided", "cams"])
def test_one_camera_zero_extrinsic_is_the_ordinary_rgbd_pass(engine_mod, mode):
    E = engine_mod
    n, H = 4, 64
    coords, pix, depth, gt_cv, gt_jp = RD.synth(n, seed=5, holes=0.2, cams=_intr(n, mode))
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    eng.set_coord_derivatives("implicit")
    keep = []
    _setup(eng, n, mode, keep)
    # the ordinary RGB-D pass: outputs, covariance, implicit backward
    keep.append(_set_depth(eng, depth))
    ref = _ordinary(eng, coords, pix, gt_jp, frame0=3, keep=keep)
    ref_unc = _unc(E, eng, n)
    ref_bw = eng.backward(coords, pix, gt_jp)
    eng.set_cell_depth_device(n, 0)
    # the same through a rig of one camera
    keep.append(_set_depth(eng, depth, 1))
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
    for key in ("dloss_dref", "dref_dhyp", "score_grads"):
        assert np.array_equal(_bits(got_bw[key]), _bits(getattr(ref_bw, key))), key
    # the direct term of the rig's RGB-D IFT agrees with the ordinary one in its last bits only, on the same cells
    assert np.array_equal(got_bw["dref_dobj"] != 0, ref_bw.dref_dobj != 0)
    assert _near(got_bw["dref_dobj"], ref_bw.dref_dobj, 1e-12)
    assert _near(got_bw["dobj"], ref_bw.dloss_dobj, 1e-12)
    assert np.abs(ref_bw.dloss_dobj).max() > 0


@pytest.mark.parametrize("C", [2, 4, 8])
def test_rgbd_rig_samples_as_ordinary_frames_and_refines_as_the_oracle(engine_mod, C):
    """hyp_pose against an ordinary RGB-D pass over the same frames and depth, bit for bit; the refinement against the CPU
    restatement from the device's soft-argmax pose (inlier maps and steps identical, the pose to test_gpu_rgbd.py's 1e-3)
    on rigs whose refinement tested no cell within 1e-4 px of the threshold; cells without depth never fitted; and
    dref_dobj against the host IFT of the rig Kabsch fit over the last step's cells."""
    from oracle import oracle as O
    E = engine_mod
    R, H = 3, 64
    n = R * C
    coords, pix, depth, ext, gt, _ = RR.scene(C, R, seed=C, holes=0.15)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=4)
    keep = [_set_depth(eng, depth, C)]
    dev = _rig(eng, coords, pix, ext, C, gt, frame0=2, keep=keep)
    got = Rig(eng, coords, pix, ext, C, gt, frame0=2).backward(seed=np.ones((R, 6)))
    eng.set_rig_cell_depth_device(n, C, 0)
    keep.append(_set_depth(eng, depth))
    ref = _ordinary(eng, coords, pix, frame0=2)
    eng.close()
    assert np.array_equal(_bits(dev["hyp_pose"]), _bits(ref.hyp_pose))
    assert not np.any(dev["inlier_map"][~(np.isfinite(depth) & (depth > 0))])
    assert dev["correct"].all(), (dev["rot_err"], dev["t_err"])
    cfg = O.default_config(n_hyps=H)
    intr = _intr(C, "uniform")
    compared = 0
    for r in range(R):
        fr = slice(r * C, (r + 1) * C)
        ey = RR.eye(pix[fr], depth[fr], intr)
        steps = int(dev["steps_done"][r])
        assert steps == eng.cfg.ref_steps and dev["status"][r] & (BAD_RIG | NO_DEPTH | REFINE_ABORTED) == 0
        cam, cell, margin, run = RR.last_step_cells(cfg, coords[fr], pix[fr], intr, ext[fr], ey, dev["avg_pose"][r], steps)
        if margin <= 1e-4:
            continue
        compared += 1
        assert np.array_equal(run["inlier_map"], dev["inlier_map"][fr]), r
        assert run["steps_done"] == steps
        assert np.abs(run["ref_pose"] - dev["ref_pose"][r]).max() <= 1e-3
        D = got["dref_dobj"][r].reshape(6, C, N, 3)
        want = np.zeros((C, N), bool)
        want[cam, cell] = True
        assert np.array_equal(np.abs(D).max(axis=(0, 3)) > 0, want)
        assert 50 <= len(cell) <= C * cfg.inlier_count
        host = RR.ift(cam, coords[fr][cam, cell], ey[cam, cell], ext[fr], dev["ref_pose"][r])
        assert host is not None
        assert _near(D[:, cam, cell, :].transpose(1, 0, 2), host, 1e-9)
    assert compared >= R - 1, compared


def test_holes(engine_mod):
    """Rig 0's camera 1 has no depth: DSAC_ST_NO_DEPTH, and the rig refines from the other cameras as the oracle does.  Rig
    1 has no depth anywhere: its refinement aborts, with no NaN in any output, its backward or its covariance."""
    from oracle import oracle as O
    E = engine_mod
    C, R, H = 3, 2, 64
    n = R * C
    coords, pix, depth, ext, gt, _ = RR.scene(C, R, seed=21)
    depth[1] = np.nan
    depth[C:] = np.nan
    eng = E.Engine(max_frames=n, n_hyps=H)
    keep = [_set_depth(eng, depth, C)]
    dev = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    unc = _rig_unc(eng, n, C)
    bw = Rig(eng, coords, pix, ext, C, gt).backward()
    eng.close()
    st = dev["status"]
    assert st[0] & NO_DEPTH and not st[0] & (BAD_RIG | REFINE_ABORTED) and dev["steps_done"][0] == eng.cfg.ref_steps
    assert st[1] & NO_DEPTH and st[1] & REFINE_ABORTED and not st[1] & BAD_RIG and dev["steps_done"][1] == 0
    assert not dev["inlier_map"][1].any() and not dev["inlier_map"][C:].any()
    for k, v in dev.items():
        assert np.isfinite(v).all(), k
    for k, v in list(unc.items()) + list(bw.items()):
        assert np.isfinite(v).all(), k
    assert unc["ok"][0] == 1 and unc["ok"][1] == 0 and unc["n_fit"][1] == 0
    assert dev["correct"][0] == 1
    intr = _intr(C, "uniform")
    cfg = O.default_config(n_hyps=H)
    o = RR.refine(cfg, coords[:C], pix[:C], intr, ext[:C], RR.eye(pix[:C], depth[:C], intr), dev["avg_pose"][0])
    assert o["min_margin"] > 1e-4
    assert np.array_equal(o["inlier_map"], dev["inlier_map"][:C])
    assert np.abs(o["ref_pose"] - dev["ref_pose"][0]).max() <= 1e-3


@pytest.mark.parametrize("n,C", [(24, 4), (1024, 4)])
def test_rgbd_rigs_do_not_depend_on_the_batch(engine_mod, n, C):
    """1024 frames take the sampler's two-lane path; each rig alone (frame0 at its first frame) gives the same bits."""
    E = engine_mod
    H = 64
    R = n // C
    coords, pix, depth, ext, gt, _ = RR.scene(C, R, seed=3, holes=0.1)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    keep = [_set_depth(eng, depth, C)]
    allr = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    for r in sorted({0, 1, R // 2, R - 1}):
        fr = slice(r * C, (r + 1) * C)
        keep.append(_set_depth(eng, depth[fr], C))
        one = _rig(eng, coords[fr], pix[fr], ext[fr], C, gt[r:r + 1], frame0=r * C, keep=keep)
        for k, v in one.items():
            whole = allr[k][fr] if k in ("hyp_pose", "inlier_map") else allr[k][r:r + 1]
            assert np.array_equal(_bits(v), _bits(whole)), (r, k)
    eng.close()


@pytest.mark.parametrize("gated", [False, True])
def test_rig_priors_with_rig_depth(engine_mod, gated):
    """One camera behind a zero extrinsic with rig priors and rig depth is the ordinary RGB-D pass with per-frame priors,
    its covariance included, bit for bit."""
    E = engine_mod
    n, H, k = 4, 64, 3
    coords, pix, depth, gt_cv, gt_jp = RD.synth(n, seed=8, holes=0.1)
    poses, info = _priors(np.random.default_rng(2), gt_cv, k, gated)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    keep = [_set_depth(eng, depth)] + _set_priors(eng, n, poses, info)
    ref = _ordinary(eng, coords, pix, gt_jp, keep=keep)
    ref_unc = _unc(E, eng, n)
    eng.set_pose_priors_device(n, 0, None)
    eng.set_cell_depth_device(n, 0)
    keep += [_set_depth(eng, depth, 1)] + _set_rig_priors(eng, n, 1, poses, info)
    rig = _rig(eng, coords, pix, np.zeros((n, 6)), 1, gt_jp, keep=keep)
    got_unc = _rig_unc(eng, n, 1)
    eng.close()
    assert np.array_equal(_bits(rig["hyp_pose"]), _bits(ref.hyp_pose))
    for key in ("scores", "sf", "avg_pose", "ref_pose", "inlier_map", "status"):
        assert np.array_equal(_bits(rig[key]), _bits(getattr(ref, key).astype(rig[key].dtype))), key
    for key in UNC:
        assert np.array_equal(_bits(got_unc[key]), _bits(ref_unc[key])), key
    assert rig["correct"].all()


def test_rgbd_rig_tracker_loop(engine_mod):
    """The tracker loop of "Rig tracking" with rig depth, over a sequence of RGB-D rig scenes: each step's prior is the last
    refined rig pose, gated by its covariance inflated by a motion noise wide enough for the next scene's pose; every step
    is correct and its covariance defined."""
    from dsac_b200 import autograd as A
    E = engine_mod
    C, H, steps = 4, 64, 4
    eng = E.Engine(max_frames=C, n_hyps=H, n_streams=2)
    prior = None
    for s in range(steps):
        coords, pix, depth, ext, gt, true = RR.scene(C, 1, seed=100 + s)
        pred = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda()
        out = A.rig_pose(eng, pred, _dev(pix, np.int32), _dev(ext, np.float64), C, gt_jp=_dev(gt, np.float64),
                         rig_priors=prior, cell_depth=_dev(depth, np.float32))
        unc = A.rig_pose_uncertainty(eng, C, C)
        torch.cuda.synchronize()
        assert int(out["correct"][0]) == 1 and int(unc["ok"][0]) == 1, s
        assert not int(out["status"][0]) & (BAD_RIG | 128)
        # the next step's scene is another random pose: a wide motion noise keeps the gate from rejecting it
        info = torch.linalg.inv(unc["cov_xi"] + torch.diag(torch.tensor([4.0] * 3 + [1e7] * 3, dtype=torch.float64, device="cuda")))
        prior = (out["ref_pose"][:, None].clone(), info[:, None].contiguous(), 16.81)
    eng.close()


def test_rig_resolves_a_two_cluster_camera(engine_mod):
    """test_gpu_rig.py's two-cluster rig with the depth of each cell's eye point: camera 0 alone, as an RGB-D frame, takes
    the wrong pose; the RGB-D rig refines to the true one."""
    E = engine_mod
    C, H = 4, 128
    coords, pix, ext, true, wrong = _two_cluster_rig(E, C)
    rng = np.random.default_rng(9)
    depth = rng.uniform(1500.0, 4000.0, size=(C, N)).astype(np.float32)
    f, cx, cy = 525.0, 320.0, 240.0
    for c in range(C):   # the eye depth of the pose (true or wrong) under which a cell reprojects onto its pixel
        for pose in (true, wrong):
            cam = _compose(ext[c], pose)
            X = Rotation.from_rotvec(cam[:3]).apply(coords[c].astype(np.float64)) + cam[3:]
            uv = np.stack([f * X[:, 0] / X[:, 2] + cx, f * X[:, 1] / X[:, 2] + cy], 1)
            on = np.linalg.norm(uv - pix[c], axis=1) < 2.0
            depth[c, on] = X[on, 2]
    eng = E.Engine(max_frames=C, n_hyps=H, n_streams=2)
    keep = [_set_depth(eng, depth[:1])]
    cam0 = _ordinary(eng, coords[:1], pix[:1], _jp(_compose(ext[0], true))[None], keep=keep)
    eng.set_cell_depth_device(1, 0)
    keep.append(_set_depth(eng, depth, C))
    rig = _rig(eng, coords, pix, ext, C, _jp(true)[None], keep=keep)
    eng.close()
    assert cam0.correct[0] == 0
    assert rig["correct"][0] == 1, (rig["rot_err"], rig["t_err"])
    assert rig["steps_done"][0] == eng.cfg.ref_steps and not rig["status"][0] & BAD_RIG


def test_refusals(engine_mod):
    E = engine_mod
    C, R, H = 2, 2, 32
    n = R * C
    coords, pix, depth, ext, gt, _ = RR.scene(C, R, seed=4)
    eng = E.Engine(max_frames=n, n_hyps=H)
    lib = E.load()
    lg = _dev(np.random.default_rng(1).normal(size=(n, N)), np.float32)
    eng.set_sampling_logits_device(n, lg.data_ptr())
    keep = [lg]
    dc, dp, de = _dev(coords, np.int16), _dev(pix, np.int32), _dev(ext, np.float64)
    dd = _dev(depth, np.float32)

    def refused(fn, text):
        with pytest.raises(RuntimeError, match="\\(-1\\)"):
            fn()
        assert text in lib.dsac_last_error(eng.h).decode(), lib.dsac_last_error(eng.h).decode()

    refused(lambda: eng.set_rig_cell_depth_device(n + 1, C, dd.data_ptr()), "out of range")
    refused(lambda: eng.set_rig_cell_depth_device(n, 0, dd.data_ptr()), "out of range")
    refused(lambda: eng.set_rig_cell_depth_device(n - 1, C, dd.data_ptr()), "not a multiple")
    keep.append(_set_depth(eng, depth, C))
    # a rig pass over another C or n
    refused(lambda: eng.forward_rig_device(n, 1, dc.data_ptr(), dp.data_ptr(), de.data_ptr()), "rig cell depth")
    refused(lambda: eng.forward_rig_device(C, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr()), "is for 4 frames of 2 cameras")
    # every other forward entry point
    refused(lambda: eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, None, 0), "dsac_set_rig_cell_depth_device")
    refused(lambda: eng.forward_dsac_device(n, dc.data_ptr(), dp.data_ptr(), 0, None, 0), "dsac_set_rig_cell_depth_device")
    refused(lambda: eng.forward(coords, pix), "dsac_set_rig_cell_depth_device")
    # per-frame cell depth: the rig pass keeps its refusal
    keep.append(_set_depth(eng, depth))
    refused(lambda: eng.forward_rig_device(n, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr()), "cell depth or pose priors")
    eng.set_cell_depth_device(n, 0)
    # the rig consumers after the rig depth changed
    r = Rig(eng, coords, pix, ext, C, gt)
    f64 = dict(dtype=torch.float64, device="cuda")
    buf, seed = torch.zeros((n, N, 3), **f64), torch.ones((R, 6), **f64)
    consumers = {
        "dsac_backward_rig_device": lambda: eng.backward_rig_device(n, None, buf.data_ptr()),
        "dsac_backward_rig_pose_device": lambda: eng.backward_rig_pose_device(n, seed.data_ptr(), buf.data_ptr()),
        "dsac_rig_refined_jp6_device": lambda: eng.rig_refined_jp6_device(n, buf.data_ptr()),
        "dsac_rig_pose_uncertainty_device": lambda: eng.rig_pose_uncertainty_device(n, C, cov_xi=buf.data_ptr()),
    }
    for fn in consumers.values():   # (the pass is usable before the change)
        fn()
    torch.cuda.synchronize()
    logp = torch.zeros(n, **f64)
    eng.sampling_log_prob_device(n, logp.data_ptr())
    keep.append(_set_depth(eng, depth, C))
    for who, fn in consumers.items():
        refused(fn, "the rig cell depth was changed (dsac_set_rig_cell_depth_device) after the forward pass")
    refused(lambda: eng.sampling_log_prob_device(n, logp.data_ptr()), "the rig cell depth was changed after the last pass")
    # the engine stays usable: a rig pass and its consumers run again
    r2 = Rig(eng, coords, pix, ext, C, gt)
    assert np.array_equal(_bits(r2.host()["ref_pose"]), _bits(r.host()["ref_pose"]))
    for fn in consumers.values():
        fn()
    eng.set_rig_cell_depth_device(n, C, None)
    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, None, 0)
    torch.cuda.synchronize()
    assert eng.last_pass(n) == "softam"
    eng.close()


def test_autograd_with_cell_depth_equals_the_entry_points(engine_mod):
    E = engine_mod
    from dsac_b200 import autograd as A
    C, R, H = 2, 2, 64
    n = R * C
    coords, pix, depth, ext, gt, _ = RR.scene(C, R, seed=12, holes=0.1)
    eng = E.Engine(max_frames=n, n_hyps=H)
    dp, de, dg, dd = _dev(pix, np.int32), _dev(ext, np.float64), _dev(gt, np.float64), _dev(depth, np.float32)
    pred = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda().requires_grad_(True)
    out = A.rig_pose(eng, pred.detach(), dp, de, C, gt_jp=dg, cell_depth=dd)
    torch.cuda.synchronize()
    ref = _rig(eng, coords, pix, ext, C, gt)   # the setting is sticky
    for k, v in out.items():
        assert np.array_equal(_bits(v.cpu().numpy()), _bits(ref[k])), k
    loss = A.rig_softam_loss(eng, pred, dp, de, C, dg, clamp=0.1, cell_depth=dd)
    loss.sum().backward()
    want = Rig(eng, coords, pix, ext, C, gt).backward(clamp=0.1, diag=False)["dpred"]
    assert np.array_equal(_bits(pred.grad.cpu().numpy()), _bits(want))
    assert np.abs(want).max() > 0
    pred2 = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda().requires_grad_(True)
    pose = A.rig_softam_pose(eng, pred2, dp, de, C, clamp=0.1, cell_depth=dd)
    w = torch.linspace(-1.0, 1.0, R * 6, dtype=torch.float64, device="cuda").reshape(R, 6)
    (pose * w).sum().backward()
    want = Rig(eng, coords, pix, ext, C).backward(seed=w.cpu().numpy(), clamp=0.1, diag=False)["dpred"]
    assert np.array_equal(_bits(pred2.grad.cpu().numpy()), _bits(want))
    with pytest.raises(ValueError, match="cell_depth"):
        A.rig_pose(eng, pred.detach(), dp, de, C, cell_depth=dd[:, :10])
    # clearing returns the rig passes to RGB
    eng.set_rig_cell_depth_device(n, C, None)
    rgb = _rig(eng, coords, pix, ext, C, gt)
    eng.close()
    assert not np.array_equal(_bits(rgb["ref_pose"]), _bits(ref["ref_pose"]))
