"""Rig gradients (dsac_backward_rig_device, dsac_backward_rig_pose_device, dsac_rig_refined_jp6_device) on the GPU: one
camera with a zero extrinsic is the ordinary implicit backward; the direct term is the host IFT of the rig fit; the seed
and loss forms agree; rigs are independent of their batch and of other calls; bad and aborted rigs; the refusals; and
the autograd functions rig_softam_loss / rig_softam_pose."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import rig_grad_oracle as RG

pytestmark = pytest.mark.gpu
N = 1600
BAD_RIG, REFINE_ABORTED = 256, 2


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _compose(ext, pose):
    Rc, R = Rotation.from_rotvec(ext[:3]), Rotation.from_rotvec(pose[:3])
    return np.concatenate([(Rc * R).as_rotvec(), Rc.apply(pose[3:]) + ext[3:]])


def _jp(pose):
    R = Rotation.from_rotvec(pose[:3]).as_matrix().copy()
    R[1:] = -R[1:]
    return np.concatenate([R.ravel(), [pose[3], -pose[4], -pose[5]]])


def _scene(E, C, R, seed=0, inliers=0.6):
    """R consistent rigs of C ring cameras: each camera sees `inliers` of its cells at the rig's true pose (0.5 px noise),
    the rest random scene points.  (coords, pix, ext [n][6], gt_rig [R][12])."""
    rng = np.random.default_rng(seed)
    n = R * C
    _, pix, _, _ = E.synth_frames(n)
    coords = np.empty((n, N, 3), np.int16)
    ext = np.concatenate([RG.ring(C, seed=seed + r) for r in range(R)])
    gt = np.empty((R, 12))
    f, cx, cy = 525.0, 320.0, 240.0
    for r in range(R):
        true = np.concatenate([Rotation.from_euler("xyz", rng.normal(scale=0.2, size=3)).as_rotvec(),
                               rng.normal(scale=300.0, size=3) + [0.0, 0.0, 1500.0]])
        gt[r] = _jp(true)
        for c in range(C):
            fr = r * C + c
            u = pix[fr, :, 0] + rng.normal(scale=0.5, size=N)
            v = pix[fr, :, 1] + rng.normal(scale=0.5, size=N)
            d = rng.uniform(1500.0, 4000.0, size=N)
            Xc = np.stack([(u - cx) / f * d, (v - cy) / f * d, d], 1)
            cam = _compose(ext[fr], true)
            X = Rotation.from_rotvec(cam[:3]).inv().apply(Xc - cam[3:])
            out = rng.uniform(size=N) >= inliers
            X[out] = rng.uniform(-4000.0, 4000.0, size=(out.sum(), 3))
            coords[fr] = np.clip(np.round(X), -32767, 32767).astype(np.int16)
    return coords, pix, ext, gt


class Rig:
    """A rig pass on device copies of host inputs, kept alive for the backward, and the rig backward's outputs."""

    def __init__(self, eng, coords, pix, ext, C, gt=None, frame0=0):
        self.eng, self.C, self.n = eng, C, len(coords)
        self.R, self.P = self.n // C, C * eng.cfg.n_hyps
        self.inputs = [_dev(coords, np.int16), _dev(pix, np.int32), _dev(ext, np.float64)]
        self.gt = _dev(gt, np.float64) if gt is not None else None
        f64 = dict(dtype=torch.float64, device="cuda")
        i32 = dict(dtype=torch.int32, device="cuda")
        self.out = {"ref_pose": torch.zeros((self.R, 6), **f64), "avg_pose": torch.zeros((self.R, 6), **f64),
                    "status": torch.zeros(self.R, **i32), "steps_done": torch.zeros(self.R, **i32),
                    "hyp_pose": torch.zeros((self.n, eng.cfg.n_hyps, 6), **f64), "rig_hyp": torch.zeros((self.R, self.P, 6), **f64),
                    "sf": torch.zeros((self.R, self.P), **f64), "inlier_map": torch.zeros((self.n, N), **i32)}
        if gt is not None:
            self.out["loss"] = torch.zeros(self.R, **f64)
        dc, dp, de = self.inputs
        eng.forward_rig_device(self.n, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr(), 0, self.gt.data_ptr() if gt is not None else None,
                               frame0, **{k: v.data_ptr() for k, v in self.out.items()})
        torch.cuda.synchronize()

    def host(self):
        return {k: v.cpu().numpy() for k, v in self.out.items()}

    def jp6(self):
        o = torch.zeros((self.R, 6), dtype=torch.float64, device="cuda")
        self.eng.rig_refined_jp6_device(self.n, o.data_ptr())
        torch.cuda.synchronize()
        return o.cpu().numpy()

    def backward(self, seed=None, loss_grad=None, clamp=0.0, diag=True):
        f64 = dict(dtype=torch.float64, device="cuda")
        dobj = torch.full((self.n, N, 3), np.nan, **f64)
        dpred = torch.full((self.n, N, 3), np.nan, dtype=torch.float32, device="cuda")
        d = {"dloss_dref": torch.zeros((self.R, 6), **f64), "dref_dhyp": torch.zeros((self.R, 6, 6), **f64),
             "score_grads": torch.zeros((self.R, self.P), **f64), "dref_dobj": torch.zeros((self.R, 6, self.C * N * 3), **f64)} if diag else {}
        ptrs = {k: v.data_ptr() for k, v in d.items()}
        if seed is not None:
            s = _dev(seed, np.float64)
            self.eng.backward_rig_pose_device(self.n, s.data_ptr(), dobj.data_ptr(), dpred.data_ptr(), clamp, **ptrs)
        else:
            g = _dev(loss_grad, np.float64) if loss_grad is not None else None
            self.eng.backward_rig_device(self.n, g.data_ptr() if g is not None else None, dobj.data_ptr(), dpred.data_ptr(), clamp, **ptrs)
        torch.cuda.synchronize()
        out = {k: v.cpu().numpy() for k, v in d.items()}
        out["dobj"], out["dpred"] = dobj.cpu().numpy(), dpred.cpu().numpy()
        return out


def _near(a, b, rel):
    scale = max(np.abs(a).max(), np.abs(b).max(), 1e-300)
    return np.abs(a - b).max() <= rel * scale


CASES = [("uniform", 0, 0.0), ("uniform", 1, 1e-4), ("guided", 0, 1e-4), ("guided", 1, 0.0), ("cams", 0, 0.0), ("cams", 1, 1e-4)]


@pytest.mark.parametrize("mode,fix_q4,clamp", CASES)
def test_one_camera_zero_extrinsic_is_the_ordinary_implicit_backward(engine_mod, mode, fix_q4, clamp):
    E = engine_mod
    n, H = 4, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=2)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2, fix_q4=fix_q4, grad_clamp=clamp)
    eng.set_coord_derivatives("implicit")
    keep = []
    if mode == "guided":
        lg = _dev(np.random.default_rng(3).normal(size=(n, N)), np.float32)
        eng.set_sampling_logits_device(n, lg.data_ptr())
        keep.append(lg)
    if mode == "cams":
        cams = np.tile([[525.0, 320.0, 240.0]], (n, 1))
        cams[1::2] = [580.0, 310.5, 250.25]
        eng.set_cameras(cams)
    # the ordinary pass and its implicit backward, loss and seeded forms
    dc, dp, dg = _dev(coords, np.int16), _dev(pix, np.int32), _dev(gt_jp, np.float64)
    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 3)
    ref = eng.backward(coords, pix, gt_jp)
    jp_ord = torch.zeros((n, 6), dtype=torch.float64, device="cuda")
    eng.refined_jp6_device(n, jp_ord.data_ptr())
    seed = np.random.default_rng(5).normal(size=(n, 6))
    ds = _dev(seed, np.float64)
    rows_seed = torch.zeros((n, N, 3), dtype=torch.float64, device="cuda")
    eng.backward_pose_device(n, ds.data_ptr(), rows_seed.data_ptr())
    torch.cuda.synchronize()
    jp_ord, rows_seed = jp_ord.cpu().numpy(), rows_seed.cpu().numpy()
    # the rig pass of one camera per rig, zero extrinsics
    rig = Rig(eng, coords, pix, np.zeros((n, 6)), 1, gt_jp, frame0=3)
    assert np.array_equal(_bits(rig.jp6()), _bits(jp_ord))
    got = rig.backward()
    got_seed = rig.backward(seed=seed, diag=False)
    eng.close()
    if clamp > 0:
        assert np.abs(ref.score_grads).max() > clamp   # the clamp bites
    assert np.array_equal(_bits(got["dloss_dref"]), _bits(ref.dloss_dref))
    assert np.array_equal(_bits(got["dref_dhyp"]), _bits(ref.dref_dhyp))
    assert np.array_equal(_bits(got["score_grads"]), _bits(ref.score_grads))
    assert np.array_equal(_bits(got["dref_dobj"]), _bits(ref.dref_dobj))
    # the support scatters sum in another order: the rows agree to rounding
    assert _near(got["dobj"], ref.dloss_dobj, 1e-12)
    assert _near(got_seed["dobj"], rows_seed, 1e-12)
    assert np.abs(ref.dloss_dobj).max() > 0


@pytest.mark.parametrize("C", [2, 3, 4])
def test_direct_term_is_the_host_ift_of_the_rig_fit(engine_mod, C):
    """dref_dobj against the host form of k_refine_ift_rig (rig_grad_shim.cpp) at the device's refined pose, over the cells
    of the last accepted refinement step as the CPU rig oracle selects them from the device's soft-argmax pose: its inlier
    map after k steps minus that after k - 1.  Those cells, and no others, carry dref_dobj.  A rig whose refinement tested
    a cell within 1e-4 px of the threshold is skipped, as tests/test_gpu_rig.py skips it (either decision is right)."""
    from oracle import oracle as O
    E = engine_mod
    R, H = 2, 64
    coords, pix, ext, gt = _scene(E, C, R, seed=C)
    eng = E.Engine(max_frames=R * C, n_hyps=H)
    rig = Rig(eng, coords, pix, ext, C, gt)
    out = rig.host()
    got = rig.backward(seed=np.ones((R, 6)))
    eng.close()
    cfg = eng.cfg
    compared = 0
    for r in range(R):
        steps = int(out["steps_done"][r])
        assert steps > 0 and not out["status"][r] & BAD_RIG
        fr = slice(r * C, (r + 1) * C)
        intr = np.tile([[cfg.focal, cfg.cx, cfg.cy]], (C, 1))
        cam, cell, margin, run = RG.last_step_cells(O.default_config(n_hyps=H), coords[fr], pix[fr], intr, ext[fr],
                                                    out["hyp_pose"][fr], out["avg_pose"][r], steps)
        if margin <= 1e-4:
            continue
        compared += 1
        assert np.array_equal(run["inlier_map"], out["inlier_map"][fr])
        D = got["dref_dobj"][r].reshape(6, C, N, 3)
        want = np.zeros((C, N), bool)
        want[cam, cell] = True
        assert np.array_equal(np.abs(D).max(axis=(0, 3)) > 0, want)    # the recorded cells, and zero elsewhere
        assert 50 <= len(cell) <= C * cfg.inlier_count
        host = RG.rig_ift(cam, coords[fr][cam, cell], pix[fr][cam, cell], ext[fr], intr, out["ref_pose"][r])
        assert host is not None
        assert _near(D[:, cam, cell, :].transpose(1, 0, 2), host, 1e-9)
    assert compared >= 1


@pytest.mark.parametrize("C,ref_steps,fix_q4,clamp", [(2, 8, 0, 0.1), (2, 0, 0, 0.1), (3, 0, 1, 1e-4), (4, 0, 0, 0.1)])
def test_whole_chain_matches_a_numpy_restatement(engine_mod, C, ref_steps, fix_q4, clamp):
    """dLoss/dObj of the rig backward against rig_grad_oracle.restate_rows: the path I support through L_j, and path II
    scored at every (camera frame, slot) with its support carried through K_c,j across the rig's cameras, restated in
    numpy from the device's dl, dRefineHyp, dref_dobj and score output gradients, with the dPNP of an ordinary implicit
    backward over the same frames (the same hypotheses, bit for bit).  On these scenes a refinement to convergence does
    not depend on its start, so dRefineHyp, and with it dLdAvg, the score output gradients, the support term and path II,
    nearly vanish: ref_steps 8 checks the direct term in the sum, ref_steps 0 (the refined pose is the soft-argmax pose)
    makes every other term carry the gradient.  fix_q4 1 and a clamp that bites cover both column layouts and the clamp."""
    E = engine_mod
    R, H = 2, 32
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=20 + C)
    eng = E.Engine(max_frames=n, n_hyps=H, fix_q4=fix_q4, grad_clamp=clamp, ref_steps=ref_steps)
    eng.set_coord_derivatives("implicit")
    dc, dp, dg = _dev(coords, np.int16), _dev(pix, np.int32), _dev(np.repeat(gt, C, 0), np.float64)
    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 0)
    ordinary = eng.fetch(n)
    ref = eng.backward(coords, pix, np.repeat(gt, C, 0))
    rig = Rig(eng, coords, pix, ext, C, gt)
    out = rig.host()
    got = rig.backward()
    cfg = eng.cfg
    eng.close()
    assert np.array_equal(_bits(out["hyp_pose"]), _bits(ordinary.hyp_pose))
    assert not np.any(out["status"] & BAD_RIG)
    if ref_steps:
        assert np.all(out["steps_done"] > 0)
    else:
        assert not np.any(got["dref_dobj"]) and np.abs(got["score_grads"]).max() > 1e-6
    if clamp < 0.1:
        assert np.abs(got["score_grads"]).max() > clamp   # the clamp bites
    want, dldavg = RG.restate_rows(cfg, C, coords, pix, ext, out["rig_hyp"], out["sf"], out["hyp_pose"], ordinary.img_idx,
                                   ref.dpnp, got["dloss_dref"], got["dref_dhyp"], got["dref_dobj"], got["score_grads"])
    # the score output gradients over the pool follow from dLdAvg as bw_combine_body forms them
    hf = (dldavg[:, None, :3] * out["rig_hyp"][..., :3]).sum(-1) + (dldavg[:, None, 3:] * (out["rig_hyp"][..., 3:] / 1000)).sum(-1)
    sog = out["sf"] * (hf - (out["sf"] * hf).sum(1, keepdims=True))
    assert _near(got["score_grads"], sog, 1e-10)
    assert _near(got["dobj"].reshape(n, -1), want, 1e-8), np.abs(got["dobj"].reshape(n, -1) - want).max() / np.abs(want).max()
    # every camera frame has a gradient
    assert all(np.abs(want[f]).max() > 0 for f in range(n))


def test_seed_reproduces_the_loss_form_and_is_linear(engine_mod):
    E = engine_mod
    C, R, H = 3, 2, 64
    coords, pix, ext, gt = _scene(E, C, R, seed=9)
    eng = E.Engine(max_frames=R * C, n_hyps=H, grad_clamp=0.0)   # no clamp: the chain is linear in its seed
    rig = Rig(eng, coords, pix, ext, C, gt)
    loss = rig.backward()
    seeded = rig.backward(seed=loss["dloss_dref"])
    doubled = rig.backward(seed=2 * loss["dloss_dref"])
    eng.close()
    assert _near(seeded["dobj"], loss["dobj"], 1e-14)
    assert np.array_equal(_bits(doubled["dobj"]), _bits(2 * seeded["dobj"]))
    assert np.abs(loss["dobj"]).max() > 0


def test_rigs_are_independent_of_the_batch_and_of_other_calls(engine_mod):
    E = engine_mod
    C, R, H = 2, 4, 64
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=4)
    eng = E.Engine(max_frames=n, n_hyps=H)
    rig = Rig(eng, coords, pix, ext, C, gt)
    jp = rig.jp6()
    a = rig.backward()
    b = rig.backward()
    assert np.array_equal(_bits(rig.jp6()), _bits(jp))
    for k in a:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k
    for r in (0, 2):
        fr = slice(r * C, (r + 1) * C)
        one = Rig(eng, coords[fr], pix[fr], ext[fr], C, gt[r:r + 1], frame0=r * C).backward()
        assert np.array_equal(_bits(one["dobj"]), _bits(a["dobj"][fr])), r
        assert np.array_equal(_bits(one["dref_dobj"]), _bits(a["dref_dobj"][r:r + 1])), r
    # a later ordinary pass gives the same results with or without a rig backward before it
    dc, dp = _dev(coords, np.int16), _dev(pix, np.int32)
    Rig(eng, coords, pix, ext, C, gt)
    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, None, 0)
    plain = eng.fetch(n)
    Rig(eng, coords, pix, ext, C, gt).backward()
    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, None, 0)
    after = eng.fetch(n)
    eng.close()
    for k in ("hyp_pose", "scores", "sf", "avg_pose", "ref_pose", "inlier_map", "status"):
        assert np.array_equal(_bits(getattr(after, k)), _bits(getattr(plain, k))), k


def test_bad_and_aborted_rigs(engine_mod):
    E = engine_mod
    C, R, H = 2, 3, 64
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=6)
    eng = E.Engine(max_frames=n, n_hyps=H)
    good = Rig(eng, coords, pix, ext, C, gt).backward()
    bad_ext = ext.copy()
    bad_ext[3, 1] = np.nan
    rig = Rig(eng, coords, pix, bad_ext, C, gt)
    assert [bool(s & BAD_RIG) for s in rig.host()["status"]] == [False, True, False]
    bad = rig.backward()
    again = rig.backward()
    for k in bad:
        assert np.array_equal(_bits(again[k]), _bits(bad[k])), k
    assert not np.any(bad["dobj"][2:4]) and not np.any(bad["dpred"][2:4])
    for k in ("dref_dhyp", "score_grads", "dref_dobj"):
        assert not np.any(bad[k][1]), k
    keep = np.r_[0:2, 4:6]
    assert np.array_equal(_bits(bad["dobj"][keep]), _bits(good["dobj"][keep]))
    # a rig whose cameras see random points only: no refinement step is accepted, so no direct term
    noise = coords.copy()
    noise[2:4] = np.random.default_rng(1).integers(-4000, 4000, size=(2, N, 3)).astype(np.int16)
    rig = Rig(eng, noise, pix, ext, C, gt)
    st = rig.host()
    got = rig.backward()
    eng.close()
    assert st["status"][1] & REFINE_ABORTED and st["steps_done"][1] == 0
    assert not np.any(got["dref_dobj"][1])
    assert np.isfinite(got["dobj"]).all() and np.isfinite(got["dpred"]).all()


def test_refusals(engine_mod):
    E = engine_mod
    C, R, H = 2, 2, 32
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=2)
    eng = E.Engine(max_frames=n, n_hyps=H)
    buf = torch.zeros((n, N, 3), dtype=torch.float64, device="cuda")
    seed = torch.zeros((R, 6), dtype=torch.float64, device="cuda")
    calls = {
        "dsac_backward_rig_device": lambda: eng.backward_rig_device(n, None, buf.data_ptr()),
        "dsac_backward_rig_pose_device": lambda: eng.backward_rig_pose_device(n, seed.data_ptr(), buf.data_ptr()),
        "dsac_rig_refined_jp6_device": lambda: eng.rig_refined_jp6_device(n, seed.data_ptr()),
    }

    def refused(fn, text):
        with pytest.raises(RuntimeError, match="\\(-1\\)"):
            fn()
        assert text in E.load().dsac_last_error(eng.h).decode(), E.load().dsac_last_error(eng.h).decode()

    for who, fn in calls.items():   # no pass yet
        refused(fn, "%s must follow a dsac_forward_rig_device over the same %d frames" % (who, n))
    dc, dp, dg = _dev(coords, np.int16), _dev(pix, np.int32), _dev(np.tile(gt, (C, 1)), np.float64)
    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 0)
    for who, fn in calls.items():
        refused(fn, "must follow a dsac_forward_rig_device")
    eng.forward_dsac_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr())
    for who, fn in calls.items():
        refused(fn, "must follow a dsac_forward_rig_device")
    rig = Rig(eng, coords, pix, ext, C, gt)
    for fn in calls.values():
        fn()
    torch.cuda.synchronize()
    refused(lambda: eng.backward_rig_device(n - C, None, buf.data_ptr()), "must follow")
    refused(lambda: eng.backward_rig_pose_device(n, None, buf.data_ptr()), "null d_grad_ref")
    refused(lambda: eng.rig_refined_jp6_device(n, None), "null output")
    eng.set_cameras(np.tile([[525.0, 320.0, 240.0]], (n, 1)))
    for fn in calls.values():
        refused(fn, "the cameras were changed (dsac_set_cameras) after the forward pass")
    eng.set_cameras(None)
    Rig(eng, coords, pix, ext, C)   # without ground truth: the seeded form only
    refused(calls["dsac_backward_rig_device"], "needs the rig ground truth")
    calls["dsac_backward_rig_pose_device"]()
    eng.set_stages(E.STAGE_SAMPLE | E.STAGE_SCORE | E.STAGE_REFINE)
    Rig(eng, coords, pix, ext, C, gt)   # ground truth without the EVAL stage
    refused(calls["dsac_backward_rig_device"], "needs the rig ground truth")
    eng.set_stages(E.STAGE_ALL)
    Rig(eng, coords, pix, ext, C, gt)
    res = eng.forward_submit(coords, pix, np.tile(gt, (C, 1)))
    refused(calls["dsac_backward_rig_device"], "has not been awaited")
    eng.forward_wait()
    assert res.ref_pose.shape == (n, 6)
    torch.cuda.synchronize()
    del rig
    eng.close()


def _autograd_case(E, C=2, R=2, H=64):
    coords, pix, ext, gt = _scene(E, C, R, seed=12)
    return coords, pix, ext, gt, E.Engine(max_frames=R * C, n_hyps=H)


def test_autograd_matches_the_entry_points(engine_mod):
    E = engine_mod
    from dsac_b200 import autograd as A
    C = 2
    coords, pix, ext, gt, eng = _autograd_case(E, C)
    n, R = len(coords), len(gt)
    dp, de, dg = _dev(pix, np.int32), _dev(ext, np.float64), _dev(gt, np.float64)
    pred = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda().requires_grad_(True)
    loss = A.rig_softam_loss(eng, pred, dp, de, C, dg, clamp=0.1)
    assert loss.shape == (R,) and loss.dtype == torch.float64
    loss.sum().backward()
    want = Rig(eng, coords, pix, ext, C, gt).backward(clamp=0.1, diag=False)["dpred"]
    assert np.array_equal(_bits(pred.grad.cpu().numpy()), _bits(want))
    assert np.abs(want).max() > 0
    # the pose form, seeded by the gradient of a function of the pose
    pred2 = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda().requires_grad_(True)
    pose = A.rig_softam_pose(eng, pred2, dp, de, C, clamp=0.1)
    assert pose.shape == (R, 6)
    w = torch.linspace(-1.0, 1.0, R * 6, dtype=torch.float64, device="cuda").reshape(R, 6)
    (pose * w).sum().backward()
    want = Rig(eng, coords, pix, ext, C).backward(seed=w.cpu().numpy(), clamp=0.1, diag=False)["dpred"]
    assert np.array_equal(_bits(pred2.grad.cpu().numpy()), _bits(want))
    # a non-contiguous prediction gives the same gradient
    strided = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda().permute(0, 2, 1).contiguous().permute(0, 2, 1)
    strided.requires_grad_(True)
    assert not strided.is_contiguous()
    A.rig_softam_loss(eng, strided, dp, de, C, dg, clamp=0.1).sum().backward()
    assert torch.equal(strided.grad, pred.grad)
    eng.close()


def test_autograd_guard_after_another_forward(engine_mod):
    E = engine_mod
    from dsac_b200 import autograd as A
    C = 2
    coords, pix, ext, gt, eng = _autograd_case(E, C)
    dp, de, dg = _dev(pix, np.int32), _dev(ext, np.float64), _dev(gt, np.float64)
    pred = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda().requires_grad_(True)
    loss = A.rig_softam_loss(eng, pred, dp, de, C, dg)
    A.rig_pose(eng, pred, dp, de, C)
    with pytest.raises(RuntimeError, match="another forward pass"):
        loss.sum().backward()
    pose = A.rig_softam_pose(eng, pred, dp, de, C)
    A.rig_softam_pose(eng, pred, dp, de, C)
    with pytest.raises(RuntimeError, match="another forward pass"):
        pose.sum().backward()
    eng.close()
