"""Multi-camera rigs at the limits of the API on the GPU: eight cameras (DSAC_MAX_RIG_CAMERAS), pools of up to C H = 1024
slots (DSAC_MAX_HYPS), pools that are not a multiple of the score tile or of 8, every camera with its own intrinsics, and
16 rig priors in a full pool.  The forward, the whole backward chain, its direct IFT term, the rig covariance and the
RGB-D rig covariance against the host references the smaller rig tests use (tests/rig_oracle.py, rig_grad_oracle.py,
rig_tracking_oracle.py, rig_rgbd_oracle.py), at those tests' tolerances; and 128 full-pool rigs of eight cameras in one
two-lane batch against the same rigs among other neighbours."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import rig_grad_oracle as RG
import rig_oracle as RO
import rig_rgbd_oracle as RR
import rig_tracking_oracle as RT
from ift_oracle import DFLIP
from test_gpu_pose_uncertainty import support_errors
from test_gpu_rig import _bits, _compose, _jp
from test_gpu_rig_grad import Rig, _near
from test_gpu_rig_tracking import _priors, _rig, _rig_unc, _set_rig_priors

pytestmark = pytest.mark.gpu
N = 1600
REFINE_ABORTED, BAD_PRIOR, BAD_RIG = 2, 128, 256


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _distinct_cams(n, C):
    """Per-frame intrinsics [n][3] in which every camera of a rig has its own f, cx and cy (and the rigs differ in f);
    every value is exact in fp32."""
    c, r = np.arange(n) % C, np.arange(n) // C
    return np.stack([500.0 + 12.5 * c + 0.25 * (r % 4), 312.0 + 2.25 * c, 236.0 + 1.5 * c], 1)


def _intr(n, C, cams):
    return _distinct_cams(n, C) if cams else np.tile([[525.0, 320.0, 240.0]], (n, 1))


def _engine(E, n, H, mode, intr, **kw):
    """An engine for n frames of H hypotheses; mode "cams" sets the per-frame intrinsics, "guided" sampling logits.
    Returns the engine and the device buffers to keep."""
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2, **kw)
    keep = []
    if mode == "cams":
        eng.set_cameras(intr)
    if mode == "guided":
        lg = _dev(np.random.default_rng(3).normal(size=(n, N)), np.float32)
        eng.set_sampling_logits_device(n, lg.data_ptr())
        keep.append(lg)
    torch.cuda.synchronize()
    return eng, keep


def _truth(gt):
    """The cv rig poses of jp ground truths [R][12]."""
    return np.stack([np.concatenate([Rotation.from_matrix(np.diag([1, -1, -1]) @ g[:9].reshape(3, 3)).as_rotvec(),
                                     g[9:] * [1, -1, -1]]) for g in gt])


# Per-camera-intrinsics forms of the rig tests' helpers: test_gpu_rig_grad.py's _scene, rig_rgbd_oracle.scene and
# rig_grad_oracle.restate_rows take one camera for every frame.  These take intr [n][3] (f, cx, cy) per camera frame and
# are otherwise the same; with every row (525, 320, 240) they give those helpers' results.

def _scene(E, C, R, seed=0, inliers=0.6, intr=None):
    """test_gpu_rig_grad.py's R consistent rigs of C ring cameras, each camera frame projecting through its own intr row
    (None: the default camera).  (coords, pix, ext [n][6], gt_rig [R][12])."""
    rng = np.random.default_rng(seed)
    n = R * C
    intr = _intr(n, C, False) if intr is None else intr
    _, pix, _, _ = E.synth_frames(n)
    coords = np.empty((n, N, 3), np.int16)
    ext = np.concatenate([RG.ring(C, seed=seed + r) for r in range(R)])
    gt = np.empty((R, 12))
    for r in range(R):
        true = np.concatenate([Rotation.from_euler("xyz", rng.normal(scale=0.2, size=3)).as_rotvec(),
                               rng.normal(scale=300.0, size=3) + [0.0, 0.0, 1500.0]])
        gt[r] = _jp(true)
        for c in range(C):
            fr = r * C + c
            f, cx, cy = intr[fr]
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


def _rgbd_scene(C, R, intr, seed=0, inliers=0.6, holes=0.0, noise=0.5):
    """rig_rgbd_oracle.scene's R consistent RGB-D rigs of C ring cameras, each camera frame with its own intr row.
    (coords, pix, depth, ext, gt_rig, true)."""
    rng = np.random.default_rng(seed)
    n = R * C
    pix = np.zeros((n, N, 2), np.int32)
    xs, ys = (np.arange(N) % 40) * 16 + 8, (np.arange(N) // 40) * 12 + 6
    coords = np.empty((n, N, 3), np.int16)
    depth = np.empty((n, N), np.float32)
    ext = np.concatenate([RG.ring(C, seed=seed + r) for r in range(R)])
    gt, true = np.empty((R, 12)), np.empty((R, 6))
    for r in range(R):
        true[r] = np.concatenate([Rotation.from_euler("xyz", rng.normal(scale=0.2, size=3)).as_rotvec(),
                                  rng.normal(scale=300.0, size=3) + [0.0, 0.0, 1500.0]])
        gt[r] = _jp(true[r])
        for c in range(C):
            fr = r * C + c
            f, cx, cy = intr[fr]
            pix[fr, :, 0] = xs + rng.integers(-4, 5, N)
            pix[fr, :, 1] = ys + rng.integers(-3, 4, N)
            u = pix[fr, :, 0] + rng.normal(scale=noise, size=N)
            v = pix[fr, :, 1] + rng.normal(scale=noise, size=N)
            d = rng.uniform(1500.0, 4000.0, size=N)
            Xc = np.stack([(u - cx) / f * d, (v - cy) / f * d, d], 1)
            Rc, tc = Rotation.from_rotvec(ext[fr, :3]), ext[fr, 3:]
            cam_R, cam_t = Rc * Rotation.from_rotvec(true[r, :3]), Rc.apply(true[r, 3:]) + tc
            X = cam_R.inv().apply(Xc - cam_t)
            out = rng.uniform(size=N) >= inliers
            X[out] = rng.uniform(-4000.0, 4000.0, size=(out.sum(), 3))
            coords[fr] = np.clip(np.round(X), -32767, 32767).astype(np.int16)
            dd = d.astype(np.float32)
            dd[rng.uniform(size=N) < holes] = np.nan
            depth[fr] = dd
    return coords, pix, depth, ext, gt, true


def _restate_rows(cfg, C_, coords, pix, ext, intr, rig_hyp, sf, hyp_pose, img_idx, dpnp, dl, dref_dhyp, dref_dobj, sog):
    """rig_grad_oracle.restate_rows with camera frame f's reprojections through intr[f]: dLoss/dObj [n][N * 3] of the rig
    backward (path I direct and support, path II direct and support; see there), and dLdAvg [R][6]."""
    thr, alpha, beta, clamp, fix_q4 = float(cfg.thr2d), cfg.alpha, cfg.beta, cfg.grad_clamp, cfg.fix_q4
    n, H = hyp_pose.shape[:2]
    R_, P = n // C_, C_ * H
    rows = np.zeros((n, N * 3))
    dldavg = np.einsum("rk,rki->ri", dl, dref_dhyp.reshape(R_, 6, 6))
    Rcs = RG.rot(ext[:, :3])
    # path I direct
    for r in range(R_):
        rows[r * C_:(r + 1) * C_] += (dl[r] @ dref_dobj[r].reshape(6, C_ * N * 3)).reshape(C_, N * 3)
    # path II: w and the direct part, per camera frame
    W = np.zeros((n, P, 6))
    for fr in range(n):
        r = fr // C_
        f, cx, cy = intr[fr]
        Rr, tr = RG.rot(rig_hyp[r, :, :3]), rig_hyp[r, :, 3:]
        Rk, tk = Rcs[fr] @ Rr, tr @ Rcs[fr].T + ext[fr, 3:]
        Rj, tj = DFLIP @ Rk, tk * RG.FLIP                             # [P][3][3], [P][3] in jp
        go = sog[r] if clamp <= 0 else np.clip(sog[r], -clamp, clamp)
        Yw = coords[fr].astype(np.float32).astype(np.float64)          # [N][3]
        pu = pix[fr, :, 0].astype(np.float32).astype(np.float64)
        pv = pix[fr, :, 1].astype(np.float32).astype(np.float64)
        X, Y, Z = Yw[:, 0], Yw[:, 1], Yw[:, 2]
        # the reprojection error of the diffmap, with k_score's roundings, in the cv pose of the same camera pose
        xc = ((Rj[:, 0, 0, None] * X + Rj[:, 0, 1, None] * Y) + Rj[:, 0, 2, None] * Z) + tj[:, 0, None]
        yc = ((-Rj[:, 1, 0, None] * X + -Rj[:, 1, 1, None] * Y) + -Rj[:, 1, 2, None] * Z) + -tj[:, 1, None]
        zc = ((-Rj[:, 2, 0, None] * X + -Rj[:, 2, 1, None] * Y) + -Rj[:, 2, 2, None] * Z) + -tj[:, 2, None]
        iz = np.where(zc != 0, 1.0 / np.where(zc != 0, zc, 1.0), 1.0)
        pfu, pfv = ((xc * iz) * f + cx).astype(np.float32), ((yc * iz) * f + cy).astype(np.float32)
        du, dv = (pu.astype(np.float32) - pfu).astype(np.float64), (pv.astype(np.float32) - pfv).astype(np.float64)
        e = np.minimum(np.sqrt(du * du + dv * dv), 100.0).astype(np.float32).astype(np.float64)
        sg = 1.0 / (1.0 + np.exp(-beta * (thr - e)))
        g = go[:, None] * (-alpha * beta * sg * (1.0 - sg))            # [P][N] d score / d error
        # the error's derivative through the jp projection
        Xj = np.einsum("pik,nk->pni", Rj, Yw) + tj[:, None, :]
        ex, ey, ez = Xj[..., 0], Xj[..., 1], Xj[..., 2]
        ok = np.abs(ez) >= 1e-8
        ez = np.where(ok, ez, 1.0)
        px, py = -f * ex / ez + cx, f * ey / ez + cy
        ddx, ddy = pu - px, pv - py
        err = np.sqrt(ddx * ddx + ddy * ddy)
        ok &= err <= 100.0
        a0, a1 = -ddx / (err + 1e-8), -ddy / (err + 1e-8)              # d error / d (px, py), as k_dscore regularises it
        G = np.stack([a0 * (-f / ez), a1 * (f / ez), a0 * (f * ex / ez ** 2) + a1 * (-f * ey / ez ** 2)], -1)
        G *= np.where(ok, g, 0.0)[..., None]                            # [P][N][3] d score / d X_jp
        acc = np.einsum("pni,pik->nk", G, Rj)                           # d / dY
        cols = RG._q4(np.arange(N), fix_q4)
        rows[fr].reshape(N, 3)[cols] += acc
        rod = RG.log(Rj)
        W[fr, :, 3:] = G.sum(1)
        for m in range(3):
            d = np.zeros(3)
            d[m] = 1e-7
            dR = (RG.rot(rod + d) - RG.rot(rod - d)) / 2e-7            # [P][3][3]
            W[fr, :, m] = np.einsum("pni,pik,nk->p", G, dR, Yw)
    # the support scatters
    for fr in range(n):
        r, c2 = divmod(fr, C_)
        L = RG.lift_jac(Rcs[fr], ext[fr, 3:], hyp_pose[fr])            # [H][6][6]
        u2 = np.zeros((H, 6))
        for c in range(C_):
            K = RG.cross_jac(Rcs[r * C_ + c], ext[r * C_ + c, 3:], Rcs[fr], ext[fr, 3:], hyp_pose[fr])
            u2 += np.einsum("hk,hkm->hm", W[r * C_ + c, c2 * H:(c2 + 1) * H], K)
        u1 = sf[r, c2 * H:(c2 + 1) * H, None] * np.einsum("k,hkm->hm", dldavg[r], L)
        s1 = np.einsum("hk,hkq->hq", u1, dpnp[fr])                      # [H][12]
        s2 = np.einsum("hk,hkq->hq", u2, dpnp[fr])
        for h in range(H):
            for q in range(4):
                cell = img_idx[fr, h, q]
                if cell < 0:
                    continue
                rows[fr, cell * 3:cell * 3 + 3] += s1[h, q * 3:q * 3 + 3]
                col = RG._q4(cell, fix_q4) * 3
                rows[fr, col:col + 3] += s2[h, q * 3:q * 3 + 3]
    return rows, dldavg


def _agrees_with_the_rig_oracle(dev, coords, pix, intr, ext, gt, C, H, pool=None):
    """test_gpu_rig.py::test_device_agrees_with_the_rig_oracle's assertions and tolerances, rig by rig; pool: a mask of
    the slots whose lifted pose is compared (all when None)."""
    from oracle import oracle as O
    R = len(gt)
    pool = np.ones(C * H, bool) if pool is None else pool
    cfg = O.default_config(n_hyps=H)
    compared = 0
    for r in range(R):
        fr = slice(r * C, (r + 1) * C)
        o = RO.forward(cfg, coords[fr], pix[fr], intr[fr], ext[fr], dev["hyp_pose"][fr], gt[r], start=dev["avg_pose"][r])
        assert np.abs(o["rig_hyp"][pool, :3] - dev["rig_hyp"][r][pool, :3]).max() <= 1e-9
        assert np.abs(o["rig_hyp"][pool, 3:] - dev["rig_hyp"][r][pool, 3:]).max() <= 1e-6
        assert np.abs(o["scores"] - dev["scores"][r]).max() <= 1e-5 * np.abs(o["scores"]).max()
        assert np.abs(O.softmax(dev["scores"][r]) - dev["sf"][r]).max() <= 1e-12
        assert np.abs(o["sf"] - dev["sf"][r]).max() <= 1e-4
        bound = (np.abs(o["sf"] - dev["sf"][r])[:, None] * np.abs(o["rig_hyp"])).sum(0)
        assert (np.abs(o["avg_pose"] - dev["avg_pose"][r]) <= bound + 1e-9 * np.abs(o["avg_pose"]) + 1e-12).all()
        if o["min_margin"] <= 1e-4:
            continue
        compared += 1
        assert np.array_equal(o["inlier_map"], dev["inlier_map"][fr]), r
        assert o["steps_done"] == dev["steps_done"][r]
        assert np.abs(o["ref_pose"][:3] - dev["ref_pose"][r][:3]).max() <= 1e-6
        assert np.abs(o["ref_pose"][3:] - dev["ref_pose"][r][3:]).max() <= 1e-3
        assert abs(o["rot_err"] - dev["rot_err"][r]) <= 1e-4 and abs(o["t_err"] - dev["t_err"][r]) <= 1e-2
        assert o["correct"] == dev["correct"][r]
    assert compared >= R - 1, compared


FORWARD = [(8, 128, "uniform"), (8, 32, "cams"), (2, 512, "guided"), (5, 200, "uniform"), (7, 146, "uniform")]


@pytest.mark.parametrize("C,H,mode", FORWARD)
def test_forward_agrees_with_the_rig_oracle(engine_mod, C, H, mode):
    """Full pools (8 x 128, 2 x 512), eight cameras each with its own intrinsics, and pools of 1000 and 1022 slots (not a
    multiple of the score tile or of 8), four rigs each, against the CPU rig oracle."""
    E = engine_mod
    R = 4
    n = R * C
    intr = _intr(n, C, mode == "cams")
    coords, pix, ext, gt = _scene(E, C, R, seed=40 + C, intr=intr)
    eng, keep = _engine(E, n, H, mode, intr)
    dev = _rig(eng, coords, pix, ext, C, gt)
    eng.close()
    assert not np.any(dev["status"] & BAD_RIG)
    assert dev["correct"].all(), (dev["rot_err"], dev["t_err"])
    _agrees_with_the_rig_oracle(dev, coords, pix, intr, ext, gt, C, H)


@pytest.mark.parametrize("gated", [False, True])
def test_sixteen_rig_priors_in_a_full_pool(engine_mod, gated):
    """C = 8, H = 128 with DSAC_MAX_PRIORS rig priors: pool slot c H + H - k + i holds rig prior i's bits for every camera
    c, and the rest of the pool, its scores, the soft-argmax and the refinement agree with the CPU rig oracle as in
    test_forward_agrees_with_the_rig_oracle."""
    E = engine_mod
    C, H, R, k = 8, 128, 2, E.MAX_PRIORS
    n = R * C
    intr = _intr(n, C, False)
    coords, pix, ext, gt = _scene(E, C, R, seed=60 + gated, intr=intr)
    rp, info = _priors(np.random.default_rng(7), _truth(gt), k, gated)
    eng, keep = _engine(E, n, H, "uniform", intr)
    keep += _set_rig_priors(eng, n, C, rp, info)
    dev = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    eng.close()
    assert not np.any(dev["status"] & (BAD_PRIOR | BAD_RIG))
    for r in range(R):
        for c in range(C):
            assert np.array_equal(_bits(dev["rig_hyp"][r, c * H + H - k:(c + 1) * H]), _bits(rp[r])), (r, c)
    sampled = np.arange(C * H) % H < H - k
    _agrees_with_the_rig_oracle(dev, coords, pix, intr, ext, gt, C, H, pool=sampled)


BACKWARD = [(8, 32, "uniform", 0, 0, 1e-4), (8, 32, "uniform", 8, 1, 0.1),
            (2, 512, "uniform", 0, 1, 0.1), (2, 512, "uniform", 8, 0, 0.1),
            (4, 256, "cams", 0, 0, 1e-4), (4, 256, "cams", 8, 1, 0.1)]


@pytest.mark.parametrize("C,H,mode,ref_steps,fix_q4,clamp", BACKWARD)
def test_whole_chain_matches_the_numpy_restatement(engine_mod, C, H, mode, ref_steps, fix_q4, clamp):
    """test_gpu_rig_grad.py::test_whole_chain_matches_a_numpy_restatement at eight cameras, a full pool of two cameras and
    a full pool of four cameras with their own intrinsics, at its tolerances."""
    E = engine_mod
    R = 2
    n = R * C
    intr = _intr(n, C, mode == "cams")
    coords, pix, ext, gt = _scene(E, C, R, seed=80 + C, intr=intr)
    eng, keep = _engine(E, n, H, mode, intr, fix_q4=fix_q4, grad_clamp=clamp, ref_steps=ref_steps)
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
    want, dldavg = _restate_rows(cfg, C, coords, pix, ext, intr, out["rig_hyp"], out["sf"], out["hyp_pose"], ordinary.img_idx,
                                 ref.dpnp, got["dloss_dref"], got["dref_dhyp"], got["dref_dobj"], got["score_grads"])
    hf = (dldavg[:, None, :3] * out["rig_hyp"][..., :3]).sum(-1) + (dldavg[:, None, 3:] * (out["rig_hyp"][..., 3:] / 1000)).sum(-1)
    sog = out["sf"] * (hf - (out["sf"] * hf).sum(1, keepdims=True))
    assert _near(got["score_grads"], sog, 1e-10)
    assert _near(got["dobj"].reshape(n, -1), want, 1e-8), np.abs(got["dobj"].reshape(n, -1) - want).max() / np.abs(want).max()
    # every camera frame has a gradient
    assert all(np.abs(want[f]).max() > 0 for f in range(n))


@pytest.mark.parametrize("mode", ["uniform", "cams"])
def test_direct_term_at_eight_cameras_is_the_host_ift(engine_mod, mode):
    """test_gpu_rig_grad.py::test_direct_term_is_the_host_ift_of_the_rig_fit at C = 8, with and without per-camera
    intrinsics: the selection entries cam << 11 | cell reach camera 7."""
    from oracle import oracle as O
    E = engine_mod
    C, R, H = 8, 2, 64
    n = R * C
    intr = _intr(n, C, mode == "cams")
    coords, pix, ext, gt = _scene(E, C, R, seed=100, intr=intr)
    eng, keep = _engine(E, n, H, mode, intr)
    rig = Rig(eng, coords, pix, ext, C, gt)
    out = rig.host()
    got = rig.backward(seed=np.ones((R, 6)))
    cfg = eng.cfg
    eng.close()
    compared = 0
    for r in range(R):
        steps = int(out["steps_done"][r])
        assert steps > 0 and not out["status"][r] & BAD_RIG
        fr = slice(r * C, (r + 1) * C)
        cam, cell, margin, run = RG.last_step_cells(O.default_config(n_hyps=H), coords[fr], pix[fr], intr[fr], ext[fr],
                                                    out["hyp_pose"][fr], out["avg_pose"][r], steps)
        if margin <= 1e-4:
            continue
        compared += 1
        assert np.array_equal(run["inlier_map"], out["inlier_map"][fr])
        assert set(cam) == set(range(C))   # every camera, the last one included, has cells in the fit
        D = got["dref_dobj"][r].reshape(6, C, N, 3)
        want = np.zeros((C, N), bool)
        want[cam, cell] = True
        assert np.array_equal(np.abs(D).max(axis=(0, 3)) > 0, want)
        assert 50 <= len(cell) <= C * cfg.inlier_count
        host = RG.rig_ift(cam, coords[fr][cam, cell], pix[fr][cam, cell], ext[fr], intr[fr], out["ref_pose"][r])
        assert host is not None
        assert _near(D[:, cam, cell, :].transpose(1, 0, 2), host, 1e-9)
    assert compared >= 1


def _support_bracket(coords, pix, ext, intr, pose, thr):
    """test_gpu_rig_tracking.py's support bracket: (cells below thr2d in every camera at the composed poses, cells within
    1e-4 px of it in fp64 or k_score's fp32 arithmetic, or on different sides of it in the two)."""
    sure = amb = 0
    for c in range(len(ext)):
        e64, e32 = support_errors(coords[c], pix[c], _compose(ext[c], pose), intr[c])
        a = (np.abs(e64 - thr) <= 1e-4) | (np.abs(e32 - thr) <= 1e-4) | ((e64 < thr) != (e32 < thr))
        sure += int(((e64 < thr) & ~a).sum())
        amb += int(a.sum())
    return sure, amb


@pytest.mark.parametrize("C,H", [(5, 64), (8, 64), (2, 512)])
def test_rig_covariance_with_per_camera_intrinsics(engine_mod, C, H):
    """test_gpu_rig_tracking.py::test_rig_covariance_matches_the_host_over_the_oracle_cells at five and eight cameras and at
    a full pool of two, every camera with its own intrinsics (k_pose_uncertainty_rig_cam)."""
    from oracle import oracle as O
    E = engine_mod
    R = 2
    n = R * C
    intr = _intr(n, C, True)
    coords, pix, ext, gt = _scene(E, C, R, seed=120 + C, intr=intr)
    eng, keep = _engine(E, n, H, "cams", intr)
    rig = _rig(eng, coords, pix, ext, C, keep=keep)
    unc = _rig_unc(eng, n, C)
    cfg = eng.cfg
    eng.close()
    compared = 0
    for r in range(R):
        steps = int(rig["steps_done"][r])
        fr = slice(r * C, (r + 1) * C)
        cam, cell, margin, run = RG.last_step_cells(O.default_config(n_hyps=H), coords[fr], pix[fr], intr[fr], ext[fr],
                                                    rig["hyp_pose"][fr], rig["avg_pose"][r], steps)
        sure, amb = _support_bracket(coords[fr], pix[fr], ext[fr], intr[fr], rig["ref_pose"][r], cfg.thr2d)
        assert sure <= unc["support"][r] <= sure + amb
        if margin <= 1e-4:
            continue
        compared += 1
        assert unc["n_fit"][r] == len(cell)
        ok, cxi, cjp, s2 = RT.rig_cov(cam, coords[fr][cam, cell], pix[fr][cam, cell], ext[fr], intr[fr], rig["ref_pose"][r])
        assert ok and unc["ok"][r] == 1
        for key, h in (("cov_xi", cxi), ("cov_jp6", cjp)):
            assert np.abs(unc[key][r] - h).max() <= 1e-9 * np.abs(h).max(), key
        assert abs(unc["sigma2"][r] - s2) <= 1e-9 * s2
    assert compared >= 1


@pytest.mark.parametrize("mode", ["uniform", "cams"])
@pytest.mark.parametrize("C", [2, 8])
def test_rgbd_rig_covariance_matches_the_host(engine_mod, C, mode):
    """k_pose_uncertainty_rig_rgbd (and, with per-camera intrinsics, its _cam form) against rig_rgbd_oracle.cov over the
    cells of the last accepted step of the CPU RGB-D rig refinement from the device's soft-argmax pose, with 15 % of the
    cells without depth.  The fit and the host are the same fp64 arithmetic summed in other orders: the 1e-9 relative bound
    of the RGB rig covariance.  The support is the reprojection count with or without depth: the RGB rig's bracket."""
    from oracle import oracle as O
    E = engine_mod
    R, H = 2, 64
    n = R * C
    intr = _intr(n, C, mode == "cams")
    coords, pix, depth, ext, gt, _ = _rgbd_scene(C, R, intr, seed=140 + C, holes=0.15)
    eng, keep = _engine(E, n, H, mode, intr)
    d = _dev(depth, np.float32)
    eng.set_rig_cell_depth_device(n, C, d.data_ptr())
    keep.append(d)
    dev = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    unc = _rig_unc(eng, n, C)
    cfg = eng.cfg
    eng.close()
    assert not np.any(dev["inlier_map"][~(np.isfinite(depth) & (depth > 0))])
    ocfg = O.default_config(n_hyps=H)
    compared = 0
    for r in range(R):
        fr = slice(r * C, (r + 1) * C)
        steps = int(dev["steps_done"][r])
        assert steps == cfg.ref_steps and dev["status"][r] & (BAD_RIG | REFINE_ABORTED) == 0
        assert dev["correct"][r] == 1
        ey = RR.eye(pix[fr], depth[fr], intr[fr])
        cam, cell, margin, run = RR.last_step_cells(ocfg, coords[fr], pix[fr], intr[fr], ext[fr], ey, dev["avg_pose"][r], steps)
        sure, amb = _support_bracket(coords[fr], pix[fr], ext[fr], intr[fr], dev["ref_pose"][r], cfg.thr2d)
        assert sure <= unc["support"][r] <= sure + amb
        if margin <= 1e-4:
            continue
        compared += 1
        assert np.array_equal(run["inlier_map"], dev["inlier_map"][fr]), r
        assert unc["n_fit"][r] == len(cell)
        ok, cxi, cjp, s2 = RR.cov(cam, coords[fr][cam, cell], ey[cam, cell], ext[fr], dev["ref_pose"][r])
        assert ok and unc["ok"][r] == 1
        for key, h in (("cov_xi", cxi), ("cov_jp6", cjp)):
            assert np.abs(unc[key][r] - h).max() <= 1e-9 * np.abs(h).max(), key
        assert abs(unc["sigma2"][r] - s2) <= 1e-9 * s2
    assert compared >= 1


def _backward_rows(eng, n, R, P, clamp):
    """dsac_backward_rig_device with the score gradients as its only diagnostic: (dLoss/dObj [n][N][3], sog [R][P])."""
    f64 = dict(dtype=torch.float64, device="cuda")
    dobj = torch.full((n, N, 3), np.nan, **f64)
    sog = torch.zeros((R, P), **f64)
    eng.backward_rig_device(n, None, dobj.data_ptr(), None, clamp, score_grads=sog.data_ptr())
    torch.cuda.synchronize()
    return dobj.cpu().numpy(), sog.cpu().numpy()


def test_full_pool_rigs_do_not_depend_on_the_batch(engine_mod):
    """128 rigs of eight cameras with their own intrinsics and full pools (n = 1024: the sampler's two-lane path, and
    dscore_groups at its minimum, one group of the 1024 slots per frame), against the same batch with every rig but 0, 63
    and 127 replaced by another scene: those three rigs' forward outputs, dLoss/dObj and score gradients are bit for bit.
    The neighbours change and the batch size does not, so the sampler's kernels and the backward's dscore groups (the
    order of the fp64 sums over the pool) are the same.  A rig run alone is not compared bit for bit, for two reasons
    outside the rig kernels: with fewer than 128 sampler streams k1_solve solves each flagged candidate on four lanes, and
    a few of those poses differ from the one-lane solve's in their last bits (the same minimal sets; on these scenes up to
    4e-14 rad and 1.4e-10 mm, in the ordinary pass as in the rig pass); and eight frames alone take 32 dscore groups of 32
    slots, so k_dscore_rig adds each frame's direct part in another order."""
    E = engine_mod
    C, H, n = 8, 128, 1024
    R, P = n // C, C * H
    intr = _intr(n, C, True)
    eng, keep = _engine(E, n, H, "cams", intr)
    runs = []
    for seed in (160, 161):
        coords, pix, ext, gt = _scene(E, C, R, seed=seed, intr=intr)
        if runs:   # the second batch: the first's rigs 0, 63 and 127 among other rigs
            first = runs[0]["inputs"]
            for r in (0, 63, 127):
                fr = slice(r * C, (r + 1) * C)
                coords[fr], pix[fr], ext[fr], gt[r] = first[0][fr], first[1][fr], first[2][fr], first[3][r]
        out = _rig(eng, coords, pix, ext, C, gt, keep=keep)
        rig = Rig(eng, coords, pix, ext, C, gt)   # keeps the pass's inputs alive for its backward
        dobj, sog = _backward_rows(eng, n, R, P, 0.1)
        assert out["correct"].mean() > 0.9 and not np.any(out["status"] & BAD_RIG)
        assert np.isfinite(dobj).all()
        runs.append(dict(inputs=(coords, pix, ext, gt), out=out, dobj=dobj, sog=sog))
        del rig
    eng.close()
    a, b = runs
    assert not np.array_equal(a["inputs"][0][C:2 * C], b["inputs"][0][C:2 * C])
    for r in (0, 63, 127):
        fr = slice(r * C, (r + 1) * C)
        for k, v in a["out"].items():
            rows = fr if k in ("hyp_pose", "inlier_map") else slice(r, r + 1)
            assert np.array_equal(_bits(v[rows]), _bits(b["out"][k][rows])), (r, k)
        assert np.abs(a["dobj"][fr]).max() > 0
        assert np.array_equal(_bits(a["dobj"][fr]), _bits(b["dobj"][fr])), r
        assert np.array_equal(_bits(a["sog"][r]), _bits(b["sog"][r])), r
