"""Rig score hooks (dsac_set_rig_score_hooks) on the GPU: the score seam for the rig passes and the rig backward.

The scorer is test_gpu_score_seam_modes.py's float64 sigmoid scorer, alpha' sum_i sigmoid(beta' (thr2d - d_ji)) with
alpha' = 0.3 and beta' = 1.5, and its analytic adjoint -alpha' beta' s (1 - s) g, while the engine keeps its defaults
(alpha 0.1, beta 0.5).  So an unhooked rig engine built with alpha' and beta' is a reference for a hooked rig, and an
engine that ignored what the hook wrote, or dropped its adjoint, is off by a factor, not by rounding.

1. One camera with a zero extrinsic is the ordinary pass under the same hooks as per-frame hooks, bit for bit.
2. Several cameras: the error images against float64 reprojections at the composed poses, one call per pass, and the
   hooked rig against the unhooked alpha' / beta' rig.
3. The layout of the camera scores, 4. the backward's linearity in the hook's adjoint, 5. hooks with RGB-D rigs, rig
   priors and guided sampling, 6. the score CNN, 7. the rules and refusals."""
import ctypes as Cc

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import rig_grad_oracle as RG

pytestmark = pytest.mark.gpu
N = 1600
A1, B1, THR = 0.3, 1.5, 10.0


class _W:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}


def _stream(s):
    return torch.cuda.ExternalStream(s) if s else torch.cuda.default_stream()


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
    """R consistent rigs of C ring cameras (test_gpu_rig_grad.py's): (coords, pix, ext [n][6], gt_rig [R][12], depth [n][N])."""
    rng = np.random.default_rng(seed)
    n = R * C
    _, pix, _, _ = E.synth_frames(n)
    coords = np.empty((n, N, 3), np.int16)
    depth = np.empty((n, N), np.float32)
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
            depth[fr] = d
            Xc = np.stack([(u - cx) / f * d, (v - cy) / f * d, d], 1)
            cam = _compose(ext[fr], true)
            X = Rotation.from_rotvec(cam[:3]).inv().apply(Xc - cam[3:])
            out = rng.uniform(size=N) >= inliers
            X[out] = rng.uniform(-4000.0, 4000.0, size=(out.sum(), 3))
            coords[fr] = np.clip(np.round(X), -32767, 32767).astype(np.int16)
    return coords, pix, ext, gt, depth


class Scorer:
    """The float64 sigmoid scorer as rig score hooks (rig=True) or as the per-frame seam.  Frames are scored one at a time
    on the stream the engine passes.  fixed: [n][P] scores to write instead; temper: a factor on the scores written (the
    adjoint does not see it); scale: c of the backward hook's c * adjoint;
    seen / written / grads: host copies of the error images, the scores written and the score gradients received;
    fail_forward / fail_backward: the hook returns 1."""

    def __init__(self, eng, rig=True, fixed=None, scale=1.0):
        self.eng, self.fixed, self.scale, self.temper = eng, fixed, scale, 1.0
        self.calls, self.bw_calls, self.seen, self.written, self.grads = [], [], None, None, None
        self.fail_forward = self.fail_backward = False
        if rig:
            eng.set_rig_score_hooks(self.forward, self.backward)
        else:
            eng.set_score_hook(self.forward)
            eng.set_score_backward_hook(self.backward)

    def forward(self, dm, n, P, sc, stream):
        self.calls.append((n, P))
        if self.fail_forward:
            return 1
        try:
            with torch.cuda.stream(_stream(stream)):
                d = torch.as_tensor(_W(dm, (n, P, N), "<f4"), device="cuda")
                s = torch.as_tensor(_W(sc, (n, P), "<f8"), device="cuda")
                if self.fixed is not None:
                    s.copy_(torch.from_numpy(np.ascontiguousarray(self.fixed, np.float64)).cuda())
                else:
                    for f in range(n):
                        s[f].copy_(self.temper * A1 * torch.sigmoid(B1 * (THR - d[f].double())).sum(1))
                self.seen, self.written = d.cpu().numpy(), s.cpu().numpy()
        except Exception as ex:   # an exception cannot cross the C callback: the engine sees the nonzero return
            print("rig score hook:", repr(ex))
            return 1
        return 0

    def backward(self, dm, sg, n, P, out, stream):
        self.bw_calls.append((n, P))
        if self.fail_backward:
            return 1
        with torch.cuda.stream(_stream(stream)):
            d = torch.as_tensor(_W(dm, (n, P, N), "<f4"), device="cuda")
            g = torch.as_tensor(_W(sg, (n, P), "<f8"), device="cuda")
            o = torch.as_tensor(_W(out, (n, P, N), "<f8"), device="cuda")
            for f in range(n):
                s = torch.sigmoid(B1 * (THR - d[f].double()))
                o[f].copy_(g[f][:, None] * (-A1 * B1 * self.scale) * s * (1 - s))
            self.grads = g.cpu().numpy()
        return 0


F64 = dict(dtype=torch.float64, device="cuda")
I32 = dict(dtype=torch.int32, device="cuda")


class Rig:
    """A rig pass on device copies of host inputs, kept alive for the backward, and the rig backward's outputs."""

    def __init__(self, eng, coords, pix, ext, C, gt=None, frame0=0):
        self.eng, self.C, self.n = eng, C, len(coords)
        H = eng.cfg.n_hyps
        self.R, self.P = self.n // C, C * H
        self.inputs = [_dev(coords, np.int16), _dev(pix, np.int32), _dev(ext, np.float64)]
        self.gt = _dev(gt, np.float64) if gt is not None else None
        R, P, n = self.R, self.P, self.n
        self.out = {"hyp_pose": torch.zeros((n, H, 6), **F64), "rig_hyp": torch.zeros((R, P, 6), **F64),
                    "scores": torch.zeros((R, P), **F64), "sf": torch.zeros((R, P), **F64), "entropy": torch.zeros(R, **F64),
                    "avg_pose": torch.zeros((R, 6), **F64), "ref_pose": torch.zeros((R, 6), **F64),
                    "inlier_map": torch.zeros((n, N), **I32), "steps_done": torch.zeros(R, **I32), "status": torch.zeros(R, **I32)}
        if gt is not None:
            self.out["loss"] = torch.zeros(R, **F64)
        dc, dp, de = self.inputs
        eng.forward_rig_device(n, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr(), 0, self.gt.data_ptr() if gt is not None else None,
                               frame0, **{k: v.data_ptr() for k, v in self.out.items()})
        torch.cuda.synchronize()
        self.res = {k: v.cpu().numpy() for k, v in self.out.items()}

    def backward(self, seed=None, clamp=0.0):
        dobj = torch.full((self.n, N, 3), np.nan, **F64)
        d = {"dloss_dref": torch.zeros((self.R, 6), **F64), "dref_dhyp": torch.zeros((self.R, 6, 6), **F64),
             "score_grads": torch.zeros((self.R, self.P), **F64), "dref_dobj": torch.zeros((self.R, 6, self.C * N * 3), **F64)}
        ptrs = {k: v.data_ptr() for k, v in d.items()}
        if seed is not None:
            s = _dev(seed, np.float64)
            self.eng.backward_rig_pose_device(self.n, s.data_ptr(), dobj.data_ptr(), None, clamp, **ptrs)
        else:
            self.eng.backward_rig_device(self.n, None, dobj.data_ptr(), None, clamp, **ptrs)
        torch.cuda.synchronize()
        out = {k: v.cpu().numpy() for k, v in d.items()}
        out["dobj"] = dobj.cpu().numpy()
        return out


def _near(a, b, rel):
    scale = max(np.abs(a).max(), np.abs(b).max(), 1e-300)
    return np.abs(a - b).max() <= rel * scale


def _refused(E, eng, fn, text):
    with pytest.raises(RuntimeError, match="\\(-1\\)"):
        fn()
    err = E.load().dsac_last_error(eng.h).decode()
    assert text in err, err


# ------------------------------------------------------------------ 1. one camera


@pytest.mark.parametrize("mode,clamp", [("uniform", 0.0), ("uniform", 1e-4), ("cams", 0.0)])
def test_one_camera_is_the_ordinary_hooked_pass(engine_mod, mode, clamp):
    E = engine_mod
    n, H = 4, 64
    coords, pix, _, gt_jp = E.synth_frames(n, n_streams=2)
    engines = []
    for _ in range(2):
        eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2, grad_clamp=clamp)
        eng.set_coord_derivatives("implicit")
        if mode == "cams":
            cams = np.tile([[525.0, 320.0, 240.0]], (n, 1))
            cams[1::2] = [580.0, 310.5, 250.25]
            eng.set_cameras(cams)
        engines.append(eng)
    eng_o, eng_r = engines
    so, sr = Scorer(eng_o, rig=False), Scorer(eng_r)
    # the ordinary pass and its implicit backward under the per-frame seam
    dc, dp, dg = _dev(coords, np.int16), _dev(pix, np.int32), _dev(gt_jp, np.float64)
    eng_o.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 3)
    ref = eng_o.fetch(n)
    torch.cuda.synchronize()
    bw = eng_o.backward(coords, pix, gt_jp)
    # the rig pass of one camera per rig, zero extrinsics, under the rig hooks
    rig = Rig(eng_r, coords, pix, np.zeros((n, 6)), 1, gt_jp, frame0=3)
    got = rig.backward()
    assert sr.calls == [(n, H)] and sr.bw_calls == [(n, H)]
    assert np.array_equal(_bits(sr.seen), _bits(so.seen))
    assert np.array_equal(_bits(sr.written), _bits(so.written))
    assert np.array_equal(_bits(rig.res["rig_hyp"]), _bits(ref.hyp_pose))
    for k in ("scores", "sf", "entropy", "avg_pose", "ref_pose", "inlier_map", "loss"):
        assert np.array_equal(_bits(rig.res[k]), _bits(getattr(ref, k).astype(rig.res[k].dtype))), k
    assert np.array_equal(rig.res["steps_done"], ref.ref_steps_done)
    assert np.array_equal(_bits(sr.grads), _bits(so.grads))
    if clamp > 0:
        assert np.abs(bw.score_grads).max() > clamp   # the clamp bites
    for k in ("dloss_dref", "dref_dhyp", "score_grads", "dref_dobj"):
        assert np.array_equal(_bits(got[k]), _bits(getattr(bw, k))), k
    # the support scatters sum in another order: the rows agree to rounding
    assert _near(got["dobj"], bw.dloss_dobj, 1e-12)
    assert np.abs(bw.dloss_dobj).max() > 0
    for eng in engines:
        eng.close()


# ------------------------------------------------------------------ 2. several cameras


def _reproject(coords, pix, cam, pose):
    """float64 reprojection errors [N] of a frame's cells at a cv pose, clamped at 100 as k_score clamps them."""
    f, cx, cy = cam
    X = Rotation.from_rotvec(pose[:3]).apply(coords.astype(np.float64)) + pose[3:]
    z = np.where(X[:, 2] == 0, 1.0, X[:, 2])
    u, v = f * X[:, 0] / z + cx, f * X[:, 1] / z + cy
    return np.minimum(np.hypot(pix[:, 0] - u, pix[:, 1] - v), 100.0)


@pytest.mark.parametrize("C", [2, 4, 8])
def test_several_cameras_against_numpy_and_the_unhooked_rig(engine_mod, C):
    E = engine_mod
    R, H = 2, 16
    n, P = R * C, C * H
    coords, pix, ext, gt, _ = _scene(E, C, R, seed=C)
    cams = np.tile([[525.0, 320.0, 240.0]], (n, 1))
    cams[1::2] = [540.0, 322.5, 238.0]
    eng = E.Engine(max_frames=n, n_hyps=H)
    eng.set_cameras(cams)
    sc = Scorer(eng)
    rig = Rig(eng, coords, pix, ext, C, gt)
    got = rig.backward(clamp=0.0)
    eng.close()
    assert sc.calls == [(n, P)] and sc.bw_calls == [(n, P)]
    # the error images the hook saw: every camera frame against its rig's pool at the composed pose
    worst = 0.0
    for f in range(n):
        r = f // C
        for j in range(0, P, 3):
            want = _reproject(coords[f], pix[f], cams[f], _compose(ext[f], rig.res["rig_hyp"][r, j]))
            worst = max(worst, float((np.abs(sc.seen[f, j] - want) / (1.0 + want)).max()))
    print("C=%d error images: %.3g" % (C, worst))
    assert worst <= 1e-4
    # the unhooked rig engine scoring in closed form with alpha' and beta'
    ref_eng = E.Engine(max_frames=n, n_hyps=H, alpha=A1, beta=B1)
    ref_eng.set_cameras(cams)
    ref = Rig(ref_eng, coords, pix, ext, C, gt)
    want = ref.backward(clamp=0.0)
    ref_eng.close()
    assert np.array_equal(_bits(rig.res["rig_hyp"]), _bits(ref.res["rig_hyp"]))
    smax = np.abs(ref.res["scores"]).max()
    ds = np.abs(rig.res["scores"] - ref.res["scores"]).max()
    print("C=%d scores %.3g of %.3g" % (C, ds, smax))
    assert ds <= (1e-5 + B1 * 2e-3) * smax
    assert np.abs(rig.res["sf"] - ref.res["sf"]).max() <= max(1e-4, 2 * ds)
    ok = rig.res["status"] == ref.res["status"]
    assert ok.all()
    rot = [(Rotation.from_rotvec(a[:3]) * Rotation.from_rotvec(b[:3]).inv()).magnitude()
           for a, b in zip(rig.res["ref_pose"], ref.res["ref_pose"])]
    assert max(rot) <= 1e-5 and np.abs(rig.res["ref_pose"][:, 3:] - ref.res["ref_pose"][:, 3:]).max() <= 1e-2
    # a rig's softmax is about C times sharper than a frame's: score gradients that underflow to 0 in one may be 1e-200
    # in the other
    assert np.abs(got["score_grads"] - want["score_grads"]).max() <= 1e-2 * np.abs(want["score_grads"]).max() + 1e-12
    assert _near(got["dobj"], want["dobj"], 2e-2)
    assert np.abs(want["dobj"]).max() > 0


# ------------------------------------------------------------------ 3. layout


def test_camera_score_layout(engine_mod):
    E = engine_mod
    C, R, H = 4, 2, 8
    n, P = R * C, C * H
    coords, pix, ext, gt, _ = _scene(E, C, R, seed=11)
    fixed = np.random.default_rng(4).uniform(-3.0, 3.0, size=(n, P))
    eng = E.Engine(max_frames=n, n_hyps=H)
    sc = Scorer(eng, fixed=fixed)
    rig = Rig(eng, coords, pix, ext, C)
    want = np.empty((R, P))
    for r in range(R):
        s = fixed[r * C].copy()
        for c in range(1, C):
            s = s + fixed[r * C + c]
        want[r] = s
    assert np.array_equal(_bits(rig.res["scores"]), _bits(want))
    sf = np.exp(want - want.max(1, keepdims=True))
    sf /= sf.sum(1, keepdims=True)
    assert np.allclose(rig.res["sf"], sf, rtol=1e-12, atol=1e-300)
    # scoring only camera c's frames moves the soft-argmax onto camera c's slots
    for c in range(C):
        only = np.zeros((n, P))
        only[c::C, c * H:(c + 1) * H] = 50.0 + np.arange(H) * 1e-3
        sc.fixed = only
        res = Rig(eng, coords, pix, ext, C).res
        mass = res["sf"][:, c * H:(c + 1) * H].sum(1)
        assert (mass > 1 - 1e-12).all(), (c, mass)
        block = res["rig_hyp"][:, c * H:(c + 1) * H]
        avg = (res["sf"][:, c * H:(c + 1) * H, None] * block).sum(1)
        assert np.allclose(res["avg_pose"], avg, rtol=1e-9, atol=1e-9)
    eng.close()


# ------------------------------------------------------------------ 4. adjoint


@pytest.mark.parametrize("clamp", [0.0, 1e-12])   # the score gradients of this one-step refinement are about 1e-12
def test_backward_is_linear_in_the_hooks_adjoint(engine_mod, clamp):
    """c * adjoint for c in {0, 1, 2}: path II doubles (to 1e-12 relative), everything upstream of the hook is
    bit-identical.  The forward hook writes the sigmoid scorer's scores times 0.02, so that the rig softmax spreads over the
    good slots (at full scale it puts all its mass on one slot), and the refinement takes one step, so that its replays from
    perturbed starts do not all converge to the same bits: otherwise dRefineHyp, and with it every score gradient, is 0."""
    E = engine_mod
    C, R, H = 3, 2, 16
    n = R * C
    coords, pix, ext, gt, _ = _scene(E, C, R, seed=5)
    eng = E.Engine(max_frames=n, n_hyps=H, grad_clamp=clamp, ref_steps=1)
    sc = Scorer(eng)
    sc.temper = 0.02
    out = {}
    for s in (0.0, 1.0, 2.0):
        sc.scale = s
        rig = Rig(eng, coords, pix, ext, C, gt)
        out[s] = rig.backward()
        # the hook receives the rig's clamped score gradients, once per camera frame
        g = out[s]["score_grads"]
        if clamp > 0:
            g = np.clip(g, -clamp, clamp)
        assert np.array_equal(_bits(sc.grads), _bits(np.repeat(g, C, axis=0)))
    eng.close()
    if clamp > 0:
        assert np.abs(out[1.0]["score_grads"]).max() > clamp
    for k in ("dloss_dref", "dref_dhyp", "score_grads", "dref_dobj"):
        assert np.array_equal(_bits(out[0.0][k]), _bits(out[1.0][k])) and np.array_equal(_bits(out[1.0][k]), _bits(out[2.0][k])), k
    p1 = out[0.0]["dobj"]
    p2, p2x2 = out[1.0]["dobj"] - p1, out[2.0]["dobj"] - p1
    assert np.abs(p2).max() > 0
    d = np.abs(p2x2 - 2 * p2).max() / max(np.abs(2 * p2).max(), np.abs(p1).max())
    print("linearity: %.3g" % d)
    assert d <= 1e-12


# ------------------------------------------------------------------ 5. combinations


def test_hooks_with_rgbd_rigs_priors_and_guided_sampling(engine_mod):
    E = engine_mod
    C, R, H, k = 2, 2, 16, 2
    n, P = R * C, C * H
    coords, pix, ext, gt, depth = _scene(E, C, R, seed=8)
    lg = _dev(np.random.default_rng(3).normal(size=(n, N)), np.float32)
    dd = _dev(depth, np.float32)
    # k rig priors per rig near its true pose (the cv form of the jp ground truth)
    flip = np.array([1.0, -1.0, -1.0])
    pri = np.stack([[np.concatenate([RG.log(np.diag(flip) @ g[:9].reshape(3, 3)), g[9:] * flip]) + 1e-3 * i for i in range(k)]
                    for g in gt])
    dpr = _dev(pri, np.float64)
    runs = {}
    for hooked in (False, True):
        eng = E.Engine(max_frames=n, n_hyps=H)
        eng.set_sampling_logits_device(n, lg.data_ptr())
        eng.set_rig_cell_depth_device(n, C, dd.data_ptr())
        eng.set_rig_pose_priors_device(n, C, k, dpr.data_ptr())
        sc = Scorer(eng) if hooked else None
        rig = Rig(eng, coords, pix, ext, C, gt)
        logp = torch.zeros(n, **F64)
        eng.sampling_log_prob_device(n, logp.data_ptr())
        got = rig.backward()
        torch.cuda.synchronize()
        runs[hooked] = (rig.res, logp.cpu().numpy(), got, sc)
        eng.close()
    (r0, l0, g0, _), (r1, l1, g1, sc) = runs[False], runs[True]
    assert sc.calls == [(n, P)] and sc.bw_calls == [(n, P)]
    assert np.array_equal(_bits(l0), _bits(l1))   # sampling does not see the score
    assert np.array_equal(_bits(r0["hyp_pose"]), _bits(r1["hyp_pose"]))
    assert np.array_equal(_bits(r0["rig_hyp"]), _bits(r1["rig_hyp"]))
    # the prior slots are scored by the hook like any other slot
    for c in range(C):
        for j in range(k):
            slot = c * H + H - k + j
            assert np.array_equal(_bits(r1["rig_hyp"][:, slot]), _bits(pri[:, j]))
            for f in range(c, n, C):
                want = A1 * (1.0 / (1.0 + np.exp(-B1 * (THR - sc.seen[f, slot].astype(np.float64))))).sum()
                assert abs(sc.written[f, slot] - want) <= 1e-9 * abs(want)
    assert not np.array_equal(r0["scores"], r1["scores"])
    assert np.isfinite(r1["ref_pose"]).all() and np.isfinite(g1["dobj"]).all() and np.abs(g1["dobj"]).max() > 0


# ------------------------------------------------------------------ 6. the score CNN


def test_score_cnn_through_the_rig(engine_mod):
    E = engine_mod
    from dsac_b200 import autograd as A
    from dsac_b200.score_cnn import ScoreCNN
    saved = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    n, H = 2, 32
    coords, pix, _, gt_jp = E.synth_frames(n)
    dp, dg = _dev(pix, np.int32), _dev(gt_jp, np.float64)
    grads = []
    for rig in (False, True):
        eng = E.Engine(max_frames=n, n_hyps=H)
        cnn = ScoreCNN(seed=0)
        pred = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda().requires_grad_(True)
        if rig:
            eng.set_rig_score_hooks(cnn, cnn.backward)
            ext = torch.zeros((n, 6), **F64)
            loss = A.rig_softam_loss(eng, pred, dp, ext, 1, dg)
        else:
            eng.set_score_hook(cnn)
            eng.set_score_backward_hook(cnn.backward)
            loss = A.softam_loss(eng, pred, dp, dg, derivatives="implicit")
        loss.sum().backward()
        torch.cuda.synchronize()
        grads.append(([p.grad.detach().cpu().numpy() for p in cnn.model.parameters()], loss.detach().cpu().numpy(),
                      pred.grad.cpu().numpy()))
        eng.close()
    (g0, l0, d0), (g1, l1, d1) = grads
    assert np.array_equal(_bits(l0), _bits(l1))
    for a, b in zip(g0, g1):
        assert np.array_equal(_bits(a), _bits(b))
    assert _near(d1, d0, 1e-6)
    assert any(np.abs(a).max() > 0 for a in g0)
    # four cameras: finite, nonzero parameter gradients
    C, R = 4, 2
    coords, pix, ext, gt, _ = _scene(E, C, R, seed=21)
    eng = E.Engine(max_frames=R * C, n_hyps=H)
    cnn = ScoreCNN(seed=0)
    eng.set_rig_score_hooks(cnn, cnn.backward)
    pred = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda().requires_grad_(True)
    A.rig_softam_loss(eng, pred, _dev(pix, np.int32), _dev(ext, np.float64), C, _dev(gt, np.float64)).sum().backward()
    torch.cuda.synchronize()
    g = [p.grad.detach().cpu().numpy() for p in cnn.model.parameters()]
    assert all(np.isfinite(a).all() for a in g) and any(np.abs(a).max() > 0 for a in g)
    eng.close()
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved


# ------------------------------------------------------------------ 7. rules


def test_rules_and_refusals(engine_mod):
    E = engine_mod
    lib = E.load()
    C, R, H = 2, 2, 16
    n = R * C
    coords, pix, ext, gt, _ = _scene(E, C, R, seed=3)
    eng = E.Engine(max_frames=n, n_hyps=H)
    plain = Rig(eng, coords, pix, ext, C, gt).res   # the never-hooked engine's pass, below
    sc = Scorer(eng)
    # exactly one hook NULL
    fwd = E.SCORE_HOOK(lambda *a: 0)
    bwd = E.SCORE_BACKWARD_HOOK(lambda *a: 0)
    for a, b in ((Cc.cast(fwd, Cc.c_void_p), None), (None, Cc.cast(bwd, Cc.c_void_p))):
        _refused(E, eng, lambda: eng._check(lib.dsac_set_rig_score_hooks(eng.h, a, b, None)), "are set together")
    with pytest.raises(ValueError):
        eng.set_rig_score_hooks(sc.forward, None)
    # the hooks are still those of sc: the ordinary and DSAC forwards refuse, naming the setter
    dc, dp, dg = _dev(coords, np.int16), _dev(pix, np.int32), _dev(np.tile(gt, (C, 1)), np.float64)
    text = "rig score hooks are registered (dsac_set_rig_score_hooks)"
    _refused(E, eng, lambda: eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 0), text)
    _refused(E, eng, lambda: eng.forward(coords, pix, np.tile(gt, (C, 1))), text)
    _refused(E, eng, lambda: eng.forward_dsac(coords, pix, np.tile(gt, (C, 1))), text)
    _refused(E, eng, lambda: eng.forward_dsac_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr()), text)
    # a hooked pass; the backward refuses after the hooks changed or were cleared, the pose queries do not read the score
    rig = Rig(eng, coords, pix, ext, C, gt)
    rig.backward()
    jp = torch.zeros((R, 6), **F64)
    unc = {k: torch.zeros((R, 6, 6), **F64) for k in ("cov_jp6", "cov_xi")}
    unc.update(sigma2=torch.zeros(R, **F64), n_fit=torch.zeros(R, **I32), support=torch.zeros(R, **I32), ok=torch.zeros(R, **I32))
    Scorer(eng)   # other trampolines: other hooks
    for fn in (lambda: rig.backward(), lambda: rig.backward(seed=np.ones((R, 6)))):
        _refused(E, eng, fn, "the rig score hooks changed (dsac_set_rig_score_hooks) after the forward pass, which called other hooks")
    eng.set_rig_score_hooks(None, None)
    _refused(E, eng, lambda: rig.backward(), "the rig score hooks changed")
    eng.rig_refined_jp6_device(n, jp.data_ptr())
    eng.rig_pose_uncertainty_device(n, C, **{k: v.data_ptr() for k, v in unc.items()})
    torch.cuda.synchronize()
    assert np.isfinite(jp.cpu().numpy()).all() and np.isfinite(unc["cov_xi"].cpu().numpy()).all()
    assert (unc["support"].cpu().numpy() > 0).all()
    # an unhooked pass refuses a backward once hooks are registered
    unhooked = Rig(eng, coords, pix, ext, C, gt)
    sc = Scorer(eng)
    _refused(E, eng, lambda: unhooked.backward(), "which was scored in closed form")
    # a failing forward hook: DSAC_ERR_ARG and no pass held
    sc.fail_forward = True
    with pytest.raises(RuntimeError, match="\\(-1\\)"):
        Rig(eng, coords, pix, ext, C, gt)
    assert "the rig score hook returned 1" in lib.dsac_last_error(eng.h).decode()
    _refused(E, eng, lambda: eng.rig_refined_jp6_device(n, jp.data_ptr()), "must follow a dsac_forward_rig_device")
    _refused(E, eng, lambda: rig.backward(), "must follow a dsac_forward_rig_device")
    # a failing backward hook
    sc.fail_forward = False
    rig = Rig(eng, coords, pix, ext, C, gt)
    sc.fail_backward = True
    _refused(E, eng, lambda: rig.backward(), "the rig score backward hook returned 1")
    sc.fail_backward = False
    rig.backward()
    # the per-frame score hook still makes the rig pass refuse
    eng.set_score_hook(lambda *a: 0)
    with pytest.raises(RuntimeError, match="\\(-1\\)"):
        Rig(eng, coords, pix, ext, C, gt)
    assert "a score hook is registered" in lib.dsac_last_error(eng.h).decode()
    eng.set_score_hook(None)
    # cleared: the ordinary forward runs again and a rig pass is the never-hooked engine's, bit for bit
    eng.set_rig_score_hooks(None, None)
    eng.forward(coords, pix, np.tile(gt, (C, 1)))
    again = Rig(eng, coords, pix, ext, C, gt).res
    for k, v in plain.items():
        assert np.array_equal(_bits(v), _bits(again[k])), k
    eng.close()
