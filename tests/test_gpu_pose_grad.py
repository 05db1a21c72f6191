"""Pose-valued outputs: dsac_refined_jp6_device, the seeded backward entry points dsac_backward_pose_device and
dsac_backward_dsac_pose_device, and softam_pose / dsac_hypotheses of dsac_b200/autograd.py, against the loss rounds, the
oracle's seeded chains and themselves (selection, linearity)."""
import numpy as np
import pytest
import seeded_oracle as S

pytestmark = pytest.mark.gpu


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _rel(a, b, floor=1e-300):
    return np.abs(a - b).max() / max(floor, np.abs(b).max())


def _gt6(O, gt_jp):
    return np.concatenate([O.rodrigues_inv(gt_jp[:9]), gt_jp[9:]])


def _jp6(eng, n, shape):
    import torch
    out = torch.full(shape, np.nan, dtype=torch.float64, device="cuda")
    eng.refined_jp6_device(n, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _pose_backward(eng, n, seed, clamp=0.0, want_pred=False):
    """dsac_backward_pose_device -> (dLoss/dObj, coordinate-CNN gradient or None) on host."""
    import torch
    dobj = torch.full((n, 1600, 3), np.nan, dtype=torch.float64, device="cuda")
    pred = torch.full((n, 1600, 3), np.nan, dtype=torch.float32, device="cuda") if want_pred else None
    d_seed = _dev(seed)
    eng.backward_pose_device(n, d_seed.data_ptr(), dobj.data_ptr(), pred.data_ptr() if want_pred else None, clamp,
                             torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return dobj.cpu().numpy(), (pred.cpu().numpy() if want_pred else None)


def _dsac_pose_backward(eng, n, H, seed, grad_sf, d_dloss_dpred=None, clamp=0.0):
    import torch
    outs = {"dloss_dobj": torch.full((n, 1600, 3), np.nan, dtype=torch.float64, device="cuda"),
            "path1": torch.full((n, 1600, 3), np.nan, dtype=torch.float64, device="cuda"),
            "path2": torch.full((n, 1600, 3), np.nan, dtype=torch.float64, device="cuda"),
            "score_grads": torch.full((n, H), np.nan, dtype=torch.float64, device="cuda"),
            "n_selected": torch.full((n,), -1, dtype=torch.int32, device="cuda"),
            "n_refine_jobs": torch.full((n,), -1, dtype=torch.int32, device="cuda")}
    ds = _dev(seed) if seed is not None else None
    dg = _dev(grad_sf) if grad_sf is not None else None
    eng.backward_dsac_pose_device(n, ds.data_ptr() if ds is not None else None, dg.data_ptr() if dg is not None else None,
                                  d_dloss_dpred, clamp, torch.cuda.current_stream().cuda_stream,
                                  **{k: v.data_ptr() for k, v in outs.items()})
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in outs.items()}


def test_refined_jp6_matches_oracle_jp6(engine_mod, oracle):
    """After both pass kinds: the jp 6-vector of every fetched cv refined pose, to 1e-12; misuse is refused."""
    E, O = engine_mod, oracle
    nf, H = 3, 32
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    fw = eng.forward(coords, pix, gt_jp)
    got = _jp6(eng, nf, (nf, 6))
    want = np.stack([O.jp6(p[:3], p[3:]) for p in fw.ref_pose])
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    with pytest.raises(RuntimeError):
        _jp6(eng, nf - 1, (nf, 6))
    fd = eng.forward_dsac(coords, pix, None, random_draw=True)
    got = _jp6(eng, nf, (nf, H, 6))
    want = np.stack([[O.jp6(p[:3], p[3:]) for p in fd.ref_pose[f]] for f in range(nf)])
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    assert np.isfinite(got).all()


def test_softam_pose_backward_with_the_loss_seed_equals_the_loss_backward(engine_mod):
    """dloss_dref of a pass with ground truth, as the seed of a second engine whose forward had no ground truth: the
    same dLoss/dObj bit for bit."""
    import torch
    E = engine_mod
    nf, H = 6, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, frame0=2)
    ref = E.Engine(max_frames=nf, n_hyps=H)
    ref.forward(coords, pix, gt_jp, frame0=2)
    bw = ref.backward(coords, pix, gt_jp, full=False)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    dc, dp = _dev(coords), _dev(pix)
    eng.forward_device(nf, dc.data_ptr(), dp.data_ptr(), 0, None, 2, torch.cuda.current_stream().cuda_stream)
    got, _ = _pose_backward(eng, nf, bw.dloss_dref)
    assert np.array_equal(got, bw.dloss_dobj)
    assert np.abs(got).max() > 0


@pytest.mark.parametrize("H", [64, 256])
@pytest.mark.parametrize("fix_q4", [0, 1])
def test_softam_pose_backward_matches_oracle(engine_mod, oracle, H, fix_q4):
    E, O = engine_mod, oracle
    nf = 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H, fix_q4=fix_q4)
    fwd = eng.forward(coords, pix)
    seed = np.random.default_rng(H + fix_q4).normal(0, 1, (nf, 6))
    got, _ = _pose_backward(eng, nf, seed)
    for f in range(nf):
        cfg = O.default_config(seed=1305 + f, n_hyps=H, fix_q4=fix_q4)
        ofw = O.forward(cfg, coords[f], pix[f])
        assert np.array_equal(ofw.img_idx, fwd.img_idx[f])
        obw = S.backward_seeded(O, cfg, coords[f], pix[f], ofw, seed[f])
        assert np.isfinite(got[f]).all()
        assert _rel(got[f], obw.dloss_dobj, floor=1e-6) <= 1e-3   # the dLoss/dObj band of test_gpu_backward.py
        assert np.abs(got[f]).max() > 0


def _dsac_pass(E, nf, H, frame0=0, gt=True, random_draw=False):
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, frame0=frame0)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    fw = eng.forward_dsac(coords, pix, gt_jp if gt else None, random_draw=random_draw, frame0=frame0)
    return eng, fw, coords, pix, gt_jp


def test_dsac_pose_backward_with_expected_loss_seeds_equals_the_loss_backward(engine_mod, oracle):
    """seed_h = sf_h dLossMax_h on the device's refined poses, grad_sf = losses: the loss round's selection, jobs and
    score gradients exactly, dLoss/dObj to 1e-12 of max-abs (sf enters before the sum over the pose, not after)."""
    E, O = engine_mod, oracle
    nf, H = 4, 48
    eng, fw, coords, pix, gt_jp = _dsac_pass(E, nf, H, frame0=3, random_draw=True)
    bw = eng.backward_dsac(nf)
    ref6 = _jp6(eng, nf, (nf, H, 6))
    seed = np.stack([[fw.sf[f, h] * O.dloss_max(ref6[f, h], _gt6(O, gt_jp[f])) for h in range(H)] for f in range(nf)])
    got = _dsac_pose_backward(eng, nf, H, seed, fw.losses)
    assert np.array_equal(got["n_selected"], bw.n_selected) and bw.n_selected.min() >= 1
    assert np.array_equal(got["n_refine_jobs"], bw.n_refine_jobs)
    assert np.array_equal(got["score_grads"], bw.score_grads)
    assert np.abs(got["dloss_dobj"] - bw.dloss_dobj).max() <= 1e-12 * np.abs(bw.dloss_dobj).max()


@pytest.mark.parametrize("H", [16, 48])
def test_dsac_pose_backward_matches_oracle(engine_mod, oracle, H):
    """Random seeds on a random half of the hypotheses and a random dOuter/dsf, against orc_backward_dsac_seeded fed the
    engine's forward state; the tolerances of test_dsac_variant_backward_matches_oracle."""
    E, O = engine_mod, oracle
    nf = 2
    eng, fw, coords, pix, gt_jp = _dsac_pass(E, nf, H, gt=False)
    rng = np.random.default_rng(H)
    seed = rng.normal(0, 1, (nf, H, 6)) * (rng.random((nf, H, 1)) < 0.5)
    seed[np.arange(nf), np.argmax(fw.sf, axis=1)] = rng.normal(0, 1, (nf, 6))   # the likeliest hypothesis is always seeded
    grad_sf = rng.normal(0, 1, (nf, H))
    got = _dsac_pose_backward(eng, nf, H, seed, grad_sf)
    for f in range(nf):
        cfg = O.default_config(seed=1305 + f, n_hyps=H)
        ofw = O.ForwardDsac(cfg)
        ofw.hyp_rvec[:] = fw.hyp_pose[f][:, :3]; ofw.hyp_tvec[:] = fw.hyp_pose[f][:, 3:]
        ofw.img_idx[:] = fw.img_idx[f]; ofw.sf[:] = fw.sf[f]; ofw.ref_pose[:] = fw.ref_pose[f]
        obw = S.backward_dsac_seeded(O, cfg, coords[f], pix[f], ofw, seed[f], grad_sf[f])
        assert obw.n_selected == got["n_selected"][f] and obw.n_selected >= 1
        assert obw.n_refine_jobs == got["n_refine_jobs"][f]
        assert _rel(got["score_grads"][f], obw.score_grads, floor=1e-12) <= 1e-9
        assert np.abs(obw.path1).max() > 0 and np.abs(obw.path2).max() > 0
        assert _rel(got["path1"][f], obw.path1) <= 1e-5
        assert np.median(np.abs(got["path1"][f] - obw.path1)) <= 1e-10 * np.abs(obw.path1).max()
        assert _rel(got["path2"][f], obw.path2) <= 1e-6
        assert _rel(got["dloss_dobj"][f], obw.dloss_dobj) <= 1e-5


def test_dsac_pose_backward_selection(engine_mod):
    """Zero seeds refine nothing; seeding only the drawn hypothesis selects it iff sf > 1e-4; null seeds zero their path."""
    E = engine_mod
    nf, H = 4, 32
    eng, fw, coords, pix, gt_jp = _dsac_pass(E, nf, H, gt=False, random_draw=True)
    zero = _dsac_pose_backward(eng, nf, H, np.zeros((nf, H, 6)), None)
    assert (zero["n_refine_jobs"] == 0).all() and (zero["n_selected"] == 0).all()
    assert not zero["path1"].any() and not zero["path2"].any() and not zero["score_grads"].any()
    seed = np.zeros((nf, H, 6))
    pick = fw.hyp_idx
    seed[np.arange(nf), pick] = np.random.default_rng(0).normal(0, 1, (nf, 6))
    one = _dsac_pose_backward(eng, nf, H, seed, None)
    assert np.array_equal(one["n_selected"], (fw.sf[np.arange(nf), pick] > 1e-4).astype(np.int32))
    assert not one["path2"].any()
    full = _dsac_pose_backward(eng, nf, H, np.ones((nf, H, 6)), None)
    assert (one["n_refine_jobs"] <= full["n_refine_jobs"]).all() and (full["n_selected"] > one["n_selected"]).any()
    sf_only = _dsac_pose_backward(eng, nf, H, None, np.random.default_rng(1).normal(0, 1, (nf, H)))
    assert (sf_only["n_refine_jobs"] == 0).all() and not sf_only["path1"].any() and np.abs(sf_only["path2"]).max() > 0


def test_seeded_backward_is_linear_in_the_seed(engine_mod, oracle):
    """Doubling every seed doubles dLoss/dObj bit for bit (no score gradient reaches grad_clamp); b(x) + b(y) = b(x + y)
    to 1e-12 of max-abs.  Both pipelines."""
    E, O = engine_mod, oracle
    nf, H = 2, 32
    rng = np.random.default_rng(5)
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    assert eng.cfg.grad_clamp > 0
    eng.forward(coords, pix)
    x, y = rng.normal(0, 1e-3, (nf, 6)), rng.normal(0, 1e-3, (nf, 6))
    for f in range(nf):   # no score gradient of these seeds reaches grad_clamp
        cfg = O.default_config(seed=1305 + f, n_hyps=H)
        ofw = O.forward(cfg, coords[f], pix[f])
        for s in (2 * x[f], y[f], x[f] + y[f]):
            assert np.abs(S.backward_seeded(O, cfg, coords[f], pix[f], ofw, s).score_grads).max() < 0.5 * eng.cfg.grad_clamp
    bx, by = _pose_backward(eng, nf, x)[0], _pose_backward(eng, nf, y)[0]
    assert np.array_equal(_pose_backward(eng, nf, 2 * x)[0], 2 * bx)
    bxy = _pose_backward(eng, nf, x + y)[0]
    assert np.abs(bx + by - bxy).max() <= 1e-12 * np.abs(bxy).max() and np.abs(bxy).max() > 0

    eng, fw, coords, pix, gt_jp = _dsac_pass(E, nf, H, gt=False)
    x, y = rng.normal(0, 1, (nf, H, 6)), rng.normal(0, 1, (nf, H, 6))
    gx, gy = rng.normal(0, 1e-2, (nf, H)), rng.normal(0, 1e-2, (nf, H))
    r1, r2 = _dsac_pose_backward(eng, nf, H, x, gx), _dsac_pose_backward(eng, nf, H, 2 * x, 2 * gx)
    assert np.abs(r2["score_grads"]).max() < eng.cfg.grad_clamp
    assert np.array_equal(r2["dloss_dobj"], 2 * r1["dloss_dobj"])
    r3, r4 = _dsac_pose_backward(eng, nf, H, y, gy), _dsac_pose_backward(eng, nf, H, x + y, gx + gy)
    assert np.abs(r1["dloss_dobj"] + r3["dloss_dobj"] - r4["dloss_dobj"]).max() <= 1e-12 * np.abs(r4["dloss_dobj"]).max()


def test_pose_entry_points_refuse_misuse(engine_mod):
    """The wrong pass kind, a frame count other than the forward's and a pending submitted pass are refused."""
    import torch
    E = engine_mod
    nf, H = 2, 16
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    seed6, seedH, gsf, jp6 = _dev(np.ones((nf, 6))), _dev(np.ones((nf, H, 6))), _dev(np.ones((nf, H))), _dev(np.zeros((nf, 6)))
    s = torch.cuda.current_stream().cuda_stream
    eng.forward(coords, pix)
    with pytest.raises(RuntimeError, match=r"\(-1\)"):
        eng.backward_dsac_pose_device(nf, seedH.data_ptr(), gsf.data_ptr(), stream=s)
    with pytest.raises(RuntimeError, match=r"\(-1\)"):
        eng.backward_pose_device(nf - 1, seed6.data_ptr(), stream=s)
    eng.forward_dsac(coords, pix, None)
    with pytest.raises(RuntimeError, match=r"\(-1\)"):
        eng.backward_pose_device(nf, seed6.data_ptr(), stream=s)
    with pytest.raises(RuntimeError, match=r"\(-1\)"):
        eng.backward_dsac_pose_device(nf - 1, seedH.data_ptr(), gsf.data_ptr(), stream=s)
    eng.forward_submit(coords, pix)
    for call in (lambda: eng.backward_pose_device(nf, seed6.data_ptr(), stream=s),
                 lambda: eng.refined_jp6_device(nf, jp6.data_ptr(), s)):
        with pytest.raises(RuntimeError, match=r"\(-1\)"):
            call()
    eng.forward_wait()
    torch.cuda.synchronize()


def _prediction(coords, seed=0, noise_mm=0.0):
    import torch
    rng = np.random.default_rng(seed)
    p = coords.astype(np.float32) / np.float32(1000) + (rng.normal(0, noise_mm, coords.shape) / 1000).astype(np.float32)
    return torch.from_numpy(p).cuda()


def _rounded(eng, pred, nf):
    import torch
    q = torch.empty((nf, 1600, 3), dtype=torch.int16, device="cuda")
    eng.coords_from_prediction_device(nf, pred.detach().data_ptr(), q.data_ptr())
    torch.cuda.synchronize()
    return q


def test_softam_pose_autograd(engine_mod):
    """prediction.grad of (softam_pose * W).sum() = float32(clip(dLoss/dObj(seed = W), +-0.1)) bit for bit; with W the
    engine's dLossMax it is softam_loss's gradient bit for bit."""
    import torch
    from dsac_b200.autograd import softam_loss, softam_pose
    E = engine_mod
    nf, H, frame0 = 8, 64, 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, frame0=frame0)
    pred = _prediction(coords, seed=1, noise_mm=3.0).requires_grad_(True)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    dpix, dgt = _dev(pix), _dev(gt_jp)
    W = _dev(np.random.default_rng(2).normal(0, 1, (nf, 6)))
    pose = softam_pose(eng, pred, dpix, frame0=frame0)
    assert pose.shape == (nf, 6) and pose.dtype == torch.float64
    (pose * W).sum().backward()
    torch.cuda.synchronize()
    q = _rounded(eng, pred, nf)
    ref = E.Engine(max_frames=nf, n_hyps=H)
    ref.forward_device(nf, q.data_ptr(), dpix.data_ptr(), 0, None, frame0, torch.cuda.current_stream().cuda_stream)
    assert np.array_equal(_jp6(ref, nf, (nf, 6)), pose.detach().cpu().numpy())
    dobj, _ = _pose_backward(ref, nf, W.cpu().numpy())
    got = pred.grad.cpu().numpy()
    assert np.array_equal(got, np.clip(dobj, -0.1, 0.1).astype(np.float32)) and np.abs(got).max() > 0

    ref.forward(q.cpu().numpy(), pix, gt_jp, frame0=frame0)
    dref = ref.backward(q.cpu().numpy(), pix, gt_jp, full=False).dloss_dref
    pred.grad = None
    (softam_pose(eng, pred, dpix, frame0=frame0) * _dev(dref)).sum().backward()
    g_pose = pred.grad.clone()
    pred.grad = None
    softam_loss(eng, pred, dpix, dgt, frame0=frame0).sum().backward()
    assert torch.equal(g_pose, pred.grad)


def test_dsac_hypotheses_autograd(engine_mod):
    """L = (sf * (ref * W).sum(-1)).sum(): prediction.grad matches the C entry seeded by the same torch ops (the DSAC
    tolerance of test_autograd_hand_off); an output without gradient skips its path."""
    import torch
    from dsac_b200.autograd import dsac_hypotheses
    E = engine_mod
    nf, H, frame0 = 6, 64, 1
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, frame0=frame0)
    pred = _prediction(coords, seed=3, noise_mm=3.0).requires_grad_(True)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    dpix = _dev(pix)
    W = _dev(np.random.default_rng(4).normal(0, 1, (nf, H, 6)))
    sf, ref6 = dsac_hypotheses(eng, pred, dpix, frame0=frame0)
    assert sf.shape == (nf, H) and ref6.shape == (nf, H, 6)
    (sf * (ref6 * W).sum(-1)).sum().backward()
    torch.cuda.synchronize()
    g_ref = sf.detach()[..., None] * W
    g_sf = (ref6.detach() * W).sum(-1)
    q = _rounded(eng, pred, nf)
    ref = E.Engine(max_frames=nf, n_hyps=H)
    ref.forward_dsac_device(nf, q.data_ptr(), dpix.data_ptr(), 0, None, True, frame0, torch.cuda.current_stream().cuda_stream)
    want_t = torch.empty((nf, 1600, 3), dtype=torch.float32, device="cuda")
    ref.backward_dsac_pose_device(nf, g_ref.data_ptr(), g_sf.data_ptr(), want_t.data_ptr(), 0.1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    want, got = want_t.cpu().numpy(), pred.grad.cpu().numpy()
    assert np.abs(got - want).max() <= 1e-5 * max(1e-12, np.abs(want).max())
    assert np.mean(got == want) > 0.99 and np.abs(got).max() > 0

    pred.grad = None
    _, ref6 = dsac_hypotheses(eng, pred, dpix, frame0=frame0)
    (ref6 * W).sum().backward()     # no gradient reaches sf: path II is skipped
    assert torch.isfinite(pred.grad).all() and pred.grad.abs().max() > 0


def test_pose_autograd_misuse_raises(engine_mod):
    import torch
    from dsac_b200.autograd import dsac_hypotheses, softam_pose
    E = engine_mod
    nf = 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=16)
    pred = _prediction(coords).requires_grad_(True)
    dpix = _dev(pix)
    for fn in (softam_pose, lambda *a: dsac_hypotheses(*a)[1]):
        out = fn(eng, pred, dpix)
        fn(eng, pred.detach(), dpix)          # a second pass on the same engine
        with pytest.raises(RuntimeError, match="another forward pass"):
            out.sum().backward()
        with pytest.raises(ValueError, match="is on cpu"):
            fn(eng, pred, torch.from_numpy(pix))


def test_sgd_through_softam_pose_lowers_a_user_pose_loss(engine_mod, oracle):
    """A learnable per-cell offset added to noisy predictions of fixed frames, trained with SGD through softam_pose on a
    user-written L2 distance to the ground-truth jp 6-vector."""
    import torch
    from dsac_b200.autograd import softam_pose
    E, O = engine_mod, oracle
    nf = 16
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    gt6 = _dev(np.stack([_gt6(O, g) for g in gt_jp]))
    base = _prediction(coords, seed=2, noise_mm=20.0)
    eng = E.Engine(max_frames=nf, n_hyps=64)
    dpix = _dev(pix)
    offset = torch.zeros((1, E.N, 3), dtype=torch.float32, device="cuda", requires_grad=True)
    opt = torch.optim.SGD([offset], lr=SGD_LR)

    def pose_loss(pose):
        return torch.linalg.vector_norm(pose - gt6, dim=-1).mean()

    losses = []
    for _ in range(SGD_STEPS):
        opt.zero_grad()
        loss = pose_loss(softam_pose(eng, base + offset, dpix))
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    with torch.no_grad():
        final = float(pose_loss(softam_pose(eng, base + offset, dpix)))
    assert final < losses[0], (losses, final)


SGD_LR, SGD_STEPS = 0.3, 3
