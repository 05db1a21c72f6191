"""Guided sampling (dsac_set_sampling_logits_device) on the GPU against its CPU restatement (tests/guided_oracle.py):
the integer tables, the sampled minimal sets and everything after them, the log-probability of a pass's draw and its
gradient; batch-split invariance, misuse, and the autograd surface."""
import numpy as np
import pytest
import torch

import guided_oracle as G

pytestmark = pytest.mark.gpu
N = 1600


def _inlier_logits(O, coords, pix, gt_cv, mass=0.9):
    """Logits that put `mass` of every frame's weight on its inlier cells (reprojection error < thr2d under the
    ground-truth pose), float32 [n][N]."""
    out = np.zeros((len(coords), N), np.float32)
    for f in range(len(coords)):
        inl = O.diff_map(coords[f], pix[f], gt_cv[f, :3], gt_cv[f, 3:]) < 10
        k = max(int(inl.sum()), 1)
        out[f] = np.where(inl, np.log(mass / k), np.log((1 - mass) / max(N - k, 1))).astype(np.float32)
    return out


def _logits(n, seed=3, scale=1.0):
    return (np.random.default_rng(seed).standard_normal((n, N)) * scale).astype(np.float32)


def _set(eng, logits):
    d = torch.from_numpy(logits).cuda()
    eng.set_sampling_logits_device(len(logits), d.data_ptr())
    torch.cuda.synchronize()
    return d


@pytest.mark.parametrize("T,H", [(1, 64), (3, 64), (1, 256), (3, 256)])
def test_forward_matches_guided_oracle(engine_mod, oracle, T, H):
    E, O = engine_mod, oracle
    n = 4
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=T)
    logits = _logits(n)
    logits[1] = _inlier_logits(O, coords[1:2], pix[1:2], gt_cv[1:2])[0]
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=T)
    d = _set(eng, logits)
    q = torch.empty((n, N), dtype=torch.int32, device="cuda")
    eng.sampling_table_device(n, q.data_ptr())
    res = eng.forward(coords, pix, gt_jp, frame0=5)
    logp = torch.empty(n, dtype=torch.float64, device="cuda")
    eng.sampling_log_prob_device(n, logp.data_ptr())
    gl = torch.linspace(0.5, 2.0, n, dtype=torch.float64, device="cuda")
    grad = torch.empty((n, N), dtype=torch.float32, device="cuda")
    eng.sampling_log_prob_backward_device(n, gl.data_ptr(), grad.data_ptr())
    grad2 = torch.empty_like(grad)
    eng.sampling_log_prob_backward_device(n, gl.data_ptr(), grad2.data_ptr())
    logp2 = torch.empty_like(logp)
    eng.sampling_log_prob_device(n, logp2.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(grad, grad2) and torch.equal(logp, logp2)
    cfg = O.default_config(n_hyps=H, n_streams=T)
    for f in range(n):
        w, qo, cum, bad = G.table(logits[f])
        assert not bad and np.array_equal(q[f].cpu().numpy().view(np.uint32), qo), f
        fw, ncand = G.forward(O, cfg, cum, 5 + f, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
        assert np.array_equal(fw.img_idx, res.img_idx[f]), f
        assert np.array_equal(fw.cand_idx, res.cand_idx[f]), f
        assert fw.n_candidates == res.n_candidates[f], f
        assert res.status[f] == 0
        assert np.abs(fw.scores - res.scores[f]).max() <= 1e-5 * np.abs(fw.scores).max()
        assert np.abs(fw.ref - res.ref_pose[f]).max() <= 1e-3
        assert abs(fw.loss - res.loss[f]) <= 1e-3 * max(1.0, abs(fw.loss))
        lp, go = G.log_prob(w, cum, T, 1305, 5 + f, ncand)
        assert abs(logp[f].item() - lp) <= 1e-10 * abs(lp)
        want = (gl[f].item() * go).astype(np.float32)
        assert np.allclose(grad[f].cpu().numpy(), want, rtol=1e-5, atol=1e-6 * np.abs(want).max())
    del d
    eng.close()


def _rel(a, b, floor=1e-300):
    return np.abs(a - b).max() / max(floor, np.abs(b).max())


@pytest.mark.parametrize("random_draw", [0, 1])
def test_dsac_variant_matches_guided_oracle(engine_mod, oracle, random_draw):
    """The DSAC variant after a guided draw: sampled sets, softmax, the drawn hypothesis (MT19937 stream 0 of the frame,
    read right after stream_skip), every refined pose, the losses and the expected loss, with the tolerances of the
    uniform path's test."""
    E, O = engine_mod, oracle
    n, H, T = 3, 32, 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=T)
    logits = _logits(n, 4)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=T)
    _set(eng, logits)
    res = eng.forward_dsac(coords, pix, gt_jp, random_draw=bool(random_draw), want_inlier_maps=True)
    cfg = O.default_config(n_hyps=H, n_streams=T)
    for f in range(n):
        _, _, cum, _ = G.table(logits[f])
        o = G.forward_dsac(O, cfg, cum, f, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], bool(random_draw))
        assert np.array_equal(o.img_idx, res.img_idx[f]), f
        assert o.hyp_idx == res.hyp_idx[f], f
        assert np.array_equal(o.steps_done, res.steps_done[f])
        assert np.array_equal(o.inlier_maps, res.inlier_maps[f])
        assert np.abs(o.ref_pose[:, :3] - res.ref_pose[f][:, :3]).max() <= 1e-8
        assert np.abs(o.ref_pose[:, 3:] - res.ref_pose[f][:, 3:]).max() <= 1e-5
        assert np.abs(o.losses - res.losses[f]).max() <= 1e-6 * max(1.0, np.abs(o.losses).max())
        assert np.abs(o.sf - res.sf[f]).max() <= 1e-4
        assert abs(o.expected_loss - res.expected_loss[f]) <= 1e-3 * max(1.0, abs(o.expected_loss))
        assert abs(o.rot_err - res.rot_err[f]) <= 1e-6 and abs(o.t_err - res.t_err[f]) <= 1e-4 and o.correct == res.correct[f]
    eng.close()


def test_backward_through_a_guided_pass(engine_mod, oracle):
    """The coordinate backward of both pipelines after a guided forward equals the oracle's backward applied to the
    guided oracle's forward (tolerances of the uniform path's tests).  For the DSAC variant the oracle takes the engine's
    sf, as the uniform test does: the fp32 score moves sf by up to 1e-4, which would move the sf > 1e-4 selection."""
    E, O = engine_mod, oracle
    n, H = 2, 32
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    logits = _logits(n, 8)
    eng = E.Engine(max_frames=n, n_hyps=H)
    _set(eng, logits)
    fwd = eng.forward(coords, pix, gt_jp)
    bw = eng.backward(coords, pix, gt_jp)
    cfg = O.default_config(n_hyps=H)
    for f in range(n):
        _, _, cum, _ = G.table(logits[f])
        ofw, _ = G.forward(O, cfg, cum, f, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
        assert np.array_equal(ofw.img_idx, fwd.img_idx[f])
        obw = O.backward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw)
        assert _rel(bw.dloss_dref[f], obw.dloss_dref) <= 1e-9
        assert _rel(bw.dref_dhyp[f], obw.dref_dhyp, floor=1e-3) <= 1e-7
        assert _rel(bw.dpnp[f], obw.dpnp) <= 1e-7
        assert _rel(bw.score_grads[f], obw.score_grads, floor=1e-6) <= 1e-4
        assert _rel(bw.dloss_dobj[f], obw.dloss_dobj, floor=1e-6) <= 1e-3 and np.abs(bw.dloss_dobj[f]).max() > 0
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    bwd = eng.backward_dsac(n)
    for f in range(n):
        _, _, cum, _ = G.table(logits[f])
        ofw = G.forward_dsac(O, cfg, cum, f, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], False)
        assert np.array_equal(ofw.img_idx, fw.img_idx[f])
        ofw.sf[:] = fw.sf[f]
        obw = O.backward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw)
        assert obw.n_selected == bwd.n_selected[f] and obw.n_selected >= 1
        assert _rel(bwd.path1[f], obw.path1) <= 1e-5
        assert _rel(bwd.path2[f], obw.path2) <= 1e-6
        assert _rel(bwd.dloss_dobj[f], obw.dloss_dobj) <= 1e-5
    eng.close()


@pytest.mark.parametrize("max_candidates", [1 << 20, 1400])
def test_short_streams_continue_in_guided_steps(engine_mod, oracle, monkeypatch, max_candidates):
    """One round only (DSAC_K1_ROUNDS=1): streams the round leaves short continue in k1_gtail, 256 guided candidates at a
    time, and with a small max_candidates run out there.  Sets, candidate indices, counts and the exhausted bit equal
    the guided oracle's."""
    E, O = engine_mod, oracle
    monkeypatch.setenv("DSAC_K1_ROUNDS", "1")
    n, H, T = 4, 64, 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=T)
    logits = _logits(n, 9)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=T, max_candidates=max_candidates)
    _set(eng, logits)
    res = eng.forward(coords, pix, gt_jp)
    cfg = O.default_config(n_hyps=H, n_streams=T, max_candidates=max_candidates)
    exhausted = 0
    for f in range(n):
        _, _, cum, _ = G.table(logits[f])
        fw, ncand = G.forward(O, cfg, cum, f, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
        assert np.array_equal(fw.img_idx, res.img_idx[f]), f
        assert np.array_equal(fw.cand_idx, res.cand_idx[f]), f
        assert fw.n_candidates == res.n_candidates[f], f
        assert bool(res.status[f] & E.ST_SAMPLER_EXHAUSTED) == (fw.status == -1), f
        exhausted += fw.status == -1
        if fw.status != -1:
            assert np.abs(fw.ref - res.ref_pose[f]).max() <= 1e-3
    assert (exhausted > 0) == (max_candidates < 1 << 20)
    eng.close()


def test_batch_split_invariance(engine_mod, oracle):
    """One 1024-frame guided batch (two lanes) equals the same frames run as four calls with frame0 offsets, bit for bit;
    the same with per-frame cameras."""
    E, O = engine_mod, oracle
    n, H = 1024, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    logits = _logits(n, 5)
    cams = np.tile(np.array([[525.0, 320.0, 240.0], [585.0, 324.5, 236.25]]), (n // 2, 1))
    for use_cams in (False, True):
        eng = E.Engine(max_frames=n, n_hyps=H)
        if use_cams:
            eng.set_cameras(cams)
        _set(eng, logits)
        whole = eng.forward(coords, pix, gt_jp)
        part = E.Engine(max_frames=256, n_hyps=H)
        for k in range(4):
            sl = slice(256 * k, 256 * (k + 1))
            if use_cams:
                part.set_cameras(cams[sl])
            _set(part, logits[sl])
            r = part.forward(coords[sl], pix[sl], gt_jp[sl], frame0=256 * k)
            for name in ("img_idx", "cand_idx", "n_candidates", "hyp_pose", "scores", "ref_pose", "status"):
                assert np.array_equal(getattr(whole, name)[sl], getattr(r, name)), (use_cams, k, name)
        eng.close()
        part.close()


def test_misuse_and_bad_weights(engine_mod):
    E = engine_mod
    n = 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    eng = E.Engine(max_frames=n, n_hyps=64)
    d = torch.zeros((n, N), dtype=torch.float32, device="cuda")
    buf = torch.empty(n, dtype=torch.float64, device="cuda")
    g = torch.empty((n, N), dtype=torch.float32, device="cuda")
    with pytest.raises(RuntimeError):
        eng.set_sampling_logits_device(n + 1, d.data_ptr())          # n out of range
    eng.forward(coords, pix, gt_jp)
    with pytest.raises(RuntimeError):
        eng.sampling_log_prob_device(n, buf.data_ptr())               # the pass was not guided
    bad = torch.zeros((n, N), dtype=torch.float32, device="cuda")
    bad[1, 7] = float("nan")
    bad[2, 3:] = float("-inf")
    eng.set_sampling_logits_device(n, bad.data_ptr())
    with pytest.raises(RuntimeError):
        eng.forward(coords[:2], pix[:2], gt_jp[:2])                   # n differs from the setting
    res = eng.forward(coords, pix, gt_jp)
    assert res.status[0] == 0 and res.status[1] & E.ST_BAD_WEIGHTS and res.status[2] & E.ST_BAD_WEIGHTS
    assert (res.img_idx[1:] == -1).all() and (res.cand_idx[1:] == -1).all() and (res.hyp_pose[1:] == 0).all()
    with pytest.raises(RuntimeError):
        eng.sampling_log_prob_device(n - 1, buf.data_ptr())           # n differs from the pass
    eng.sampling_log_prob_device(n, buf.data_ptr())
    eng.sampling_log_prob_backward_device(n, buf.data_ptr(), g.data_ptr())
    torch.cuda.synchronize()
    assert buf[1].item() == 0 and buf[2].item() == 0 and (g[1:] == 0).all()
    eng.set_sampling_logits_device(n, d.data_ptr())
    with pytest.raises(RuntimeError):
        eng.sampling_log_prob_device(n, buf.data_ptr())               # the logits changed since the pass
    eng.forward_submit(coords, pix, gt_jp)
    for call in (lambda: eng.set_sampling_logits_device(n, d.data_ptr()), lambda: eng.sampling_log_prob_device(n, buf.data_ptr())):
        with pytest.raises(RuntimeError):
            call()                                                    # a submitted pass is pending
    eng.forward_wait()
    eng.sampling_log_prob_device(n, buf.data_ptr())
    eng.set_sampling_logits_device(n, None)
    res = eng.forward(coords, pix, gt_jp)                             # back to the reference sampler
    ref = E.Engine(max_frames=n, n_hyps=64).forward(coords, pix, gt_jp)
    assert np.array_equal(res.img_idx, ref.img_idx)
    eng.close()


def test_autograd(engine_mod, oracle):
    E, O = engine_mod, oracle
    from dsac_b200 import autograd as A
    n, H = 4, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    eng = E.Engine(max_frames=n, n_hyps=H)
    pred = (torch.from_numpy(coords.astype(np.float32)) / 1000).cuda().requires_grad_(True)
    pix_t = torch.from_numpy(pix).cuda()
    gt = torch.from_numpy(gt_jp).cuda()
    logits = torch.from_numpy(_logits(n, 6)).cuda().requires_grad_(True)
    for fn in (lambda: A.softam_loss(eng, pred, pix_t, gt, sampling_logits=logits),
               lambda: A.dsac_expected_loss(eng, pred, pix_t, gt, sampling_logits=logits),
               lambda: A.softam_pose(eng, pred, pix_t, sampling_logits=logits).sum(1),
               lambda: A.dsac_hypotheses(eng, pred, pix_t, sampling_logits=logits)[0][:, 0]):
        logits.grad = None
        pred.grad = None
        out = fn()
        logp = A.sampling_log_prob(eng, logits)
        (out + (out.detach() - out.detach().mean()) * logp).sum().backward()
        assert logits.grad is not None and torch.isfinite(logits.grad).all() and pred.grad is not None
        assert abs(logits.grad.double().sum(1)).max().item() <= 1e-3 * logits.grad.abs().max().item() + 1e-6
    with pytest.raises(RuntimeError):
        A.sampling_log_prob(eng, logits.detach().clone())             # not the tensor the pass was sampled with
    A.softam_loss(eng, pred, pix_t, gt, sampling_logits=logits)
    with torch.no_grad():
        logits.add_(0)                                                # modified since the pass
    with pytest.raises(RuntimeError):
        A.sampling_log_prob(eng, logits)
    with pytest.raises(ValueError):
        A.softam_loss(eng, pred, pix_t, gt, sampling_logits=logits.double())
    eng.close()


def test_reinforce_lowers_candidates(engine_mod, oracle):
    """A short deterministic REINFORCE loop on free logits: reward = -candidates per frame, baseline = the mean over 8
    replicas of each frame (distinct frame0 keys), Adam.  The softmax mass on inlier cells rises and the candidates per
    frame fall."""
    E, O = engine_mod, oracle
    nf, R, H = 4, 8, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    inl = np.stack([O.diff_map(coords[f], pix[f], gt_cv[f, :3], gt_cv[f, 3:]) < 10 for f in range(nf)])
    inl_t = torch.from_numpy(inl).cuda()
    eng = E.Engine(max_frames=nf * R, n_hyps=H)
    rep = lambda a: np.repeat(a, R, axis=0)
    c_r, p_r, g_r = rep(coords), rep(pix), rep(gt_jp)
    free = torch.zeros((nf, N), dtype=torch.float32, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([free], lr=0.3)
    hist = []
    for it in range(40):
        logits = free.repeat_interleave(R, 0).detach().requires_grad_(True)
        d = logits.detach().contiguous()
        eng.set_sampling_logits_device(nf * R, d.data_ptr())
        res = eng.forward(c_r, p_r, g_r, frame0=it * nf * R)
        cand = torch.from_numpy(res.n_candidates.astype(np.float64)).cuda()
        A = -cand
        adv = A - A.view(nf, R).mean(1).repeat_interleave(R)
        logp = torch.empty(nf * R, dtype=torch.float64, device="cuda")
        eng.sampling_log_prob_device(nf * R, logp.data_ptr())
        grad = torch.empty((nf * R, N), dtype=torch.float32, device="cuda")
        eng.sampling_log_prob_backward_device(nf * R, (-adv / (nf * R)).contiguous().data_ptr(), grad.data_ptr())
        opt.zero_grad()
        free.grad = grad.view(nf, R, N).sum(1)
        opt.step()
        mass = (torch.softmax(free.detach().double(), 1) * inl_t).sum(1).mean().item()
        hist.append((cand.mean().item(), mass))
    eng.close()
    first, last = np.mean([h[0] for h in hist[:5]]), np.mean([h[0] for h in hist[-5:]])
    # measured once on an H100 80GB HBM3 (700 W): candidates per frame 4778.2 over the first five steps, 3087.9 over the
    # last five (ratio 0.646); inlier mass 0.2894 -> 0.3912.  The loop is deterministic; the thresholds leave margin.
    assert hist[-1][1] > hist[0][1] + 0.05, hist
    assert last < 0.8 * first, hist
