"""RGB-D localisation (dsac_set_cell_depth_device) on the GPU against its CPU restatement (tests/rgbd_oracle.py): the
sampled minimal sets, scores and the Kabsch refinement, with depth holes, per-frame cameras, guided sampling and frames
without depth; invariance to the sampler's schedule; returning to RGB; misuse."""
import numpy as np
import pytest
import torch

import guided_oracle as G
import rgbd_oracle as R

pytestmark = pytest.mark.gpu
N = 1600


def _set(eng, depth):
    d = torch.from_numpy(np.ascontiguousarray(depth, np.float32)).cuda()
    eng.set_cell_depth_device(len(depth), d.data_ptr())
    torch.cuda.synchronize()
    return d


def _check_frames(O, cfg, res, coords, pix, depth, gt_jp, frame0, cams=None, cums=None):
    """Compare every frame with the oracle; frames the oracle marks fragile are skipped and counted."""
    fragile = 0
    for f in range(len(coords)):
        c = cams[f] if cams is not None else (cfg.f, cfg.cx, cfg.cy)
        cf = O.default_config(n_hyps=cfg.n_hyps, n_streams=cfg.n_streams, f=c[0], cx=c[1], cy=c[2])
        ey, have = R.eye(pix[f], depth[f], *c)
        fw, ncand = R.forward(O, cf, frame0 + f, coords[f], pix[f], ey, None if cums is None else cums[f], gt_jp[f, :9], gt_jp[f, 9:])
        if have < 4:
            assert fw.status == -2
            assert res.status[f] & 64 and (res.img_idx[f] == -1).all() and res.n_candidates[f] == 0, f
            continue
        if fw.n_fragile:
            fragile += 1
            continue
        assert np.array_equal(fw.img_idx, res.img_idx[f]), f
        assert np.array_equal(fw.cand_idx, res.cand_idx[f]), f
        assert fw.n_candidates == res.n_candidates[f], f
        assert not res.status[f] & 64
        exhausted = bool(res.status[f] & 1)
        assert exhausted == (fw.status == -1), f
        hp = np.concatenate([fw.hyp_rvec, fw.hyp_tvec], 1)
        assert _rel(res.hyp_pose[f], hp, floor=1e-3) <= 1e-9, f
        assert np.abs(fw.scores - res.scores[f]).max() <= 1e-5 * np.abs(fw.scores).max()
        assert np.abs(fw.sf - res.sf[f]).max() <= 1e-4
        assert np.abs(fw.ref - res.ref_pose[f]).max() <= 1e-3
        assert abs(fw.loss - res.loss[f]) <= 1e-3 * max(1.0, abs(fw.loss))
        assert abs(fw.rot_err - res.rot_err[f]) <= 1e-3 and abs(fw.t_err - res.t_err[f]) <= 1e-2 and fw.correct == res.correct[f]
    return fragile


def _rel(a, b, floor=1e-300):
    return np.abs(a - b).max() / max(floor, np.abs(b).max())


@pytest.mark.parametrize("T,H", [(1, 64), (3, 64), (1, 256), (3, 256)])
@pytest.mark.parametrize("per_frame_cams", [False, True])
def test_forward_matches_rgbd_oracle(engine_mod, oracle, T, H, per_frame_cams):
    E, O = engine_mod, oracle
    n = 4
    cams = np.array([[525.0, 320.0, 240.0], [580.0, 310.5, 250.25], [500.0, 330.0, 236.0], [540.0, 320.0, 240.0]]) if per_frame_cams else None
    coords, pix, depth, _, gt_jp = R.synth(n, seed=11 + T, holes=0.15, cams=cams)
    depth[3, 4:] = np.nan                      # frame 3: 4 cells with depth
    if T == 3:
        depth[2, 3:] = np.nan                  # frame 2: 3 cells with depth, DSAC_ST_NO_DEPTH
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=T, max_candidates=20000)
    if cams is not None:
        eng.set_cameras(cams)
    d = _set(eng, depth)
    res = eng.forward(coords, pix, gt_jp, frame0=5)
    cfg = O.default_config(n_hyps=H, n_streams=T)
    fragile = _check_frames(O, cfg, res, coords, pix, depth, gt_jp, 5, cams)
    print("fragile frames skipped:", fragile)
    del d
    eng.close()


def test_guided_rgbd_with_inf_on_holes(engine_mod, oracle):
    E, O = engine_mod, oracle
    n, H, T = 3, 64, 3
    coords, pix, depth, _, gt_jp = R.synth(n, seed=21, holes=0.15)
    logits = np.random.default_rng(5).standard_normal((n, N)).astype(np.float32)
    logits[~np.isfinite(depth)] = -np.inf
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=T, max_candidates=20000)
    dl = torch.from_numpy(logits).cuda()
    eng.set_sampling_logits_device(n, dl.data_ptr())
    d = _set(eng, depth)
    res = eng.forward(coords, pix, gt_jp, frame0=2)
    cums = [G.table(logits[f])[2] for f in range(n)]
    fragile = _check_frames(O, O.default_config(n_hyps=H, n_streams=T), res, coords, pix, depth, gt_jp, 2, cums=cums)
    print("fragile frames skipped:", fragile)
    # the draw never picks a cell without depth, so far fewer candidates than the uniform draw needs
    eng.set_sampling_logits_device(0, None)
    uni = eng.forward(coords, pix, gt_jp, frame0=2)
    assert res.n_candidates.sum() < uni.n_candidates.sum()
    del d, dl
    eng.close()


def _run(E, monkeypatch, env, coords, pix, depth, gt_jp, T, H, max_candidates):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = E.Engine(max_frames=len(coords), n_hyps=H, n_streams=T, max_candidates=max_candidates)
    d = _set(eng, depth)
    res = eng.forward(coords, pix, gt_jp, frame0=1)
    for k in env:
        monkeypatch.delenv(k)
    del d
    eng.close()
    return res


@pytest.mark.parametrize("max_candidates", [20000, 300])
def test_schedules_are_bit_identical(engine_mod, monkeypatch, max_candidates):
    """800 frames x 2 streams: portioned, overlapped rounds and two lanes by default, so every variable compares a
    schedule the engine really chooses with another."""
    E = engine_mod
    n, H, T = 800, 64, 2
    coords, pix, depth, _, gt_jp = R.synth(n, seed=31, holes=0.3, rho=0.4)
    base = _run(E, monkeypatch, {}, coords, pix, depth, gt_jp, T, H, max_candidates)
    for env in ({"DSAC_K1_MODE": "mono"}, {"DSAC_K1_ROUNDS": "1"}, {"DSAC_K1_SPEC": "0"}, {"DSAC_K1_LANES": "0"}):
        other = _run(E, monkeypatch, env, coords, pix, depth, gt_jp, T, H, max_candidates)
        for name in ("img_idx", "cand_idx", "n_candidates", "status", "hyp_pose", "scores", "ref_pose", "loss"):
            assert np.array_equal(getattr(base, name), getattr(other, name), equal_nan=True), (env, name)


def test_batch_split_invariance(engine_mod):
    E = engine_mod
    n, H, T = 1024, 64, 2
    coords, pix, depth, _, gt_jp = R.synth(n, seed=41, holes=0.15)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=T, max_candidates=20000)
    d = _set(eng, depth)
    whole = eng.forward(coords, pix, gt_jp, frame0=0)
    for k in range(4):
        s = slice(256 * k, 256 * (k + 1))
        _set(eng, depth[s])
        part = eng.forward(coords[s], pix[s], gt_jp[s], frame0=256 * k)
        for name in ("img_idx", "cand_idx", "n_candidates", "hyp_pose", "ref_pose", "loss"):
            assert np.array_equal(getattr(whole, name)[s], getattr(part, name)), (k, name)
    del d
    eng.close()


def test_cleared_depth_is_rgb(engine_mod):
    E = engine_mod
    n = 3
    coords, pix, depth, _, gt_jp = R.synth(n, seed=51)
    ref_eng = E.Engine(max_frames=n, n_hyps=64, n_streams=2)
    want = ref_eng.forward(coords, pix, gt_jp, frame0=0)
    eng = E.Engine(max_frames=n, n_hyps=64, n_streams=2)
    d = _set(eng, depth)
    rgbd = eng.forward(coords, pix, gt_jp, frame0=0)
    eng.set_cell_depth_device(0, None)
    got = eng.forward(coords, pix, gt_jp, frame0=0)
    for name in ("img_idx", "cand_idx", "n_candidates", "hyp_pose", "scores", "ref_pose", "loss", "status"):
        assert np.array_equal(getattr(want, name), getattr(got, name)), name
    assert not np.array_equal(rgbd.hyp_pose, want.hyp_pose)
    del d
    eng.close()
    ref_eng.close()


@pytest.mark.parametrize("random_draw", [0, 1])
def test_dsac_variant_matches_rgbd_oracle(engine_mod, oracle, random_draw):
    """Sampled sets, softmax, the drawn hypothesis, every refined pose (one k_refine_rgbd job per hypothesis), the losses
    and the expected loss, with the tolerances of the uniform path's test."""
    E, O = engine_mod, oracle
    n, H, T = 3, 32, 3
    coords, pix, depth, _, gt_jp = R.synth(n, seed=61, holes=0.1)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=T)
    d = _set(eng, depth)
    res = eng.forward_dsac(coords, pix, gt_jp, random_draw=bool(random_draw), want_inlier_maps=True)
    cfg = O.default_config(n_hyps=H, n_streams=T)
    for f in range(n):
        ey, _ = R.eye(pix[f], depth[f])
        o = R.forward_dsac(O, cfg, f, coords[f], pix[f], ey, gt_jp[f, :9], gt_jp[f, 9:], bool(random_draw))
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
    del d
    eng.close()


@pytest.mark.parametrize("H", [1, 32])
def test_backward_matches_rgbd_oracle(engine_mod, oracle, H):
    """The soft-argmax backward of an RGB-D pass: refinement jobs through k_refine_rgbd, dPNP through k_dkabsch."""
    E, O = engine_mod, oracle
    n = 2
    coords, pix, depth, _, gt_jp = R.synth(n, seed=81, holes=0.1)
    eng = E.Engine(max_frames=n, n_hyps=H)
    d = _set(eng, depth)
    fwd = eng.forward(coords, pix, gt_jp)
    bw = eng.backward(coords, pix, gt_jp)
    cfg = O.default_config(n_hyps=H)
    for f in range(n):
        cf = O.default_config(n_hyps=H, seed=1305)
        ey, _ = R.eye(pix[f], depth[f])
        ofw, _ = R.forward(O, cf, f, coords[f], pix[f], ey, None, gt_jp[f, :9], gt_jp[f, 9:])
        assert np.array_equal(ofw.img_idx, fwd.img_idx[f])
        obw = R.backward(O, cfg, coords[f], pix[f], ey, gt_jp[f, :9], gt_jp[f, 9:], ofw)
        assert _rel(bw.dloss_dref[f], obw.dloss_dref) <= 1e-9
        assert _rel(bw.dref_dhyp[f], obw.dref_dhyp, floor=1e-3) <= 1e-7
        assert _rel(bw.dref_dobj[f], obw.dref_dobj, floor=1e-3) <= 1e-7
        assert _rel(bw.dpnp[f], obw.dpnp) <= 1e-7
        assert np.abs(bw.dpnp[f][:, :, 9:]).max() == 0
        tol = 1e-7 if H == 1 else 1e-3   # one hypothesis: sf is exactly 1 and path II vanishes, so no fp32 score error
        assert _rel(bw.dloss_dobj[f], obw.dloss_dobj, floor=1e-6) <= tol
        assert np.abs(bw.dloss_dobj[f]).max() > 0
    del d
    eng.close()


def test_backward_dsac_matches_rgbd_oracle(engine_mod, oracle):
    """The DSAC variant's backward of an RGB-D pass: path I's jobs start from k_dsac_job_kabsch and refine through
    k_refine_rgbd, path II through k_dkabsch."""
    E, O = engine_mod, oracle
    n, H, T = 2, 16, 1
    coords, pix, depth, _, gt_jp = R.synth(n, seed=91, holes=0.1)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=T)
    d = _set(eng, depth)
    eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    bw = eng.backward_dsac(n)
    cfg = O.default_config(n_hyps=H, n_streams=T)
    for f in range(n):
        ey, _ = R.eye(pix[f], depth[f])
        ofw = R.forward_dsac(O, cfg, f, coords[f], pix[f], ey, gt_jp[f, :9], gt_jp[f, 9:], True)
        obw = R.backward_dsac(O, cfg, coords[f], pix[f], ey, gt_jp[f, :9], gt_jp[f, 9:], ofw)
        assert bw.n_selected[f] == obw.n_selected and bw.n_refine_jobs[f] == obw.n_refine_jobs
        assert _rel(bw.path1[f], obw.path1) <= 1e-5   # the RGB path's tolerance (test_gpu_backward.py)
        assert np.median(np.abs(bw.path1[f] - obw.path1)) <= 1e-10 * np.abs(obw.path1).max()
        assert np.abs(obw.path1).max() > 0
        assert _rel(bw.dloss_dobj[f], obw.dloss_dobj, floor=1e-6) <= 1e-3
    del d
    eng.close()


@pytest.mark.parametrize("variant", ["softam", "dsac"])
def test_autograd_equals_device(engine_mod, variant):
    """prediction.grad of a loss with cell_depth= equals the _device entry points' dLoss/dPred on the same pass."""
    from dsac_b200 import autograd as A
    E = engine_mod
    n, H = 4, 32
    coords, pix, depth, _, gt_jp = R.synth(n, seed=101, holes=0.1)
    pred = torch.from_numpy(coords.astype(np.float32) / np.float32(1000)).cuda().requires_grad_()
    dpix, dgt, dd = torch.from_numpy(pix).cuda(), torch.from_numpy(gt_jp).cuda(), torch.from_numpy(depth).cuda()
    eng = E.Engine(max_frames=n, n_hyps=H)
    fn = A.softam_loss if variant == "softam" else A.dsac_expected_loss
    loss = fn(eng, pred, dpix, dgt, cell_depth=dd)
    loss.sum().backward()
    ref = E.Engine(max_frames=n, n_hyps=H)
    ref.set_cell_depth_device(n, dd.data_ptr())
    s = torch.cuda.current_stream().cuda_stream
    q = torch.empty((n, E.N, 3), dtype=torch.int16, device="cuda")
    ref.coords_from_prediction_device(n, pred.detach().data_ptr(), q.data_ptr(), s)
    g = torch.ones(n, dtype=torch.float64, device="cuda")
    got = torch.empty((n, E.N, 3), dtype=torch.float32, device="cuda")
    if variant == "softam":
        ref.forward_device(n, q.data_ptr(), dpix.data_ptr(), 0, dgt.data_ptr(), 0, s)
        ref.backward_device(n, g.data_ptr(), None, got.data_ptr(), 0.1, s)
    else:
        el = torch.empty(n, dtype=torch.float64, device="cuda")
        ref.forward_dsac_device(n, q.data_ptr(), dpix.data_ptr(), 0, dgt.data_ptr(), True, 0, s, expected_loss=el.data_ptr())
        ref.backward_dsac_device(n, g.data_ptr(), got.data_ptr(), 0.1, s)
    torch.cuda.synchronize()
    assert torch.equal(pred.grad, got)
    assert pred.grad.abs().max() > 0
    eng.close()
    ref.close()


def test_misuse(engine_mod):
    from dsac_b200 import autograd as A
    E = engine_mod
    n = 2
    coords, pix, depth, _, gt_jp = R.synth(n, seed=71)
    eng = E.Engine(max_frames=n, n_hyps=32, n_streams=1)
    dd = torch.from_numpy(depth).cuda()
    with pytest.raises(Exception):
        eng.set_cell_depth_device(n + 1, dd.data_ptr())       # n > max_frames
    eng.set_cell_depth_device(1, dd.data_ptr())
    with pytest.raises(Exception):
        eng.forward(coords, pix, gt_jp)                       # 2 frames, the setting has 1
    eng.set_cell_depth_device(n, dd.data_ptr())
    eng.forward(coords, pix, gt_jp)
    eng.set_cell_depth_device(n, dd.data_ptr())
    with pytest.raises(Exception):
        eng.backward(coords, pix, gt_jp)                      # the setting changed after the pass
    pred = torch.from_numpy(coords.astype(np.float32) / 1000).cuda().requires_grad_()
    pix_t, gt_t = torch.from_numpy(pix).cuda(), torch.from_numpy(gt_jp).cuda()
    pose = A.softam_pose(eng, pred, pix_t, cell_depth=dd)
    pose.sum().backward()                                     # the seeded pose backward of an RGB-D pass
    assert torch.isfinite(pred.grad).all()
    loss = A.softam_loss(eng, pred, pix_t, gt_t, cell_depth=dd)
    eng.set_cell_depth_device(n, dd.data_ptr())               # the setting changed after the pass
    with pytest.raises(Exception):
        loss.sum().backward()
    with pytest.raises(ValueError):
        A.softam_pose(eng, pred, pix_t, cell_depth=dd[:1])
    eng.close()
