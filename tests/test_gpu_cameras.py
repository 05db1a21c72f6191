"""Per-frame cameras (dsac_set_cameras): one batch may mix focal lengths and principal points.

The engine's scheduling is bit-transparent and sampler streams are keyed by the global frame, so the central property
needs no oracle: frame g of a mixed batch equals, bit for bit, frame g run alone (frame0 = g) on an engine created with
that frame's camera in dsac_config.  The oracle comparison guards against a per-frame path that is wrong in the same
way in both engines.

One thing the comparison has to respect, cameras or not: k1_solve takes one thread per flagged candidate from 128
(frame, stream) pairs on and four lanes per candidate below, and the two instantiations round a hypothesis pose
differently in its last bits (1e-11 mm).  So a batch is compared with single-frame engines that take the same
instantiation: fewer than 128 pairs in the batch, or DSAC_K1_SOLVE4=0 for both."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CAMS = [(525.0, 320.0, 240.0), (585.0, 324.5, 236.25), (1800.0, 511.5, 400.0)]
FWD = ("img_idx", "cand_idx", "n_candidates", "hyp_pose", "scores", "sf", "avg_pose", "ref_pose", "inlier_map", "loss",
       "status", "diffmaps")
BWD = ("dloss_dobj", "dloss_dref", "dref_dhyp", "score_grads", "dpnp")
DSAC_FWD = ("hyp_pose", "img_idx", "sf", "entropy", "ref_pose", "losses", "steps_done", "expected_loss", "hyp_idx",
            "rot_err", "t_err", "correct", "status")
DSAC_BWD = ("dloss_dobj", "path1", "path2", "score_grads", "n_selected", "n_refine_jobs")


def _mixed(E, n, T=1, cams=CAMS):
    """Frames 0..n-1, frame g synthesised for (and to be run with) camera g mod len(cams); frame0 = g throughout."""
    cam = np.array([cams[g % len(cams)] for g in range(n)], np.float64)
    parts = [E.synth_frames(1, frame0=g, n_streams=T, focal=cam[g, 0], cx=cam[g, 1], cy=cam[g, 2]) for g in range(n)]
    coords, pix, _, gt_jp = (np.concatenate([p[k] for p in parts]) for k in range(4))
    return coords, pix, gt_jp, cam


def _cfg(cam):
    return dict(focal=float(cam[0]), cx=float(cam[1]), cy=float(cam[2]))


def _same(got, g, want, names):
    """Frame g of the batch result `got` against the single-frame result `want`, bit for bit."""
    for k in names:
        a, b = getattr(got, k), getattr(want, k)
        if a is None and b is None:
            continue
        assert np.array_equal(a[g], b[0]), (k, g)


@pytest.mark.parametrize("nf,T,dm", [(12, 1, 1), (3, 1, 1), (12, 8, 1), (6, 16, 1), (12, 1, 0)])
def test_mixed_batch_equals_per_camera_engines(engine_mod, nf, T, dm):
    E = engine_mod
    H = 256
    coords, pix, gt_jp, cam = _mixed(E, nf, T)
    eng = E.Engine(max_frames=nf, n_hyps=H, n_streams=T, write_diffmaps=dm)
    eng.set_cameras(cam)
    res = eng.forward(coords, pix, gt_jp, want_diffmaps=bool(dm))
    eng.close()
    assert (res.status == 0).all()
    for g in range(nf):
        one = E.Engine(max_frames=1, n_hyps=H, n_streams=T, write_diffmaps=dm, **_cfg(cam[g]))
        _same(res, g, one.forward(coords[g:g + 1], pix[g:g + 1], gt_jp[g:g + 1], frame0=g, want_diffmaps=bool(dm)), FWD)
        one.close()


def test_mixed_batch_matches_oracle(engine_mod, oracle):
    """Tolerances of test_gpu_forward.py; the fp32 ones (diffmaps, refined translation) scale with the focal length."""
    E, O = engine_mod, oracle
    nf, H = 6, 64
    coords, pix, gt_jp, cam = _mixed(E, nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.set_cameras(cam)
    res = eng.forward(coords, pix, gt_jp, want_diffmaps=True)
    eng.close()
    for g in range(nf):
        s = max(1.0, cam[g, 0] / 525.0)
        cfg = O.default_config(seed=1305 + g, n_hyps=H, f=cam[g, 0], cx=cam[g, 1], cy=cam[g, 2])
        fw = O.forward(cfg, coords[g], pix[g], gt_jp[g, :9], gt_jp[g, 9:])
        assert np.array_equal(fw.img_idx, res.img_idx[g]) and np.array_equal(fw.cand_idx, res.cand_idx[g])
        assert fw.n_candidates == res.n_candidates[g]
        assert np.abs(fw.hyp_rvec - res.hyp_pose[g][:, :3]).max() <= 1e-9
        assert np.abs(fw.hyp_tvec - res.hyp_pose[g][:, 3:]).max() <= 1e-6
        assert np.abs(fw.diffmaps - res.diffmaps[g]).max() <= 2e-3 * s
        assert np.abs(fw.scores - res.scores[g]).max() <= 1e-5 * np.abs(fw.scores).max()
        assert np.abs(fw.avg - res.avg_pose[g]).max() <= 1e-3
        assert np.array_equal(fw.inlier_map, res.inlier_map[g])
        assert np.abs(fw.ref[:3] - res.ref_pose[g][:3]).max() <= 1e-6
        assert np.abs(fw.ref[3:] - res.ref_pose[g][3:]).max() <= 1e-3 * s
        assert abs(fw.loss - res.loss[g]) <= 1e-4


def test_uniform_cameras_equal_no_cameras(engine_mod):
    """n copies of the config's camera give what an engine that never set cameras gives, forward and both backward
    passes; set_cameras(None) after a mixed batch restores the config's camera."""
    E = engine_mod
    nf, H = 4, 64
    coords, pix, _, gt_jp = E.synth_frames(nf)
    same_cam = np.tile(np.array(CAMS[0]), (nf, 1))
    plain, eng = E.Engine(max_frames=nf, n_hyps=H), E.Engine(max_frames=nf, n_hyps=H)
    eng.set_cameras(same_cam)
    want, got = plain.forward(coords, pix, gt_jp, want_diffmaps=True), eng.forward(coords, pix, gt_jp, want_diffmaps=True)
    for k in FWD:
        assert np.array_equal(getattr(want, k), getattr(got, k)), k
    wb, gb = plain.backward(coords, pix, gt_jp, full=False), eng.backward(coords, pix, gt_jp, full=False)
    for k in ("dloss_dobj", "dloss_dref", "dref_dhyp", "score_grads"):
        assert np.array_equal(getattr(wb, k), getattr(gb, k)), k
    wd, gd = plain.forward_dsac(coords, pix, gt_jp), eng.forward_dsac(coords, pix, gt_jp)
    for k in DSAC_FWD:
        assert np.array_equal(getattr(wd, k), getattr(gd, k)), k
    wdb, gdb = plain.backward_dsac(nf), eng.backward_dsac(nf)
    for k in DSAC_BWD:
        assert np.array_equal(getattr(wdb, k), getattr(gdb, k)), k
    mcoords, mpix, mgt, mcam = _mixed(E, nf)
    eng.set_cameras(mcam)
    eng.forward(mcoords, mpix, mgt)
    eng.set_cameras(None)
    again = eng.forward(coords, pix, gt_jp, want_diffmaps=True)
    for k in FWD:
        assert np.array_equal(getattr(want, k), getattr(again, k)), k
    plain.close()
    eng.close()


@pytest.mark.parametrize("mode", ["split", "mono"])
def test_batch_splitting_keeps_the_frames_cameras(engine_mod, monkeypatch, mode):
    """800 frames: the two half-batch lanes of the split sampler; with the monolithic sampler, the tail split (whole
    waves / partial wave), whose second part starts at a non-zero frame offset."""
    E = engine_mod
    if mode == "mono":
        monkeypatch.setenv("DSAC_K1_MODE", "mono")
    monkeypatch.setenv("DSAC_K1_SOLVE4", "0")   # the single-frame engines solve with k1_solve too (module docstring)
    nf, H = 800, 64
    coords, pix, gt_jp, cam = _mixed(E, nf, cams=CAMS[1:])
    eng = E.Engine(max_frames=nf, n_hyps=H, write_diffmaps=0)
    eng.set_cameras(cam)
    res = eng.forward(coords, pix, gt_jp)
    eng.close()
    for g in (0, 1, 399, 400, 401, 799):
        one = E.Engine(max_frames=1, n_hyps=H, write_diffmaps=0, **_cfg(cam[g]))
        _same(res, g, one.forward(coords[g:g + 1], pix[g:g + 1], gt_jp[g:g + 1], frame0=g), FWD)
        one.close()


def _rel(a, b, floor=1e-300):
    return np.abs(a - b).max() / max(floor, np.abs(b).max())


@pytest.mark.parametrize("fix_q4", [0, 1])
def test_softam_backward_of_a_mixed_batch(engine_mod, oracle, fix_q4):
    E, O = engine_mod, oracle
    nf, H = 6, 32
    coords, pix, gt_jp, cam = _mixed(E, nf)
    eng = E.Engine(max_frames=nf, n_hyps=H, fix_q4=fix_q4)
    eng.set_cameras(cam)
    eng.forward(coords, pix, gt_jp)
    bw = eng.backward(coords, pix, gt_jp)
    eng.close()
    for g in range(nf):
        one = E.Engine(max_frames=1, n_hyps=H, fix_q4=fix_q4, **_cfg(cam[g]))
        one.forward(coords[g:g + 1], pix[g:g + 1], gt_jp[g:g + 1], frame0=g)
        _same(bw, g, one.backward(coords[g:g + 1], pix[g:g + 1], gt_jp[g:g + 1]), BWD)
        one.close()
    g = 2   # the 1800-pixel camera, against the oracle at the tolerances of test_gpu_backward.py
    cfg = O.default_config(seed=1305 + g, n_hyps=H, fix_q4=fix_q4, f=cam[g, 0], cx=cam[g, 1], cy=cam[g, 2])
    ofw = O.forward(cfg, coords[g], pix[g], gt_jp[g, :9], gt_jp[g, 9:])
    obw = O.backward(cfg, coords[g], pix[g], gt_jp[g, :9], gt_jp[g, 9:], ofw)
    assert _rel(bw.dloss_dref[g], obw.dloss_dref) <= 1e-9
    assert _rel(bw.dref_dhyp[g], obw.dref_dhyp, floor=1e-3) <= 1e-7
    assert _rel(bw.dpnp[g], obw.dpnp) <= 1e-7
    assert _rel(bw.dloss_dobj[g], obw.dloss_dobj, floor=1e-6) <= 1e-3
    assert np.abs(bw.dloss_dobj[g]).max() > 0


@pytest.mark.parametrize("random_draw", [True, False])
def test_dsac_variant_of_a_mixed_batch(engine_mod, random_draw):
    E = engine_mod
    nf, H = 4, 32
    coords, pix, gt_jp, cam = _mixed(E, nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.set_cameras(cam)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=random_draw, want_inlier_maps=True)
    bw = eng.backward_dsac(nf)
    eng.close()
    assert np.abs(bw.dloss_dobj).max() > 0
    for g in range(nf):
        one = E.Engine(max_frames=1, n_hyps=H, **_cfg(cam[g]))
        _same(fw, g, one.forward_dsac(coords[g:g + 1], pix[g:g + 1], gt_jp[g:g + 1], random_draw=random_draw, frame0=g,
                                      want_inlier_maps=True), DSAC_FWD + ("inlier_maps",))
        _same(bw, g, one.backward_dsac(1), DSAC_BWD)
        one.close()


class _PerFrameCNN:
    """ScoreCNN applied frame by frame, so that the library convolutions see the same shapes in a batch and in a
    single-frame engine; keeps a copy of the diffmaps the engine handed over."""

    def __init__(self):
        import torch
        from dsac_b200.score_cnn import ScoreCNN
        torch.backends.cudnn.deterministic = True
        self.cnn, self.seen = ScoreCNN(), None

    def forward(self, dm, n, H, sc, stream):
        import torch
        from dsac_b200.score_cnn import _DevPtr
        for f in range(n):
            self.cnn(dm + f * H * 1600 * 4, 1, H, sc + f * H * 8, stream)
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            self.seen = torch.as_tensor(_DevPtr(dm, (n, H, 1600), "<f4"), device="cuda").clone()
        return 0

    def backward(self, dm, sg, n, H, out, stream):
        for f in range(n):
            self.cnn.backward(dm + f * H * 1600 * 4, sg + f * H * 8, 1, H, out + f * H * 1600 * 8, stream)
        return 0


def test_score_seam_sees_the_per_frame_cameras(engine_mod):
    import torch
    E = engine_mod
    nf, H = 3, 16
    coords, pix, gt_jp, cam = _mixed(E, nf)
    hook = _PerFrameCNN()

    def run(eng, c, p, g, frame0):
        eng.set_score_hook(hook.forward)
        eng.set_score_backward_hook(hook.backward)
        fw = eng.forward(c, p, g, frame0=frame0, want_diffmaps=True)
        bw = eng.backward(c, p, g, full=False)
        torch.cuda.synchronize()
        seen = hook.seen.cpu().numpy()
        eng.close()
        return fw, bw, seen

    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.set_cameras(cam)
    fw, bw, seen = run(eng, coords, pix, gt_jp, 0)
    assert np.array_equal(seen, fw.diffmaps)
    for g in range(nf):
        ofw, obw, oseen = run(E.Engine(max_frames=1, n_hyps=H, **_cfg(cam[g])), coords[g:g + 1], pix[g:g + 1], gt_jp[g:g + 1], g)
        assert np.array_equal(seen[g], oseen[0])
        assert np.array_equal(fw.scores[g], ofw.scores[0])
        assert np.array_equal(bw.dloss_dobj[g], obw.dloss_dobj[0])
    assert np.abs(bw.dloss_dobj).max() > 0


def test_autograd_cameras_keyword(engine_mod):
    import torch
    from dsac_b200.autograd import dsac_expected_loss, dsac_hypotheses, softam_loss, softam_pose
    E = engine_mod
    nf, H = 3, 32
    coords, pix, gt_jp, cam = _mixed(E, nf)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    pred = coords.astype(np.float32) / np.float32(1000)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    ones = [E.Engine(max_frames=1, n_hyps=H, **_cfg(cam[g])) for g in range(nf)]

    def value_and_grad(fn, e, lo, hi, frame0, cameras):
        p = dev(pred[lo:hi]).requires_grad_(True)
        out = fn(e, p, dev(pix[lo:hi]), dev(gt_jp[lo:hi]), frame0, cameras)
        out.sum().backward()
        torch.cuda.synchronize()
        return out.detach().cpu().numpy(), p.grad.cpu().numpy()

    fns = [
        lambda e, p, px, gt, f0, c: softam_loss(e, p, px, gt, frame0=f0, cameras=c),
        lambda e, p, px, gt, f0, c: dsac_expected_loss(e, p, px, gt, frame0=f0, cameras=c),
        lambda e, p, px, gt, f0, c: softam_pose(e, p, px, frame0=f0, cameras=c),
        lambda e, p, px, gt, f0, c: dsac_hypotheses(e, p, px, frame0=f0, cameras=c)[1],
    ]
    for k, fn in enumerate(fns):
        out, grad = value_and_grad(fn, eng, 0, nf, 0, torch.from_numpy(cam))
        assert np.abs(grad).max() > 0
        for g in range(nf):
            o1, g1 = value_and_grad(fn, ones[g], g, g + 1, g, None)
            assert np.array_equal(out[g], o1[0]), (k, g)
            if k % 2 == 0:
                assert np.array_equal(grad[g], g1[0]), (k, g)
            else:
                # The DSAC variant's device backward is compared as test_gpu_training.py's hand-off test compares it.  Seeded
                # by the poses it also differs between a batch and a single frame in a few clamped entries (a sign at the
                # clamp, with or without cameras), so there only the share of equal entries is checked.
                if k == 1:
                    assert np.abs(grad[g] - g1[0]).max() <= 1e-5 * max(1e-12, np.abs(g1[0]).max()), (k, g)
                assert np.mean(grad[g] == g1[0]) > 0.99, (k, g)
    # the cameras belong to the pass: changing them before backward() is refused
    p = dev(pred).requires_grad_(True)
    loss = softam_loss(eng, p, dev(pix), dev(gt_jp), cameras=cam)
    eng.set_cameras(cam[::-1])
    with pytest.raises(RuntimeError, match="cameras were changed"):
        loss.sum().backward()
    for e in ones + [eng]:
        e.close()


def test_argument_errors_leave_the_engine_usable(engine_mod):
    E = engine_mod
    nf, H = 3, 32
    coords, pix, gt_jp, cam = _mixed(E, nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.set_cameras(cam)
    want = eng.forward(coords, pix, gt_jp)

    def bad(cams, match):
        with pytest.raises(RuntimeError, match=match):
            eng.set_cameras(cams)

    bad(np.tile(cam, (2, 1)), "out of range")                      # n > max_frames
    bad(np.zeros((0, 3)), "out of range")
    for i, v in ((0, 0.0), (1, -525.0), (2, np.nan), (1, np.inf)):
        c = cam.copy()
        c[i, 0] = v
        bad(c, "camera %d is invalid" % i)
    c = cam.copy()
    c[2, 1] = np.nan
    bad(c, "camera 2 is invalid")
    with pytest.raises(RuntimeError, match="differs from the 3 cameras"):
        eng.forward(coords[:2], pix[:2], gt_jp[:2])
    eng.forward_submit(coords, pix, gt_jp)
    bad(cam, "has not been awaited")
    eng.forward_wait()
    got = eng.forward(coords, pix, gt_jp)                          # every refused call left the cameras as they were
    for k in FWD[:-1]:
        assert np.array_equal(getattr(want, k), getattr(got, k)), k
    eng.backward(coords, pix, gt_jp, full=False)
    eng.set_cameras(cam)
    with pytest.raises(RuntimeError, match="cameras were changed"):
        eng.backward(coords, pix, gt_jp, full=False)
    eng.close()


def test_set_cameras_allocates_nothing_per_call(engine_mod):
    """The camera buffers are sized once for max_frames.  Free device memory is compared with ">=": an engine that an
    earlier test left to the garbage collector may be destroyed at any moment, which only ever adds free memory."""
    import gc
    import torch
    E = engine_mod
    gc.collect()
    nmax, H = 16, 32
    coords, pix, gt_jp, cam = _mixed(E, nmax)

    def passes(eng, calls):
        free = []
        for i in range(calls):
            n = 1 + (i * 7) % nmax
            eng.set_cameras(cam[:n] if i % 5 else None)
            m = n if i % 5 else nmax
            eng.forward(coords[:m], pix[:m], gt_jp[:m])
            torch.cuda.synchronize()
            free.append(torch.cuda.mem_get_info()[0])
        return free

    warm = E.Engine(max_frames=nmax, n_hyps=H)   # loads every kernel the passes below launch
    passes(warm, 6)
    warm.close()
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info()[0]
    eng = E.Engine(max_frames=nmax, n_hyps=H)
    free = passes(eng, 20)
    assert all(b >= a for a, b in zip(free, free[1:])), free
    eng.close()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] >= before
