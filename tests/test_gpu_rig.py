"""Multi-camera rigs (dsac_forward_rig_device) on the GPU: C = 1 with a zero extrinsic is the ordinary pass bit for bit;
every frame samples as in an ordinary pass; a pool slot's score is the sum of the scores an ordinary pass gives its
composed poses; rigs are independent of the batch around them; a rig resolves a camera's two-cluster ambiguity; the
refusals, the pass kind and bad extrinsics."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

pytestmark = pytest.mark.gpu
N = 1600
BAD_RIG = 256


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _rig(eng, coords, pix, ext, C, gt_rig=None, frame0=0, fields=None):
    """dsac_forward_rig_device on host arrays; returns host copies of every output."""
    n = len(coords)
    R, P, H = n // C, C * eng.cfg.n_hyps, eng.cfg.n_hyps
    keep = [_dev(coords, np.int16), _dev(pix, np.int32), _dev(ext, np.float64)]
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
    eng.forward_rig_device(n, C, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), 0,
                           gt.data_ptr() if gt is not None else None, frame0, **{k: v.data_ptr() for k, v in out.items()})
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _ordinary(eng, coords, pix, gt_jp=None, frame0=0):
    n = len(coords)
    dc, dp = _dev(coords, np.int16), _dev(pix, np.int32)
    dg = _dev(gt_jp, np.float64) if gt_jp is not None else None
    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr() if dg is not None else None, frame0)
    res = eng.fetch(n)
    torch.cuda.synchronize()
    return res


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _cams(n):
    cams = np.tile([[525.0, 320.0, 240.0]], (n, 1))
    cams[1::2] = [580.0, 310.5, 250.25]
    return cams


def _setup(eng, n, mode, keep):
    if mode == "guided":
        lg = _dev(np.random.default_rng(3).normal(size=(n, N)), np.float32)
        eng.set_sampling_logits_device(n, lg.data_ptr())
        keep.append(lg)
    if mode == "cams":
        eng.set_cameras(_cams(n))
    torch.cuda.synchronize()


def _ring(C, seed=0):
    """cam_from_rig of a ring of C cameras: camera c turned by c * 360 / C degrees about y, 80 mm off the rig centre."""
    rng = np.random.default_rng(seed)
    ext = np.zeros((C, 6))
    for c in range(C):
        R = Rotation.from_euler("xyz", [rng.normal(scale=0.03), 2 * np.pi * c / C, rng.normal(scale=0.03)])
        ext[c, :3] = R.as_rotvec()
        ext[c, 3:] = [80.0 * np.sin(2 * np.pi * c / C), rng.normal(scale=5.0), 80.0 * np.cos(2 * np.pi * c / C)]
    return ext


def _compose(ext, pose):
    """The camera pose (cv) of rig pose `pose` through cam_from_rig `ext`."""
    Rc, R = Rotation.from_rotvec(ext[:3]), Rotation.from_rotvec(pose[:3])
    return np.concatenate([(Rc * R).as_rotvec(), Rc.apply(pose[3:]) + ext[3:]])


def _jp(pose):
    """The jp 12-vector (R row-major, t) of a cv pose, as the evaluation reads gt_jp (jp::cv2our)."""
    R = Rotation.from_rotvec(pose[:3]).as_matrix().copy()
    R[1:] = -R[1:]
    return np.concatenate([R.ravel(), [pose[3], -pose[4], -pose[5]]])


@pytest.mark.parametrize("mode", ["uniform", "guided", "cams"])
def test_one_camera_zero_extrinsic_is_the_ordinary_pass(engine_mod, mode):
    E = engine_mod
    n, H = 6, 128
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=2)
    assert np.allclose(np.stack([_jp(p) for p in gt_cv]), gt_jp, atol=1e-9)
    keep = []
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    _setup(eng, n, mode, keep)
    ref = _ordinary(eng, coords, pix, gt_jp, frame0=5)
    rig = _rig(eng, coords, pix, np.zeros((n, 6)), 1, gt_jp, frame0=5)
    eng.close()
    assert np.array_equal(_bits(rig["hyp_pose"]), _bits(ref.hyp_pose))
    assert np.array_equal(_bits(rig["rig_hyp"]), _bits(ref.hyp_pose))
    for k in ("scores", "sf", "entropy", "avg_pose", "ref_pose", "inlier_map", "loss", "rot_err", "t_err", "correct", "status"):
        assert np.array_equal(_bits(rig[k]), _bits(getattr(ref, k).astype(rig[k].dtype))), (mode, k)
    assert np.array_equal(rig["steps_done"], ref.ref_steps_done)
    assert rig["correct"].sum() > 0


@pytest.mark.parametrize("C,mode", [(2, "uniform"), (4, "guided"), (3, "cams")])
def test_frames_sample_as_in_the_ordinary_pass(engine_mod, C, mode):
    E = engine_mod
    n, H = 4 * C, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=4)
    keep = []
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=4)
    _setup(eng, n, mode, keep)
    ext = np.tile(_ring(C), (n // C, 1))
    rig = _rig(eng, coords, pix, ext, C, frame0=2)
    ref = _ordinary(eng, coords, pix, frame0=2)
    eng.close()
    assert np.array_equal(_bits(rig["hyp_pose"]), _bits(ref.hyp_pose))
    # the lift composed with the extrinsic returns each camera's hypothesis
    R = n // C
    for r in range(R):
        for j in range(0, C * H, 7):
            c, h = divmod(j, H)
            back = _compose(ext[r * C + c], rig["rig_hyp"][r, j])
            hp = ref.hyp_pose[r * C + c, h]
            assert np.allclose(back[3:], hp[3:], atol=1e-7)
            assert (Rotation.from_rotvec(back[:3]) * Rotation.from_rotvec(hp[:3]).inv()).magnitude() < 1e-9
    assert np.isfinite(rig["ref_pose"]).all()


def test_pool_score_is_the_sum_of_camera_scores(engine_mod):
    """The reference is an ordinary engine whose n_hyps = C H slots are all pose priors: the rig pool composed into each
    camera.  The rig builds each composed pose's fp32 rows from its fp64 rotation matrix, the priors from numpy's rvec of
    it through rodrigues: the rows may differ in the last float bit, so the scores agree to 1e-5 relative, not bitwise."""
    E = engine_mod
    C, H, R = 2, 8, 3
    n = R * C
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    ext = np.tile(_ring(C, seed=4), (R, 1))
    eng = E.Engine(max_frames=n, n_hyps=H)
    rig = _rig(eng, coords, pix, ext, C)
    eng.close()
    pri = np.empty((n, C * H, 6))
    for r in range(R):
        for c in range(C):
            for j in range(C * H):
                pri[r * C + c, j] = _compose(ext[r * C + c], rig["rig_hyp"][r, j])
    ref_eng = E.Engine(max_frames=n, n_hyps=C * H)
    p = _dev(pri, np.float64)
    ref_eng.set_pose_priors_device(n, C * H, p.data_ptr())
    ref = ref_eng.forward(coords, pix)
    ref_eng.close()
    want = np.zeros((R, C * H))
    for r in range(R):
        want[r] = ref.scores[r * C]
        for c in range(1, C):
            want[r] = want[r] + ref.scores[r * C + c]
    assert np.allclose(rig["scores"], want, rtol=1e-5, atol=1e-6)
    sf = np.exp(want - want.max(1, keepdims=True))
    sf /= sf.sum(1, keepdims=True)
    assert np.allclose(rig["sf"], sf, rtol=1e-4, atol=1e-9)


@pytest.mark.parametrize("n,C", [(24, 4), (1024, 4)])
def test_rigs_do_not_depend_on_the_batch(engine_mod, n, C):
    """1024 frames take the sampler's two-lane path; each rig alone (frame0 at its first frame) gives the same bits."""
    E = engine_mod
    H = 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=2)
    R = n // C
    ext = np.concatenate([_ring(C, seed=r % 5) for r in range(R)])
    gt_rig = np.stack([_jp(gt_cv[r * C]) for r in range(R)])
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    eng.set_cameras(_cams(n))
    allr = _rig(eng, coords, pix, ext, C, gt_rig)
    for r in sorted({0, 1, R // 2, R - 1}):
        fr = slice(r * C, (r + 1) * C)
        eng.set_cameras(_cams(n)[fr])
        one = _rig(eng, coords[fr], pix[fr], ext[fr], C, gt_rig[r:r + 1], frame0=r * C)
        for k, v in one.items():
            whole = allr[k][fr] if k in ("hyp_pose", "inlier_map") else allr[k][r:r + 1]
            assert np.array_equal(_bits(v), _bits(whole)), (r, k)
    eng.close()


def _two_cluster_rig(E, C=4, seed=7):
    """One rig whose camera 0 sees 40 % cells of a wrong rig pose (1 m, 30 degrees away) and 30 % of the true one; the
    other cameras see the true pose in 60 % of their cells.  The rest are random scene points."""
    rng = np.random.default_rng(seed)
    _, pix, _, _ = E.synth_frames(C)
    ext = _ring(C, seed=1)
    true = np.concatenate([Rotation.from_euler("xyz", [0.1, -0.2, 0.05]).as_rotvec(), [300.0, -150.0, 2000.0]])
    wrong_R = Rotation.from_rotvec([0.0, np.radians(30.0), 0.0]) * Rotation.from_rotvec(true[:3])
    wrong = np.concatenate([wrong_R.as_rotvec(), true[3:] + [1000.0, 0.0, 0.0]])
    coords = np.empty((C, N, 3), np.int16)
    f, cx, cy = 525.0, 320.0, 240.0
    for c in range(C):
        u = pix[c, :, 0] + rng.normal(scale=0.3, size=N)
        v = pix[c, :, 1] + rng.normal(scale=0.3, size=N)
        d = rng.uniform(1500.0, 4000.0, size=N)
        Xc = np.stack([(u - cx) / f * d, (v - cy) / f * d, d], 1)
        kind = rng.uniform(size=N)
        src = np.where(kind < (0.4 if c == 0 else 0.0), 1, np.where(kind < (0.7 if c == 0 else 0.6), 0, 2))
        X = np.empty((N, 3))
        for which, pose in ((0, true), (1, wrong)):
            cam = _compose(ext[c], pose)
            Rm = Rotation.from_rotvec(cam[:3])
            m = src == which
            X[m] = Rm.inv().apply(Xc[m] - cam[3:])
        m = src == 2
        X[m] = rng.uniform(-4000.0, 4000.0, size=(m.sum(), 3))
        coords[c] = np.clip(np.round(X), -32767, 32767).astype(np.int16)
    return coords, pix, ext, true, wrong


def test_rig_resolves_a_two_cluster_camera(engine_mod):
    E = engine_mod
    C, H = 4, 128
    coords, pix, ext, true, wrong = _two_cluster_rig(E, C)
    eng = E.Engine(max_frames=C, n_hyps=H, n_streams=2)
    cam0 = _ordinary(eng, coords[:1], pix[:1], _jp(_compose(ext[0], true))[None])
    rig = _rig(eng, coords, pix, ext, C, _jp(true)[None])
    eng.close()
    assert cam0.correct[0] == 0
    assert rig["correct"][0] == 1, (rig["rot_err"], rig["t_err"])
    assert rig["steps_done"][0] == eng.cfg.ref_steps and not rig["status"][0] & BAD_RIG


def test_bad_extrinsic_spoils_its_rig_only(engine_mod):
    E = engine_mod
    C, R, H = 2, 3, 32
    n = C * R
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    ext = np.tile(_ring(C), (R, 1))
    gt_rig = np.stack([_jp(gt_cv[r * C]) for r in range(R)])
    eng = E.Engine(max_frames=n, n_hyps=H)
    good = _rig(eng, coords, pix, ext, C, gt_rig)
    ext[3, 4] = np.nan
    bad = _rig(eng, coords, pix, ext, C, gt_rig)
    eng.close()
    assert [bool(s & BAD_RIG) for s in bad["status"]] == [False, True, False]
    for k, v in bad.items():
        if k == "hyp_pose":
            assert np.array_equal(_bits(v), _bits(good[k]))
            continue
        rows = slice(2, 4) if k == "inlier_map" else slice(1, 2)
        keep = np.ones(len(v), bool)
        keep[rows] = False
        assert np.array_equal(_bits(v[keep]), _bits(good[k][keep])), k
        if k != "status":
            assert not np.any(v[rows]), k


def test_refusals_and_pass_kind(engine_mod):
    E = engine_mod
    C, n, H = 2, 4, 32
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    ext = np.tile(_ring(C), (n // C, 1))
    eng = E.Engine(max_frames=n, n_hyps=H)
    lg = _dev(np.random.default_rng(1).normal(size=(n, N)), np.float32)
    eng.set_sampling_logits_device(n, lg.data_ptr())
    _ordinary(eng, coords, pix, gt_jp)
    assert eng.last_pass(n) == "softam"
    dc, dp, de = _dev(coords, np.int16), _dev(pix, np.int32), _dev(ext, np.float64)

    def call(nf=n, nc=C, **kw):
        eng.forward_rig_device(nf, nc, dc.data_ptr(), dp.data_ptr(), de.data_ptr(), **kw)

    def refused(fn, text):
        with pytest.raises(RuntimeError, match="\\(-1\\)"):
            fn()
        assert text in E.load().dsac_last_error(eng.h).decode()
        assert eng.last_pass(n) == "softam"

    refused(lambda: call(nc=3), "not a multiple")
    refused(lambda: call(nc=0), "out of range")
    refused(lambda: call(nf=n, nc=E.MAX_RIG_CAMERAS + 1), "out of range")
    big = E.Engine(max_frames=n, n_hyps=512)
    with pytest.raises(RuntimeError, match="exceeds 1024"):
        big.forward_rig_device(n, 4, dc.data_ptr(), dp.data_ptr(), de.data_ptr())
    big.close()
    eng.set_score_hook(lambda dm, nn, hh, sc, st: 0)
    refused(lambda: call(), "score hook")
    eng.set_score_hook(None)
    depth = _dev(np.full((n, N), 2000.0), np.float32)
    eng.set_cell_depth_device(n, depth.data_ptr())
    refused(lambda: call(), "cell depth or pose priors")
    eng.set_cell_depth_device(n, 0)
    pri = _dev(np.tile(gt_cv[:, None], (1, 1, 1)), np.float64)
    eng.set_pose_priors_device(n, 1, pri.data_ptr())
    refused(lambda: call(), "cell depth or pose priors")
    eng.set_pose_priors_device(n, 1, 0)
    _ordinary(eng, coords, pix, gt_jp)
    eng.set_stages(E.STAGE_SAMPLE | E.STAGE_SCORE)
    refused(lambda: call(), "stage mask")
    eng.set_stages(E.STAGE_ALL)
    assert E.load().dsac_forward_rig_device(eng.h, n, C, 0, dc.data_ptr(), dp.data_ptr(), 0, de.data_ptr(), None, None, None) == -1
    assert "null output" in E.load().dsac_last_error(eng.h).decode()
    assert eng.last_pass(n) == "softam"
    res = eng.forward_submit(coords, pix, gt_jp)
    refused(lambda: call(), "has not been awaited")
    eng.forward_wait()
    assert res.ref_pose.shape == (n, 6)

    call()
    torch.cuda.synchronize()
    assert eng.last_pass(n) == "rig"
    buf = torch.zeros((n, H, 36), dtype=torch.float64, device="cuda")
    consumers = {
        "dsac_backward_device": lambda: eng.backward_device(n, d_dloss_dpred=buf.data_ptr()),
        "dsac_backward_pose_device": lambda: eng.backward_pose_device(n, buf.data_ptr(), d_dloss_dpred=buf.data_ptr()),
        "dsac_backward_dsac_device": lambda: eng.backward_dsac_device(n, buf.data_ptr(), buf.data_ptr()),
        "dsac_backward_dsac_pose_device": lambda: eng.backward_dsac_pose_device(n, buf.data_ptr(), d_dloss_dpred=buf.data_ptr()),
        "dsac_refined_jp6_device": lambda: eng.refined_jp6_device(n, buf.data_ptr()),
        "dsac_pose_uncertainty_device": lambda: eng.pose_uncertainty_device(n, cov_xi=buf.data_ptr()),
        "dsac_pose_modes_device": lambda: eng.pose_modes_device(n, 2, 0.1, 100.0, n_modes=buf.data_ptr()),
    }
    for who, fn in consumers.items():
        with pytest.raises(RuntimeError, match="must follow"):
            fn()
    # the draws are the ordinary ones: their log-probability stays valid
    logp = torch.zeros(n, dtype=torch.float64, device="cuda")
    eng.sampling_log_prob_device(n, logp.data_ptr())
    torch.cuda.synchronize()
    assert torch.isfinite(logp).all()
    eng.close()


def test_autograd_rig_pose(engine_mod):
    E = engine_mod
    from dsac_b200 import autograd as A
    C, n, H = 2, 4, 32
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    ext = np.tile(_ring(C), (n // C, 1))
    gt_rig = np.stack([_jp(gt_cv[r * C]) for r in range(n // C)])
    eng = E.Engine(max_frames=n, n_hyps=H)
    pred = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda()
    out = A.rig_pose(eng, pred, _dev(pix, np.int32), _dev(ext, np.float64), C, gt_jp=_dev(gt_rig, np.float64))
    torch.cuda.synchronize()
    ref = _rig(eng, coords, pix, ext, C, gt_rig)
    eng.close()
    for k, v in out.items():
        assert not v.requires_grad
        assert np.array_equal(_bits(v.cpu().numpy()), _bits(ref[k])), k


@pytest.mark.parametrize("C,mode", [(2, "uniform"), (3, "cams"), (4, "guided")])
def test_device_agrees_with_the_rig_oracle(engine_mod, C, mode):
    """The CPU restatement (tests/rig_oracle.py) from the device's own frame hypotheses: pool, scores and sf at
    test_gpu_forward.py's tolerances.  The soft-argmax pose is linear in sf, so it is held to the bound that sf's own
    deviation gives, sum_j |dsf_j| |pose_j| (a rig's softmax is about C times sharper, so this is looser than one camera's
    1e-3).  The refinement is checked on its own: the oracle refines from the device's soft-argmax pose, and the inlier maps
    must be identical and the refined pose within test_gpu_forward.py's tolerances, on rigs whose refinement tested no cell
    within 1e-4 px of the threshold.  From the same start the two refinements' poses differ by rounding only (their fp64
    sums run in different orders), which moves an error by orders of magnitude less than 1e-4 px; a cell closer to the
    threshold than that may be decided either way."""
    import rig_oracle as RO
    from oracle import oracle as O
    E = engine_mod
    H, R = 32, 4
    n = R * C
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=2)
    ext = np.concatenate([_ring(C, seed=r) for r in range(R)])
    gt_rig = np.stack([_jp(gt_cv[r * C]) for r in range(R)])
    keep = []
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    _setup(eng, n, mode, keep)
    dev = _rig(eng, coords, pix, ext, C, gt_rig)
    eng.close()
    intr = _cams(n) if mode == "cams" else np.tile([[525.0, 320.0, 240.0]], (n, 1))
    cfg = O.default_config(n_hyps=H)
    compared = 0
    for r in range(R):
        fr = slice(r * C, (r + 1) * C)
        o = RO.forward(cfg, coords[fr], pix[fr], intr[fr], ext[fr], dev["hyp_pose"][fr], gt_rig[r], start=dev["avg_pose"][r])
        assert np.abs(o["rig_hyp"][:, :3] - dev["rig_hyp"][r][:, :3]).max() <= 1e-9
        assert np.abs(o["rig_hyp"][:, 3:] - dev["rig_hyp"][r][:, 3:]).max() <= 1e-6
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


def test_rig_pose_takes_a_non_contiguous_prediction(engine_mod):
    E = engine_mod
    from dsac_b200 import autograd as A
    C, n, H = 2, 4, 32
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    ext = _dev(np.tile(_ring(C), (n // C, 1)), np.float64)
    pred = torch.from_numpy(coords.astype(np.float32) / 1000.0).cuda()
    strided = pred.permute(0, 2, 1).contiguous().permute(0, 2, 1)   # [n][N][3] with channels-first storage
    assert not strided.is_contiguous()
    eng = E.Engine(max_frames=n, n_hyps=H)
    a = A.rig_pose(eng, pred, _dev(pix, np.int32), ext, C)
    b = A.rig_pose(eng, strided, _dev(pix, np.int32), ext, C)
    torch.cuda.synchronize()
    eng.close()
    for k in a:
        assert torch.equal(a[k], b[k]), k
