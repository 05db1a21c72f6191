"""Pose modes on the GPU (dsac_pose_modes_device): after a DSAC-variant pass and after a soft-argmax pass over the same
inputs (the same hypothesis pool), the selection and merge equal the numpy restatement of tests/test_pose_modes_host.py
bit for bit on the engine's own pool; every mode's pose and steps_done equal the DSAC variant's ref_pose and steps_done
of its seed's slot, and its covariance the pose uncertainty entry f H + hyp of that pass.  Radii are chosen inside gaps of
the pool's pairwise distances, before and after refinement, so that no nearness decision rests on the last bits.  Also
every engine setting, two-cluster frames, the invariances and the refusals."""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import test_pose_modes_host as MH

pytestmark = pytest.mark.gpu
N = 1600
UNC = ("cov_xi", "sigma2", "n_fit", "support", "ok")
FIELDS = ("n_modes", "hyp", "pose", "score", "mass", "members", "steps_done") + UNC
CAMS = np.array([[525.0, 320.0, 240.0], [900.0, 300.5, 250.0], [2500.0, 330.0, 200.0]])


def modes(eng, n, M, rot, trans):
    import torch
    from dsac_b200 import autograd as A
    out = A.pose_modes(eng, n, M, rot, trans)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def uncertainty(eng, n):
    import torch
    from dsac_b200 import autograd as A
    out = A.pose_uncertainty(eng, n)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _same(a, b):
    for k in FIELDS:
        assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k


def _pairwise(poses):
    """All pairwise rotation angles and translation distances of cv poses [k][6] (numpy, both orders)."""
    R = MH.rotations(poses).reshape(-1, 3, 3)
    t = np.asarray(poses).reshape(-1, 6)[:, 3:]
    M = np.einsum("aij,bkj->abik", R, R)
    v = 0.5 * np.stack([M[..., 2, 1] - M[..., 1, 2], M[..., 0, 2] - M[..., 2, 0], M[..., 1, 0] - M[..., 0, 1]], -1)
    c = 0.5 * (M[..., 0, 0] + M[..., 1, 1] + M[..., 2, 2] - 1.0)
    th = np.arctan2(np.sqrt((v * v).sum(-1)), c)
    d = np.sqrt(((t[:, None, :] - t[None, :, :]) ** 2).sum(-1))
    return th.ravel(), d.ravel()


def _gap(values, target):
    """A radius near target at least 1e-6 relative from every value (the values' own rounding is far below that)."""
    v = np.sort(values[np.isfinite(values)])
    for k in range(2000):
        r = target * (1.0 + 0.01 * k) if k % 2 == 0 else target / (1.0 + 0.01 * k)
        i = np.searchsorted(v, r)
        lo = v[i - 1] if i > 0 else -np.inf
        hi = v[i] if i < len(v) else np.inf
        if r - lo >= 1e-6 * r and hi - r >= 1e-6 * r:
            return r
    raise AssertionError("no gap near %g" % target)


def radii(pool, fw, rot, trans):
    """rot_rad, trans_mm inside gaps of every frame's pairwise distances among its slots' hypothesis poses and among their
    refined poses (empty slots included: a superset of the decisions the call makes)."""
    ths, ds = [], []
    for f in range(len(pool.scores)):
        for poses in (pool.hyp_pose[f], fw.ref_pose[f]):
            th, d = _pairwise(poses)
            ths.append(th)
            ds.append(d)
    r, t = _gap(np.concatenate(ths), rot), _gap(np.concatenate(ds), trans)
    return r, t


def expected(pool, fw, prior_k, M, rot, trans):
    """The restatement on the engine's pool, with the refined seed poses of the DSAC variant."""
    out = []
    for f in range(len(pool.scores)):
        seeds, mass, members, _ = MH.select(pool.hyp_pose[f], pool.img_idx[f], pool.scores[f], pool.sf[f], pool.status[f],
                                            prior_k, M, rot, trans)
        alive, m2, mb2 = MH.merge(fw.ref_pose[f][seeds].reshape(-1, 6), mass, members, rot, trans)
        out.append(([seeds[a] for a in alive], m2, mb2, seeds, mass))
    return out


def check(got, pool, fw, unc, prior_k, M, rot, trans):
    """Selection bit for bit against the restatement; pose, steps_done and covariance against the DSAC variant."""
    H = pool.scores.shape[1]
    for f, (hyps, mass, members, _, _) in enumerate(expected(pool, fw, prior_k, M, rot, trans)):
        k = len(hyps)
        assert got["n_modes"][f] == k, f
        assert list(got["hyp"][f, :k]) == hyps and (got["hyp"][f, k:] == -1).all(), f
        assert np.array_equal(got["mass"][f, :k], np.array(mass)), f
        assert list(got["members"][f, :k]) == members, f
        assert np.array_equal(got["score"][f, :k], pool.scores[f][hyps], equal_nan=True), f
        assert np.array_equal(got["pose"][f, :k], fw.ref_pose[f][hyps]), f
        assert np.array_equal(got["steps_done"][f, :k], fw.steps_done[f][hyps]), f
        for name in UNC:
            u = unc[name].reshape((-1,) + unc[name].shape[2:])
            assert np.array_equal(got[name][f, :k], u[f * H + np.array(hyps, int)]), (f, name)
        for name in FIELDS[1:]:
            if name != "hyp":
                assert not got[name][f, k:].any(), (f, name)


class _Pool:
    def __init__(self, res):
        for k in ("hyp_pose", "img_idx", "scores", "sf", "status"):
            setattr(self, k, getattr(res, k))


def both_pipelines(eng, n, coords, pix, gt_jp, M, rot=0.15, trans=120.0, prior_k=0, min_modes=1):
    """A DSAC-variant pass, its pose uncertainty and modes; then a soft-argmax pass on the same inputs, whose modes must be
    the same bits.  Returns the DSAC pass's modes and pool."""
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    pool = _Pool(eng.fetch(n))
    unc = uncertainty(eng, n)
    r, t = radii(pool, fw, rot, trans)
    got = modes(eng, n, M, r, t)
    check(got, pool, fw, unc, prior_k, M, r, t)
    assert got["n_modes"].sum() >= min_modes
    eng.forward(coords, pix, gt_jp)
    p2 = _Pool(eng.fetch(n))
    for k in ("hyp_pose", "img_idx", "scores", "sf"):
        assert np.array_equal(getattr(pool, k), getattr(p2, k), equal_nan=True), k
    _same(got, modes(eng, n, M, r, t))
    return got, pool, fw, (r, t)


@pytest.mark.parametrize("M", [1, 4, 16])
@pytest.mark.parametrize("T,H", [(1, 64), (3, 64), (1, 256), (3, 256), (1, 1024), (3, 1024)])
def test_selection_refinement_and_covariance_match(engine_mod, T, H, M):
    E = engine_mod
    nf = 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, n_streams=T)
    eng = E.Engine(max_frames=nf, n_hyps=H, n_streams=T)
    got, _, _, _ = both_pipelines(eng, nf, coords, pix, gt_jp, M, min_modes=nf)
    assert (got["ok"][got["hyp"] >= 0] == 1).any()


def test_per_frame_cameras(engine_mod):
    import rgbd_oracle as R
    E = engine_mod
    nf, H = 3, 64
    coords, pix, _, _, gt_jp = R.synth(nf, seed=92, cams=CAMS)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.set_cameras(CAMS)
    both_pipelines(eng, nf, coords, pix, gt_jp, 4, min_modes=nf)


def test_rgbd_with_holes_and_a_frame_without_depth(engine_mod):
    import torch
    import rgbd_oracle as R
    E = engine_mod
    nf, H = 3, 64
    coords, pix, depth, _, gt_jp = R.synth(nf, seed=93, holes=0.15)
    depth[2] = np.nan
    eng = E.Engine(max_frames=nf, n_hyps=H)
    d = torch.from_numpy(np.ascontiguousarray(depth, np.float32)).cuda()
    eng.set_cell_depth_device(nf, d.data_ptr())
    torch.cuda.synchronize()
    got, pool, _, _ = both_pipelines(eng, nf, coords, pix, gt_jp, 4, min_modes=2)
    assert pool.status[2] & E.ST_NO_DEPTH and got["n_modes"][2] == 0 and got["n_modes"][:2].min() >= 1
    del d


def test_guided_sampling_with_a_bad_weights_frame(engine_mod):
    import torch
    E = engine_mod
    nf, H = 3, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    logits = np.random.default_rng(3).standard_normal((nf, N)).astype(np.float32)
    logits[1, 11] = np.nan
    eng = E.Engine(max_frames=nf, n_hyps=H)
    d = torch.from_numpy(logits).cuda()
    eng.set_sampling_logits_device(nf, d.data_ptr())
    torch.cuda.synchronize()
    got, pool, _, _ = both_pipelines(eng, nf, coords, pix, gt_jp, 4)
    assert pool.status[1] & E.ST_BAD_WEIGHTS and got["n_modes"][1] == 0 and got["n_modes"][0] >= 1
    del d


def test_pose_priors_and_a_bad_prior_frame(engine_mod):
    """Two priors per frame: the ground truth (a near-certain seed) and a pose 1 m off; frame 2's second prior is not
    finite, so that frame samples nothing and has no modes."""
    import torch
    E = engine_mod
    nf, H, k = 3, 64, 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    poses = np.stack([gt_cv, gt_cv + [0, 0, 0, 1000.0, 0, 0]], 1)
    poses[2, 1, 0] = np.nan
    eng = E.Engine(max_frames=nf, n_hyps=H)
    p = torch.from_numpy(np.ascontiguousarray(poses)).cuda()
    eng.set_pose_priors_device(nf, k, p.data_ptr())
    torch.cuda.synchronize()
    got, pool, _, _ = both_pipelines(eng, nf, coords, pix, gt_jp, 4, prior_k=k)
    assert pool.status[2] & E.ST_BAD_PRIOR and got["n_modes"][2] == 0
    assert (got["hyp"][:2] >= H - k).any()   # a prior slot is a seed
    del p


def test_exhausted_streams_leave_empty_slots_out(engine_mod):
    E = engine_mod
    parts = [E.synth_frames(2, rho=0.02), E.synth_frames(2, frame0=10)]
    coords, pix, gt_jp = (np.concatenate([p[k] for p in parts]) for k in (0, 1, 3))
    nf, H = len(coords), 64
    eng = E.Engine(max_frames=nf, n_hyps=H, max_candidates=20000)
    got, pool, _, _ = both_pipelines(eng, nf, coords, pix, gt_jp, 16)
    empty = pool.img_idx[:, :, 0] < 0
    assert empty.any() and (pool.status & E.ST_SAMPLER_EXHAUSTED).any()
    for f in range(nf):
        assert not empty[f][got["hyp"][f][got["hyp"][f] >= 0]].any()
        assert got["members"][f].sum() <= (~empty[f]).sum()


def test_score_hook_ranking(engine_mod):
    """A hook that scores by minus the inlier count: the ranking, and so the seeds, follow the hooked scores."""
    import torch
    E = engine_mod
    nf, H = 3, 64

    class W:
        def __init__(self, ptr, shape, typestr):
            self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}

    def hook(dm, n, h, sc, stream):
        with torch.cuda.stream(torch.cuda.ExternalStream(stream) if stream else torch.cuda.default_stream()):
            d = torch.as_tensor(W(dm, (n, h, N), "<f4"), device="cuda")
            s = torch.as_tensor(W(sc, (n, h), "<f8"), device="cuda")
            s.copy_(-(d < 10.0).sum(-1).to(torch.float64))
        return 0

    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H, write_diffmaps=1)
    eng.set_score_hook(hook)
    got, pool, _, _ = both_pipelines(eng, nf, coords, pix, gt_jp, 4)
    for f in range(nf):
        assert got["score"][f, 0] == pool.scores[f].max()
    eng.set_score_hook(None)


def test_two_lane_batch_split_and_repeat(engine_mod):
    """1024 frames (the two-lane forward); a split batch and a repeated call give the same bits."""
    E = engine_mod
    n, H, M = 1024, 64, 4
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    eng = E.Engine(max_frames=n, n_hyps=H)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    unc = uncertainty(eng, n)
    sub = slice(0, 8)   # the frames checked against the restatement
    sp = _Pool(eng.fetch(n))
    for k in ("hyp_pose", "img_idx", "scores", "sf", "status"):
        setattr(sp, k, getattr(sp, k)[sub])
    r, t = radii(sp, fw, 0.15, 120.0)
    whole = modes(eng, n, M, r, t)
    _same(whole, modes(eng, n, M, r, t))
    check({k: v[sub] for k, v in whole.items()}, sp, fw, unc, 0, M, r, t)
    eng.forward(coords, pix, gt_jp)
    soft = modes(eng, n, M, r, t)
    _same(whole, soft)
    for k in range(4):
        s = slice(256 * k, 256 * (k + 1))
        eng.forward(coords[s], pix[s], gt_jp[s], frame0=256 * k)
        part = modes(eng, 256, M, r, t)
        for name in FIELDS:
            assert np.array_equal(whole[name][s], part[name], equal_nan=True), (k, name)


def _two_cluster_frames(n, seed, noise=0.0):
    """Cells 40 % consistent with pose A, 30 % with pose B (30 degrees and 1 m from A), 30 % outliers; the consistent
    scene coordinates carry `noise` mm of Gaussian noise besides the rounding to mm."""
    from dsac_b200 import engine as E
    rng = np.random.default_rng(seed)
    _, pix, gt_cv, _ = E.synth_frames(n)
    coords = np.empty((n, N, 3), np.int16)
    A, B = [], []
    for f in range(n):
        a = np.concatenate([Rotation.random(random_state=seed + f).as_rotvec() * 0.3, rng.normal(scale=200, size=3)])
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        rb = Rotation.from_rotvec(np.radians(30) * axis) * Rotation.from_rotvec(a[:3])
        d = rng.normal(size=3)
        b = np.concatenate([rb.as_rotvec(), a[3:] + 1000.0 * d / np.linalg.norm(d)])
        p = pix[f].astype(np.float64)
        z = rng.uniform(2000, 5000, size=N)
        X = np.stack([(p[:, 0] - 320.0) / 525.0 * z, (p[:, 1] - 240.0) / 525.0 * z, z], 1)
        lab = rng.permutation(np.repeat([0, 1, 2], [640, 480, 480]))
        Y = rng.uniform(-3000, 3000, size=(N, 3))
        for k, q in ((0, a), (1, b)):
            Rm = Rotation.from_rotvec(q[:3]).as_matrix()
            Y[lab == k] = (X[lab == k] - q[3:]) @ Rm + rng.normal(scale=noise, size=((lab == k).sum(), 3))
        coords[f] = np.clip(np.rint(Y), -32767, 32767).astype(np.int16)
        A.append(a)
        B.append(b)
    return coords, pix, np.array(A), np.array(B)


def _close(p, q, deg, mm):
    return MH.angle(MH.rotations(p)[0], MH.rotations(q)[0]) <= np.radians(deg) and MH.dist(p[3:], q[3:]) <= mm


@pytest.mark.parametrize("pipeline", ["softam", "dsac"])
def test_two_clusters_give_two_modes(engine_mod, pipeline):
    E = engine_mod
    n, H = 4, 256
    coords, pix, A, B = _two_cluster_frames(n, 41)
    eng = E.Engine(max_frames=n, n_hyps=H)
    if pipeline == "dsac":
        eng.forward_dsac(coords, pix, None, random_draw=True)
    else:
        eng.forward(coords, pix)
    got = modes(eng, n, 4, np.radians(10), 100.0)
    for f in range(n):
        k = got["n_modes"][f]
        assert k >= 2, f
        assert _close(got["pose"][f, 0], A[f], 5, 50) and _close(got["pose"][f, 1], B[f], 5, 50), f
        for i in range(k):
            for j in range(i):
                assert not _close(got["pose"][f, i], got["pose"][f, j], 10, 100)
        assert got["mass"][f].sum() <= 1 + 1e-12 and got["mass"][f, 0] > got["mass"][f, 1] > 0
    # with 10 mm of noise and a small radius, minimal sets give many seeds that refine onto the same pose: they merge, and
    # their mass stays
    coords, pix, A, B = _two_cluster_frames(n, 41, noise=10.0)
    if pipeline == "dsac":
        eng.forward_dsac(coords, pix, None, random_draw=True)
    else:
        eng.forward(coords, pix)
    pool = _Pool(eng.fetch(n))
    small = modes(eng, n, 16, np.radians(0.5), 5.0)
    merged = 0
    for f in range(n):
        seeds, mass, _, _ = MH.select(pool.hyp_pose[f], pool.img_idx[f], pool.scores[f], pool.sf[f], pool.status[f], 0, 16,
                                      np.radians(0.5), 5.0)
        k = small["n_modes"][f]
        merged += len(seeds) - k
        assert abs(small["mass"][f, :k].sum() - sum(mass)) <= 1e-12
    assert merged > 0


@pytest.mark.parametrize("mode", ["central", "implicit"])
def test_call_on_another_stream_changes_no_later_result(engine_mod, mode):
    import torch
    E = engine_mod
    nf, H, M = 3, 64, 4
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    dc, dp, dg = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (coords, pix, gt_jp))
    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.set_coord_derivatives(mode)
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    lg = torch.ones(nf, dtype=torch.float64, device="cuda")
    out = {k: torch.zeros((nf, M, 36) if k == "cov_xi" else (nf, M, 6) if k == "pose" else (nf,) if k == "n_modes" else (nf, M),
                          dtype=torch.float64 if k in ("pose", "score", "mass", "cov_xi", "sigma2") else torch.int32, device="cuda")
           for k in FIELDS}
    ptrs = {k: v.data_ptr() for k, v in out.items()}
    torch.cuda.synchronize()

    def softam(with_call):
        g = torch.zeros((nf, N, 3), dtype=torch.float64, device="cuda")
        eng.forward_device(nf, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 0, s0.cuda_stream)
        if with_call:
            eng.pose_modes_device(nf, M, 0.15, 120.0, s1.cuda_stream, **ptrs)
        eng.backward_device(nf, lg.data_ptr(), g.data_ptr(), None, 0.0, s0.cuda_stream)
        torch.cuda.synchronize()
        return g.cpu().numpy(), uncertainty(eng, nf)

    def dsac(with_call):
        outs = {k: torch.zeros((nf, N, 3), dtype=torch.float64, device="cuda") for k in ("dloss_dobj", "path1", "path2")}
        eng.forward_dsac_device(nf, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), True, 0, s0.cuda_stream)
        if with_call:
            eng.pose_modes_device(nf, M, 0.15, 120.0, s1.cuda_stream, **ptrs)
        eng.backward_dsac_device(nf, lg.data_ptr(), None, 0.0, s0.cuda_stream, **{k: v.data_ptr() for k, v in outs.items()})
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in outs.items()}, uncertainty(eng, nf)

    for run in (softam, dsac):
        a, ua = run(False)
        b, ub = run(True)
        if isinstance(a, dict):
            for k in a:
                assert np.array_equal(a[k], b[k]), k
        else:
            assert np.array_equal(a, b)
        for k in ua:
            assert np.array_equal(ua[k], ub[k]), k
        assert out["n_modes"].sum().item() >= nf
        first = {k: v.cpu().numpy() for k, v in out.items()}
        eng.pose_modes_device(nf, M, 0.15, 120.0, s1.cuda_stream, **ptrs)   # a second call: the same bits
        torch.cuda.synchronize()
        for k in FIELDS:
            assert np.array_equal(first[k], out[k].cpu().numpy()), k


def test_refusals_leave_the_engine_usable(engine_mod):
    import torch
    E = engine_mod
    nf, H = 3, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    buf = torch.zeros(nf, dtype=torch.int32, device="cuda")

    def call(n=nf, M=4, rot=0.15, trans=120.0):
        eng.pose_modes_device(n, M, rot, trans, n_modes=buf.data_ptr())

    with pytest.raises(RuntimeError):
        call()                                                     # no forward
    eng.forward(coords, pix, gt_jp)
    ref = modes(eng, nf, 4, 0.15, 120.0)
    assert eng.lib.dsac_pose_modes_device(eng.h, nf, 4, 0.15, 120.0, None, None) != 0   # d_out NULL
    for bad in [dict(n=nf - 1), dict(M=0), dict(M=17), dict(rot=-1e-3), dict(rot=math.nan), dict(trans=math.inf),
                dict(trans=-1.0)]:
        with pytest.raises(RuntimeError):
            call(**bad)
    _same(ref, modes(eng, nf, 4, 0.15, 120.0))
    small = E.Engine(max_frames=nf, n_hyps=2)
    small.forward(coords, pix, gt_jp)
    with pytest.raises(RuntimeError):
        small.pose_modes_device(nf, 3, 0.15, 120.0, n_modes=buf.data_ptr())   # max_modes > n_hyps
    assert modes(small, nf, 2, 0.15, 120.0)["n_modes"].min() >= 1
    eng.set_cameras(np.tile([525.0, 320.0, 240.0], (nf, 1)))
    with pytest.raises(RuntimeError):
        call()                                                     # cameras changed since the pass
    eng.set_cameras(None)
    eng.forward(coords, pix, gt_jp)
    _same(ref, modes(eng, nf, 4, 0.15, 120.0))
    depth = torch.full((nf, N), 1000.0, dtype=torch.float32, device="cuda")
    eng.set_cell_depth_device(nf, depth.data_ptr())
    eng.set_cell_depth_device(nf, None)
    with pytest.raises(RuntimeError):
        call()                                                     # cell depth changed since the pass
    eng.forward(coords, pix, gt_jp)
    p = torch.from_numpy(np.ascontiguousarray(np.stack([gt_cv], 1))).cuda()
    eng.set_pose_priors_device(nf, 1, p.data_ptr())
    with pytest.raises(RuntimeError):
        call()                                                     # priors changed since the pass
    eng.set_pose_priors_device(nf, 0, None)
    eng.set_stages(E.STAGE_SAMPLE)
    eng.forward(coords, pix, gt_jp)
    with pytest.raises(RuntimeError):
        call()                                                     # the pass skipped scoring
    eng.set_stages(E.STAGE_ALL)
    eng.forward(coords, pix, gt_jp)
    _same(ref, modes(eng, nf, 4, 0.15, 120.0))
    eng.forward_submit(coords, pix, gt_jp)
    with pytest.raises(RuntimeError):
        call()                                                     # a submitted pass is pending
    eng.forward_wait()
    _same(ref, modes(eng, nf, 4, 0.15, 120.0))


def test_autograd_helper_shapes(engine_mod):
    import torch
    from dsac_b200 import autograd as A
    E = engine_mod
    nf, H, M = 2, 64, 5
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    pred = torch.from_numpy(coords.astype(np.float32) / np.float32(1000)).cuda().requires_grad_()
    pix_t = torch.from_numpy(np.ascontiguousarray(pix)).cuda()
    eng = E.Engine(max_frames=nf, n_hyps=H)
    for run in (lambda: A.softam_pose(eng, pred, pix_t), lambda: A.dsac_hypotheses(eng, pred, pix_t)):
        run()
        m = A.pose_modes(eng, nf, M, 0.15, 120.0)
        assert m["n_modes"].shape == (nf,) and m["n_modes"].dtype == torch.int32
        assert m["pose"].shape == (nf, M, 6) and m["cov_xi"].shape == (nf, M, 6, 6)
        for k in ("score", "mass", "sigma2"):
            assert m[k].shape == (nf, M) and m[k].dtype == torch.float64
        for k in ("hyp", "members", "steps_done", "n_fit", "support", "ok"):
            assert m[k].shape == (nf, M) and m[k].dtype == torch.int32
        assert not any(v.requires_grad for v in m.values())
        assert (m["n_modes"] >= 1).all() and (m["ok"][:, 0] == 1).all()
