"""Rig pose modes on the GPU (dsac_rig_pose_modes_device): with one camera and a zero extrinsic, the ordinary pass's pose
modes bit for bit in every setting; with two to eight cameras (pools of up to 1024 slots, per-camera intrinsics), the
selection and merge against the numpy restatement of tests/test_rig_pose_modes_host.py over the engine's own pool, each
seed's refinement against the CPU rig oracle started from the seed's lifted pose, and its covariance against the host
covariance over the oracle's last-step cells, at the rig tests' tolerances.  Also two-cluster rigs, spoiled rigs, rig
score hooks, batch invariance, side effects, refusals and a multi-hypothesis rig tracker."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import rig_grad_oracle as RG
import rig_oracle as RO
import rig_rgbd_oracle as RR
import rig_tracking_oracle as RT
import test_pose_modes_host as MH
from test_gpu_pose_modes import _pairwise
from test_gpu_rig import _bits, _compose
from test_gpu_rig_grad import Rig
from test_gpu_rig_limits import _engine, _intr, _rgbd_scene, _scene, _support_bracket, _truth
from test_gpu_rig_tracking import _ordinary, _priors, _rig, _rig_unc, _set_priors, _set_rig_priors
from test_rig_pose_modes_host import occupied_rig, select_rig

pytestmark = pytest.mark.gpu
N = 1600
BAD_PRIOR, BAD_RIG, NO_DEPTH = 128, 256, 64
UNC = ("cov_xi", "sigma2", "n_fit", "support", "ok")
FIELDS = ("n_modes", "hyp", "pose", "score", "mass", "members", "steps_done") + UNC


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def rig_modes(eng, n, C, M, rot, trans):
    from dsac_b200 import autograd as A
    out = A.rig_pose_modes(eng, n, C, M, rot, trans)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def modes(eng, n, M, rot, trans):
    from dsac_b200 import autograd as A
    out = A.pose_modes(eng, n, M, rot, trans)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def img_idx(eng, n):
    """The frames' img_idx [n][H][4] of the engine's last pass (device_view)."""
    H = eng.cfg.n_hyps
    v = eng.device_view()
    t = torch.empty((n, H, 4), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    src = torch.as_tensor(_Ptr(v.img_idx, (n, H, 4), "<i4"), device="cuda")
    t.copy_(src)
    torch.cuda.synchronize()
    return t.cpu().numpy()


class _Ptr:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}


def _same(a, b, rows=slice(None)):
    for k in FIELDS:
        assert np.array_equal(_bits(a[k][rows]), _bits(b[k][rows])), k


# ------------------------------------------------------------------------------------------------ one camera

@pytest.mark.parametrize("mode", ["uniform", "guided", "cams", "rgbd", "priors"])
def test_one_camera_is_pose_modes(engine_mod, mode):
    """C = 1 with a zero extrinsic: rig_pose_modes after the rig pass is pose_modes after the ordinary pass, in all twelve
    fields, bit for bit.  rgbd: rig cell depth against per-frame cell depth; priors: gated rig priors against per-frame
    priors; cams: per-frame cameras; guided: guided sampling."""
    E = engine_mod
    n, H, C = 4, 64, 1
    intr = _intr(n, 4, mode == "cams")
    if mode == "rgbd":
        coords, pix, depth, _, gt, _ = _rgbd_scene(1, n, intr, seed=11, holes=0.1)
    else:
        coords, pix, _, gt = _scene(E, 1, n, seed=12, intr=intr)
    eng, keep = _engine(E, n, H, "cams" if mode == "cams" else "guided" if mode == "guided" else "uniform", intr)
    ext = np.zeros((n, 6))
    if mode == "rgbd":
        d = _dev(depth, np.float32)
        keep.append(d)
        eng.set_cell_depth_device(n, d.data_ptr())
    if mode == "priors":
        poses, info = _priors(np.random.default_rng(5), _truth(gt), 2, True)
        keep += _set_priors(eng, n, poses, info)
    _ordinary(eng, coords, pix, gt, keep=keep)
    ref = {M: modes(eng, n, M, 0.15, 120.0) for M in (4, 16)}
    if mode == "rgbd":
        eng.set_cell_depth_device(n, None)
        eng.set_rig_cell_depth_device(n, C, d.data_ptr())
    if mode == "priors":
        eng.set_pose_priors_device(n, 0, None)
        keep += _set_rig_priors(eng, n, C, poses, info)
    _rig(eng, coords, pix, ext, C, gt, keep=keep)
    got = {M: rig_modes(eng, n, C, M, 0.15, 120.0) for M in (4, 16)}
    eng.close()
    for M in (4, 16):
        _same(got[M], ref[M])
        assert got[M]["n_modes"].min() >= 1 and (got[M]["ok"][:, 0] == 1).all()
    if mode == "priors":
        assert (got[4]["hyp"] >= H - 2).any()


# ------------------------------------------------------------------------------------------------ against the oracles

def _gap_ok(values, r, rel):
    v = values[np.isfinite(values)]
    return v.size == 0 or np.abs(v - r).min() >= rel * r


def _choose(pairs, refined, rel_pool=1e-6, rel_ref=1e-4):
    """The first (rot, trans) candidate inside gaps of the pool's pairwise distances (the walk) and of the oracle-refined
    seeds' (the merge, whose poses agree with the device's only to the oracle tolerance)."""
    for rot in (0.15, 0.17, 0.2, 0.12, 0.25, 0.1):
        for trans in (120.0, 140.0, 160.0, 100.0, 200.0, 90.0):
            if all(_gap_ok(th, rot, rel_pool) and _gap_ok(d, trans, rel_pool) for th, d in pairs):
                ref = refined(rot, trans)
                if all(_gap_ok(th, rot, rel_ref) and _gap_ok(d, trans, rel_ref) for th, d in ref):
                    return rot, trans
    raise AssertionError("no radii in the gaps")


def _oracle_seed(cfg, coords, pix, intr, ext, hyp_pose, start, rgbd_eye):
    if rgbd_eye is not None:
        return RR.refine(cfg, coords, pix, intr, ext, rgbd_eye, start)
    return RO.forward(cfg, coords, pix, intr, ext, hyp_pose, start=start)


def _check_against_oracles(dev, idx, coords, pix, intr, ext, C, H, M, prior_k=0, eye=None):
    """Every rig's modes against the restatement, the rig oracle and the host covariance."""
    from oracle import oracle as O
    R = len(dev["pool"]["rig_hyp"])
    pool = dev["pool"]
    cfg = O.default_config(n_hyps=H)
    compared = 0
    for r in range(R):
        fr = slice(r * C, (r + 1) * C)
        ey = RR.eye(pix[fr], eye[fr], intr[fr]) if eye is not None else None
        sel = lambda rot, trans: select_rig(pool["rig_hyp"][r], idx[fr], pool["scores"][r], pool["sf"][r], pool["status"][r],
                                            prior_k, M, rot, trans)
        cache = {}

        def seed_runs(seeds):
            for s in seeds:
                if s not in cache:
                    cache[s] = _oracle_seed(cfg, coords[fr], pix[fr], intr[fr], ext[fr], dev["hyp_pose"][fr], pool["rig_hyp"][r][s], ey)
            return [cache[s] for s in seeds]

        def refined(rot, trans):
            runs = seed_runs(sel(rot, trans)[0])
            return [_pairwise(np.array([o["ref_pose"] for o in runs]))] if runs else []

        occ = occupied_rig(idx[fr], pool["status"][r], prior_k)
        rot, trans = _choose([_pairwise(pool["rig_hyp"][r][occ])], refined)
        got = rig_modes(dev["eng"], len(coords), C, M, rot, trans)
        seeds, mass, members, _ = sel(rot, trans)
        runs = seed_runs(seeds)
        alive, m2, mb2 = MH.merge(np.array([o["ref_pose"] for o in runs]).reshape(-1, 6), mass, members, rot, trans)
        k = len(alive)
        assert got["n_modes"][r] == k, r
        assert list(got["hyp"][r, :k]) == [seeds[a] for a in alive] and (got["hyp"][r, k:] == -1).all(), r
        assert np.array_equal(got["mass"][r, :k], np.array(m2)), r
        assert list(got["members"][r, :k]) == mb2, r
        assert np.array_equal(got["score"][r, :k], pool["scores"][r][[seeds[a] for a in alive]]), r
        for name in FIELDS[1:]:
            if name != "hyp":
                assert not got[name][r, k:].any(), (r, name)
        for i, a in enumerate(alive):
            o = runs[a]
            start = pool["rig_hyp"][r][seeds[a]]
            pose = got["pose"][r, i]
            if o["min_margin"] <= 1e-4:
                continue
            assert o["steps_done"] == got["steps_done"][r, i], (r, i)
            assert np.abs(o["ref_pose"][:3] - pose[:3]).max() <= 1e-6
            assert np.abs(o["ref_pose"][3:] - pose[3:]).max() <= 1e-3
            steps = int(got["steps_done"][r, i])
            sure, amb = _support_bracket(coords[fr], pix[fr], ext[fr], intr[fr], pose, cfg.thr2d)
            assert sure <= got["support"][r, i] <= sure + amb
            if steps == 0:
                assert got["n_fit"][r, i] == 0
                continue
            if ey is not None:
                cam, cell, margin, _ = RR.last_step_cells(cfg, coords[fr], pix[fr], intr[fr], ext[fr], ey, start, steps)
            else:
                cam, cell, margin, _ = RG.last_step_cells(cfg, coords[fr], pix[fr], intr[fr], ext[fr], dev["hyp_pose"][fr], start,
                                                          steps)
                cfg.ref_steps = O.default_config(n_hyps=H).ref_steps
            if margin <= 1e-4:
                continue
            compared += 1
            assert got["n_fit"][r, i] == len(cell)
            if ey is not None:
                ok, cxi, _, s2 = RR.cov(cam, coords[fr][cam, cell], ey[cam, cell], ext[fr], pose)
            else:
                ok, cxi, _, s2 = RT.rig_cov(cam, coords[fr][cam, cell], pix[fr][cam, cell], ext[fr], intr[fr], pose)
            assert got["ok"][r, i] == int(ok)
            if ok:
                assert np.abs(got["cov_xi"][r, i] - cxi).max() <= 1e-9 * np.abs(cxi).max()
                assert abs(got["sigma2"][r, i] - s2) <= 1e-9 * s2
    assert compared >= 1
    return got


ORACLE = [(2, 64, "uniform", 4), (4, 64, "cams", 4), (8, 128, "cams", 16), (2, 512, "uniform", 4)]


@pytest.mark.parametrize("C,H,mode,M", ORACLE)
def test_modes_match_the_oracles(engine_mod, C, H, mode, M):
    """Two, four and eight cameras, per-camera intrinsics, and full pools of 8 x 128 and 2 x 512 slots."""
    E = engine_mod
    R = 2
    n = R * C
    intr = _intr(n, C, mode == "cams")
    coords, pix, ext, gt = _scene(E, C, R, seed=60 + C, inliers=0.35, intr=intr)
    eng, keep = _engine(E, n, H, mode, intr)
    pool = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    idx = img_idx(eng, n)
    _check_against_oracles({"eng": eng, "pool": pool, "hyp_pose": pool["hyp_pose"]}, idx, coords, pix, intr, ext, C, H, M)
    eng.close()


def test_rgbd_modes_match_the_oracle(engine_mod):
    E = engine_mod
    C, R, H, M = 4, 2, 64, 4
    n = R * C
    intr = _intr(n, C, True)
    coords, pix, depth, ext, gt, _ = _rgbd_scene(C, R, intr, seed=70, inliers=0.35, holes=0.15)
    eng, keep = _engine(E, n, H, "cams", intr)
    d = _dev(depth, np.float32)
    eng.set_rig_cell_depth_device(n, C, d.data_ptr())
    keep.append(d)
    pool = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    idx = img_idx(eng, n)
    _check_against_oracles({"eng": eng, "pool": pool, "hyp_pose": pool["hyp_pose"]}, idx, coords, pix, intr, ext, C, H, M,
                           eye=depth)
    eng.close()


# ------------------------------------------------------------------------------------------------ two clusters

def _two_cluster_rigs(E, C, R, seed):
    """R rigs in which every camera sees 40 % of its cells from rig pose A, 30 % from rig pose B (30 degrees and 1 m from
    A) and 30 % random scene points."""
    rng = np.random.default_rng(seed)
    n = R * C
    _, pix, _, _ = E.synth_frames(n)
    coords = np.empty((n, N, 3), np.int16)
    ext = np.concatenate([RG.ring(C, seed=seed + r) for r in range(R)])
    A, B = np.empty((R, 6)), np.empty((R, 6))
    for r in range(R):
        A[r] = np.concatenate([Rotation.from_euler("xyz", rng.normal(scale=0.2, size=3)).as_rotvec(),
                               rng.normal(scale=200.0, size=3) + [0.0, 0.0, 1500.0]])
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        rb = Rotation.from_rotvec(np.radians(30.0) * axis) * Rotation.from_rotvec(A[r, :3])
        dvec = rng.normal(size=3)
        B[r] = np.concatenate([rb.as_rotvec(), A[r, 3:] + 1000.0 * dvec / np.linalg.norm(dvec)])
        for c in range(C):
            fr = r * C + c
            u = pix[fr, :, 0] + rng.normal(scale=0.3, size=N)
            v = pix[fr, :, 1] + rng.normal(scale=0.3, size=N)
            z = rng.uniform(1500.0, 4000.0, size=N)
            Xc = np.stack([(u - 320.0) / 525.0 * z, (v - 240.0) / 525.0 * z, z], 1)
            lab = rng.permutation(np.repeat([0, 1, 2], [640, 480, 480]))
            X = rng.uniform(-4000.0, 4000.0, size=(N, 3))
            for k, q in ((0, A[r]), (1, B[r])):
                cam = _compose(ext[fr], q)
                X[lab == k] = Rotation.from_rotvec(cam[:3]).inv().apply(Xc[lab == k] - cam[3:])
            coords[fr] = np.clip(np.round(X), -32767, 32767).astype(np.int16)
    return coords, pix, ext, A, B


def _close(p, q, deg, mm):
    return MH.angle(MH.rotations(p)[0], MH.rotations(q)[0]) <= np.radians(deg) and MH.dist(p[3:], q[3:]) <= mm


@pytest.mark.parametrize("C", [2, 4])
def test_two_clusters_in_every_camera_give_two_modes(engine_mod, C):
    E = engine_mod
    R, H = 3, 128
    n = R * C
    coords, pix, ext, A, B = _two_cluster_rigs(E, C, R, seed=80 + C)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    keep = []
    _rig(eng, coords, pix, ext, C, keep=keep)
    got = rig_modes(eng, n, C, 4, np.radians(10.0), 100.0)
    eng.close()
    for r in range(R):
        k = got["n_modes"][r]
        assert k >= 2, r
        assert _close(got["pose"][r, 0], A[r], 5, 50), r
        b = [i for i in range(1, k) if _close(got["pose"][r, i], B[r], 5, 50)]
        assert b, r
        assert got["mass"][r, 0] > got["mass"][r, b[0]] > 0
        assert got["mass"][r].sum() <= 1 + 1e-12
        assert (got["ok"][r, :k] == 1).all()


# ------------------------------------------------------------------------------------------------ spoiled rigs, holes

def test_spoiled_rigs_get_no_modes_and_leave_their_neighbours(engine_mod):
    """Rig 1: a non-finite extrinsic; rig 2: a non-finite rig prior.  Both get n_modes 0 and zero rows; rigs 0 and 3 are
    bit-identical to the same pass with every rig sound."""
    E = engine_mod
    C, R, H, M = 2, 4, 64, 4
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=90)
    rp, info = _priors(np.random.default_rng(1), _truth(gt), 1, True)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    keep = _set_rig_priors(eng, n, C, rp, info)
    _rig(eng, coords, pix, ext, C, gt, keep=keep)
    sound = rig_modes(eng, n, C, M, 0.15, 120.0)
    bad_ext, bad_rp = ext.copy(), rp.copy()
    bad_ext[3, 1] = np.nan
    bad_rp[2, 0, 5] = np.inf
    keep += _set_rig_priors(eng, n, C, bad_rp, info)
    pool = _rig(eng, coords, pix, bad_ext, C, gt, keep=keep)
    got = rig_modes(eng, n, C, M, 0.15, 120.0)
    eng.close()
    assert pool["status"][1] & BAD_RIG and pool["status"][2] & BAD_PRIOR
    for r in (1, 2):
        assert got["n_modes"][r] == 0 and (got["hyp"][r] == -1).all()
        for k in FIELDS[2:]:
            assert not got[k][r].any(), (r, k)
    for r in (0, 3):
        _same(got, sound, rows=r)
        assert got["n_modes"][r] >= 1


def test_rgbd_rig_with_a_camera_without_depth(engine_mod):
    E = engine_mod
    C, R, H = 3, 2, 64
    n = R * C
    intr = _intr(n, C, False)
    coords, pix, depth, ext, gt, true = _rgbd_scene(C, R, intr, seed=95, holes=0.1)
    depth[1] = np.nan   # rig 0's camera 1
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
    d = _dev(depth, np.float32)
    eng.set_rig_cell_depth_device(n, C, d.data_ptr())
    keep = [d]
    pool = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    got = rig_modes(eng, n, C, 4, 0.15, 120.0)
    eng.close()
    assert pool["status"][0] & NO_DEPTH and not pool["status"][0] & (BAD_RIG | BAD_PRIOR)
    for r in range(R):
        k = got["n_modes"][r]
        assert k >= 1 and got["ok"][r, 0] == 1, r
        assert _close(got["pose"][r, 0], true[r], 1, 20), r
    # the camera without depth contributes no seed: its slots hold zero poses (lifted) and sampled nothing
    assert not ((got["hyp"][0] >= H) & (got["hyp"][0] < 2 * H)).any()


# ------------------------------------------------------------------------------------------------ score hooks

def test_rig_score_hooks_rank_the_pool(engine_mod):
    """Rig score hooks that return minus the camera's inlier count: the ranking and score follow the hooked rig scores."""
    E = engine_mod
    C, R, H, M = 2, 2, 64, 4
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=100)
    eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)

    def fwd(dm, nn, P, sc, stream):
        with torch.cuda.stream(torch.cuda.ExternalStream(stream) if stream else torch.cuda.default_stream()):
            d = torch.as_tensor(_Ptr(dm, (nn, P, N), "<f4"), device="cuda")
            s = torch.as_tensor(_Ptr(sc, (nn, P), "<f8"), device="cuda")
            s.copy_(-(d < 10.0).sum(-1).to(torch.float64))
        return 0

    def bwd(dm, sg, nn, P, out, stream):
        return 0

    eng.set_rig_score_hooks(fwd, bwd)
    keep = []
    pool = _rig(eng, coords, pix, ext, C, gt, keep=keep)
    idx = img_idx(eng, n)
    got = rig_modes(eng, n, C, M, 0.15, 120.0)
    eng.set_rig_score_hooks(None, None)
    again = rig_modes(eng, n, C, M, 0.15, 120.0)   # the hooks are not read
    eng.close()
    _same(got, again)
    for r in range(R):
        fr = slice(r * C, (r + 1) * C)
        seeds, mass, members, owner = select_rig(pool["rig_hyp"][r], idx[fr], pool["scores"][r], pool["sf"][r],
                                                 pool["status"][r], 0, M, 0.15, 120.0)
        assert got["hyp"][r, 0] == seeds[0]
        assert got["score"][r, 0] == pool["scores"][r][owner >= 0].max() == pool["scores"][r][seeds[0]]
        assert pool["scores"][r][seeds[0]] <= 0   # minus an inlier count


# ------------------------------------------------------------------------------------------------ batch, lanes, side effects

def test_a_rigs_modes_do_not_depend_on_the_batch(engine_mod):
    """1024 frames (the sampler's two lanes) of 256 rigs of 4 cameras, M = 4: 1024 jobs.  Rigs 0, 100 and 255 give the same
    bits when every other rig of the batch is replaced, and a repeated call gives the same bits."""
    E = engine_mod
    C, H, M, n = 4, 64, 4, 1024
    R = n // C
    a = _scene(E, C, 8, seed=110)
    b = _scene(E, C, 8, seed=111)
    reps = R // 8
    coords, pix, ext, gt = (np.tile(x, (reps,) + (1,) * (x.ndim - 1)) for x in a)
    other = [np.tile(x, (reps,) + (1,) * (x.ndim - 1)) for x in b]
    eng = E.Engine(max_frames=n, n_hyps=H)
    keep = []
    _rig(eng, coords, pix, ext, C, gt, keep=keep, fields=("status",))
    whole = rig_modes(eng, n, C, M, 0.15, 120.0)
    _same(whole, rig_modes(eng, n, C, M, 0.15, 120.0))
    mixed = [x.copy() for x in other]
    for r in (0, 100, 255):
        fr = slice(r * C, (r + 1) * C)
        for dst, src in zip(mixed, (coords, pix, ext)):
            dst[fr] = src[fr]
        mixed[3][r] = gt[r]
    _rig(eng, *mixed[:3], C, mixed[3], keep=keep, fields=("status",))
    got = rig_modes(eng, n, C, M, 0.15, 120.0)
    eng.close()
    for r in (0, 100, 255):
        _same(got, whole, rows=r)
    assert (whole["n_modes"] >= 1).mean() > 0.9


def test_call_on_another_stream_changes_no_later_result(engine_mod):
    """A modes call on another stream between the pass and the rig backward and covariance changes neither's bits, nor the
    refined rig poses the engine holds."""
    E = engine_mod
    C, R, H, M = 3, 2, 64, 4
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=120)
    rp, info = _priors(np.random.default_rng(2), _truth(gt), 2, True)
    eng = E.Engine(max_frames=n, n_hyps=H)
    keep = _set_rig_priors(eng, n, C, rp, info)
    side = torch.cuda.Stream()
    out = {k: torch.zeros((R, M, 6, 6) if k == "cov_xi" else (R, M, 6) if k == "pose" else (R,) if k == "n_modes" else (R, M),
                          dtype=torch.float64 if k in ("pose", "score", "mass", "cov_xi", "sigma2") else torch.int32, device="cuda")
           for k in FIELDS}
    results = []
    for with_call in (False, True):
        rig = Rig(eng, coords, pix, ext, C, gt)
        jp = rig.jp6()
        if with_call:
            eng.rig_pose_modes_device(n, C, M, 0.15, 120.0, side.cuda_stream, **{k: v.data_ptr() for k, v in out.items()})
        bw = rig.backward()
        unc = _rig_unc(eng, n, C)
        results.append((jp, bw, unc, rig.jp6()))
    torch.cuda.synchronize()
    first = {k: v.cpu().numpy() for k, v in out.items()}
    eng.rig_pose_modes_device(n, C, M, 0.15, 120.0, side.cuda_stream, **{k: v.data_ptr() for k, v in out.items()})
    torch.cuda.synchronize()
    eng.close()
    (jp0, bw0, unc0, _), (jp1, bw1, unc1, jp1b) = results
    assert np.array_equal(_bits(jp0), _bits(jp1)) and np.array_equal(_bits(jp1), _bits(jp1b))
    for k in bw0:
        assert np.array_equal(_bits(bw0[k]), _bits(bw1[k])), k
    for k in unc0:
        assert np.array_equal(_bits(unc0[k]), _bits(unc1[k])), k
    assert first["n_modes"].min() >= 1
    _same(first, {k: v.cpu().numpy() for k, v in out.items()})


# ------------------------------------------------------------------------------------------------ refusals

def test_refusals_leave_the_engine_usable(engine_mod):
    E = engine_mod
    C, R, H = 2, 2, 32
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=130)
    eng = E.Engine(max_frames=n, n_hyps=H)
    buf = torch.zeros(R, dtype=torch.int32, device="cuda")
    keep = []

    def call(nf=n, nc=C, M=4, rot=0.15, trans=120.0):
        eng.rig_pose_modes_device(nf, nc, M, rot, trans, n_modes=buf.data_ptr())

    def refused(fn, text):
        with pytest.raises(RuntimeError, match=text):
            fn()

    refused(call, "must follow a dsac_forward_rig_device")              # no pass
    _ordinary(eng, coords, pix, keep=keep)
    refused(call, "must follow a dsac_forward_rig_device")              # an ordinary pass
    _rig(eng, coords, pix, ext, C, gt, keep=keep)
    ref = rig_modes(eng, n, C, 4, 0.15, 120.0)
    refused(lambda: eng.pose_modes_device(n, 4, 0.15, 120.0, n_modes=buf.data_ptr()), "must follow a forward pass")
    refused(lambda: call(nf=n - C), "must follow")
    refused(lambda: call(nc=1), "n_cameras 1 differs")
    refused(lambda: call(M=0), "max_modes 0 out of range")
    refused(lambda: call(M=17), "max_modes 17 out of range")
    refused(lambda: call(rot=-1e-3), "finite and >= 0")
    refused(lambda: call(rot=math.nan), "finite and >= 0")
    refused(lambda: call(trans=math.inf), "finite and >= 0")
    assert eng.lib.dsac_rig_pose_modes_device(eng.h, n, C, 4, 0.15, 120.0, None, None) != 0
    _same(ref, rig_modes(eng, n, C, 4, 0.15, 120.0))
    rp, _ = _priors(np.random.default_rng(0), _truth(gt), 1, False)
    keep += _set_rig_priors(eng, n, C, rp, None)
    refused(call, "rig pose priors were changed")
    eng.set_rig_pose_priors_device(n, C, 0, None)
    _rig(eng, coords, pix, ext, C, gt, keep=keep)
    depth = _dev(np.full((n, N), 2000.0), np.float32)
    eng.set_rig_cell_depth_device(n, C, depth.data_ptr())
    refused(call, "rig cell depth")
    eng.set_rig_cell_depth_device(n, C, None)
    _rig(eng, coords, pix, ext, C, gt, keep=keep)
    eng.set_cameras(np.tile([525.0, 320.0, 240.0], (n, 1)))
    refused(call, "cameras")
    eng.set_cameras(None)
    _rig(eng, coords, pix, ext, C, gt, keep=keep)
    _same(ref, rig_modes(eng, n, C, 4, 0.15, 120.0))
    small = E.Engine(max_frames=n, n_hyps=2)
    _rig(small, coords, pix, ext, C, gt, keep=keep)
    with pytest.raises(RuntimeError, match="max_modes 3 out of range"):
        small.rig_pose_modes_device(n, C, 3, 0.15, 120.0, n_modes=buf.data_ptr())
    assert rig_modes(small, n, C, 2, 0.15, 120.0)["n_modes"].min() >= 1
    small.close()
    eng.forward_submit(coords, pix, None)
    refused(call, "has not been awaited")
    eng.forward_wait()
    _rig(eng, coords, pix, ext, C, gt, keep=keep)
    _same(ref, rig_modes(eng, n, C, 4, 0.15, 120.0))
    eng.close()


# ------------------------------------------------------------------------------------------------ tracker, autograd

def test_multi_hypothesis_rig_tracker(engine_mod):
    """A rig whose cameras all see two clusters, moving 2 degrees and 60 mm per step: the tracker feeds every rig mode back
    as a rig prior with information inv(cov_xi + Q) (unused entries repeat mode 0).  The best mode stays on the true pose
    at every step."""
    from dsac_b200 import autograd as A
    E = engine_mod
    C, H, M = 4, 128, 4
    coords, pix, ext, true, wrong = _two_cluster_rigs(E, C, 1, seed=140)
    eng = E.Engine(max_frames=C, n_hyps=H, n_streams=2)
    Q = torch.tensor(np.diag([1e-3] * 3 + [100.0 ** 2] * 3), device="cuda")
    pix_t = torch.tensor(pix, dtype=torch.int32, device="cuda")
    ext_t = torch.tensor(ext, dtype=torch.float64, device="cuda")
    prior = None
    for step in range(5):
        Am = Rotation.from_rotvec([0.0, np.radians(2.0 * step), 0.0])
        b = np.array([60.0 * step, 0.0, 0.0])
        moved = np.clip(np.round(Am.apply(coords.reshape(-1, 3).astype(np.float64)) + b), -32767, 32767).astype(np.int16)
        Rt = Rotation.from_rotvec(true[0, :3]) * Am.inv()
        pose = np.concatenate([Rt.as_rotvec(), true[0, 3:] - Rt.apply(b)])
        pred = torch.tensor(moved.reshape(coords.shape).astype(np.float32) / 1000.0, device="cuda")
        out = A.rig_pose(eng, pred, pix_t, ext_t, C, frame0=100 * step, rig_priors=prior)
        m = A.rig_pose_modes(eng, C, C, M, np.radians(10.0), 100.0)
        torch.cuda.synchronize()
        assert not out["status"][0].item() & (BAD_PRIOR | BAD_RIG)
        k = int(m["n_modes"][0].item())
        assert k >= 2, step
        poses = m["pose"].cpu().numpy()[0]
        assert _close(poses[0], pose, 2, 30), (step, poses[0], pose)
        assert m["ok"][0, 0].item() == 1
        used = torch.arange(M, device="cuda") < k
        pp = torch.where(used[None, :, None], m["pose"], m["pose"][:, :1])
        cov = torch.where(used[None, :, None, None], m["cov_xi"], m["cov_xi"][:, :1])
        info = torch.linalg.inv(cov + Q)
        prior = (pp.contiguous(), info.contiguous(), 16.81)
    eng.close()


def test_autograd_helper_shapes(engine_mod):
    from dsac_b200 import autograd as A
    E = engine_mod
    C, R, H, M = 2, 3, 64, 5
    n = R * C
    coords, pix, ext, gt = _scene(E, C, R, seed=150)
    eng = E.Engine(max_frames=n, n_hyps=H)
    pred = torch.from_numpy(coords.astype(np.float32) / np.float32(1000)).cuda().requires_grad_()
    pix_t = torch.from_numpy(np.ascontiguousarray(pix)).cuda()
    ext_t = torch.from_numpy(ext).cuda()
    A.rig_softam_pose(eng, pred, pix_t, ext_t, C)
    m = A.rig_pose_modes(eng, n, C, M, 0.15, 120.0)
    torch.cuda.synchronize()
    assert m["n_modes"].shape == (R,) and m["n_modes"].dtype == torch.int32
    assert m["pose"].shape == (R, M, 6) and m["cov_xi"].shape == (R, M, 6, 6)
    for k in ("score", "mass", "sigma2", "pose", "cov_xi"):
        assert m[k].dtype == torch.float64
    for k in ("score", "mass", "sigma2"):
        assert m[k].shape == (R, M)
    for k in ("hyp", "members", "steps_done", "n_fit", "support", "ok"):
        assert m[k].shape == (R, M) and m[k].dtype == torch.int32
    assert not any(v.requires_grad for v in m.values())
    assert (m["n_modes"] >= 1).all() and (m["ok"][:, 0] == 1).all()
    eng.close()
