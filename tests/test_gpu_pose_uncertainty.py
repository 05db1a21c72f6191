"""Pose uncertainty on the GPU (dsac_pose_uncertainty_device): for every refined pose of both pipelines the covariance,
sigma2 and n_fit equal the host build of ift_fit_covariance (tests/host_shim/unc_shim.cpp) over the cell set the
oracle's refinement replay records (tests/ift_oracle.py), at the forward's refined pose; the support equals a count of
the cells below thr2d.  Also per-frame cameras, RGB-D, guided sampling and aborted refinements, the scheduling
invariances, the refusals, and that the call changes no later backward.

Two limits, on purpose.  The pose the call's own recording replay ends with is not an output of the engine, so it is not
compared bit for bit with the forward's ref_pose: the covariance, which the engine evaluates at the replay's pose, is
compared at 1e-9 with the host build evaluated at ref_pose, which catches a replay that drifted but not one that differs
in the last bits.  And support is counted in k_score's fp32 arithmetic (the contract), so the count is bounded, not
matched cell by cell: besides cells within 1e-4 px of thr2d, a cell may count differently from fp64 where fp32 rounding,
restated in numpy, puts its error on the other side of thr2d (check_support)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600
FIELDS = ("cov_jp6", "cov_xi", "sigma2", "n_fit", "support", "ok")
CAMS = np.array([[525.0, 320.0, 240.0], [900.0, 300.5, 250.0], [2500.0, 330.0, 200.0]])


@pytest.fixture(scope="module")
def shim():
    so = os.path.join(tempfile.mkdtemp(prefix="unc_shim_"), "libunc_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "unc_shim.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f64(a):
    return np.ascontiguousarray(a, np.float64)


def pose_uncertainty_tensors(eng, n):
    from dsac_b200 import autograd as A
    return A.pose_uncertainty(eng, n)


def uncertainty(eng, n):
    """pose_uncertainty's tensors on the host, flattened to one entry per job."""
    import torch
    out = pose_uncertainty_tensors(eng, n)
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    jobs = res["ok"].size
    return {k: v.reshape(jobs, 6, 6) if k.startswith("cov") else v.reshape(jobs) for k, v in res.items()}


def host_covariance(shim, Y, e, pose, cam, rgbd):
    cxi, cjp, s2 = np.zeros(36), np.zeros(36), C.c_double(-1.0)
    ok = shim.shim_ift_fit_covariance(len(Y), _p(_f64(Y)), _p(_f64(e)), _p(_f64(pose)), C.c_double(cam[0]), C.c_double(cam[1]),
                                      C.c_double(cam[2]), int(rgbd), _p(cxi), _p(cjp), C.byref(s2))
    return bool(ok), cxi.reshape(6, 6), cjp.reshape(6, 6), s2.value


def _fma(a, b, c):
    # a b + c rounded once to float32: the product of two floats is exact in double, so only the sum rounds twice
    return (a.astype(np.float64) * b.astype(np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def support_errors(c3, p2, pose, cam):
    """(fp64 reprojection errors, k_score's fp32 arithmetic restated in numpy) of the 1600 cells at the cv pose."""
    f, cx, cy = cam
    R = Rotation.from_rotvec(pose[:3]).as_matrix()
    t = np.asarray(pose[3:], np.float64)
    Y = c3.astype(np.float64)
    X = Y @ R.T + t
    z = np.where(X[:, 2] != 0, X[:, 2], 1.0)
    e64 = np.minimum(np.hypot(p2[:, 0] - (f * X[:, 0] / z + cx), p2[:, 1] - (f * X[:, 1] / z + cy)), 100.0)
    rows = np.array([[f * R[0, 0], f * R[0, 1], f * R[0, 2], f * t[0]], [f * R[1, 0], f * R[1, 1], f * R[1, 2], f * t[1]],
                     [R[2, 0], R[2, 1], R[2, 2], t[2]]]).astype(np.float32)
    Xf, Yf, Zf = (c3[:, k].astype(np.float32) for k in range(3))
    pu = p2[:, 0].astype(np.float32) - np.float32(cx)
    pv = p2[:, 1].astype(np.float32) - np.float32(cy)
    proj = [_fma(r[0], Xf, _fma(r[1], Yf, _fma(r[2], Zf, r[3]))) for r in rows]
    zs = np.where(proj[2] != 0, proj[2], np.float32(1))
    du, dv = _fma(pu, zs, -proj[0]), _fma(pv, zs, -proj[1])
    A = _fma(du, du, dv * dv)
    q = _fma(A, zs * zs, np.float32(1e-30))
    e32 = np.minimum(A * (1.0 / np.sqrt(q.astype(np.float64))).astype(np.float32), np.float32(100))
    return e64, e32.astype(np.float64)


def check_support(sup, c3, p2, pose, cam, thr):
    """The engine's count may differ from the fp64 count only at cells within 1e-4 px of thr2d, in fp64 or in k_score's
    fp32 arithmetic, or whose fp32 error falls on the other side of thr2d than the fp64 one."""
    e64, e32 = support_errors(c3, p2, pose, cam)
    amb = (np.abs(e64 - thr) <= 1e-4) | (np.abs(e32 - thr) <= 1e-4) | ((e64 < thr) != (e32 < thr))
    sure = int(((e64 < thr) & ~amb).sum())
    assert sure <= sup <= sure + int(amb.sum()), (sup, sure, int(amb.sum()))


def check_job(shim, got, j, S, c3, e, pose, cam, rgbd, p2, thr):
    """Entry j of the engine's outputs against the host build over the cells S at the refined cv pose."""
    assert got["n_fit"][j] == len(S), (j, got["n_fit"][j], len(S))
    ok, cxi, cjp, s2 = host_covariance(shim, c3[S], e[S], pose, cam, rgbd) if len(S) else (False, 0, 0, 0.0)
    assert got["ok"][j] == int(ok), j
    if ok:
        for k, h in (("cov_xi", cxi), ("cov_jp6", cjp)):
            assert np.abs(got[k][j] - h).max() <= 1e-9 * np.abs(h).max(), (j, k, np.abs(got[k][j] - h).max() / np.abs(h).max())
        assert abs(got["sigma2"][j] - s2) <= 1e-9 * s2
        assert np.array_equal(got["cov_xi"][j], got["cov_xi"][j].T)
    else:
        assert not got["cov_xi"][j].any() and not got["cov_jp6"][j].any() and got["sigma2"][j] == 0
    check_support(got["support"][j], c3, p2, pose, cam, thr)
    return ok


def check_pose(oracle_pose, pose):
    """The oracle's replay reaches the engine's refined pose within the forward's parity tolerances (test_gpu_forward.py):
    the two LM implementations are not bit-identical for every hypothesis, and the covariance is compared at the engine's
    pose."""
    assert np.abs(oracle_pose[:3] - pose[:3]).max() <= 1e-6 and np.abs(oracle_pose[3:] - pose[3:]).max() <= 1e-3


def _pixels(pix, f):
    p = np.asarray(pix).reshape(-1, N, 2)
    return p[0] if len(p) == 1 else p[f]


def _e_rgb(p2):
    return np.concatenate([p2.astype(np.float64), np.zeros((N, 1))], 1)


def check_softam(O, I, shim, eng, fwd, got, coords, pix, cams=None):
    """Every frame of a soft-argmax pass: S and the pose from the oracle's replay from the engine's avg_pose."""
    n_ok = 0
    for f in range(len(coords)):
        cam = tuple(cams[f]) if cams is not None else (eng.cfg.focal, eng.cfg.cx, eng.cfg.cy)
        cfg = O.default_config(n_hyps=eng.cfg.n_hyps, f=cam[0], cx=cam[1], cy=cam[2])
        perm = O.refine_permutations(cfg.ref_steps)
        c3, p2 = coords[f].reshape(N, 3), _pixels(pix, f)
        pose, S, _ = I.refine_record(cfg, c3, p2, perm, fwd.n_perm_steps[f], fwd.avg_pose[f])
        check_pose(pose, fwd.ref_pose[f])
        n_ok += check_job(shim, got, f, S, c3.astype(np.float64), _e_rgb(p2), fwd.ref_pose[f], cam, False, p2, eng.cfg.thr2d)
    return n_ok


def check_dsac(O, I, shim, eng, fw, got, coords, pix, cams=None):
    """Every hypothesis of a DSAC-variant pass: S and the pose from the oracle's replay from the hypothesis' pose."""
    H = eng.cfg.n_hyps
    n_ok = 0
    for f in range(len(coords)):
        cam = tuple(cams[f]) if cams is not None else (eng.cfg.focal, eng.cfg.cx, eng.cfg.cy)
        cfg = O.default_config(n_hyps=H, f=cam[0], cx=cam[1], cy=cam[2])
        perm = O.refine_permutations(cfg.ref_steps)
        c3, p2 = coords[f].reshape(N, 3), _pixels(pix, f)
        for h in range(H):
            pose, S, _ = I.refine_record(cfg, c3, p2, perm, cfg.ref_steps, fw.hyp_pose[f, h])
            check_pose(pose, fw.ref_pose[f, h])
            n_ok += check_job(shim, got, f * H + h, S, c3.astype(np.float64), _e_rgb(p2), fw.ref_pose[f, h], cam, False, p2,
                              eng.cfg.thr2d)
    return n_ok


def _same(a, b):
    for k in FIELDS:
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("T,H", [(1, 64), (3, 64), (1, 256), (3, 256)])
def test_softam_matches_oracle_set_and_host(engine_mod, oracle, shim, T, H):
    import ift_oracle as I
    E = engine_mod
    nf = 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H, n_streams=T)
    fwd = eng.forward(coords, pix, gt_jp)
    got = uncertainty(eng, nf)
    assert check_softam(oracle, I, shim, eng, fwd, got, coords, pix) == nf
    _same(got, uncertainty(eng, nf))   # a repeated call gives the same bits


@pytest.mark.parametrize("T,H", [(1, 64), (3, 256)])
@pytest.mark.parametrize("random_draw", [0, 1])
def test_dsac_variant_matches_oracle_set_and_host(engine_mod, oracle, shim, T, H, random_draw):
    import ift_oracle as I
    E = engine_mod
    nf = 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H, n_streams=T)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=bool(random_draw))
    got = uncertainty(eng, nf)
    assert got["ok"].shape == (nf * H,)
    assert check_dsac(oracle, I, shim, eng, fw, got, coords, pix) >= nf * H // 4
    _same(got, uncertainty(eng, nf))


def test_per_frame_cameras_both_pipelines(engine_mod, oracle, shim):
    import ift_oracle as I
    import rgbd_oracle as R
    E = engine_mod
    nf, H = 3, 64
    coords, pix, _, _, gt_jp = R.synth(nf, seed=92, cams=CAMS)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.set_cameras(CAMS)
    fwd = eng.forward(coords, pix, gt_jp)
    assert check_softam(oracle, I, shim, eng, fwd, uncertainty(eng, nf), coords, pix, CAMS) >= 2
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    assert check_dsac(oracle, I, shim, eng, fw, uncertainty(eng, nf), coords, pix, CAMS) >= nf * H // 4


@pytest.mark.parametrize("cams", [False, True])
def test_rgbd_with_holes_and_a_frame_without_depth(engine_mod, oracle, shim, cams):
    """S and the pose from the RGB-D oracle's Kabsch refinement replay (tests/rgbd_record.py), independent of the engine's
    recording; e the eye points.  Both pipelines, depth holes, and a frame without depth (nothing sampled, n_fit 0)."""
    import torch
    import rgbd_oracle as R
    import rgbd_record as RR
    E, O = engine_mod, oracle
    nf, H = 3, 64
    cam_tab = CAMS if cams else None
    coords, pix, depth, _, gt_jp = R.synth(nf, seed=93, holes=0.15, cams=cam_tab)
    depth[2] = np.nan
    eng = E.Engine(max_frames=nf, n_hyps=H)
    if cams:
        eng.set_cameras(cam_tab)
    d = torch.from_numpy(np.ascontiguousarray(depth, np.float32)).cuda()
    eng.set_cell_depth_device(nf, d.data_ptr())
    torch.cuda.synchronize()

    def frame(f):
        cam = tuple(cam_tab[f]) if cams else (525.0, 320.0, 240.0)
        cfg = O.default_config(n_hyps=H, f=cam[0], cx=cam[1], cy=cam[2])
        c3, p2 = coords[f].reshape(N, 3), pix[f].reshape(N, 2)
        ey, _ = R.eye(p2, depth[f], *cam)
        return cam, cfg, O.refine_permutations(cfg.ref_steps), c3, p2, ey

    fwd = eng.forward(coords, pix, gt_jp)
    assert fwd.status[2] & E.ST_NO_DEPTH
    got = uncertainty(eng, nf)
    n_ok = 0
    for f in range(nf):
        cam, cfg, perm, c3, p2, ey = frame(f)
        pose, S, _ = RR.refine_record(cfg, c3, p2, ey, perm, fwd.n_perm_steps[f], fwd.avg_pose[f])
        check_pose(pose, fwd.ref_pose[f])
        n_ok += check_job(shim, got, f, S, c3.astype(np.float64), ey, fwd.ref_pose[f], cam, True, p2, eng.cfg.thr2d)
    assert n_ok == 2 and got["n_fit"][2] == 0 and got["ok"][2] == 0
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    g2 = uncertainty(eng, nf)
    n_ok = 0
    for f in range(nf):
        cam, cfg, perm, c3, p2, ey = frame(f)
        for h in range(H):
            pose, S, _ = RR.refine_record(cfg, c3, p2, ey, perm, cfg.ref_steps, fw.hyp_pose[f, h])
            check_pose(pose, fw.ref_pose[f, h])
            n_ok += check_job(shim, g2, f * H + h, S, c3.astype(np.float64), ey, fw.ref_pose[f, h], cam, True, p2, eng.cfg.thr2d)
    assert not g2["ok"].reshape(nf, H)[2].any() and not g2["n_fit"].reshape(nf, H)[2].any() and n_ok >= H // 2
    del d


def test_guided_sampling_with_a_bad_weights_frame(engine_mod, oracle, shim):
    import torch
    import ift_oracle as I
    E = engine_mod
    nf, H = 3, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    logits = np.random.default_rng(3).standard_normal((nf, N)).astype(np.float32)
    logits[1, 11] = np.nan
    eng = E.Engine(max_frames=nf, n_hyps=H)
    d = torch.from_numpy(logits).cuda()
    eng.set_sampling_logits_device(nf, d.data_ptr())
    torch.cuda.synchronize()
    fwd = eng.forward(coords, pix, gt_jp)
    assert fwd.status[1] & E.ST_BAD_WEIGHTS
    got = uncertainty(eng, nf)
    check_softam(oracle, I, shim, eng, fwd, got, coords, pix)
    assert got["ok"][0] == 1 and got["ok"][2] == 1
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    g2 = uncertainty(eng, nf)
    check_dsac(oracle, I, shim, eng, fw, g2, coords, pix)
    assert not g2["ok"].reshape(nf, H)[1].any() and not g2["n_fit"].reshape(nf, H)[1].any()   # empty hypotheses
    del d


def test_aborted_refinement(engine_mod, oracle, shim):
    """Frames with few inliers: refinements that stop early or accept no step."""
    import ift_oracle as I
    E = engine_mod
    parts = [E.synth_frames(2, rho=0.02), E.synth_frames(6, frame0=10, rho=0.05)]
    coords, pix, gt_jp = (np.concatenate([p[k] for p in parts]) for k in (0, 1, 3))
    nf, H = len(coords), 64
    eng = E.Engine(max_frames=nf, n_hyps=H, max_candidates=20000)
    fwd = eng.forward(coords, pix, gt_jp)
    assert (fwd.status & E.ST_REFINE_ABORTED).any()
    got = uncertainty(eng, nf)
    check_softam(oracle, I, shim, eng, fwd, got, coords, pix)
    aborted = (fwd.ref_steps_done == 0)
    assert (got["n_fit"][aborted] == 0).all() and (got["ok"][aborted] == 0).all()


def test_batch_split_and_repeat_are_bit_identical(engine_mod):
    E = engine_mod
    n, H = 1024, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    eng = E.Engine(max_frames=n, n_hyps=H)
    eng.forward(coords, pix, gt_jp, frame0=0)
    whole = uncertainty(eng, n)
    _same(whole, uncertainty(eng, n))
    assert whole["ok"].sum() > n // 2
    for k in range(4):
        s = slice(256 * k, 256 * (k + 1))
        eng.forward(coords[s], pix[s], gt_jp[s], frame0=256 * k)
        part = uncertainty(eng, 256)
        for name in FIELDS:
            assert np.array_equal(whole[name][s], part[name]), (k, name)


def test_refusals_leave_the_engine_usable(engine_mod):
    import torch
    E = engine_mod
    nf, H = 3, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    buf = torch.zeros(nf, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        eng.pose_uncertainty_device(nf, ok=buf.data_ptr())             # no forward
    eng.forward(coords, pix, gt_jp)
    assert eng.lib.dsac_pose_uncertainty_device(eng.h, nf, None, None) != 0   # d_out NULL
    ref = uncertainty(eng, nf)
    with pytest.raises(RuntimeError):
        eng.pose_uncertainty_device(nf - 1, ok=buf.data_ptr())         # a different n
    _same(ref, uncertainty(eng, nf))
    eng.set_cameras(np.tile([525.0, 320.0, 240.0], (nf, 1)))
    with pytest.raises(RuntimeError):
        eng.pose_uncertainty_device(nf, ok=buf.data_ptr())             # cameras changed since the pass
    eng.set_cameras(None)
    eng.forward(coords, pix, gt_jp)
    _same(ref, uncertainty(eng, nf))
    depth = torch.full((nf, N), 1000.0, dtype=torch.float32, device="cuda")
    eng.set_cell_depth_device(nf, depth.data_ptr())
    eng.set_cell_depth_device(nf, None)
    with pytest.raises(RuntimeError):
        eng.pose_uncertainty_device(nf, ok=buf.data_ptr())             # cell depth changed since the pass
    eng.forward(coords, pix, gt_jp)
    _same(ref, uncertainty(eng, nf))
    eng.forward_submit(coords, pix, gt_jp)
    with pytest.raises(RuntimeError):
        eng.pose_uncertainty_device(nf, ok=buf.data_ptr())             # a submitted pass is pending
    eng.forward_wait()
    _same(ref, uncertainty(eng, nf))


@pytest.mark.parametrize("H", [1, 64])
def test_refused_forward_keeps_the_pass_and_its_shapes(engine_mod, H):
    """A forward the engine refuses leaves the pass it holds, and pose_uncertainty sizes its outputs from that pass
    (dsac_last_pass), not from the last forward attempted.  H = 1: [n][1] after the DSAC variant, [n] after soft-argmax."""
    import torch
    E = engine_mod
    nf = 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf + 2)
    dc, dp = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (coords, pix))
    eng = E.Engine(max_frames=nf, n_hyps=H)
    with pytest.raises(RuntimeError):
        eng.last_pass(nf)                                               # no pass yet
    eng.forward_dsac(coords[:nf], pix[:nf], gt_jp[:nf], random_draw=True)
    assert eng.last_pass(nf) == "dsac"
    ref = uncertainty(eng, nf)
    assert ref["ok"].shape == (nf * H,)
    with pytest.raises(RuntimeError):
        eng.forward_device(nf + 2, dc.data_ptr(), dp.data_ptr(), 0, None, 0)   # n beyond max_frames: refused
    with pytest.raises(RuntimeError):
        eng.forward(coords, pix, gt_jp)                                  # the same through the host-buffer entry point
    assert eng.last_pass(nf) == "dsac"
    u = pose_uncertainty_tensors(eng, nf)
    assert tuple(u["cov_xi"].shape) == (nf, H, 6, 6) and tuple(u["ok"].shape) == (nf, H)
    torch.cuda.synchronize()
    _same(ref, {k: v.cpu().numpy().reshape((nf * H, 6, 6) if k.startswith("cov") else (nf * H,)) for k, v in u.items()})
    # the reverse: a soft-argmax pass, then a refused DSAC-variant forward
    eng.forward(coords[:nf], pix[:nf], gt_jp[:nf])
    ref = uncertainty(eng, nf)
    with pytest.raises(RuntimeError):
        eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    assert eng.last_pass(nf) == "softam"
    u = pose_uncertainty_tensors(eng, nf)
    assert tuple(u["cov_xi"].shape) == (nf, 6, 6) and tuple(u["ok"].shape) == (nf,)
    torch.cuda.synchronize()
    _same(ref, {k: v.cpu().numpy().reshape((nf, 6, 6) if k.startswith("cov") else (nf,)) for k, v in u.items()})
    with pytest.raises(RuntimeError):
        pose_uncertainty_tensors(eng, nf - 1)                                  # no pass over nf - 1 frames


@pytest.mark.parametrize("mode", ["central", "implicit"])
def test_call_on_another_stream_changes_no_backward(engine_mod, mode):
    """forward, pose uncertainty on a second stream, backward: the same bits as forward, backward."""
    import torch
    E = engine_mod
    nf, H = 3, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    dc, dp, dg = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (coords, pix, gt_jp))
    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.set_coord_derivatives(mode)
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    lg = torch.ones(nf, dtype=torch.float64, device="cuda")
    unc = {k: torch.zeros((nf * H, 36) if k.startswith("cov") else (nf * H,), dtype=torch.float64 if k in ("cov_jp6", "cov_xi", "sigma2")
                          else torch.int32, device="cuda") for k in FIELDS}
    ptrs = {k: v.data_ptr() for k, v in unc.items()}
    torch.cuda.synchronize()

    def softam(with_call):
        out = torch.zeros((nf, N, 3), dtype=torch.float64, device="cuda")
        eng.forward_device(nf, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 0, s0.cuda_stream)
        if with_call:
            eng.pose_uncertainty_device(nf, s1.cuda_stream, **ptrs)
        eng.backward_device(nf, lg.data_ptr(), out.data_ptr(), None, 0.0, s0.cuda_stream)
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def dsac(with_call):
        outs = {k: torch.zeros((nf, N, 3), dtype=torch.float64, device="cuda") for k in ("dloss_dobj", "path1", "path2")}
        eng.forward_dsac_device(nf, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), True, 0, s0.cuda_stream)
        if with_call:
            eng.pose_uncertainty_device(nf, s1.cuda_stream, **ptrs)
        eng.backward_dsac_device(nf, lg.data_ptr(), None, 0.0, s0.cuda_stream, **{k: v.data_ptr() for k, v in outs.items()})
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in outs.items()}

    a = softam(False)
    assert np.array_equal(a, softam(True))
    assert unc["ok"][:nf].sum().item() == nf
    b = dsac(False)
    c = dsac(True)
    for k in b:
        assert np.array_equal(b[k], c[k]), k
    assert unc["ok"].sum().item() > 0


def test_autograd_helper_shapes(engine_mod):
    import torch
    from dsac_b200 import autograd as A
    E = engine_mod
    nf, H = 2, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    pred = torch.from_numpy(coords.astype(np.float32) / np.float32(1000)).cuda().requires_grad_()
    pix_t = torch.from_numpy(np.ascontiguousarray(pix)).cuda()
    eng = E.Engine(max_frames=nf, n_hyps=H)
    pose = A.softam_pose(eng, pred, pix_t)
    u = A.pose_uncertainty(eng, nf)
    assert u["cov_jp6"].shape == (nf, 6, 6) and u["cov_xi"].shape == (nf, 6, 6) and u["sigma2"].shape == (nf,)
    assert u["ok"].dtype == torch.int32 and u["support"].shape == (nf,) and not u["cov_jp6"].requires_grad
    assert (u["ok"] == 1).all() and pose.requires_grad
    # the jp covariance is the xi one pushed through d jp6 / d xi: equal traces of the translation blocks (D t)
    assert torch.allclose(torch.diagonal(u["cov_jp6"], dim1=1, dim2=2)[:, 3:], torch.diagonal(u["cov_xi"], dim1=1, dim2=2)[:, 3:])
    sf, ref = A.dsac_hypotheses(eng, pred, pix_t)
    u = A.pose_uncertainty(eng, nf)
    assert u["cov_xi"].shape == (nf, H, 6, 6) and u["n_fit"].shape == (nf, H)
