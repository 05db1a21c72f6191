"""Pose covariance of a refined pose (dsac_b200/csrc/ift.cuh's ift_fit_covariance, compiled for the host) against an
independent numpy fp64 computation -- Jacobians by central differences of the residuals, taken directly in the xi chart and
separately in the jp 6-vector -- its documented refusals, and its calibration: on synthetic fits with Gaussian noise of
known sigma the predicted covariance matches the spread of 2000 frozen-set solves."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import ift_oracle as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DFLIP = np.diag([1.0, -1.0, -1.0])


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


def covariance(shim, Y, e, R, t, cam, rgbd):
    """(ok, cov_xi [6][6], cov_jp6 [6][6], sigma2) of ift_fit_covariance at the cv pose (R, t)."""
    pose = _f64(np.concatenate([Rotation.from_matrix(R).as_rotvec(), t]))
    cxi, cjp, s2 = np.zeros(36), np.zeros(36), C.c_double(-1.0)
    ok = shim.shim_ift_fit_covariance(len(Y), _p(_f64(Y)), _p(_f64(e)), _p(pose), C.c_double(cam[0]), C.c_double(cam[1]),
                                      C.c_double(cam[2]), int(rgbd), _p(cxi), _p(cjp), C.byref(s2))
    return bool(ok), cxi.reshape(6, 6), cjp.reshape(6, 6), s2.value


def residuals(Y, e, R, t, cam, rgbd):
    f, cx, cy = cam
    X = Y @ R.T + t
    if rgbd:
        return (X - e).reshape(-1)
    return (np.stack([f * X[:, 0] / X[:, 2] + cx, f * X[:, 1] / X[:, 2] + cy], 1) - e[:, :2]).reshape(-1)


def _jacobian(fun, steps):
    """Five-point central differences of fun (R^6 -> R^k) at 0 with per-coordinate steps."""
    cols = []
    for a in range(6):
        d = np.zeros(6)
        d[a] = steps[a]
        cols.append((8 * (fun(d) - fun(-d)) - (fun(2 * d) - fun(-2 * d))) / (12 * steps[a]))
    return np.stack(cols, 1)


def numpy_covariances(Y, e, R, t, cam, rgbd):
    """(cov_xi, cov_jp6, sigma2): sigma2 (J^T J)^-1 with J by central differences in each chart."""
    steps = [1e-3] * 3 + [1.0] * 3
    J_xi = _jacobian(lambda d: residuals(Y, e, Rotation.from_rotvec(d[:3]).as_matrix() @ R, t + d[3:], cam, rgbd), steps)
    jp = np.concatenate([Rotation.from_matrix(DFLIP @ R).as_rotvec(), DFLIP @ t])

    def from_jp(d):
        v = jp + d
        return residuals(Y, e, DFLIP @ Rotation.from_rotvec(v[:3]).as_matrix(), DFLIP @ v[3:], cam, rgbd)

    J_jp = _jacobian(from_jp, steps)
    r = residuals(Y, e, R, t, cam, rgbd)
    s2 = r @ r / ((3 if rgbd else 2) * len(Y) - 6)
    return s2 * np.linalg.inv(J_xi.T @ J_xi), s2 * np.linalg.inv(J_jp.T @ J_jp), s2


def _scene(rng, m, R, t, cam, noise, rgbd):
    f, cx, cy = cam
    uv = np.stack([rng.uniform(20, 620, m), rng.uniform(20, 460, m)], 1)
    d = rng.uniform(800, 4000, m)
    Xc = np.stack([(uv[:, 0] - cx) * d / f, (uv[:, 1] - cy) * d / f, d], 1)
    Y = np.round((Xc - t) @ R)                 # int16-grid scene coordinates
    e = Xc + rng.normal(0, noise, Xc.shape) if rgbd else np.concatenate([np.round(uv + rng.normal(0, noise, uv.shape)), np.zeros((m, 1))], 1)
    return Y, e


def _pose(rng, near_pi):
    if near_pi:   # jp rotation within 1e-4 rad of pi
        ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
        R = DFLIP @ Rotation.from_rotvec((np.pi - rng.uniform(1e-5, 1e-4)) * ax).as_matrix()
    else:
        R = Rotation.from_rotvec(rng.uniform(-0.5, 0.5, 3)).as_matrix()
    return R, np.array([rng.uniform(-300, 300), rng.uniform(-300, 300), rng.uniform(-200, 200)])


CASES = [  # (f, cx, cy), near pi, rgbd
    ((525.0, 320.0, 240.0), True, False),
    ((525.0, 320.0, 240.0), False, False),
    ((300.0, 250.0, 300.0), True, False),
    ((2500.0, 410.5, 170.25), True, False),
    ((1200.0, 333.0, 211.5), False, False),
    ((900.0, 250.0, 300.0), True, True),
    ((525.0, 320.0, 240.0), False, True),
    ((2500.0, 410.5, 170.25), False, True),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_covariance_matches_numpy_central_differences(shim, case):
    cam, near_pi, rgbd = CASES[case]
    rng = np.random.default_rng(300 + case)
    R0, t0 = _pose(rng, near_pi)
    Y, e = _scene(rng, 100, R0, t0, cam, 3.0 if rgbd else 1.5, rgbd)
    R, t = I.frozen_fit(Y, e, R0, t0, cam, rgbd, iters=20)
    if near_pi:
        assert np.pi - np.linalg.norm(I.jp6(R, t)[:3]) < 3e-3
    ok, cxi, cjp, s2 = covariance(shim, Y, e, R, t, cam, rgbd)
    assert ok
    nxi, njp, ns2 = numpy_covariances(Y, e, R, t, cam, rgbd)
    assert abs(s2 - ns2) <= 1e-12 * ns2
    assert np.abs(cxi - nxi).max() <= 1e-7 * np.abs(nxi).max(), np.abs(cxi - nxi).max() / np.abs(nxi).max()
    assert np.abs(cjp - njp).max() <= 1e-7 * np.abs(njp).max(), np.abs(cjp - njp).max() / np.abs(njp).max()
    assert np.array_equal(cxi, cxi.T) and np.array_equal(cjp, cjp.T)
    assert np.linalg.eigvalsh(cxi).min() > 0


def test_covariance_away_from_the_fit_uses_the_same_formula(shim):
    """The definition holds at any pose the call is given: sigma2 from the residuals there, the Gauss-Newton information."""
    cam = (700.0, 300.0, 260.0)
    rng = np.random.default_rng(41)
    R0, t0 = _pose(rng, False)
    Y, e = _scene(rng, 60, R0, t0, cam, 2.0, False)
    R = Rotation.from_rotvec([0.01, -0.02, 0.005]).as_matrix() @ R0
    t = t0 + np.array([5.0, -3.0, 20.0])
    ok, cxi, cjp, s2 = covariance(shim, Y, e, R, t, cam, False)
    nxi, njp, ns2 = numpy_covariances(Y, e, R, t, cam, False)
    assert ok and abs(s2 - ns2) <= 1e-12 * ns2
    assert np.abs(cxi - nxi).max() <= 1e-7 * np.abs(nxi).max()
    assert np.abs(cjp - njp).max() <= 1e-7 * np.abs(njp).max()


def _refused(res):
    ok, cxi, cjp, s2 = res
    return not ok and not cxi.any() and not cjp.any() and s2 == 0.0


def test_degenerate_fits_give_false_and_zeros(shim):
    cam = (525.0, 320.0, 240.0)
    rng = np.random.default_rng(9)
    R0, t0 = _pose(rng, False)
    # m at the degree-of-freedom limit: 2m - 6 = 0 (RGB, m = 3), 3m - 6 = 0 (RGB-D, m = 2); one more cell is enough
    Y, e = _scene(rng, 4, R0, t0, cam, 1.0, False)
    assert _refused(covariance(shim, Y[:3], e[:3], R0, t0, cam, False))
    assert covariance(shim, Y, e, R0, t0, cam, False)[0]
    Y, e = _scene(rng, 3, R0, t0, cam, 1.0, True)
    assert _refused(covariance(shim, Y[:2], e[:2], R0, t0, cam, True))
    assert covariance(shim, Y, e, R0, t0, cam, True)[0]
    assert _refused(covariance(shim, np.zeros((0, 3)), np.zeros((0, 3)), R0, t0, cam, False))
    # collinear cells: the rotation about their line is free
    Y = np.array([[0, 0, 1000], [100, 0, 1000], [200, 0, 1000], [300, 0, 1000], [400, 0, 1000]], np.float64)
    t = np.array([-200.0, 0.0, 1500.0])
    X = Y + t
    uv = np.stack([525 * X[:, 0] / X[:, 2] + 320, 525 * X[:, 1] / X[:, 2] + 240, np.zeros(5)], 1)
    assert _refused(covariance(shim, Y, uv + rng.normal(0, 0.5, uv.shape) * [1, 1, 0], np.eye(3), t, cam, False))
    assert _refused(covariance(shim, Y, X + rng.normal(0, 2.0, X.shape), np.eye(3), t, cam, True))
    # non-finite input: a scene coordinate, an observation, the pose
    Y, e = _scene(rng, 30, R0, t0, cam, 1.0, False)
    for rgbd in (False, True):
        Yb = Y.copy(); Yb[4, 1] = np.nan
        assert _refused(covariance(shim, Yb, e, R0, t0, cam, rgbd))
        eb = e.copy(); eb[7, 0] = np.inf
        assert _refused(covariance(shim, Y, eb, R0, t0, cam, rgbd))
        assert _refused(covariance(shim, Y, e, R0, t0 * np.array([1, np.nan, 1]), cam, rgbd))


@pytest.mark.parametrize("rgbd", [False, True])
def test_covariance_is_calibrated(shim, rgbd):
    """A fixed cell set with a known pose, Gaussian noise of known sigma on the pixels (RGB) or the eye points (RGB-D), 2000
    frozen-set solves: the predicted covariance matches the empirical one, and the normalised errors are chi-square(6)."""
    rng = np.random.default_rng(2024 + rgbd)
    cam = (585.0, 322.5, 236.0)
    m, sigma, draws = 100, (4.0 if rgbd else 1.0), 2000
    R_true = Rotation.from_rotvec([0.3, -0.2, 0.1]).as_matrix()
    t_true = np.array([80.0, -40.0, 150.0])
    f, cx, cy = cam
    uv = np.stack([rng.uniform(20, 620, m), rng.uniform(20, 460, m)], 1)
    d = rng.uniform(800, 4000, m)
    Xc = np.stack([(uv[:, 0] - cx) * d / f, (uv[:, 1] - cy) * d / f, d], 1)
    Y = (Xc - t_true) @ R_true
    clean = Xc if rgbd else np.concatenate([uv, np.zeros((m, 1))], 1)
    errs, covs = np.zeros((draws, 6)), np.zeros((draws, 6, 6))
    for k in range(draws):
        e = clean.copy()
        if rgbd:
            e += rng.normal(0, sigma, e.shape)
        else:
            e[:, :2] += rng.normal(0, sigma, (m, 2))
        R, t = I.frozen_fit(Y, e, R_true, t_true, cam, rgbd, iters=8)
        ok, cxi, _, s2 = covariance(shim, Y, e, R, t, cam, rgbd)
        assert ok
        errs[k] = np.concatenate([Rotation.from_matrix(R @ R_true.T).as_rotvec(), t - t_true])
        covs[k] = cxi
    pred = covs.mean(0)
    emp = errs.T @ errs / draws
    w, V = np.linalg.eigh(pred)
    isq = V @ np.diag(w ** -0.5) @ V.T
    ev = np.linalg.eigvalsh(isq @ emp @ isq)
    assert 0.85 <= ev.min() and ev.max() <= 1.15, ev
    nees = np.mean([errs[k] @ np.linalg.solve(covs[k], errs[k]) for k in range(draws)])
    assert abs(nees - 6.0) <= 0.5, nees


def test_entry_point_is_exported(engine_mod):
    lib = engine_mod.load()
    assert hasattr(lib, "dsac_pose_uncertainty_device")
    assert "dsac_pose_uncertainty_device" in engine_mod.EXPORTS


def test_rgbd_recording_replay_is_the_oracle_refinement(oracle):
    """tests/host_shim/rgbd_record.cpp, the independent set S of the GPU tests' RGB-D passes: its pose is the RGB-D
    oracle's refined pose bit for bit, from the oracle's own average and permutations."""
    import rgbd_oracle as R
    import rgbd_record as RR
    coords, pix, depth, _, _ = R.synth(3, seed=93, holes=0.15)
    for g in range(3):
        cfg = oracle.default_config(n_hyps=16)
        ey, _ = R.eye(pix[g], depth[g])
        fw, _ = R.forward(oracle, cfg, g, coords[g], pix[g], ey)
        pose, S, done = RR.refine_record(cfg, coords[g], pix[g], ey, fw.pixel_idxs, fw.n_perm_steps, np.array(fw.avg))
        assert np.array_equal(pose, np.array(fw.ref))
        assert done == fw.ref_steps_done and (done == 0) == (len(S) == 0)
        assert len(np.unique(S)) == len(S) and np.isfinite(ey[S]).all()
