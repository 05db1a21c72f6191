"""Implicit-function scene-coordinate derivatives (dsac_b200/csrc/ift.cuh, compiled for the host) against central
differences of independent solves: a frozen-set Gauss-Newton solver in numpy for the refinement's fit, the product's P3P
and Kabsch in double for dPNP."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import adversarial_sets as adv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DFLIP = np.diag([1.0, -1.0, -1.0])


@pytest.fixture(scope="module")
def shim():
    so = os.path.join(tempfile.mkdtemp(prefix="ift_shim_"), "libift_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "ift_shim.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f64(a):
    return np.ascontiguousarray(a, np.float64)


def jp6(R, t):
    """jp 6-vector of a cv pose: (rotation vector of D R, D t)."""
    return np.concatenate([Rotation.from_matrix(DFLIP @ R).as_rotvec(), DFLIP @ t])


def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def frozen_fit(Y, e, R, t, cam, rgbd):
    """Stationary point of the fit over the frozen set by Gauss-Newton in the left chart, to a step below 1e-14."""
    f, cx, cy = cam
    for _ in range(500):
        q = Y @ R.T
        X = q + t
        rows, res = [], []
        for i in range(len(Y)):
            dX = np.concatenate([-_skew(q[i]), np.eye(3)], 1)   # dX / (w, tau)
            if rgbd:
                rows.append(dX); res.append(X[i] - e[i])
            else:
                z = X[i, 2]
                g = np.array([[f / z, 0, -f * X[i, 0] / z ** 2], [0, f / z, -f * X[i, 1] / z ** 2]])
                rows.append(g @ dX); res.append(np.array([f * X[i, 0] / z + cx, f * X[i, 1] / z + cy]) - e[i, :2])
        J, r = np.concatenate(rows), np.concatenate(res)
        step = -np.linalg.solve(J.T @ J, J.T @ r)
        R = Rotation.from_rotvec(step[:3]).as_matrix() @ R
        t = t + step[3:]
        if np.abs(step).max() < 1e-14:
            break
    return R, t


def ift_fit(shim, Y, e, R, t, cam, rgbd):
    m = len(Y)
    pose = _f64(np.concatenate([Rotation.from_matrix(R).as_rotvec(), t]))
    D = np.zeros((m, 6, 3))
    ok = shim.shim_ift_fit_deriv(m, _p(_f64(Y)), _p(_f64(e)), _p(pose), C.c_double(cam[0]), C.c_double(cam[1]),
                                 C.c_double(cam[2]), int(rgbd), _p(D))
    return bool(ok), D


def _scene(rng, m, R, t, cam, noise, rgbd):
    f, cx, cy = cam
    uv = np.stack([rng.uniform(20, 620, m), rng.uniform(20, 460, m)], 1)
    d = rng.uniform(800, 4000, m)
    Xc = np.stack([(uv[:, 0] - cx) * d / f, (uv[:, 1] - cy) * d / f, d], 1)
    Y = np.round((Xc - t) @ R)                 # int16-grid scene coordinates
    e = Xc + rng.normal(0, noise, Xc.shape) if rgbd else np.concatenate([np.round(uv + rng.normal(0, noise, uv.shape)), np.zeros((m, 1))], 1)
    return Y, e


def _pose(rng, near_pi):
    if near_pi:   # jp rotation within 1e-3 rad of pi
        ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
        Rj = Rotation.from_rotvec((np.pi - rng.uniform(1e-5, 1e-4)) * ax).as_matrix()
        R = DFLIP @ Rj
    else:
        R = Rotation.from_rotvec(rng.uniform(-0.5, 0.5, 3)).as_matrix()
    return R, np.array([rng.uniform(-300, 300), rng.uniform(-300, 300), rng.uniform(-200, 200)])


CASES = [  # (f, cx, cy), near pi, rgbd
    ((525.0, 320.0, 240.0), True, False),
    ((525.0, 320.0, 240.0), False, False),
    ((2500.0, 410.5, 170.25), True, False),
    ((900.0, 250.0, 300.0), True, True),
    ((525.0, 320.0, 240.0), False, True),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_refinement_ift_matches_frozen_set_central_differences(shim, case):
    cam, near_pi, rgbd = CASES[case]
    rng = np.random.default_rng(100 + case)
    R0, t0 = _pose(rng, near_pi)
    m = 16
    Y, e = _scene(rng, m, R0, t0, cam, 2.0 if rgbd else 1.5, rgbd)
    R, t = frozen_fit(Y, e, R0, t0, cam, rgbd)
    if near_pi:   # the fit moves the pose by the noise
        assert np.pi - np.linalg.norm(jp6(R, t)[:3]) < 3e-3
    ok, D = ift_fit(shim, Y, e, R, t, cam, rgbd)
    assert ok
    eps = 1e-3
    num = np.zeros((m, 6, 3))
    for i in range(m):
        for j in range(3):
            Yp, Ym = Y.copy(), Y.copy()
            Yp[i, j] += eps; Ym[i, j] -= eps
            Rp, tp = frozen_fit(Yp, e, R, t, cam, rgbd)
            Rm, tm = frozen_fit(Ym, e, R, t, cam, rgbd)
            num[i, :, j] = (jp6(Rp, tp) - jp6(Rm, tm)) / (2 * eps)
    scale = np.abs(num).max()
    assert np.abs(D - num).max() <= 1e-5 * scale, (np.abs(D - num).max(), scale)


def test_residual_curvature_matters(shim):
    """The Gauss-Newton Hessian alone would be off by O(residual): with noisy pixels the full Hessian is needed."""
    cam = (525.0, 320.0, 240.0)
    rng = np.random.default_rng(7)
    R0, t0 = _pose(rng, True)
    Y, e = _scene(rng, 30, R0, t0, cam, 4.0, False)
    R, t = frozen_fit(Y, e, R0, t0, cam, False)
    ok, D = ift_fit(shim, Y, e, R, t, cam, False)
    assert ok
    eps = 1e-3
    Yp, Ym = Y.copy(), Y.copy()
    Yp[3, 1] += eps; Ym[3, 1] -= eps
    num = (jp6(*frozen_fit(Yp, e, R, t, cam, False)) - jp6(*frozen_fit(Ym, e, R, t, cam, False))) / (2 * eps)
    assert np.abs(D[3, :, 1] - num).max() <= 1e-5 * np.abs(num).max()


def test_jp_jacobian_matches_central_differences(shim):
    rng = np.random.default_rng(3)
    for near_pi in (True, False, True):
        R0, t0 = _pose(rng, near_pi)
        pose = _f64(np.concatenate([Rotation.from_matrix(R0).as_rotvec(), t0]))
        Rs, M = np.zeros(9), np.zeros(36)
        shim.shim_ift_jp_jacobian(_p(pose), _p(Rs), _p(M))
        M = M.reshape(6, 6)
        num = np.zeros((6, 6))
        eps = 1e-6
        for a in range(6):
            d = np.zeros(6); d[a] = eps
            Rp = Rotation.from_rotvec(d[:3]).as_matrix() @ R0
            Rm = Rotation.from_rotvec(-d[:3]).as_matrix() @ R0
            num[:, a] = (jp6(Rp, t0 + d[3:]) - jp6(Rm, t0 - d[3:])) / (2 * eps)
        assert np.abs(M - num).max() <= 1e-6 * np.abs(num).max()


def test_degenerate_sets_give_documented_zeros(shim):
    cam = (525.0, 320.0, 240.0)
    # collinear RGB-D set: the rotation about the line is free, the Hessian is singular
    Y = np.array([[0, 0, 1000], [100, 0, 1000], [200, 0, 1000], [300, 0, 1000]], np.float64)
    e = Y + np.array([0, 0, 500.0])
    ok, D = ift_fit(shim, Y, e, np.eye(3), np.array([0, 0, 500.0]), cam, True)
    assert not ok and not D.any()
    # an indefinite Hessian: the pose rotated by pi about z away from the fit (not a stationary point; the zero rule
    # looks only at the Hessian)
    rng = np.random.default_rng(5)
    Y = rng.uniform(-500, 500, (10, 3)).round()
    Rz = Rotation.from_rotvec([0, 0, np.pi]).as_matrix()
    e = Y.copy()
    ok, D = ift_fit(shim, Y - Y.mean(0), e - e.mean(0), Rz, np.zeros(3), cam, True)
    assert not ok and not D.any()
    # no cells
    ok, D = ift_fit(shim, np.zeros((0, 3)), np.zeros((0, 3)), np.eye(3), np.array([0, 0, 1000.0]), cam, False)
    assert not ok


def _p3p_pose(shim, X4, uv4, cam):
    R, t = np.zeros(9), np.zeros(3)
    n = shim.shim_p3p_double(_p(_f64(X4)), _p(_f64(uv4)), C.c_double(cam[0]), C.c_double(cam[1]), C.c_double(cam[2]), _p(R), _p(t))
    return n > 0, R.reshape(3, 3), t


def test_dpnp_p3p_ift_matches_central_differences(shim):
    rng = np.random.default_rng(21)
    n_ok = 0
    for i in range(40):
        cam = [(525.0, 320.0, 240.0), (2500.0, 400.0, 200.0), (800.0, 300.5, 260.0)][i % 3]
        R0, t0 = _pose(rng, i % 2 == 0)
        Y, e = _scene(rng, 4, R0, t0, cam, 0.0, False)
        uv = e[:, :2]
        ok, R, t = _p3p_pose(shim, Y, uv, cam)
        # within 1e-5 rad of pi the sign of the rotation vector is a convention (rodrigues' near-pi branch), not a function
        # of the rotation: there the central differences below, through scipy, may follow the other sign
        if not ok or np.pi - np.linalg.norm(jp6(R, t)[:3]) < 1e-5:
            continue
        pose = _f64(np.concatenate([Rotation.from_matrix(R).as_rotvec(), t]))
        out = np.zeros(72)
        if not shim.shim_ift_dpnp_p3p(_p(pose), _p(_f64(Y[:3])), _p(_f64(uv[:3])), C.c_double(cam[0]), C.c_double(cam[1]),
                                      C.c_double(cam[2]), _p(out)):
            continue
        out = out.reshape(6, 12)
        eps = 1e-3
        num = np.zeros((6, 12))
        good = True
        for col in range(9):
            Yp, Ym = Y.copy(), Y.copy()
            Yp.flat[col] += eps; Ym.flat[col] -= eps
            okp, Rp, tp = _p3p_pose(shim, Yp, uv, cam)
            okm, Rm, tm = _p3p_pose(shim, Ym, uv, cam)
            if not (okp and okm):
                good = False
                break
            num[:, col] = (jp6(Rp, tp) - jp6(Rm, tm)) / (2 * eps)
        if not good:
            continue
        assert not out[:, 9:].any()
        assert np.abs(out - num).max() <= 1e-5 * np.abs(num).max(), i
        n_ok += 1
    assert n_ok >= 25


def test_dpnp_kabsch_ift_matches_central_differences(shim):
    rng = np.random.default_rng(22)
    for i in range(20):
        a = rng.uniform(-800, 800, (3, 3)).round()
        R0, t0 = _pose(rng, i % 2 == 0)
        b = a @ R0.T + t0 + np.array([0, 0, 2500]) + rng.normal(0, 3, (3, 3))
        out = np.zeros(72)
        assert shim.shim_ift_dpnp_kabsch(_p(_f64(a)), _p(_f64(b)), _p(out))
        out = out.reshape(6, 12)
        num = np.zeros((6, 12))
        eps = 1e-3
        for col in range(9):
            ap, am = a.copy(), a.copy()
            ap.flat[col] += eps; am.flat[col] -= eps
            js = []
            for x in (ap, am):
                R, t = np.zeros(9), np.zeros(3)
                shim.shim_kabsch(3, _p(_f64(x)), _p(_f64(b)), _p(R), _p(t))
                js.append(jp6(R.reshape(3, 3), t))
            num[:, col] = (js[0] - js[1]) / (2 * eps)
        assert not out[:, 9:].any()
        assert np.abs(out - num).max() <= 1e-5 * np.abs(num).max(), i


def test_dpnp_ift_adversarial_sets_finite_or_zero(shim):
    cam = (525.0, 320.0, 240.0)
    rng = np.random.default_rng(8)
    objs, imgs = zip(adv.danger_cylinder(rng, cam, 10, trials=60), adv.near_collinear(rng, cam, 10, trials=60), adv.NEAR_CAMERA_CASE)
    n = 0
    for Y, uv in zip(np.concatenate([o.reshape(-1, 12) for o in objs]), np.concatenate([i.reshape(-1, 8) for i in imgs])):
        Y = np.asarray(Y, np.float64).reshape(4, 3)
        uv = np.asarray(uv, np.float64).reshape(4, 2)
        ok, R, t = _p3p_pose(shim, Y, uv, cam)
        if ok:
            pose = _f64(np.concatenate([Rotation.from_matrix(R).as_rotvec(), t]))
            out = np.zeros(72)
            r = shim.shim_ift_dpnp_p3p(_p(pose), _p(_f64(Y[:3])), _p(_f64(uv[:3])), C.c_double(cam[0]), C.c_double(cam[1]),
                                       C.c_double(cam[2]), _p(out))
            assert np.isfinite(out).all()
            assert r or not out.any()
        out = np.zeros(72)
        r = shim.shim_ift_dpnp_kabsch(_p(_f64(Y[:3])), _p(_f64(Y[:3] + np.array([0, 0, 2000.0]))), _p(out))
        assert np.isfinite(out).all() and (r or not out.any())
        n += 1
    assert n > 50
