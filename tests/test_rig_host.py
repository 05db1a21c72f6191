"""The multi-camera rig arithmetic on the host (tests/host_shim/rig_shim.cpp): the lift inverts the composition with the
extrinsic, an identity extrinsic changes no bit, and the chained LM Jacobian of lm_point_contrib_ext matches central
differences of the projection through the extrinsic."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def shim():
    d = os.path.join(HERE, "host_shim")
    so, src = os.path.join(d, "librig_shim.so"), os.path.join(d, "rig_shim.cpp")
    deps = [src] + [os.path.join(ROOT, "dsac_b200", "csrc", f) for f in ("pose_math.cuh", "lm_math.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(x) > os.path.getmtime(so) for x in deps):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _call(fn, *arrays):
    fn(*[_p(a) for a in arrays])


def _random_pose(rng, scale=1.0):
    return np.concatenate([Rotation.random(random_state=rng).as_rotvec() * scale, rng.normal(scale=500.0, size=3)])


def test_lift_then_compose_returns_the_camera_pose(shim):
    rng = np.random.default_rng(1)
    for _ in range(200):
        ext, cam = _random_pose(rng), _random_pose(rng)
        Rc, R = Rotation.from_rotvec(ext[:3]).as_matrix(), Rotation.from_rotvec(cam[:3]).as_matrix()
        Rr, tr, Rk, tk = np.empty(9), np.empty(3), np.empty(9), np.empty(3)
        _call(shim.shim_rig_lift, Rc.ravel().copy(), ext[3:].copy(), R.ravel().copy(), cam[3:].copy(), Rr, tr)
        assert np.allclose(Rr.reshape(3, 3), Rc.T @ R, atol=1e-14)
        assert np.allclose(tr, Rc.T @ (cam[3:] - ext[3:]), atol=1e-10)
        _call(shim.shim_rig_compose, Rc.ravel().copy(), ext[3:].copy(), Rr, tr, Rk, tk)
        assert np.allclose(Rk, R.ravel(), atol=1e-14)
        assert np.allclose(tk, cam[3:], atol=1e-10)


def test_identity_extrinsic_changes_no_bit(shim):
    rng = np.random.default_rng(2)
    I, z = np.eye(3).ravel().copy(), np.zeros(3)
    for _ in range(200):
        pose = _random_pose(rng)
        R = Rotation.from_rotvec(pose[:3]).as_matrix().ravel().copy()
        t = pose[3:].copy()
        for fn in (shim.shim_rig_lift, shim.shim_rig_compose):
            Ro, to = np.empty(9), np.empty(3)
            _call(fn, I, z, R, t, Ro, to)
            assert np.array_equal(Ro, R) and np.array_equal(to, t)
        X = rng.normal(scale=1000.0, size=3)
        X[2] += 3000.0
        pix = rng.uniform(0.0, 640.0, size=2)
        a, b = np.empty(28), np.empty(28)
        shim.shim_point_contrib(_p(pose), None, None, _p(X), _p(pix), C.c_double(525.0), C.c_double(320.0), C.c_double(240.0), _p(a))
        shim.shim_point_contrib(_p(pose), _p(I), _p(z), _p(X), _p(pix), C.c_double(525.0), C.c_double(320.0), C.c_double(240.0), _p(b))
        assert np.array_equal(a, b)


def _project(param, ext, X, f, cx, cy):
    R = Rotation.from_rotvec(param[:3]).as_matrix()
    Rc = Rotation.from_rotvec(ext[:3]).as_matrix()
    Xc = Rc @ (R @ X + param[3:]) + ext[3:]
    return np.array([Xc[0] / Xc[2] * f + cx, Xc[1] / Xc[2] * f + cy])


def test_chained_jacobian_matches_central_differences(shim):
    rng = np.random.default_rng(3)
    f, cx, cy = 580.0, 310.5, 250.25
    for _ in range(50):
        ext = np.concatenate([Rotation.random(random_state=rng).as_rotvec() * 0.5, rng.normal(scale=100.0, size=3)])
        Rc = Rotation.from_rotvec(ext[:3]).as_matrix()
        param = np.concatenate([rng.normal(scale=0.5, size=3), rng.normal(scale=200.0, size=3)])
        # a scene point 2-4 m in front of the camera
        Xc = np.array([rng.normal(scale=500.0), rng.normal(scale=500.0), rng.uniform(2000.0, 4000.0)])
        R = Rotation.from_rotvec(param[:3]).as_matrix()
        X = R.T @ (Rc.T @ (Xc - ext[3:]) - param[3:])
        proj = _project(param, ext, X, f, cx, cy)
        J = np.empty((2, 6))
        for a in range(6):
            h = 1e-7 if a < 3 else 1e-4
            d = np.zeros(6)
            d[a] = h
            J[:, a] = (_project(param + d, ext, X, f, cx, cy) - _project(param - d, ext, X, f, cx, cy)) / (2 * h)
        for row in range(2):   # with the residual e = unit vector row, v[21..26] = J^T e is the Jacobian's row
            pix = proj - np.eye(2)[row]
            v = np.empty(28)
            shim.shim_point_contrib(_p(param), _p(Rc.ravel().copy()), _p(ext[3:].copy()), _p(X), _p(pix), C.c_double(f),
                                    C.c_double(cx), C.c_double(cy), _p(v))
            assert np.allclose(v[21:27], J[row], rtol=1e-5, atol=1e-6 * np.abs(J[row]).max()), (row, v[21:27], J[row])
            assert abs(v[27] - 1.0) < 1e-6
