"""The pose priors' covariance gate (dsac_b200/csrc/prior.cuh, compiled for the host) against numpy / scipy: the squared
Mahalanobis distance d^2 = xi^T Lambda xi with xi = (log(R_h R_j^T), t_h - t_j), rotations up to pi - 1e-6, the Cholesky
refusals of DSAC_ST_BAD_PRIOR, and that only the lower triangle of Lambda is read."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def shim():
    so = os.path.join(tempfile.mkdtemp(prefix="prior_shim_"), "libprior_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "prior_shim.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f64(a):
    return np.ascontiguousarray(a, np.float64)


def shim_d2(shim, priors, infos, pose):
    priors, infos, pose = _f64(priors), _f64(infos), _f64(pose)
    k = priors.shape[0]
    d2 = np.full(k, np.nan)
    ok = shim.shim_prior_d2(C.c_int(k), _p(priors), _p(infos), _p(pose), _p(d2))
    return ok, d2


def ref_d2(prior, info, pose):
    rel = Rotation.from_rotvec(pose[:3]) * Rotation.from_rotvec(prior[:3]).inv()
    xi = np.concatenate([rel.as_rotvec(), pose[3:] - prior[3:]])
    return float(xi @ info @ xi)


def random_info(rng):
    A = rng.normal(size=(6, 6))
    D = np.diag([30.0, 30.0, 30.0, 0.1, 0.1, 0.1])   # information of a few degrees and ~10 mm: rad^-2 and mm^-2
    return D @ (A @ A.T + 0.5 * np.eye(6)) @ D


def pose_at_angle(rng, prior, angle):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    rel = Rotation.from_rotvec(angle * axis)
    R = rel * Rotation.from_rotvec(prior[:3])
    return np.concatenate([R.as_rotvec(), prior[3:] + rng.normal(scale=50.0, size=3)])


@pytest.mark.parametrize("angle", [0.0, 1e-9, 1e-4, 0.3, np.pi / 2, 2.0, 3.0, np.pi - 1e-3, np.pi - 1e-6])
def test_d2_matches_scipy(shim, angle):
    rng = np.random.default_rng(int(angle * 1e6) + 7)
    for _ in range(20):
        prior = np.concatenate([Rotation.random(random_state=rng.integers(1 << 30)).as_rotvec(), rng.normal(scale=1000, size=3)])
        info = random_info(rng)
        pose = pose_at_angle(rng, prior, angle)
        ok, d2 = shim_d2(shim, prior[None], info[None], pose)
        assert ok == 1
        ref = ref_d2(prior, info, pose)
        assert abs(d2[0] - ref) <= 1e-9 * abs(ref) + 1e-300, (angle, d2[0], ref)


def test_log_is_principal_near_pi(shim):
    rng = np.random.default_rng(3)
    for angle in [np.pi - 1e-6, np.pi - 1e-8, np.pi]:
        for _ in range(20):
            axis = rng.normal(size=3)
            axis /= np.linalg.norm(axis)
            M = _f64(Rotation.from_rotvec(angle * axis).as_matrix())
            w = np.zeros(3)
            shim.shim_so3_log(_p(M), _p(w))
            assert abs(np.linalg.norm(w) - angle) <= 1e-12
            # the axis up to sign at exactly pi, where both are the principal log
            if angle < np.pi:
                assert np.abs(w - angle * axis).max() <= 1e-9
            else:
                assert min(np.abs(w - angle * axis).max(), np.abs(w + angle * axis).max()) <= 1e-9


def test_gate_is_min_over_priors(shim):
    rng = np.random.default_rng(11)
    k = 5
    priors = np.stack([np.concatenate([Rotation.random(random_state=i).as_rotvec(), rng.normal(scale=500, size=3)])
                       for i in range(k)])
    infos = np.stack([np.diag([400.0] * 3 + [1e-2] * 3) for _ in range(k)])
    for trial in range(200):
        pose = pose_at_angle(rng, priors[trial % k], rng.uniform(0, 0.3))
        ok, d2 = shim_d2(shim, priors, infos, pose)
        assert ok == 1
        chi2 = float(np.median(d2)) if trial % 2 else float(d2.min()) * (1 - 1e-12)
        passed = shim.shim_prior_gate_pass(C.c_int(k), _p(_f64(priors)), _p(_f64(infos)), C.c_double(chi2), _p(_f64(pose)))
        assert passed == int(d2.min() <= chi2)


def _cholesky_ok(shim, info):
    L = np.zeros(21)
    return shim.shim_prior_cholesky(_p(_f64(info)), _p(L)), L


def test_cholesky_refusals(shim):
    rng = np.random.default_rng(5)
    A = rng.normal(size=(6, 5))
    singular = A @ A.T                                            # rank 5
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    indefinite = Q @ np.diag([3.0, 2.0, 1.0, 1.0, 0.5, -0.1]) @ Q.T
    nan = np.eye(6)
    nan[4, 2] = np.nan
    inf = np.eye(6)
    inf[5, 5] = np.inf
    for bad in [singular, indefinite, -np.eye(6), np.zeros((6, 6)), nan, inf]:
        assert _cholesky_ok(shim, bad)[0] == 0
    ok, L = _cholesky_ok(shim, random_info(rng))
    assert ok == 1
    # a refused entry refuses the frame: d2 is not computed
    prior = np.zeros(6)
    assert shim_d2(shim, prior[None], indefinite[None], np.ones(6))[0] == 0
    # a non-finite prior pose is refused as well
    assert shim_d2(shim, np.array([[0, np.nan, 0, 0, 0, 0.0]]), np.eye(6)[None], np.ones(6))[0] == 0


def test_cholesky_factor(shim):
    rng = np.random.default_rng(9)
    info = random_info(rng)
    ok, Lp = _cholesky_ok(shim, info)
    assert ok == 1
    L = np.zeros((6, 6))
    for i in range(6):
        for j in range(i + 1):
            L[i, j] = Lp[i * (i + 1) // 2 + j]
    assert np.allclose(L, np.linalg.cholesky(info), rtol=1e-12, atol=0)


def test_reads_lower_triangle_only(shim):
    rng = np.random.default_rng(13)
    prior = np.concatenate([Rotation.random(random_state=1).as_rotvec(), [10.0, -20.0, 3000.0]])
    pose = pose_at_angle(rng, prior, 0.2)
    info = random_info(rng)
    ok, d2 = shim_d2(shim, prior[None], info[None], pose)
    assert ok == 1
    for junk in [np.nan, np.inf, -1e300, 0.0]:
        garbled = info.copy()
        garbled[np.triu_indices(6, 1)] = junk
        ok2, d2b = shim_d2(shim, prior[None], garbled[None], pose)
        assert ok2 == 1 and d2b[0] == d2[0]
