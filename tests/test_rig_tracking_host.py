"""Rig tracking's fp64 arithmetic on the host (tests/host_shim/rig_tracking_shim.cpp, the device's DSAC_HD code): the
composition of a rig prior with an extrinsic against scipy, the gate's invariance under it, the exact identity of a zero
extrinsic, and the rig fit covariance against numpy and, for one camera behind an identity, against ift_fit_covariance."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from rig_grad_oracle import ring, rot
from rig_tracking_oracle import compose, compose_np, fit_cov, lift, prior_d2, rig_cov, rig_cov_np


def _info(rng):
    A = rng.normal(size=(6, 6)) * np.array([50.0] * 3 + [0.05] * 3)
    return A @ A.T + np.diag([1e3] * 3 + [1e-3] * 3)


def _pose(rng, scale=0.8):
    return np.concatenate([Rotation.random(random_state=rng).as_rotvec() * rng.uniform(0.05, scale),
                           rng.normal(scale=600.0, size=3) + [0, 0, 2000.0]])


def test_composition_matches_scipy():
    rng = np.random.default_rng(1)
    for C_ in (2, 3, 4):
        ext = ring(C_, seed=C_)
        for _ in range(40):
            pose, info = _pose(rng), _info(rng)
            for c in range(C_):
                ok, op, oi = compose(ext[c], pose, info)
                rp, ri = compose_np(ext[c], pose, info)
                assert ok
                assert np.allclose(rot(op[:3]), rot(rp[:3]), rtol=0, atol=1e-12)
                assert np.allclose(op[3:], rp[3:], rtol=0, atol=1e-9)
                assert np.allclose(oi, ri, rtol=0, atol=1e-12 * np.abs(ri).max())


def test_camera_gate_equals_rig_gate_of_the_lifted_hypothesis():
    rng = np.random.default_rng(2)
    checked = 0
    for C_ in (2, 3, 4):
        ext = ring(C_, seed=10 + C_)
        ext[:, :3] += rng.normal(scale=0.2, size=(C_, 3))
        for _ in range(60):
            pose, info = _pose(rng), _info(rng)
            for c in range(C_):
                ok, op, oi = compose(ext[c], pose, info)
                # a camera hypothesis near the composed prior, and its lift to the rig
                hyp = np.concatenate([(Rotation.from_rotvec(rng.normal(scale=0.05, size=3)) * Rotation.from_rotvec(op[:3])).as_rotvec(),
                                      op[3:] + rng.normal(scale=30.0, size=3)])
                d_cam = prior_d2(hyp, op, oi)
                d_rig = prior_d2(lift(ext[c], hyp), pose, info)
                assert d_cam > 0 and d_rig > 0
                assert abs(d_cam - d_rig) <= 1e-9 * d_rig, (d_cam, d_rig)
                checked += 1
    assert checked > 500


def test_zero_extrinsic_composition_is_bitwise_the_identity():
    rng = np.random.default_rng(3)
    for _ in range(100):
        ext = np.concatenate([np.zeros(3), rng.normal(scale=50.0, size=3) * rng.integers(0, 2)])
        pose, info = _pose(rng, 3.0), _info(rng)
        ok, op, oi = compose(ext, pose, info)
        assert ok
        assert np.array_equal(op[:3], pose[:3]) and np.array_equal(oi, info)
        assert np.array_equal(op[3:], pose[3:] + ext[3:])
        ok, op2, _ = compose(ext, pose, None)
        assert ok and np.array_equal(op2, op)


def test_non_finite_extrinsic_is_refused():
    ok, _, _ = compose(np.array([0.1, np.nan, 0, 0, 0, 0]), np.zeros(6) + 0.1, None)
    assert not ok
    ok, _, _ = compose(np.array([0.1, 0, 0, 0, np.inf, 0]), np.zeros(6) + 0.1, _info(np.random.default_rng(0)))
    assert not ok


def _rig_cells(rng, C_, ext, fcc, pose, per=40, noise=1.5):
    R0, t0 = rot(pose[:3]), pose[3:]
    cam = np.repeat(np.arange(C_), per).astype(np.int32)
    Y, uv = np.zeros((C_ * per, 3)), np.zeros((C_ * per, 2))
    for c in range(C_):
        Rc = rot(ext[c, :3])
        Xc = np.stack([rng.normal(scale=600.0, size=per), rng.normal(scale=500.0, size=per), rng.uniform(1500.0, 4000.0, per)], 1)
        X = (Xc - ext[c, 3:]) @ Rc
        Y[c * per:(c + 1) * per] = (X - t0) @ R0
        uv[c * per:(c + 1) * per] = np.stack([fcc[c, 0] * Xc[:, 0] / Xc[:, 2] + fcc[c, 1], fcc[c, 0] * Xc[:, 1] / Xc[:, 2] + fcc[c, 2]], 1)
    return cam, Y, uv + rng.normal(scale=noise, size=uv.shape)


@pytest.mark.parametrize("C_", [1, 2, 3, 4])
def test_rig_covariance_matches_numpy(C_):
    rng = np.random.default_rng(30 + C_)
    ext = ring(C_, seed=C_)
    fcc = np.array([[525.0 + 20 * c, 320.0 - 3 * c, 240.0 + 2 * c] for c in range(C_)])
    pose = np.concatenate([rng.normal(scale=0.3, size=3), rng.normal(scale=300.0, size=3)])
    cam, Y, uv = _rig_cells(rng, C_, ext, fcc, pose)
    ok, cxi, cjp, s2 = rig_cov(cam, Y, uv, ext, fcc, pose)
    ref, s2_ref = rig_cov_np(cam, Y, uv, ext, fcc, pose)
    assert ok
    assert abs(s2 - s2_ref) <= 1e-9 * s2_ref
    assert np.allclose(cxi, ref, rtol=0, atol=1e-5 * np.abs(np.diag(ref)).max()), (cxi - ref)
    assert np.array_equal(cjp, cjp.T) and np.array_equal(cxi, cxi.T)


def test_one_camera_behind_an_identity_is_ift_fit_covariance_bit_for_bit():
    rng = np.random.default_rng(40)
    for _ in range(20):
        fcc = np.array([[rng.uniform(400, 700), rng.uniform(300, 340), rng.uniform(220, 260)]])
        pose = np.concatenate([rng.normal(scale=0.5, size=3), rng.normal(scale=300.0, size=3)])
        ext = np.zeros((1, 6))
        cam, Y, uv = _rig_cells(rng, 1, ext, fcc, pose, per=int(rng.integers(4, 128)))
        a = rig_cov(cam, Y, uv, ext, fcc, pose)
        b = fit_cov(Y, uv, fcc[0], pose)
        assert a[0] == b[0]
        for x, y in zip(a[1:], b[1:]):
            assert np.array_equal(x, y)
