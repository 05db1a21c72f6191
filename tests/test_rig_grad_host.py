"""The rig backward's fp64 arithmetic on the host (tests/host_shim/rig_grad_shim.cpp): the lift's Jacobian L and the
composition's Jacobian K against central differences of the lift and the composition, exact identities for a zero
extrinsic and for a camera's own slots, and the implicit-function derivative of a rig fit over cells of several cameras
against central differences of a frozen-set rig fit solved independently in numpy."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from ift_oracle import jp6
from rig_grad_oracle import cross_jac, cross_jp, frozen_fit_rig, lift_cv, lift_jac, ring, rig_ift
from rig_grad_oracle import log as _log, p as _p, rot as _rot, shim as _shim


@pytest.fixture(scope="module")
def shim():
    return _shim()


def test_lift_jacobian_matches_central_differences(shim):
    rng = np.random.default_rng(11)
    checked = 0
    for _ in range(200):
        e = np.concatenate([Rotation.random(random_state=rng).as_rotvec() * rng.uniform(0.1, 0.9), rng.normal(scale=100.0, size=3)])
        hyp = np.concatenate([Rotation.random(random_state=rng).as_rotvec() * rng.uniform(0.05, 0.8), rng.normal(scale=800.0, size=3)])
        Rc = _rot(e[:3])
        if np.linalg.norm(lift_cv(Rc, e[3:], hyp[None])[0, :3]) > np.pi - 0.05:
            continue   # the rotation vector's branch cut
        L = np.empty(36)
        shim.shim_rig_lift_jac(_p(Rc.ravel().copy()), _p(hyp[:3].copy()), _p(L))
        num = lift_jac(Rc, e[3:], hyp[None])[0]   # [output][input]
        assert np.allclose(L.reshape(6, 6), num, rtol=0, atol=2e-7 * np.abs(num).max()), (L.reshape(6, 6) - num)
        checked += 1
    assert checked > 150


def test_cross_jacobian_matches_central_differences(shim):
    rng = np.random.default_rng(12)
    checked = 0
    for C_ in (2, 3, 4):
        ext = ring(C_, seed=C_)
        for _ in range(60):
            # cv hypotheses of ordinary poses: small cv rotations, so their jp rotation vectors are near pi
            hyp_cv = np.concatenate([Rotation.random(random_state=rng).as_rotvec() * rng.uniform(0.05, 0.6),
                                     rng.normal(scale=500.0, size=3) + [0, 0, 2000.0]])
            x = jp6(_rot(hyp_cv[:3]), hyp_cv[3:])
            c2, c = rng.integers(C_), rng.integers(C_)
            Rc, Rc2 = _rot(ext[c, :3]), _rot(ext[c2, :3])
            out = cross_jp(Rc, ext[c, 3:], Rc2, ext[c2, 3:], x[None])[0]
            if max(np.linalg.norm(x[:3]), np.linalg.norm(out[:3])) > np.pi - 0.02:
                continue
            K = np.empty(36)
            shim.shim_rig_cross_jac(_p(Rc.ravel().copy()), _p(Rc2.ravel().copy()), _p(_rot(hyp_cv[:3]).ravel().copy()), int(c == c2), _p(K))
            num = cross_jac(Rc, ext[c, 3:], Rc2, ext[c2, 3:], hyp_cv[None])[0]
            assert np.allclose(K.reshape(6, 6), num, rtol=0, atol=2e-6 * np.abs(num).max()), (C_, c, c2, K.reshape(6, 6) - num)
            checked += 1
    assert checked > 120


def test_zero_extrinsic_and_own_camera_give_exact_identities(shim):
    rng = np.random.default_rng(13)
    I = np.eye(3).ravel().copy()
    for _ in range(50):
        r = Rotation.random(random_state=rng).as_rotvec()
        L = np.empty(36)
        shim.shim_rig_lift_jac(_p(I), _p(r.copy()), _p(L))
        assert np.array_equal(L, np.eye(6).ravel())
        Rc = _rot(Rotation.random(random_state=rng).as_rotvec()).ravel().copy()
        K = np.empty(36)
        shim.shim_rig_cross_jac(_p(Rc), _p(Rc), _p(_rot(r).ravel().copy()), 1, _p(K))
        assert np.array_equal(K, np.eye(6).ravel())


@pytest.mark.parametrize("C_", [2, 3, 4])
def test_rig_ift_matches_frozen_set_central_differences(shim, C_):
    rng = np.random.default_rng(20 + C_)
    ext = ring(C_, seed=C_)
    fcc = np.array([[525.0 + 20 * c, 320.0 - 3 * c, 240.0 + 2 * c] for c in range(C_)])
    R0, t0 = _rot(rng.normal(scale=0.3, size=3)), rng.normal(scale=300.0, size=3)
    per = 40
    cam = np.repeat(np.arange(C_), per).astype(np.int32)
    Y, uv = np.zeros((C_ * per, 3)), np.zeros((C_ * per, 2))
    for c in range(C_):
        Rc = _rot(ext[c, :3])
        Xc = np.stack([rng.normal(scale=600.0, size=per), rng.normal(scale=500.0, size=per), rng.uniform(1500.0, 4000.0, per)], 1)
        X = (Xc - ext[c, 3:]) @ Rc          # Rc^T (Xc - tc), the rig frame
        Y[c * per:(c + 1) * per] = (X - t0) @ R0   # R0^T (X - t0), the scene
        uv[c * per:(c + 1) * per] = np.stack([fcc[c, 0] * Xc[:, 0] / Xc[:, 2] + fcc[c, 1], fcc[c, 0] * Xc[:, 1] / Xc[:, 2] + fcc[c, 2]], 1)
    uv += rng.normal(scale=2.0, size=uv.shape)   # residuals, so that their curvature enters
    R, t = frozen_fit_rig(Y, uv, cam, ext, fcc, R0, t0)
    pose = np.concatenate([_log(R), t])
    D = rig_ift(cam, Y, uv, ext, fcc, pose)
    assert D is not None
    eps = 1e-3
    for i in rng.choice(len(Y), 12, replace=False):
        for j in range(3):
            Yp, Ym = Y.copy(), Y.copy()
            Yp[i, j] += eps
            Ym[i, j] -= eps
            num = (jp6(*frozen_fit_rig(Yp, uv, cam, ext, fcc, R, t)) - jp6(*frozen_fit_rig(Ym, uv, cam, ext, fcc, R, t))) / (2 * eps)
            assert np.allclose(D[i, :, j], num, rtol=0, atol=1e-6 * np.abs(num).max() + 1e-12), (i, j, D[i, :, j], num)
