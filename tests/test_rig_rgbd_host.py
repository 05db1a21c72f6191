"""The RGB-D rig arithmetic on the host (tests/host_shim/rig_rgbd_shim.cpp, the product's code built for the host): the
rig-frame eye point's exact identities, the rig Kabsch fit against the truth and against a least-squares solve of the
camera-frame objective, its implicit-function derivative against central differences of the fit over a frozen cell set,
and its covariance against numpy; and the CPU restatement of an RGB-D rig (tests/host_shim/rig_rgbd_oracle.cpp) against
the RGB-D oracle's refinement for one camera behind a zero extrinsic."""
import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation

import rgbd_oracle as RD
import rig_rgbd_oracle as RR
from ift_oracle import jp6
from rig_grad_oracle import ring, rot

N = 1600


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def test_zero_rvec_extrinsic_gives_the_difference_exactly():
    rng = np.random.default_rng(1)
    for _ in range(200):
        e = rng.normal(scale=2000.0, size=3)
        tc = rng.normal(scale=100.0, size=3)
        got = RR.rig_point(np.concatenate([[0.0, 0.0, 0.0], tc]), e)
        assert np.array_equal(_bits(got), _bits(e - tc))
        assert np.array_equal(_bits(RR.rig_point(np.zeros(6), e)), _bits(e))
        # any other extrinsic: Rc^T (e - tc)
        ext = np.concatenate([Rotation.random(random_state=rng).as_rotvec(), tc])
        assert np.allclose(RR.rig_point(ext, e), rot(ext[:3]).T @ (e - tc), rtol=0, atol=1e-9)
    e = np.array([-0.0, 5.0, np.nan])   # a signed zero, and a cell without depth
    assert np.array_equal(_bits(RR.rig_point(np.zeros(6), e)), _bits(e))


def _cells(C_, per, rng, pose, ext, noise):
    """per cells per camera of a rig at cv pose `pose`: (cam, Y scene, e camera-frame eye points)."""
    R0, t0 = rot(pose[:3]), pose[3:]
    cam = np.repeat(np.arange(C_), per).astype(np.int32)
    Y, e = np.zeros((C_ * per, 3)), np.zeros((C_ * per, 3))
    for c in range(C_):
        Rc = rot(ext[c, :3])
        Xc = np.stack([rng.normal(scale=600.0, size=per), rng.normal(scale=500.0, size=per), rng.uniform(1500.0, 4000.0, per)], 1)
        X = (Xc - ext[c, 3:]) @ Rc             # Rc^T (Xc - tc), the rig frame
        Y[c * per:(c + 1) * per] = (X - t0) @ R0   # R0^T (X - t0), the scene
        e[c * per:(c + 1) * per] = Xc
    e += rng.normal(scale=noise, size=e.shape)
    return cam, Y, e


def _pose(rng):
    return np.concatenate([Rotation.from_euler("xyz", rng.normal(scale=0.3, size=3)).as_rotvec(), rng.normal(scale=300.0, size=3)])


@pytest.mark.parametrize("C_", [2, 4, 8])
def test_rig_kabsch_recovers_the_rig_pose(C_):
    rng = np.random.default_rng(30 + C_)
    ext = ring(C_, seed=C_)
    pose = _pose(rng)
    cam, Y, e = _cells(C_, 30, rng, pose, ext, 0.0)
    got = RR.kabsch(cam, Y, e, ext)
    assert np.abs(got[:3] - pose[:3]).max() < 1e-9
    assert np.abs(got[3:] - pose[3:]).max() < 1e-9 * 1e3


@pytest.mark.parametrize("C_", [2, 4, 8])
def test_rig_kabsch_is_the_least_squares_minimiser_of_the_camera_frame_objective(C_):
    rng = np.random.default_rng(40 + C_)
    ext = ring(C_, seed=C_ + 1)
    pose = _pose(rng)
    cam, Y, e = _cells(C_, 40, rng, pose, ext, 15.0)
    got = RR.kabsch(cam, Y, e, ext)
    Rc, tc = rot(ext[cam, :3]), ext[cam, 3:]

    def res(x):
        X = Y @ rot(x[:3]).T + x[3:]
        return (np.einsum("nij,nj->ni", Rc, X) + tc - e).ravel()

    ls = least_squares(res, pose + rng.normal(scale=[0.01] * 3 + [5.0] * 3), xtol=1e-15, ftol=1e-15, gtol=1e-15).x
    assert np.abs(got - ls).max() <= 1e-6 * np.abs(ls).max()
    assert np.sum(res(got) ** 2) <= np.sum(res(ls) ** 2) * (1 + 1e-12)


@pytest.mark.parametrize("C_", [2, 4, 8])
def test_rig_rgbd_ift_matches_frozen_set_central_differences(C_):
    """The RGB-D twin of test_rig_ift_matches_frozen_set_central_differences: the fit over a frozen set is the closed-form
    rig Kabsch fit itself, so its central differences need no iterative solve."""
    rng = np.random.default_rng(50 + C_)
    ext = ring(C_, seed=C_ + 2)
    cam, Y, e = _cells(C_, 25, rng, _pose(rng), ext, 20.0)   # residuals, so that their curvature enters
    pose = RR.kabsch(cam, Y, e, ext)
    D = RR.ift(cam, Y, e, ext, pose)
    assert D is not None

    def jp(p):
        return jp6(rot(p[:3]), p[3:])

    eps = 1e-3
    for i in rng.choice(len(Y), 12, replace=False):
        for j in range(3):
            Yp, Ym = Y.copy(), Y.copy()
            Yp[i, j] += eps
            Ym[i, j] -= eps
            num = (jp(RR.kabsch(cam, Yp, e, ext)) - jp(RR.kabsch(cam, Ym, e, ext))) / (2 * eps)
            assert np.allclose(D[i, :, j], num, rtol=0, atol=1e-6 * np.abs(num).max() + 1e-12), (i, j, D[i, :, j], num)


@pytest.mark.parametrize("C_", [1, 3, 8])
def test_rig_rgbd_covariance_matches_numpy(C_):
    rng = np.random.default_rng(60 + C_)
    ext = ring(C_, seed=C_ + 3)
    cam, Y, e = _cells(C_, 30, rng, _pose(rng), ext, 10.0)
    pose = RR.kabsch(cam, Y, e, ext)
    ok, cov_xi, cov_jp6, s2 = RR.cov(cam, Y, e, ext, pose)
    assert ok
    R0, t0 = rot(pose[:3]), pose[3:]
    Rc, tc = rot(ext[cam, :3]), ext[cam, 3:]

    def res(xi):   # camera-frame residuals in the rig chart R = exp([w]x) R0, t = t0 + tau
        X = Y @ (rot(xi[:3]) @ R0).T + t0 + xi[3:]
        return (np.einsum("nij,nj->ni", Rc, X) + tc - e).ravel()

    J = np.zeros((3 * len(Y), 6))
    for a in range(6):
        d = np.zeros(6)
        d[a] = 1e-6
        J[:, a] = (res(d) - res(-d)) / 2e-6
    r = res(np.zeros(6))
    want_s2 = r @ r / (3 * len(Y) - 6)
    want = want_s2 * np.linalg.inv(J.T @ J)
    assert abs(s2 - want_s2) <= 1e-9 * want_s2
    assert np.allclose(cov_xi, want, rtol=0, atol=1e-6 * np.abs(want).max())
    assert np.array_equal(cov_xi, cov_xi.T) and np.array_equal(cov_jp6, cov_jp6.T)


def test_one_camera_behind_an_identity_is_the_rgbd_fit_covariance_bit_for_bit():
    rng = np.random.default_rng(70)
    cam, Y, e = _cells(1, 60, rng, _pose(rng), np.zeros((1, 6)), 10.0)
    pose = RR.kabsch(cam, Y, e, np.zeros((1, 6)))
    a, b = RR.cov(cam, Y, e, np.zeros((1, 6)), pose), RR.fit_cov(Y, e, pose)
    assert a[0] and b[0]
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(_bits(np.asarray(x)), _bits(np.asarray(y)))


@pytest.mark.parametrize("seed,holes", [(3, 0.0), (4, 0.3)])
def test_oracle_one_camera_zero_extrinsic_is_the_rgbd_oracle(oracle, seed, holes):
    """rig_rgbd_oracle.cpp with C = 1 and a zero extrinsic against rgbd_oracle.cpp's forward pass: the pool, scores and
    soft-argmax pose of the RGB rig restatement and the RGB-D rig refinement give its outputs bit for bit."""
    O = oracle
    coords, pix, depth, gt_cv, gt_jp = RD.synth(1, seed=seed, holes=holes)
    cfg = O.default_config(n_hyps=64, n_streams=4)
    ey, _ = RD.eye(pix[0], depth[0])
    fwd, _ = RD.forward(O, cfg, 0, coords[0], pix[0], ey)
    assert fwd.status == 0 and fwd.ref_steps_done > 0
    hyp = np.concatenate([fwd.hyp_rvec, fwd.hyp_tvec], 1)
    intr = np.array([[cfg.f, cfg.cx, cfg.cy]])
    rig = RR.forward(cfg, coords, pix, intr, np.zeros((1, 6)), hyp[None], ey[None])
    assert np.array_equal(_bits(rig["scores"]), _bits(fwd.scores))
    assert np.array_equal(_bits(rig["avg_pose"]), _bits(fwd.avg))
    assert np.array_equal(_bits(rig["ref_pose"]), _bits(fwd.ref))
    assert np.array_equal(rig["inlier_map"][0], fwd.inlier_map)
    assert rig["steps_done"] == fwd.ref_steps_done
