"""The CPU restatement of RGB-D localisation (tests/rgbd_oracle.py) on its own: eye coordinates, the Kabsch acceptance
test and the forward pass on noise-free frames."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import rgbd_oracle as R

N = 1600


@pytest.mark.parametrize("cam", [(525.0, 320.0, 240.0), (600.5, 301.25, 255.75)])
def test_eye_matches_numpy(cam):
    f, cx, cy = cam
    coords, pix, depth, _, _ = R.synth(1, seed=1, holes=0.2, cams=np.array([cam]))
    ey, have = R.eye(pix[0], depth[0], f, cx, cy)
    d = depth[0].astype(np.float64)
    ok = np.isfinite(d) & (d > 0)
    want = np.stack([(pix[0, :, 0] - cx) * d / f, (pix[0, :, 1] - cy) * d / f, d], 1)
    assert have == ok.sum()
    assert np.array_equal(ey[ok], want[ok])
    assert np.isnan(ey[~ok]).all()
    d[:3] = [0.0, -5.0, np.inf]
    ey2, _ = R.eye(pix[0], d.astype(np.float32), f, cx, cy)
    assert np.isnan(ey2[:3]).all()


def _exact_frame():
    """One noise-free frame: every cell an inlier of the pose, with depth."""
    coords, pix, depth, gt_cv, gt_jp = R.synth(1, seed=2, rho=1.0, sigma=0.0)
    return coords[0], pix[0], depth[0], gt_cv[0], gt_jp[0]


def test_accept_recovers_rigid_transform(oracle):
    coords, pix, depth, gt_cv, _ = _exact_frame()
    cfg = oracle.default_config()
    ey, _ = R.eye(pix, depth)
    # the scene points of the fixture are rounded to mm: fit the exact transform to the rounded points' eye images
    Rm = Rotation.from_rotvec(gt_cv[:3]).as_matrix()
    ey = coords.astype(np.float64) @ Rm.T + gt_cv[3:]
    ok, r, t, _ = R.accept(cfg, coords, pix, ey, [10, 700, 1400, 333])
    assert ok
    assert np.abs(r - gt_cv[:3]).max() < 1e-9
    assert np.abs(t - gt_cv[3:]).max() < 1e-9 * 1e3


def test_accept_rejects_degenerate_and_missing(oracle):
    coords, pix, depth, gt_cv, _ = _exact_frame()
    cfg = oracle.default_config()
    ey, _ = R.eye(pix, depth)
    assert R.accept(cfg, coords, pix, ey, [10, 700, 1400, 333])[0]
    assert not R.accept(cfg, coords, pix, ey, [10, 10, 1400, 333])[0]          # duplicate cell
    col = coords.copy()
    col[1400] = 2 * col[700].astype(np.int32) - col[10]                         # scene points collinear
    assert not R.accept(cfg, col, pix, ey, [10, 700, 1400, 333])[0]
    d = depth.copy()
    d[333] = np.nan                                                              # 4th cell without depth
    ey2, _ = R.eye(pix, d)
    assert not R.accept(cfg, coords, pix, ey2, [10, 700, 1400, 333])[0]
    behind = ey.copy()
    behind[:, 2] *= -1                                                           # every point behind the camera
    assert not R.accept(cfg, coords, pix, behind, [10, 700, 1400, 333])[0]


def test_forward_noise_free_is_correct(oracle):
    # (outliers that happen to reproject within thr2d would enter the refinement's 3D fit: none here)
    coords, pix, depth, _, gt_jp = R.synth(2, seed=3, rho=1.0, sigma=0.0)
    cfg = oracle.default_config(n_hyps=64, n_streams=2)
    for g in range(2):
        ey, _ = R.eye(pix[g], depth[g])
        fw, ncand = R.forward(oracle, cfg, g, coords[g], pix[g], ey, None, gt_jp[g, :9], gt_jp[g, 9:])
        assert fw.status == 0
        assert fw.correct == 1 and fw.loss < 0.1, (fw.rot_err, fw.t_err)
        assert (fw.img_idx >= 0).all() and ncand.sum() == fw.n_candidates


def test_frame_without_depth_samples_nothing(oracle):
    coords, pix, depth, _, _ = R.synth(1, seed=4)
    d = np.full(N, np.nan, np.float32)
    d[:3] = 1000
    ey, have = R.eye(pix[0], d)
    assert have == 3
    fw, ncand = R.forward(oracle, oracle.default_config(n_hyps=16), 0, coords[0], pix[0], ey)
    assert fw.status == -2 and fw.n_candidates == 0 and (fw.img_idx == -1).all()


def test_backward_reference_runs(oracle):
    """Both backward passes of the CPU reference on one RGB-D frame: finite, nonzero, and the dPNP columns of the 4th
    point are zero (the Kabsch hypothesis does not use it)."""
    coords, pix, depth, _, gt_jp = R.synth(1, seed=5, holes=0.1)
    ey, _ = R.eye(pix[0], depth[0])
    cfg = oracle.default_config(n_hyps=16, n_streams=1)
    fw, _ = R.forward(oracle, cfg, 0, coords[0], pix[0], ey, None, gt_jp[0, :9], gt_jp[0, 9:])
    bw = R.backward(oracle, cfg, coords[0], pix[0], ey, gt_jp[0, :9], gt_jp[0, 9:], fw)
    assert np.isfinite(bw.dloss_dobj).all() and np.abs(bw.dloss_dobj).max() > 0
    assert np.abs(bw.dpnp[:, :, 9:]).max() == 0 and np.abs(bw.dpnp[:, :, :9]).max() > 0
    fd = R.forward_dsac(oracle, cfg, 0, coords[0], pix[0], ey, gt_jp[0, :9], gt_jp[0, 9:], True)
    assert np.array_equal(fd.img_idx, fw.img_idx)
    bd = R.backward_dsac(oracle, cfg, coords[0], pix[0], ey, gt_jp[0, :9], gt_jp[0, 9:], fd)
    assert np.isfinite(bd.dloss_dobj).all() and bd.n_selected > 0 and np.abs(bd.path1).max() > 0


@pytest.mark.parametrize("shared", [True, False])
def test_cell_depth_helper_matches_numpy(shared):
    import torch
    from dsac_b200 import autograd as A
    rng = np.random.default_rng(9)
    n, Hh, W = 3, 48, 64
    d = rng.integers(0, 65536, (n, Hh, W)).astype(np.uint16)
    d[:, ::5, ::7] = 0
    d[:, 1::5, ::3] = 65535
    pix = rng.integers(-3, 70, (1 if shared else n, N, 2)).astype(np.int32)
    want = np.full((n, N), np.nan, np.float32)
    for f in range(n):
        p = pix[0 if shared else f]
        x, y = p[:, 0], p[:, 1]
        ok = (x >= 0) & (x < W) & (y >= 0) & (y < Hh)
        v = np.zeros(N, np.int64)
        v[ok] = d[f, y[ok], x[ok]]
        ok &= (v != 0) & (v != 65535)
        want[f, ok] = v[ok]
    for depth in (torch.from_numpy(d.astype(np.int32)), torch.from_numpy(d.view(np.int16))):   # int16 storage of uint16
        got = A.cell_depth(depth, torch.from_numpy(pix[0] if shared else pix)).numpy()
        assert np.array_equal(got, want, equal_nan=True)
