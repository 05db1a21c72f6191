"""Host references for RGB-D rigs, shared by tests/test_rig_rgbd_host.py and tests/test_gpu_rig_rgbd.py:
- lib(): the CPU restatement of one RGB-D rig's refinement (tests/host_shim/rig_rgbd_oracle.cpp), compiled from the
  unmodified oracle sources and the RGB rig restatement with the flags of the oracle's parity build;
- shim(): the product's RGB-D rig arithmetic built for the host (tests/host_shim/rig_rgbd_shim.cpp);
- the seeded synthetic RGB-D rig scene the tests use.
Both libraries are compiled once per process into a temporary directory (the tree may be read-only)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
from scipy.spatial.transform import Rotation

import rig_oracle as RO
from rig_grad_oracle import ext12, ring

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600
_lib = _shim = None


def _cxx():
    return "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="rig_rgbd_oracle_"), "librig_rgbd_oracle.so")
        subprocess.check_call([_cxx(), "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-ffp-contract=off",
                               "-shared", "-I", os.path.join(ROOT, "oracle"), "-I", os.path.join(ROOT, "tests", "host_shim"),
                               "-o", so, os.path.join(ROOT, "tests", "host_shim", "rig_rgbd_oracle.cpp"), "-lpthread"])
        _lib = C.CDLL(so)
    return _lib


def shim():
    global _shim
    if _shim is None:
        so = os.path.join(tempfile.mkdtemp(prefix="rig_rgbd_shim_"), "librig_rgbd_shim.so")
        subprocess.check_call([_cxx(), "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                               os.path.join(ROOT, "tests", "host_shim", "rig_rgbd_shim.cpp")])
        _shim = C.CDLL(so)
        _shim.shim_rig_point.restype = None
        _shim.shim_rig_kabsch.restype = None
    return _shim


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _f64(a, shape):
    return np.ascontiguousarray(a, np.float64).reshape(shape)


def eye(pix, depth, intr):
    """Eye points float64 [C][N][3] of C camera frames (k_rgbd_eye_t's rule: NaN without depth): pix [C][N][2], depth
    float32 [C][N] (mm), intr [C][3] (f, cx, cy)."""
    pix = np.asarray(pix, np.float64).reshape(-1, N, 2)
    d = np.asarray(depth, np.float32).reshape(-1, N).astype(np.float64)
    intr = np.asarray(intr, np.float64).reshape(-1, 3)
    f, cx, cy = intr[:, :1], intr[:, 1:2], intr[:, 2:]
    ok = np.isfinite(d) & (d > 0)
    out = np.stack([(pix[..., 0] - cx) * d / f, (pix[..., 1] - cy) * d / f, d], -1)
    out[~ok] = np.nan
    return out


def refine(cfg, coords, pix, intr, ext, ey, start):
    """The RGB-D rig refinement of one rig of C cameras from the cv rig pose `start`: a dict of ref_pose [6], inlier_map
    [C][N], steps_done and min_margin."""
    C_ = len(ext)
    o = {"ref_pose": np.zeros(6), "inlier_map": np.zeros((C_, N), np.int32), "steps_done": np.zeros(1, np.int32),
         "min_margin": np.zeros(1)}
    rc = lib().rig_rgbd_refine(C.byref(cfg), C_, _p(np.ascontiguousarray(coords, np.int16).reshape(C_, N, 3)),
                               _p(np.ascontiguousarray(pix, np.int32).reshape(C_, N, 2)), _p(_f64(intr, (C_, 3))),
                               _p(_f64(ext, (C_, 6))), _p(_f64(ey, (C_, N, 3))), _p(_f64(start, 6)),
                               *[_p(o[k]) for k in ("ref_pose", "inlier_map", "steps_done", "min_margin")])
    assert rc == 0
    o["steps_done"], o["min_margin"] = int(o["steps_done"][0]), float(o["min_margin"][0])
    return o


def forward(cfg, coords, pix, intr, ext, hyp_pose, ey, start=None):
    """One RGB-D rig from the frames' hypotheses: the pool, scores, sf, entropy and soft-argmax pose of the RGB rig oracle
    (the score is the same reprojection score), and the RGB-D refinement from `start` or the soft-argmax pose."""
    o = RO.forward(cfg, coords, pix, intr, ext, hyp_pose)
    for k in ("ref_pose", "inlier_map", "steps_done", "min_margin", "loss", "rot_err", "t_err", "correct"):
        del o[k]
    o.update(refine(cfg, coords, pix, intr, ext, ey, o["avg_pose"] if start is None else start))
    return o


def last_step_cells(cfg, coords, pix, intr, ext, ey, start, steps):
    """The (camera, cell) pairs of the last accepted step of the RGB-D rig refinement from `start`, `steps` accepted: the
    oracle's inlier map after `steps` steps minus that after steps - 1; the smaller threshold margin and the final run."""
    runs = []
    ref_steps = cfg.ref_steps
    for k in (steps - 1, steps):
        cfg.ref_steps = k
        runs.append(refine(cfg, coords, pix, intr, ext, ey, start))
    cfg.ref_steps = ref_steps
    diff = runs[1]["inlier_map"] - runs[0]["inlier_map"]
    assert diff.min() >= 0 and diff.max() <= 1
    cam, cell = np.nonzero(diff)
    return cam, cell, min(r["min_margin"] for r in runs), runs[1]


def rig_point(ext, e):
    """The shim's rig-frame point of camera-frame point e [3] behind the cv extrinsic ext [6]."""
    E = ext12(np.asarray(ext, np.float64).reshape(1, 6))[0]
    o = np.zeros(3)
    shim().shim_rig_point(_p(E[:9].copy()), _p(E[9:].copy()), _p(_f64(e, 3)), _p(o))
    return o


def kabsch(cam, Y, e, ext):
    """The shim's rig Kabsch fit (cv rig pose [6]) over cells (cam [m], Y [m][3], camera-frame eye points e [m][3])."""
    pose = np.zeros(6)
    shim().shim_rig_kabsch(len(Y), _p(np.ascontiguousarray(cam, np.int32)), _p(_f64(Y, (-1, 3))), _p(_f64(e, (-1, 3))),
                           _p(ext12(np.asarray(ext, np.float64).reshape(-1, 6))), _p(pose))
    return pose


def ift(cam, Y, e, ext, pose):
    """The shim's d jp6 / dY [m][6][3] of the rig Kabsch fit at the cv rig pose; None if it is not defined."""
    D = np.zeros((len(Y), 6, 3))
    ok = shim().shim_rig_rgbd_ift_deriv(len(Y), _p(np.ascontiguousarray(cam, np.int32)), _p(_f64(Y, (-1, 3))), _p(_f64(e, (-1, 3))),
                                        _p(ext12(np.asarray(ext, np.float64).reshape(-1, 6))), _p(_f64(pose, 6)), _p(D))
    return D if ok else None


def cov(cam, Y, e, ext, pose):
    """The shim's (ok, cov_xi, cov_jp6, sigma2) of the rig Kabsch fit at the cv rig pose."""
    cx, cj, s2 = np.zeros((6, 6)), np.zeros((6, 6)), np.zeros(1)
    ok = shim().shim_rig_rgbd_fit_covariance(len(Y), _p(np.ascontiguousarray(cam, np.int32)), _p(_f64(Y, (-1, 3))),
                                             _p(_f64(e, (-1, 3))), _p(ext12(np.asarray(ext, np.float64).reshape(-1, 6))),
                                             _p(_f64(pose, 6)), _p(cx), _p(cj), _p(s2))
    return bool(ok), cx, cj, s2[0]


def fit_cov(Y, e, pose):
    """ift_fit_covariance(rgbd=true) of one camera's cells: (ok, cov_xi, cov_jp6, sigma2)."""
    cx, cj, s2 = np.zeros((6, 6)), np.zeros((6, 6)), np.zeros(1)
    ok = shim().shim_fit_covariance_rgbd(len(Y), _p(_f64(Y, (-1, 3))), _p(_f64(e, (-1, 3))), _p(_f64(pose, 6)), _p(cx), _p(cj), _p(s2))
    return bool(ok), cx, cj, s2[0]


def scene(C_, R, seed=0, inliers=0.6, holes=0.0, noise=0.5, f=525.0, cx=320.0, cy=240.0):
    """R consistent RGB-D rigs of C ring cameras: every cell has depth U(1500, 4000) mm at its grid pixel, a fraction
    `inliers` of them a scene point at the rig's true pose (the eye point, with `noise` px of pixel noise), the rest random
    scene points; a fraction `holes` has no depth (NaN).  (coords [n][N][3] int16, pix [n][N][2] int32, depth [n][N]
    float32, ext [n][6], gt_rig [R][12] jp, true [R][6] cv rig poses)."""
    rng = np.random.default_rng(seed)
    n = R * C_
    pix = np.zeros((n, N, 2), np.int32)
    xs, ys = (np.arange(N) % 40) * 16 + 8, (np.arange(N) // 40) * 12 + 6
    coords = np.empty((n, N, 3), np.int16)
    depth = np.empty((n, N), np.float32)
    ext = np.concatenate([ring(C_, seed=seed + r) for r in range(R)])
    gt, true = np.empty((R, 12)), np.empty((R, 6))
    for r in range(R):
        true[r] = np.concatenate([Rotation.from_euler("xyz", rng.normal(scale=0.2, size=3)).as_rotvec(),
                                  rng.normal(scale=300.0, size=3) + [0.0, 0.0, 1500.0]])
        Rt = Rotation.from_rotvec(true[r, :3]).as_matrix().copy()
        Rt[1:] = -Rt[1:]
        gt[r] = np.concatenate([Rt.ravel(), true[r, 3:] * [1, -1, -1]])
        for c in range(C_):
            fr = r * C_ + c
            pix[fr, :, 0] = xs + rng.integers(-4, 5, N)
            pix[fr, :, 1] = ys + rng.integers(-3, 4, N)
            u = pix[fr, :, 0] + rng.normal(scale=noise, size=N)
            v = pix[fr, :, 1] + rng.normal(scale=noise, size=N)
            d = rng.uniform(1500.0, 4000.0, size=N)
            Xc = np.stack([(u - cx) / f * d, (v - cy) / f * d, d], 1)
            Rc, tc = Rotation.from_rotvec(ext[fr, :3]), ext[fr, 3:]
            Rr = Rotation.from_rotvec(true[r, :3])
            cam_R, cam_t = Rc * Rr, Rc.apply(true[r, 3:]) + tc
            X = cam_R.inv().apply(Xc - cam_t)
            out = rng.uniform(size=N) >= inliers
            X[out] = rng.uniform(-4000.0, 4000.0, size=(out.sum(), 3))
            coords[fr] = np.clip(np.round(X), -32767, 32767).astype(np.int16)
            dd = d.astype(np.float32)
            dd[rng.uniform(size=N) < holes] = np.nan
            depth[fr] = dd
    return coords, pix, depth, ext, gt, true
