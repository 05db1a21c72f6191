"""The oracle's refinement replay recording the cells its last accepted step fitted (tests/host_shim/ift_oracle.cpp),
compiled from the unmodified oracle sources plus the helper with the flags of the oracle's parity build, into a temporary
directory (the tree may be read-only); and a frozen-set solver: the stationary point of the last step's fit over a fixed
set of cells by Gauss-Newton in numpy, independent of the product's implicit-function code."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600
DFLIP = np.diag([1.0, -1.0, -1.0])
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="ift_oracle_"), "libift_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-ffp-contract=off",
                               "-shared", "-I", os.path.join(ROOT, "oracle"), "-o", so,
                               os.path.join(ROOT, "tests", "host_shim", "ift_oracle.cpp"), "-lpthread"])
        _lib = C.CDLL(so)
        _lib.ior_refine_record.argtypes = [C.c_void_p] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 4
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def refine_record(cfg, coords, pix, perm, n_perm, init):
    """(cv pose, recorded cells S in selection order, steps done) of refine() from the cv pose `init`."""
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    perm = np.ascontiguousarray(perm, np.int32).reshape(-1, N)
    init = np.ascontiguousarray(init, np.float64).reshape(6)
    pose = np.zeros(6)
    sel = np.zeros(max(cfg.inlier_count, 1), np.int32)
    cnt = C.c_int32(0)
    done = lib().ior_refine_record(C.byref(cfg), _p(coords), _p(pix), _p(perm), int(n_perm), _p(init), _p(pose), _p(sel),
                                   C.byref(cnt))
    return pose, sel[:cnt.value].copy(), done


def jp6(R, t):
    """jp 6-vector of a cv pose (R, t): (rotation vector of D R, D t)."""
    return np.concatenate([Rotation.from_matrix(DFLIP @ R).as_rotvec(), DFLIP @ t])


def frozen_fit(Y, e, R, t, cam, rgbd, iters=200):
    """Stationary point of sum |pi(R Y + t) - p|^2 (RGB, e[:, :2] = p) or sum |R Y + t - e|^2 (RGB-D) over the frozen
    set, by Gauss-Newton in the left chart, to a step below 1e-14."""
    f, cx, cy = cam
    for _ in range(iters):
        q = Y @ R.T
        X = q + t
        dX = np.zeros((len(Y), 3, 6))
        dX[:, 0, 1], dX[:, 0, 2] = q[:, 2], -q[:, 1]
        dX[:, 1, 0], dX[:, 1, 2] = -q[:, 2], q[:, 0]
        dX[:, 2, 0], dX[:, 2, 1] = q[:, 1], -q[:, 0]
        dX[:, :, 3:] = np.eye(3)
        if rgbd:
            J, r = dX, X - e
        else:
            z = X[:, 2]
            g = np.zeros((len(Y), 2, 3))
            g[:, 0, 0] = f / z; g[:, 0, 2] = -f * X[:, 0] / z ** 2
            g[:, 1, 1] = f / z; g[:, 1, 2] = -f * X[:, 1] / z ** 2
            J = g @ dX
            r = np.stack([f * X[:, 0] / z + cx, f * X[:, 1] / z + cy], 1) - e[:, :2]
        J, r = J.reshape(-1, 6), r.reshape(-1)
        step = -np.linalg.solve(J.T @ J, J.T @ r)
        R = Rotation.from_rotvec(step[:3]).as_matrix() @ R
        t = t + step[3:]
        if np.abs(step).max() < 1e-14:
            break
    return R, t


def frozen_derivative(Y, e, pose_cv, cam, rgbd, cells, eps=1e-3):
    """Central differences (eps mm) of the frozen-set solution's jp 6-vector with respect to Y[cells]: [len(cells)][6][3]."""
    R0 = Rotation.from_rotvec(pose_cv[:3]).as_matrix()
    R, t = frozen_fit(Y, e, R0, np.asarray(pose_cv[3:], np.float64), cam, rgbd)
    out = np.zeros((len(cells), 6, 3))
    for k, i in enumerate(cells):
        for j in range(3):
            Yp, Ym = Y.copy(), Y.copy()
            Yp[i, j] += eps; Ym[i, j] -= eps
            out[k, :, j] = (jp6(*frozen_fit(Yp, e, R, t, cam, rgbd)) - jp6(*frozen_fit(Ym, e, R, t, cam, rgbd))) / (2 * eps)
    return out
