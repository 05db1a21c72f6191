"""Host references of rig tracking (dsac_set_rig_pose_priors_device, dsac_rig_pose_uncertainty_device), shared by
tests/test_rig_tracking_host.py and tests/test_gpu_rig_tracking.py: the host build of the device's fp64 arithmetic
(tests/host_shim/rig_tracking_shim.cpp) and independent numpy / scipy restatements of it."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from rig_grad_oracle import _rig_residuals, ext12, log, p, rot

HERE = os.path.dirname(os.path.abspath(__file__))
_shim = None


def shim():
    global _shim
    if _shim is None:
        so = os.path.join(tempfile.mkdtemp(prefix="rig_tracking_shim_"), "librig_tracking_shim.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                               os.path.join(HERE, "host_shim", "rig_tracking_shim.cpp")])
        lib = C.CDLL(so)
        lib.shim_prior_d2.restype = C.c_double
        _shim = lib
    return _shim


def _c(a):
    return np.ascontiguousarray(a, np.float64)


def compose(ext, pose, info=None):
    """The device's composition of one rig prior (pose [6], info [6][6] or None) with one extrinsic [6]: (ok, pose, info)."""
    op, oi = np.zeros(6), np.zeros(36)
    ok = shim().shim_rig_prior_compose(p(_c(ext)), p(_c(pose)), p(_c(info)) if info is not None else None, p(op), p(oi))
    return bool(ok), op, (oi.reshape(6, 6) if info is not None else None)


def compose_np(ext, pose, info=None):
    """The same composition in scipy: (R_c R_j, R_c t_j + t_c) and B Lambda B^T, B = blockdiag(R_c, R_c)."""
    Rc = rot(ext[:3])
    R = Rc @ rot(pose[:3])
    out = np.concatenate([log(R), Rc @ pose[3:] + ext[3:]])
    if info is None:
        return out, None
    B = np.zeros((6, 6))
    B[:3, :3] = Rc
    B[3:, 3:] = Rc
    return out, B @ info @ B.T


def prior_d2(hyp, pose, info):
    """xi^T Lambda xi of the cv pose hyp against the prior (pose, info) in the device's arithmetic; -1 if refused."""
    return shim().shim_prior_d2(p(_c(hyp)), p(_c(pose)), p(_c(info)))


def lift(ext, hyp):
    """The cv rig pose of camera pose hyp [6] behind the extrinsic ext [6]: (R_c^T R_h, R_c^T (t_h - t_c))."""
    Rc = rot(ext[:3])
    return np.concatenate([log(Rc.T @ rot(hyp[:3])), Rc.T @ (hyp[3:] - ext[3:])])


def rig_cov(cam, Y, uv, ext, fcc, pose):
    """The device's rig fit covariance over cells (cam, Y, uv) at the cv rig pose: (ok, cov_xi, cov_jp6, sigma2)."""
    cx, cj, s2 = np.zeros(36), np.zeros(36), np.zeros(1)
    ok = shim().shim_rig_fit_covariance(len(Y), p(np.ascontiguousarray(cam, np.int32)), p(_c(Y)), p(_c(uv)), p(ext12(ext)),
                                        p(_c(fcc)), p(_c(pose)), p(cx), p(cj), p(s2))
    return bool(ok), cx.reshape(6, 6), cj.reshape(6, 6), s2[0]


def fit_cov(Y, uv, fcc, pose):
    """ift_fit_covariance (RGB) of one camera: (ok, cov_xi, cov_jp6, sigma2)."""
    cx, cj, s2 = np.zeros(36), np.zeros(36), np.zeros(1)
    ok = shim().shim_fit_covariance(len(Y), p(_c(Y)), p(_c(uv)), p(_c(fcc)), p(_c(pose)), p(cx), p(cj), p(s2))
    return bool(ok), cx.reshape(6, 6), cj.reshape(6, 6), s2[0]


def rig_cov_np(cam, Y, uv, ext, fcc, pose, eps=1e-6):
    """sigma2 (J^T J)^-1 in numpy, J the central differences of the rig residuals (rig_grad_oracle's model) in the chart
    R = exp([w]x) R*, t = t* + tau: (cov_xi, sigma2)."""
    R0, t0 = rot(pose[:3]), pose[3:]

    def res(xi):
        return _rig_residuals(Y, uv, cam, ext, fcc, rot(xi[:3]) @ R0, t0 + xi[3:])[3].reshape(-1)

    J = np.zeros((2 * len(Y), 6))
    for a in range(6):
        d = np.zeros(6)
        d[a] = eps if a < 3 else eps * 1e3
        J[:, a] = (res(d) - res(-d)) / (2 * d[a])
    r = res(np.zeros(6))
    s2 = r @ r / (2 * len(Y) - 6)
    return s2 * np.linalg.inv(J.T @ J), s2
