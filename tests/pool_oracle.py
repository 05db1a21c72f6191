"""The oracle's pipelines from a given hypothesis pool (tests/host_shim/pool_oracle.cpp), for the pose priors: compiled
from the unmodified oracle sources plus the helper with the flags of the oracle's parity build, into a temporary directory
(the tree may be read-only).  The result objects are oracle.oracle's, so a pool result feeds the pool backward exactly as
an oracle forward feeds the oracle backward."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="pool_oracle_"), "libpool_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-ffp-contract=off",
                               "-shared", "-I", os.path.join(ROOT, "oracle"), "-o", so,
                               os.path.join(ROOT, "tests", "host_shim", "pool_oracle.cpp"), "-lpthread"])
        _lib = C.CDLL(so)
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _frame(coords, pix, gt_R, gt_t):
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    gR = np.ascontiguousarray(gt_R, np.float64).reshape(9)
    gt = np.ascontiguousarray(gt_t, np.float64).reshape(3)
    return coords, pix, gR, gt


def forward(cfg, coords, pix, gt_R, gt_t, hyp_pose, img_idx):
    """Soft-argmax forward of the pool hyp_pose [H][6] (cv), img_idx [H][4] (-1: no minimal set): an O.Forward."""
    coords, pix, gR, gt = _frame(coords, pix, gt_R, gt_t)
    out = O.Forward(cfg, want_diffmaps=False)
    out.hyp_rvec[:] = hyp_pose[:, :3]; out.hyp_tvec[:] = hyp_pose[:, 3:]; out.img_idx[:] = img_idx; out.cand_idx[:] = -1
    lib().por_forward(C.byref(cfg), _p(coords), _p(pix), _p(gR), _p(gt), C.byref(out.raw))
    out._keep = (coords, pix)
    return out


def forward_dsac(cfg, coords, pix, gt_R, gt_t, hyp_pose, img_idx):
    """DSAC-variant forward (arg-max draw) of the pool: an O.ForwardDsac."""
    coords, pix, gR, gt = _frame(coords, pix, gt_R, gt_t)
    out = O.ForwardDsac(cfg)
    out.hyp_rvec[:] = hyp_pose[:, :3]; out.hyp_tvec[:] = hyp_pose[:, 3:]; out.img_idx[:] = img_idx
    lib().por_forward_dsac(C.byref(cfg), _p(coords), _p(pix), _p(gR), _p(gt), C.byref(out.raw))
    return out


def backward(cfg, coords, pix, gt_R, gt_t, fwd):
    coords, pix, gR, gt = _frame(coords, pix, gt_R, gt_t)
    out = O.Backward(cfg)
    lib().por_backward(C.byref(cfg), _p(coords), _p(pix), _p(gR), _p(gt), C.byref(fwd.raw), C.byref(out.raw))
    return out


def backward_dsac(cfg, coords, pix, gt_R, gt_t, fwd, n_prior):
    coords, pix, gR, gt = _frame(coords, pix, gt_R, gt_t)
    out = O.BackwardDsac(cfg)
    lib().por_backward_dsac(C.byref(cfg), _p(coords), _p(pix), _p(gR), _p(gt), C.c_int(n_prior), C.byref(fwd.raw),
                            C.byref(out.raw))
    return out
