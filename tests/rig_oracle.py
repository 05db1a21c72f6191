"""The CPU restatement of one multi-camera rig (tests/host_shim/rig_oracle.cpp): compiled from the unmodified oracle
sources plus the helper with the flags of the oracle's parity build, into a temporary directory (the tree may be
read-only)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="rig_oracle_"), "librig_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-ffp-contract=off",
                               "-shared", "-I", os.path.join(ROOT, "oracle"), "-o", so,
                               os.path.join(ROOT, "tests", "host_shim", "rig_oracle.cpp"), "-lpthread"])
        _lib = C.CDLL(so)
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def forward(cfg, coords, pix, intr, ext, hyp_pose, gt_jp=None, start=None):
    """One rig of C cameras: coords [C][N][3], pix [C][N][2], intr [C][3] (f, cx, cy), ext [C][6] (cam_from_rig),
    hyp_pose [C][H][6] (H = cfg.n_hyps), gt_jp [12] or None; start [6] or None: the pose the refinement starts from in
    place of the soft-argmax pose.  A dict of the rig's outputs as dsac_rig_out names them, plus min_margin: the smallest
    |error - thr2d| the refinement's selections tested."""
    C_ = len(ext)
    H = cfg.n_hyps
    coords = np.ascontiguousarray(coords, np.int16).reshape(C_, N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(C_, N, 2)
    intr = np.ascontiguousarray(intr, np.float64).reshape(C_, 3)
    ext = np.ascontiguousarray(ext, np.float64).reshape(C_, 6)
    hyp = np.ascontiguousarray(hyp_pose, np.float64).reshape(C_, H, 6)
    gt = np.ascontiguousarray(gt_jp, np.float64).reshape(12) if gt_jp is not None else None
    st = np.ascontiguousarray(start, np.float64).reshape(6) if start is not None else None
    o = {"rig_hyp": np.zeros((C_ * H, 6)), "scores": np.zeros(C_ * H), "sf": np.zeros(C_ * H), "entropy": np.zeros(1),
         "avg_pose": np.zeros(6), "ref_pose": np.zeros(6), "inlier_map": np.zeros((C_, N), np.int32),
         "steps_done": np.zeros(1, np.int32), "loss": np.zeros(1), "rot_err": np.zeros(1), "t_err": np.zeros(1),
         "correct": np.zeros(1, np.int32), "min_margin": np.zeros(1)}
    rc = lib().rig_forward(C.byref(cfg), C_, _p(coords), _p(pix), _p(intr), _p(ext), _p(hyp), _p(gt), _p(st),
                           *[_p(o[k]) for k in ("rig_hyp", "scores", "sf", "entropy", "avg_pose", "ref_pose", "inlier_map",
                                                "steps_done", "loss", "rot_err", "t_err", "correct", "min_margin")])
    assert rc == 0
    for k in ("entropy", "steps_done", "loss", "rot_err", "t_err", "correct", "min_margin"):
        o[k] = o[k][0]
    return o
