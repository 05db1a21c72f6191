"""The RGB-D oracle's Kabsch refinement replay recording the cells its last accepted step fitted
(tests/host_shim/rgbd_record.cpp, built on tests/host_shim/rgbd_oracle.cpp and the unmodified oracle sources with the
flags of the oracle's parity build), into a temporary directory (the tree may be read-only)."""
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
        so = os.path.join(tempfile.mkdtemp(prefix="rgbd_record_"), "librgbd_record.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-ffp-contract=off",
                               "-shared", "-I", os.path.join(ROOT, "oracle"), "-I", os.path.join(ROOT, "tests", "host_shim"),
                               "-o", so, os.path.join(ROOT, "tests", "host_shim", "rgbd_record.cpp"), "-lpthread"])
        _lib = C.CDLL(so)
        _lib.rrec_refine_record.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 4
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def refine_record(cfg, coords, pix, eye, perm, n_perm, init):
    """(cv pose, recorded cells S in selection order, steps done) of the RGB-D refinement from the cv pose `init`, with the
    camera of cfg (f, cx, cy); eye [N][3], NaN without depth."""
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    eye = np.ascontiguousarray(eye, np.float64).reshape(N, 3)
    perm = np.ascontiguousarray(perm, np.int32).reshape(-1, N)
    init = np.ascontiguousarray(init, np.float64).reshape(6)
    pose = np.zeros(6)
    sel = np.zeros(max(cfg.inlier_count, 1), np.int32)
    cnt = C.c_int32(0)
    done = lib().rrec_refine_record(C.byref(cfg), _p(coords), _p(pix), _p(eye), _p(perm), int(n_perm), _p(init), _p(pose),
                                    _p(sel), C.byref(cnt))
    return pose, sel[:cnt.value].copy(), done
