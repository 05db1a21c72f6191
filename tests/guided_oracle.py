"""Guided sampling restated on the CPU (tests/host_shim/guided_oracle.cpp), the reference the engine's guided passes are
checked against: weight table, Philox4x32-10, the draw rule, orc_forward with the guided draw, and the log-probability of
a pass's draw with its gradient.  Compiled from the unmodified oracle sources plus the shim, with the flags of the
oracle's parity build, into a temporary directory (the tree may be read-only)."""
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
        so = os.path.join(tempfile.mkdtemp(prefix="guided_oracle_"), "libguided_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-ffp-contract=off",
                               "-shared", "-I", os.path.join(ROOT, "oracle"), "-o", so,
                               os.path.join(ROOT, "tests", "host_shim", "guided_oracle.cpp"), "-lpthread"])
        _lib = C.CDLL(so)
        _lib.gor_log_prob.restype = C.c_double
        _lib.gor_log_prob.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint32, C.c_int64, C.c_void_p, C.c_void_p]
        _lib.gor_draw.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]
        _lib.gor_forward_dsac.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p]
        _lib.gor_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def philox(ctr, key):
    ctr = np.ascontiguousarray(ctr, np.uint32)
    key = np.ascontiguousarray(key, np.uint32)
    out = np.zeros(4, np.uint32)
    lib().gor_philox(_p(ctr), _p(key), _p(out))
    return out


def table(logits):
    """(w float64 [N], q uint32 [N], cum uint32 [N], bad) of one frame's logits."""
    logits = np.ascontiguousarray(logits, np.float32).reshape(N)
    w, q, cum = np.zeros(N), np.zeros(N, np.uint32), np.zeros(N, np.uint32)
    bad = lib().gor_table(_p(logits), _p(w), _p(q), _p(cum))
    return w, q, cum, bool(bad)


def draw(cum, seed, z, i):
    cells = np.zeros(4, np.int32)
    lib().gor_draw(_p(cum), seed, z, i, _p(cells))
    return cells


def forward(O, cfg, cum, g, coords, pix, gt_R=None, gt_t=None):
    """orc_forward of global frame g with the guided draw from the frame's prefix sums cum; O: oracle.oracle.  Returns
    (O.Forward result, stream_ncand [T])."""
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    out = O.Forward(cfg)
    ncand = np.zeros(max(1, cfg.n_streams), np.int64)
    gR = np.ascontiguousarray(gt_R, np.float64).reshape(9) if gt_R is not None else None
    gt = np.ascontiguousarray(gt_t, np.float64).reshape(3) if gt_t is not None else None
    out.status = lib().gor_forward(C.byref(cfg), _p(cum), g, _p(coords), _p(pix), _p(gR), _p(gt), C.byref(out.raw), _p(ncand))
    out._keep = (coords, pix)
    return out, ncand


def forward_dsac(O, cfg, cum, g, coords, pix, gt_R, gt_t, random_draw=True):
    """orc_forward_dsac of global frame g with the guided draw; O: oracle.oracle.  Returns an O.ForwardDsac."""
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    out = O.ForwardDsac(cfg)
    gR = np.ascontiguousarray(gt_R, np.float64).reshape(9)
    gt = np.ascontiguousarray(gt_t, np.float64).reshape(3)
    out.status = lib().gor_forward_dsac(C.byref(cfg), int(random_draw), _p(cum), g, _p(coords), _p(pix), _p(gR), _p(gt),
                                        C.byref(out.raw))
    out._keep = (coords, pix)
    return out


def log_prob(w, cum, T, seed, g, stream_ncand, want_grad=True):
    """(log p, d log p / d logits [N] or None) of one frame's used candidates."""
    w = np.ascontiguousarray(w, np.float64)
    ncand = np.ascontiguousarray(stream_ncand, np.int64)
    grad = np.zeros(N) if want_grad else None
    lp = lib().gor_log_prob(_p(w), _p(cum), T, seed, g, _p(ncand), _p(grad))
    return lp, grad
