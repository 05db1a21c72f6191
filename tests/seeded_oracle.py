"""The oracle's backward chains seeded by the caller (tests/host_shim/seeded_oracle.cpp), the reference the engine's
pose-valued outputs are checked against.  The library is compiled from the unmodified oracle sources plus the seeded
chains, with the flags of the oracle's parity build, into a temporary directory (the tree may be read-only)."""
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
        so = os.path.join(tempfile.mkdtemp(prefix="seeded_oracle_"), "libseeded_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-ffp-contract=off",
                               "-shared", "-I", os.path.join(ROOT, "oracle"), "-o", so,
                               os.path.join(ROOT, "tests", "host_shim", "seeded_oracle.cpp"), "-lpthread"])
        _lib = C.CDLL(so)
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def backward_seeded(O, cfg, coords, pix, fwd, seed6):
    """oracle.backward() with seed6 = dOuter/d(refined jp6) in place of dLossMax; no ground truth.  O: oracle.oracle,
    fwd: an oracle.forward() result."""
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    seed6 = np.ascontiguousarray(seed6, np.float64).reshape(6)
    out = O.Backward(cfg)
    lib().orc_backward_seeded(C.byref(cfg), _p(coords), _p(pix), C.byref(fwd.raw), _p(seed6), C.byref(out.raw))
    return out


def backward_dsac_seeded(O, cfg, coords, pix, fwd, seed=None, grad_sf=None):
    """oracle.backward_dsac() with seed [H][6] in place of sf_h dLossMax_h (over the hypotheses with sf > 1e-4 and a
    nonzero seed) and grad_sf [H] = dOuter/dsf in place of the losses; either None (its path is zero)."""
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    seed = np.ascontiguousarray(seed, np.float64).reshape(cfg.n_hyps, 6) if seed is not None else None
    grad_sf = np.ascontiguousarray(grad_sf, np.float64).reshape(cfg.n_hyps) if grad_sf is not None else None
    out = O.BackwardDsac(cfg)
    lib().orc_backward_dsac_seeded(C.byref(cfg), _p(coords), _p(pix), C.byref(fwd.raw), _p(seed), _p(grad_sf),
                                   C.byref(out.raw))
    return out
