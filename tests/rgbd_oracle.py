"""RGB-D localisation restated on the CPU (tests/host_shim/rgbd_oracle.cpp), the reference the engine's RGB-D passes are
checked against: eye coordinates, the Kabsch acceptance over the oracle's own candidate streams (uniform or guided),
the Kabsch refinement and orc_forward with both swapped.  Compiled from the unmodified oracle sources plus the shim, with
the flags of the oracle's parity build, into a temporary directory (the tree may be read-only).  Also the seeded
synthetic RGB-D frames the tests use."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, GRID = 1600, 40
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="rgbd_oracle_"), "librgbd_oracle.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-ffp-contract=off",
                               "-shared", "-I", os.path.join(ROOT, "oracle"), "-o", so,
                               os.path.join(ROOT, "tests", "host_shim", "rgbd_oracle.cpp"), "-lpthread"])
        _lib = C.CDLL(so)
        _lib.ror_eye.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_void_p]
        _lib.ror_accept.argtypes = [C.c_void_p] + [C.c_void_p] * 7
        _lib.ror_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 7
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def eye(pix, depth, f=525.0, cx=320.0, cy=240.0):
    """(eye float64 [N][3], cells with depth) of one frame."""
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    depth = np.ascontiguousarray(depth, np.float32).reshape(N)
    out = np.zeros((N, 3))
    have = lib().ror_eye(_p(pix), _p(depth), f, cx, cy, _p(out))
    return out, have


def accept(cfg, coords, pix, ey, cells):
    """(accepted, rvec, tvec, fragile count) of the minimal set `cells` (4 cell indices, draw order)."""
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    ey = np.ascontiguousarray(ey, np.float64).reshape(N, 3)
    cells = np.ascontiguousarray(cells, np.int32)
    r, t, fr = np.zeros(3), np.zeros(3), np.zeros(1, np.int64)
    ok = lib().ror_accept(C.byref(cfg), _p(coords), _p(pix), _p(ey), _p(cells), _p(r), _p(t), _p(fr))
    return bool(ok), r, t, int(fr[0])


def forward(O, cfg, g, coords, pix, ey, cum=None, gt_R=None, gt_t=None):
    """orc_forward of global frame g as an RGB-D pass (cum: the guided draw's prefix sums, None: uniform); O:
    oracle.oracle.  Returns (O.Forward result with .status, stream_ncand [T])."""
    coords = np.ascontiguousarray(coords, np.int16).reshape(N, 3)
    pix = np.ascontiguousarray(pix, np.int32).reshape(N, 2)
    ey = np.ascontiguousarray(ey, np.float64).reshape(N, 3)
    out = O.Forward(cfg)
    ncand = np.zeros(max(1, cfg.n_streams), np.int64)
    gR = np.ascontiguousarray(gt_R, np.float64).reshape(9) if gt_R is not None else None
    gt = np.ascontiguousarray(gt_t, np.float64).reshape(3) if gt_t is not None else None
    cum = np.ascontiguousarray(cum, np.uint32) if cum is not None else None
    out.status = lib().ror_forward(C.byref(cfg), _p(cum), g, _p(coords), _p(pix), _p(ey), _p(gR), _p(gt), C.byref(out.raw),
                                   _p(ncand))
    out._keep = (coords, pix, ey, cum)
    return out, ncand


def synth(n, seed=7, holes=0.0, rho=0.6, sigma=10.0, cams=None, f=525.0, cx=320.0, cy=240.0):
    """Seeded synthetic RGB-D frames: (coords int16 [n][N][3], pix int32 [n][N][2], depth float32 [n][N], gt_cv [n][6],
    gt_jp [n][12]).  Depth U(500, 3500) mm at each cell's grid pixel; a fraction rho of the cells are inliers, scene
    point R^T (X_eye - t) plus N(0, sigma) mm, the rest uniform in the scene box; a fraction `holes` has no depth (NaN).
    cams: float64 [n][3] per-frame (focal, cx, cy), or None for (f, cx, cy)."""
    rng = np.random.default_rng(seed)
    coords = np.zeros((n, N, 3), np.int16)
    pix = np.zeros((n, N, 2), np.int32)
    depth = np.zeros((n, N), np.float32)
    gt_cv = np.zeros((n, 6))
    gt_jp = np.zeros((n, 12))
    for g in range(n):
        ff, ccx, ccy = cams[g] if cams is not None else (f, cx, cy)
        xs = (np.arange(N) % GRID) * 16 + 8 + rng.integers(-4, 5, N)
        ys = (np.arange(N) // GRID) * 12 + 6 + rng.integers(-3, 4, N)
        pix[g, :, 0], pix[g, :, 1] = xs, ys
        d = rng.uniform(500, 3500, N)
        Xe = np.stack([(xs - ccx) * d / ff, (ys - ccy) * d / ff, d], 1)
        rvec = rng.normal(0, 0.4, 3)
        R = Rotation.from_rotvec(rvec).as_matrix()
        t = rng.uniform(-500, 500, 3)
        Xs = (Xe - t) @ R   # R^T (X_eye - t)
        Xs += rng.normal(0, sigma, Xs.shape)
        out = rng.random(N) >= rho
        Xs[out] = rng.uniform(-3000, 3000, (int(out.sum()), 3))
        coords[g] = np.clip(np.rint(Xs), -32767, 32767).astype(np.int16)
        d = d.astype(np.float32)
        d[rng.random(N) < holes] = np.nan
        depth[g] = d
        gt_cv[g, :3], gt_cv[g, 3:] = rvec, t
        # jp (cv2our) of the cv pose: y and z axes flipped
        Ro = R.copy()
        Ro[1:] *= -1
        gt_jp[g, :9] = Ro.reshape(9)
        gt_jp[g, 9:] = [t[0], -t[1], -t[2]]
    return coords, pix, depth, gt_cv, gt_jp


def _frame(coords, pix, ey):
    return (np.ascontiguousarray(coords, np.int16).reshape(N, 3), np.ascontiguousarray(pix, np.int32).reshape(N, 2),
            np.ascontiguousarray(ey, np.float64).reshape(N, 3))


def forward_dsac(O, cfg, g, coords, pix, ey, gt_R, gt_t, random_draw=True):
    """orc_forward_dsac of global frame g as an RGB-D pass (uniform streams); an O.ForwardDsac with .status."""
    coords, pix, ey = _frame(coords, pix, ey)
    out = O.ForwardDsac(cfg)
    gR = np.ascontiguousarray(gt_R, np.float64).reshape(9)
    gt = np.ascontiguousarray(gt_t, np.float64).reshape(3)
    lib().ror_forward_dsac.argtypes = [C.c_void_p, C.c_int, C.c_int64] + [C.c_void_p] * 6
    out.status = lib().ror_forward_dsac(C.byref(cfg), int(random_draw), g, _p(coords), _p(pix), _p(ey), _p(gR), _p(gt),
                                        C.byref(out.raw))
    out._keep = (coords, pix, ey)
    return out


def backward(O, cfg, coords, pix, ey, gt_R, gt_t, fwd):
    """orc_backward of an RGB-D pass from a forward() result; an O.Backward."""
    coords, pix, ey = _frame(coords, pix, ey)
    out = O.Backward(cfg)
    gR = np.ascontiguousarray(gt_R, np.float64).reshape(9)
    gt = np.ascontiguousarray(gt_t, np.float64).reshape(3)
    lib().ror_backward.argtypes = [C.c_void_p] * 8
    lib().ror_backward(C.byref(cfg), _p(coords), _p(pix), _p(ey), _p(gR), _p(gt), C.byref(fwd.raw), C.byref(out.raw))
    return out


def backward_dsac(O, cfg, coords, pix, ey, gt_R, gt_t, fwd):
    """orc_backward_dsac of an RGB-D pass from a forward_dsac() result; an O.BackwardDsac."""
    coords, pix, ey = _frame(coords, pix, ey)
    out = O.BackwardDsac(cfg)
    gR = np.ascontiguousarray(gt_R, np.float64).reshape(9)
    gt = np.ascontiguousarray(gt_t, np.float64).reshape(3)
    lib().ror_backward_dsac.argtypes = [C.c_void_p] * 8
    lib().ror_backward_dsac(C.byref(cfg), _p(coords), _p(pix), _p(ey), _p(gR), _p(gt), C.byref(fwd.raw), C.byref(out.raw))
    return out
