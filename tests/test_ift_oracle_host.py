"""The recording refinement replay (tests/host_shim/ift_oracle.cpp) against the oracle's own forward, and the product's
implicit-function derivative (ift.cuh compiled for the host) at the oracle's recorded set against central differences of
the numpy frozen-set solver (tests/ift_oracle.py) -- on the oracle's refinement of a synthetic frame."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import ift_oracle as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600


@pytest.fixture(scope="module")
def shim():
    so = os.path.join(tempfile.mkdtemp(prefix="ift_shim_"), "libift_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "ift_shim.cpp")])
    return C.CDLL(so)


def host_ift(shim, pose, coords, pix, cells, cam):
    Y = np.ascontiguousarray(coords[cells], np.float64)
    e = np.ascontiguousarray(np.concatenate([pix[cells].astype(np.float64), np.zeros((len(cells), 1))], 1))
    D = np.zeros((len(cells), 6, 3))
    ok = shim.shim_ift_fit_deriv(len(cells), I._p(Y), I._p(e), I._p(np.ascontiguousarray(pose, np.float64)), C.c_double(cam[0]),
                                 C.c_double(cam[1]), C.c_double(cam[2]), 0, I._p(D))
    return bool(ok), D


def test_recording_replay_is_the_oracle_refinement_and_its_ift_matches_the_frozen_set_solver(oracle, shim):
    from dsac_b200 import engine as E
    O = oracle
    coords, pix, gt_cv, gt_jp = E.synth_frames(2)
    for f in range(2):
        cfg = O.default_config(seed=1305 + f, n_hyps=64)
        ofw = O.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
        pose, S, done = I.refine_record(cfg, coords[f], pix[f], ofw.pixel_idxs, ofw.n_perm_steps, ofw.avg)
        assert done == ofw.ref_steps_done
        assert np.array_equal(pose, ofw.ref)                        # bit for bit the oracle's refined pose
        assert 50 <= len(S) <= cfg.inlier_count and len(np.unique(S)) == len(S)
        assert (ofw.inlier_map[S] > 0).all()
        c3, p2 = coords[f].reshape(N, 3).astype(np.float64), pix[f].reshape(N, 2)
        cam = (cfg.f, cfg.cx, cfg.cy)
        ok, D = host_ift(shim, pose, c3, p2, S, cam)
        assert ok
        # independent check: the frozen-set solution's central differences (every 8th cell of S)
        Y = c3[S]
        e = np.concatenate([p2[S].astype(np.float64), np.zeros((len(S), 1))], 1)
        pick = np.arange(0, len(S), 8)
        num = I.frozen_derivative(Y, e, pose, cam, False, pick)
        assert np.abs(D[pick] - num).max() <= 1e-5 * np.abs(num).max()
