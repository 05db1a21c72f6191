"""The fp32 decisions of the engine's device arithmetic (dsac_b200/csrc/*.cuh, compiled for the host) across cameras,
inlier thresholds and score parameters.  tests/test_host_math.py runs the same three checks at the default camera
(f = 525, principal point (320, 240)), thr = 10 and alpha / beta = 0.1 / 0.5 only; every margin below is built from
f, cx, cy and thr at run time, so each must hold for any camera, not only the default one.

  sampler filter (p3p_quick_inline)  ........ never rejects a candidate the exact P3P + reprojection check accepts
  refinement inlier test (reproj_below_thr_fast)  no wrong decision; fewer than 2 % of cells left to the exact arithmetic
  exact minimal-set solve (p3p_front / quartic_roots) the same accept / reject decisions with and without FMA contraction
  k_score arithmetic (score_pair_error / score_sigmoid_sum5):
      error-matrix entries ....................... <= 2e-3 px from getDiffMap's exact arithmetic (the diffmap contract)
      scores ..................................... <= alpha * N * 2^-25 + (1e-5 + beta * de) * s_exact:
          the 2^-25 floor under every sigmoid (score_sigmoid_sum5 shares one reciprocal between five sigmoids) times
          alpha and N = 1600; 1e-5 relative for the fp32 sigmoid sum (test_host_math's bound at the default camera); and
          the entries' own fp32 error de (the largest |fp32 - exact| of the hypothesis, asserted <= 2e-3 above) passed
          through the sigmoid, |d sigma / d e| = beta sigma (1 - sigma) <= beta sigma.  de grows with f (fp32 projection
          of f-scaled rows), so this term matters at long focal lengths: at f = 1500 it is what keeps a score at
          1.002 x (floor + 1e-5 s) inside its bound.

Frames come from the synthetic generator with the same camera (its sampling grid is 2 cx x 2 cy).  Run with -s to see
the measured maxima.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from dsac_b200 import synth

N = 1600
# (f, cx, cy): short and long focal lengths, a half-pixel principal point, principal points far off the 640 x 480 centre
CAMERAS = [(300.0, 320.0, 240.0), (585.0, 319.5, 239.5), (1000.0, 480.0, 360.0), (1500.0, 320.0, 240.0), (1500.0, 520.0, 90.0),
           (2500.0, 960.0, 540.0)]
THRS = [2, 5, 30]
# (thr, alpha, beta) of the score check
SCORE_PARAMS = [(2, 0.1, 0.5), (10, 0.3, 1.5), (5, 0.05, 2.0), (30, 0.1, 0.5)]


def _ids(cams):
    return ["f%g_c%g_%g" % c for c in cams]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _frames(n, cam):
    f, cx, cy = cam
    return synth.synth_frames(n, focal=f, cx=cx, cy=cy)


@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("cam", CAMERAS, ids=_ids(CAMERAS))
def test_conservative_filter_across_cameras(host_shim, cam, thr):
    """K1's fp64 filter may only say "certainly rejected" for candidates the exact P3P + reprojection check
    (cnn_softam.h:1041-1059) rejects -- with the case's camera and threshold in both."""
    f, cx, cy = cam
    coords, pix, _, _ = _frames(2, cam)
    tot = np.zeros(6, np.int64)
    for i in range(2):
        out = (C.c_longlong * 6)()
        host_shim.shim_filter_stats(_p(coords[i]), _p(pix[i]), C.c_uint32(1305 + i), C.c_uint32(6400 if i == 0 else 0),
                                    C.c_int(40000), C.c_double(f), C.c_double(cx), C.c_double(cy), C.c_int(thr), out)
        tot += np.array(list(out))
    n, acc, flagged, _, missed, _ = [int(v) for v in tot]
    print("filter f=%g c=(%g, %g) thr=%d: %d candidates, %d accepted, %d flagged, %d missed" % (f, cx, cy, thr, n, acc, flagged, missed))
    assert n == 80000 and acc > 0
    assert missed == 0


def _reproj_check(host_shim, cam, thr, rvec, tvec, coords, pix, want_err=False):
    f, cx, cy = cam
    n = len(coords)
    out = (C.c_longlong * 4)()
    err = np.zeros(n, np.float32) if want_err else None
    coords = np.ascontiguousarray(coords, np.int16); pix = np.ascontiguousarray(pix, np.int32)
    rvec = np.ascontiguousarray(rvec, np.float64); tvec = np.ascontiguousarray(tvec, np.float64)
    host_shim.shim_reproj_check(C.c_int(n), _p(rvec), _p(tvec), _p(coords), _p(pix), C.c_double(f), C.c_double(cx), C.c_double(cy),
                                C.c_int(thr), out, _p(err) if want_err else None)
    return [int(v) for v in out], err


@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("cam", CAMERAS, ids=_ids(CAMERAS))
def test_refinement_inlier_test_across_cameras(host_shim, cam, thr):
    """k_refine's "error < thr" in fp32 with a bound built from thr, |cx| + |cy| and the f-scaled pose rows; cells within
    the bound go to the exact arithmetic.  (a) poses around the generating pose, (b) one pose parameter bisected until the
    exact error of a cell crosses thr, then a cloud of poses around the crossing, (c) saturated / in-plane coordinates."""
    rng = np.random.default_rng(5 + thr)
    coords, pix, gt_cv, _ = _frames(3, cam)
    tot = np.zeros(4, np.int64)
    for f in range(3):
        for k in range(20):
            s = 0.0 if k == 0 else 10.0 ** rng.uniform(-6, -1)
            rv = gt_cv[f, :3] + rng.normal(0, s, 3)
            tv = gt_cv[f, 3:] + rng.normal(0, 1000 * s, 3)
            tot += _reproj_check(host_shim, cam, thr, rv, tv, coords[f], pix[f])[0]
    n_adv = 0
    fl = cam[0]
    quiet, _, quiet_cv, _ = synth.synth_frames(2, focal=fl, cx=cam[1], cy=cam[2], sigma=0.5)   # near-exact inliers at any f and thr
    for f in range(2):
        rv0, tv0 = quiet_cv[f, :3].copy(), quiet_cv[f, 3:].copy()
        _, e0 = _reproj_check(host_shim, cam, thr, rv0, tv0, quiet[f], pix[f], True)
        cells = np.flatnonzero(e0 < 0.5 * thr)[:25]
        for c in cells:
            cc, pp = quiet[f][c:c + 1], pix[f][c:c + 1]
            lo, hi = 0.0, 8.0 * thr * 7000.0 / fl     # shift of tvec[0] in mm: moves a cell at depth <= 7 m well past thr
            if _reproj_check(host_shim, cam, thr, rv0, tv0 + [hi, 0, 0], cc, pp)[0][3] == 1:
                continue
            for _ in range(60):
                mid = 0.5 * (lo + hi)
                if _reproj_check(host_shim, cam, thr, rv0, tv0 + [mid, 0, 0], cc, pp)[0][3] == 1:
                    lo = mid
                else:
                    hi = mid
            for d in np.concatenate([[0.0], rng.normal(0, 1e-9, 6), rng.normal(0, 1e-6, 6), rng.normal(0, 1e-4, 6), rng.normal(0, 1e-2, 6)]):
                tot += _reproj_check(host_shim, cam, thr, rv0, tv0 + [lo + d, 0, 0], cc, pp)[0]
                n_adv += 1
    cx = coords[0].copy()
    cx[::7] = 32767; cx[1::7] = -32768; cx[2::7] = 0
    for k in range(20):
        rv = rng.uniform(-3, 3, 3)
        tv = rng.uniform(-1, 1, 3) * 10.0 ** rng.uniform(0, 6)
        tot += _reproj_check(host_shim, cam, thr, rv, tv, cx, pix[0])[0]
    tot += _reproj_check(host_shim, cam, thr, np.zeros(3), np.zeros(3), cx, pix[0])[0]
    decided, undecided, wrong, inliers = [int(v) for v in tot]
    print("inlier test f=%g c=(%g, %g) thr=%d: %d decided, %d undecided (%.3g %%), %d wrong, %d adversarial poses"
          % (cam[0], cam[1], cam[2], thr, decided, undecided, 100.0 * undecided / (decided + undecided), wrong, n_adv))
    assert wrong == 0
    assert n_adv > 1000 and inliers > 500
    assert undecided < 0.02 * (decided + undecided)


@pytest.mark.parametrize("thr,alpha,beta", SCORE_PARAMS)
@pytest.mark.parametrize("cam", CAMERAS, ids=_ids(CAMERAS))
def test_score_arithmetic_across_cameras(host_shim, cam, thr, alpha, beta):
    """k_score's fp32 error and sigmoid sum with the case's camera, threshold and (alpha, beta), against getDiffMap's exact
    arithmetic and the double-precision soft-inlier score."""
    f, cx, cy = cam
    rng = np.random.default_rng(12 + thr)
    coords, pix, gt_cv, _ = _frames(3, cam)
    floor = alpha * N * 2.0 ** -25

    def frac(e32, ex, s, sx):     # the score error as a fraction of its bound
        return abs(s - sx) / (floor + (1e-5 + beta * float(np.abs(e32 - ex).max())) * sx)

    def run(rv, tv, cc, pp):
        e32, ex = np.zeros(N, np.float32), np.zeros(N, np.float32)
        s, sx = C.c_double(0), C.c_double(0)
        cc = np.ascontiguousarray(cc, np.int16); pp = np.ascontiguousarray(pp, np.int32)
        rv = np.ascontiguousarray(rv, np.float64); tv = np.ascontiguousarray(tv, np.float64)
        host_shim.shim_score_hypothesis(_p(rv), _p(tv), _p(cc), _p(pp), C.c_double(f), C.c_double(cx), C.c_double(cy), C.c_double(thr),
                                        C.c_double(alpha), C.c_double(beta), _p(e32), _p(ex), C.byref(s), C.byref(sx))
        return e32, ex, s.value, sx.value

    worst_e, worst_s = 0.0, 0.0     # worst entry error (px), worst score error as a fraction of its bound
    for fr in range(3):
        for k in range(15):
            sc = 0.0 if k == 0 else 10.0 ** rng.uniform(-5, -0.5)
            rv = gt_cv[fr, :3] + rng.normal(0, sc, 3)
            tv = gt_cv[fr, 3:] + rng.normal(0, 1000 * sc, 3)
            e32, ex, s, sx = run(rv, tv, coords[fr], pix[fr])
            worst_e = max(worst_e, float(np.abs(e32 - ex).max()))
            worst_s = max(worst_s, frac(e32, ex, s, sx))
    cz = coords[0].copy()
    cz[::3] = 0; cz[1::11, 2] = 0; cz[5::13] = 32767; cz[7::17] = -32768
    e32, ex, s, sx = run(np.zeros(3), np.zeros(3), cz, pix[0])
    assert np.isfinite(e32).all()
    worst_e = max(worst_e, float(np.abs(e32 - ex).max()))
    worst_s = max(worst_s, frac(e32, ex, s, sx))
    print("score f=%g c=(%g, %g) thr=%d alpha=%g beta=%g: entries %.3g px (bound 2e-3), scores %.3g of their bound"
          % (f, cx, cy, thr, alpha, beta, worst_e, worst_s))
    assert worst_e <= 2e-3
    assert worst_s <= 1.0


@pytest.fixture(scope="module")
def host_shim_fma(tmp_path_factory):
    """The host shim built with fused multiply-adds allowed everywhere (-mfma -ffp-contract=fast), as nvcc compiles device
    code by default; None where this CPU has no FMA instructions."""
    try:
        with open("/proc/cpuinfo") as f:
            if " fma " not in f.read().replace("\n", " "):
                return None
    except OSError:
        return None
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_shim", "host_math_shim.cpp")
    so = str(tmp_path_factory.mktemp("shim_fma") / "libhost_shim_fma.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-mfma", "-ffp-contract=fast", "-o", so, src])
    return C.CDLL(so)


# (camera, frame, sampler seed, candidates): (1500, 320, 240) frame 1 holds the minimal set of cells (17, 259, 171, 126), whose
# quartic has a near-double root: contracted, its discriminants used to decide "no real root" and the set was dropped
CONTRACTION_CASES = [((1500.0, 320.0, 240.0), 1, 1306, 27000), ((525.0, 320.0, 240.0), 0, 1305, 15000),
                     ((2500.0, 960.0, 540.0), 2, 1307, 15000), ((300.0, 320.0, 240.0), 1, 1306, 15000)]


@pytest.mark.parametrize("cam,frame,seed,n", CONTRACTION_CASES, ids=_ids([c[0] for c in CONTRACTION_CASES]))
def test_exact_solve_does_not_depend_on_contraction(host_shim, host_shim_fma, cam, frame, seed, n):
    """The exact minimal-set solve takes sign decisions on the P3P quartic's discriminants, which a fused multiply-add
    can flip next to a double root.  Its closed forms keep every product unfused (p3p_mul), so a build that contracts
    everything else must accept exactly the candidates the uncontracted build accepts, as the reference does."""
    if host_shim_fma is None:
        pytest.skip("this CPU has no FMA instructions")
    f, cx, cy = cam
    coords, pix, _, _ = synth.synth_frames(frame + 1, focal=f, cx=cx, cy=cy)
    co, px = coords[frame], pix[frame]
    cells = np.zeros((n, 4), np.int32)
    used = np.zeros(n, np.uint32)
    host_shim.shim_candidates(C.c_uint32(seed), C.c_uint32(0), n, _p(cells), _p(used))
    n_acc, differ = 0, []
    for k in range(n):
        obj = np.ascontiguousarray(co[cells[k]].reshape(-1), np.float32)
        img = np.ascontiguousarray(px[cells[k]].reshape(-1), np.float32)
        got = []
        for lib in (host_shim, host_shim_fma):
            rv, tv, fr = np.zeros(3), np.zeros(3), C.c_int(0)
            got.append(lib.shim_minimal_set(_p(obj), _p(img), C.c_double(f), C.c_double(cx), C.c_double(cy), 10, _p(rv), _p(tv),
                                            C.byref(fr)))
        n_acc += got[0]
        if got[0] != got[1]:
            differ.append((k, list(cells[k])))
    print("contraction f=%g c=(%g, %g): %d candidates, %d accepted, differing %s" % (f, cx, cy, n, n_acc, differ[:4]))
    assert n_acc > 0
    assert not differ
