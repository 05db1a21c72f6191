"""The sampler's conservative filter (p3p_lambda_core, via minimal_set_needs_full) on minimal sets that random candidates
rarely produce, compiled for the host: it may only say "certainly rejected" for candidates that the exact P3P +
reprojection check (minimal_set_hypothesis) rejects.  The families are described in tests/adversarial_sets.py, which
tests/test_gpu_device_arithmetic.py shares to run the same check with the device build of the filter.
"""
import ctypes as C

import numpy as np
import pytest

import adversarial_sets as A

CAMERAS = [(525.0, 320.0, 240.0), (1500.0, 320.0, 240.0)]
# the new families at long focal lengths and off-centre principal points as well: the fp32 tail's error grows with f and
# with the 4th pixel's distance from the principal point
NEW_CAMERAS = [(525.0, 320.0, 240.0), (1500.0, 320.0, 240.0), (2500.0, 320.0, 240.0), (1000.0, 480.0, 360.0),
               (1500.0, 520.0, 90.0)]
THRS = [2, 10, 30]


def check_batch(shim, cam, thr, obj, img):
    """(accepted, needs_full) of the host build for each set"""
    f, cx, cy = cam
    n = obj.shape[0]
    acc, need = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    shim.shim_filter_batch(n, A._p(np.ascontiguousarray(obj)), A._p(np.ascontiguousarray(img)), C.c_double(f), C.c_double(cx),
                           C.c_double(cy), thr, A._p(acc), A._p(need))
    return acc.astype(bool), need.astype(bool)


@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("cam", CAMERAS, ids=["f%g" % c[0] for c in CAMERAS])
def test_filter_adversarial_minimal_sets(host_shim, cam, thr):
    rng = np.random.default_rng(31 + thr + int(cam[0]))
    o1, i1, n_bisected = A.double_roots(rng, cam, thr, host_shim)
    o2, i2 = A.danger_cylinder(rng, cam, thr)
    o3, i3 = A.near_collinear(rng, cam, thr)
    obj, img = np.concatenate([o1, o2, o3]), np.concatenate([i1, i2, i3])
    acc, need = check_batch(host_shim, cam, thr, obj, img)
    missed = np.flatnonzero(acc & ~need)
    print("adversarial f=%g thr=%d: %d minimal sets, %d accepted, %d flagged, %d missed, %d double roots bisected"
          % (cam[0], thr, len(acc), acc.sum(), need.sum(), len(missed), n_bisected))
    assert n_bisected > 10
    assert acc.sum() > 200
    assert not len(missed), (obj[missed[:2]], img[missed[:2]])


def test_filter_near_camera_regression_case(host_shim):
    """A triangle ~20 m away and a 4th point 24 mm in front of the camera, its pixel 9.87 px from where the exact pose
    projects it: accepted.  The fp32 4th-point stage once put it beyond thr + 0.25 px and rejected it."""
    obj, img = A.NEAR_CAMERA_CASE
    acc, need = check_batch(host_shim, (525.0, 320.0, 240.0), 10, obj[None], img[None])
    assert acc[0] and need[0]


@pytest.mark.parametrize("integer", [False, True], ids=["float", "int"])
@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("cam", NEW_CAMERAS, ids=["f%g_c%g_%g" % c for c in NEW_CAMERAS])
@pytest.mark.parametrize("family", sorted(A.NEW_FAMILIES))
def test_filter_far_triangle_near_point_families(host_shim, family, cam, thr, integer):
    """near camera, tiny triangle and ill-conditioned triangles (tests/adversarial_sets.py), float and integer inputs,
    every 4th pixel 0 .. 0.5 px inside the threshold"""
    rng = np.random.default_rng([sorted(A.NEW_FAMILIES).index(family), int(cam[0]), int(cam[1]), thr, integer])
    obj, img = A.NEW_FAMILIES[family](rng, cam, thr, 600, host_shim, integer)
    acc, need = check_batch(host_shim, cam, thr, obj, img)
    missed = np.flatnonzero(acc & ~need)
    print("%s f=%g c=(%g, %g) thr=%d %s: %d minimal sets, %d accepted, %d flagged, %d missed"
          % (family, cam[0], cam[1], cam[2], thr, "int" if integer else "float", len(acc), acc.sum(), need.sum(), len(missed)))
    assert acc.sum() > 100
    assert not len(missed), (obj[missed[:2]], img[missed[:2]])
