"""The sampler's conservative filter (p3p_lambda_core, via minimal_set_needs_full) on minimal sets that random candidates
rarely produce, compiled for the host: it may only say "certainly rejected" for candidates that the exact P3P +
reprojection check (minimal_set_hypothesis) rejects.

  double roots ........ the camera moved along a path until the exact solve's number of real solutions changes, then
                        bisected onto the change (two solutions merge there)
  danger cylinder ..... the camera on, or 10^-9 .. 10^-2 off, the cylinder through the three points perpendicular to
                        their plane (the P3P Jacobian is singular on it)
  near-collinear ...... the third scene point 10^-6 .. 10^-1 of the triangle's size off the line through the other two
  threshold ........... the 4th point's pixel thr +- 10^-3 px from where the true pose projects it

Scene coordinates are rounded to float (as the engine's int16 grid converted to float would be), pixels are float.
"""
import ctypes as C

import numpy as np
import pytest

CAMERAS = [(525.0, 320.0, 240.0), (1500.0, 320.0, 240.0)]
THRS = [2, 10, 30]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _look_at(Cc, target, rng):
    z = target - Cc
    z = z / np.linalg.norm(z)
    up = rng.normal(size=3)
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    return np.stack([x, y, z])          # rows: camera axes in world coordinates (world -> camera rotation)


def _project(R, Cc, X, cam):
    f, cx, cy = cam
    Xc = (X - Cc) @ R.T
    return np.stack([f * Xc[:, 0] / Xc[:, 2] + cx, f * Xc[:, 1] / Xc[:, 2] + cy], 1)


def _make(X, R, Cc, cam, off3=(0.0, 0.0)):
    """float correspondences (obj 4 x 3, img 4 x 2) of scene points X seen from camera centre Cc with rotation R; the 4th
    pixel moved by off3 from its true projection"""
    obj = X.astype(np.float32)
    img = _project(R, Cc, obj.astype(np.float64), cam)
    img[3] += off3
    return np.ascontiguousarray(obj.reshape(-1)), np.ascontiguousarray(img.astype(np.float32).reshape(-1))


class _Check:
    def __init__(self, shim, cam, thr):
        self.shim, self.cam, self.thr = shim, cam, thr
        self.n = self.accepted = self.flagged = 0
        self.missed = []

    def __call__(self, obj, img):
        f, cx, cy = self.cam
        rv, tv, fr = np.zeros(3), np.zeros(3), C.c_int(0)
        acc = self.shim.shim_minimal_set(_p(obj), _p(img), C.c_double(f), C.c_double(cx), C.c_double(cy), self.thr, _p(rv), _p(tv),
                                         C.byref(fr))
        need = self.shim.shim_needs_full(_p(obj), _p(img), C.c_double(f), C.c_double(cx), C.c_double(cy), self.thr)
        self.n += 1
        self.accepted += acc
        self.flagged += need
        if acc and not need:
            self.missed.append((obj.copy(), img.copy()))

    def n_solutions(self, obj, img):
        f, cx, cy = self.cam
        R, t, e2 = np.zeros(9), np.zeros(3), C.c_double(0)
        return self.shim.shim_p3p_best(_p(obj), _p(img), C.c_double(f), C.c_double(cx), C.c_double(cy), _p(R), _p(t), C.byref(e2))

    def offsets(self, rng):
        """4th-pixel offsets: on the true projection, and thr -+ 1e-3 px away from it in a random direction"""
        d = rng.normal(size=2)
        d /= np.linalg.norm(d)
        return [(0.0, 0.0)] + [tuple(d * (self.thr + s)) for s in (-1e-3, 1e-3)]


def _scene(rng):
    """three scene points ~0.5 .. 1.5 m apart around the origin, a 4th one nearby"""
    X = rng.uniform(-800, 800, (4, 3))
    return X - X[:3].mean(0)


def _circle(X):
    """circumcentre, circumradius and unit normal of the triangle X[0..2]"""
    a, b = X[1] - X[0], X[2] - X[0]
    n = np.cross(a, b)
    o = X[0] + (np.dot(a, a) * np.cross(b, n) + np.dot(b, b) * np.cross(n, a)) / (2 * np.dot(n, n))
    return o, np.linalg.norm(X[0] - o), n / np.linalg.norm(n)


@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("cam", CAMERAS, ids=["f%g" % c[0] for c in CAMERAS])
def test_filter_adversarial_minimal_sets(host_shim, cam, thr):
    rng = np.random.default_rng(31 + thr + int(cam[0]))
    chk = _Check(host_shim, cam, thr)
    n_bisected = 0
    # (1) double roots: the camera centre moves on a segment; where the exact solve's solution count changes, bisect
    for trial in range(150):
        X = _scene(rng)
        C0 = rng.normal(size=3)
        C0 = C0 / np.linalg.norm(C0) * rng.uniform(1500, 4000)
        C1 = C0 + rng.normal(size=3) * 800
        R = _look_at(C0, X[:3].mean(0), rng)
        counts = [chk.n_solutions(*_make(X, R, C0 + s * (C1 - C0), cam)) for s in np.linspace(0, 1, 9)]
        k = next((i for i in range(8) if counts[i] != counts[i + 1]), None)
        if k is None:
            continue
        lo, hi = k / 8, (k + 1) / 8
        n_lo = counts[k]
        for _ in range(45):
            mid = 0.5 * (lo + hi)
            if chk.n_solutions(*_make(X, R, C0 + mid * (C1 - C0), cam)) == n_lo:
                lo = mid
            else:
                hi = mid
        n_bisected += 1
        for s in np.concatenate([[lo, hi], lo + (hi - lo) * rng.uniform(-4, 5, 4), lo + rng.normal(0, 1e-6, 4)]):
            for off in chk.offsets(rng):
                chk(*_make(X, R, C0 + s * (C1 - C0), cam, off))
    # (2) the danger cylinder through the three points
    for trial in range(200):
        X = _scene(rng)
        o, rho, nrm = _circle(X[:3])
        u = np.cross(nrm, rng.normal(size=3))
        u /= np.linalg.norm(u)
        v = np.cross(nrm, u)
        phi = rng.uniform(0, 2 * np.pi)
        eps = [0.0, 1e-9, -1e-9, 1e-6, -1e-6, 1e-4, -1e-4, 1e-2, -1e-2][trial % 9]
        Cc = o + rho * (1 + eps) * (np.cos(phi) * u + np.sin(phi) * v) + nrm * rng.choice([-1, 1]) * rng.uniform(1000, 3500)
        R = _look_at(Cc, X[:3].mean(0), rng)
        for off in chk.offsets(rng):
            chk(*_make(X, R, Cc, cam, off))
    # (3) near-collinear scene triangles
    for trial in range(200):
        X = _scene(rng)
        d = X[1] - X[0]
        perp = np.cross(d, rng.normal(size=3))
        perp /= np.linalg.norm(perp)
        X[2] = X[0] + rng.uniform(-0.5, 1.5) * d + perp * np.linalg.norm(d) * 10.0 ** rng.uniform(-6, -1)
        Cc = rng.normal(size=3)
        Cc = Cc / np.linalg.norm(Cc) * rng.uniform(1500, 4000)
        R = _look_at(Cc, X[:3].mean(0), rng)
        for off in chk.offsets(rng):
            chk(*_make(X, R, Cc, cam, off))
    print("adversarial f=%g thr=%d: %d minimal sets, %d accepted, %d flagged, %d missed, %d double roots bisected"
          % (cam[0], thr, chk.n, chk.accepted, chk.flagged, len(chk.missed), n_bisected))
    assert n_bisected > 10
    assert chk.accepted > 200
    assert not chk.missed, chk.missed[:2]
