"""Minimal sets (4 scene points, 4 pixels) on which the sampler's conservative filter is hardest to get right, shared by
the host test of the filter (tests/test_host_filter_adversarial.py) and its device twin (tests/test_gpu_device_arithmetic.py).

  double roots ........ the camera moved along a path until the exact solve's number of real solutions changes, then
                        bisected onto the change (two solutions merge there)
  danger cylinder ..... the camera on, or 10^-9 .. 10^-2 off, the cylinder through the three points perpendicular to
                        their plane (the P3P Jacobian is singular on it)
  near-collinear ...... the third scene point 10^-6 .. 10^-1 of the triangle's size off the line through the other two
  threshold ........... the 4th point's pixel thr +- 10^-3 px from where the true pose projects it (part of the three above)
  near camera ......... a triangle 10 .. 25 m away and a 4th point 8 .. 60 mm in front of the camera, its pixel near an
                        image corner: the 4th point's depth is tiny against the lengths the filter sums it from
  tiny triangle ....... sides of 5 .. 50 mm, 0.3 .. 3 m from the camera, and a 4th point 1 .. 5 m away from it: the
                        camera frame the filter builds from the triangle amplifies every error by (distance / side)
  ill-conditioned ..... the triangle's angle at point 0 with sin^2 = 10^-3 x 10^(-0.5 .. 0.5), both sides of the filter's
                        limit nn = 10^-3 s01 s02, at an acute and at an obtuse angle
For the last three the 4th pixel is 0 .. 0.2 px (float sets) or 0 .. 0.5 px (integer sets) inside thr from where the best
exact pose projects it: accepted, and as close to the threshold as the inputs allow.

Float sets: scene coordinates rounded to float, float pixels.  Integer sets: what the engine takes (int16 mm, integer
pixels).  Every generator returns (obj [n, 12], img [n, 8]) float32 arrays.
"""
import ctypes as C

import numpy as np

# the integer minimal set at the default camera (f = 525, (320, 240)), thr = 10 that the fp32 tail of the filter used to
# reject: accepted, 4th-point error 9.870 px, depths 18.9 m, 20.7 m, 20.2 m and 23.7 mm
NEAR_CAMERA_CASE = (np.array([18234, 2459, 9914, 21811, 6758, -3610, 19398, 1132, 10014, 8, 2122, 1231], np.float32),
                    np.array([310, 40, 113, 368, 341, 61, 554, 126], np.float32))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def look_at(Cc, target, rng):
    z = target - Cc
    z = z / np.linalg.norm(z)
    up = rng.normal(size=3)
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    return np.stack([x, y, z])          # rows: camera axes in world coordinates (world -> camera rotation)


def project(R, Cc, X, cam):
    f, cx, cy = cam
    Xc = (X - Cc) @ R.T
    return np.stack([f * Xc[:, 0] / Xc[:, 2] + cx, f * Xc[:, 1] / Xc[:, 2] + cy], 1)


def make(X, R, Cc, cam, off3=(0.0, 0.0)):
    """float correspondences (obj 12, img 8) of scene points X seen from camera centre Cc with rotation R; the 4th
    pixel moved by off3 from its true projection"""
    obj = X.astype(np.float32)
    img = project(R, Cc, obj.astype(np.float64), cam)
    img[3] += off3
    return np.ascontiguousarray(obj.reshape(-1)), np.ascontiguousarray(img.astype(np.float32).reshape(-1))


def n_solutions(shim, cam, obj, img):
    f, cx, cy = cam
    R, t, e2 = np.zeros(9), np.zeros(3), C.c_double(0)
    return shim.shim_p3p_best(_p(obj), _p(img), C.c_double(f), C.c_double(cx), C.c_double(cy), _p(R), _p(t), C.byref(e2))


def _offsets(rng, thr):
    """4th-pixel offsets: on the true projection, and thr -+ 1e-3 px away from it in a random direction"""
    d = rng.normal(size=2)
    d /= np.linalg.norm(d)
    return [(0.0, 0.0)] + [tuple(d * (thr + s)) for s in (-1e-3, 1e-3)]


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


def _stack(sets):
    return (np.stack([s[0] for s in sets]).astype(np.float32), np.stack([s[1] for s in sets]).astype(np.float32))


def double_roots(rng, cam, thr, shim, trials=150):
    """returns (obj, img, number of double roots bisected)"""
    sets, n_bisected = [], 0
    for trial in range(trials):
        X = _scene(rng)
        C0 = rng.normal(size=3)
        C0 = C0 / np.linalg.norm(C0) * rng.uniform(1500, 4000)
        C1 = C0 + rng.normal(size=3) * 800
        R = look_at(C0, X[:3].mean(0), rng)
        counts = [n_solutions(shim, cam, *make(X, R, C0 + s * (C1 - C0), cam)) for s in np.linspace(0, 1, 9)]
        k = next((i for i in range(8) if counts[i] != counts[i + 1]), None)
        if k is None:
            continue
        lo, hi = k / 8, (k + 1) / 8
        n_lo = counts[k]
        for _ in range(45):
            mid = 0.5 * (lo + hi)
            if n_solutions(shim, cam, *make(X, R, C0 + mid * (C1 - C0), cam)) == n_lo:
                lo = mid
            else:
                hi = mid
        n_bisected += 1
        for s in np.concatenate([[lo, hi], lo + (hi - lo) * rng.uniform(-4, 5, 4), lo + rng.normal(0, 1e-6, 4)]):
            for off in _offsets(rng, thr):
                sets.append(make(X, R, C0 + s * (C1 - C0), cam, off))
    return _stack(sets) + (n_bisected,)


def danger_cylinder(rng, cam, thr, trials=200):
    sets = []
    for trial in range(trials):
        X = _scene(rng)
        o, rho, nrm = _circle(X[:3])
        u = np.cross(nrm, rng.normal(size=3))
        u /= np.linalg.norm(u)
        v = np.cross(nrm, u)
        phi = rng.uniform(0, 2 * np.pi)
        eps = [0.0, 1e-9, -1e-9, 1e-6, -1e-6, 1e-4, -1e-4, 1e-2, -1e-2][trial % 9]
        Cc = o + rho * (1 + eps) * (np.cos(phi) * u + np.sin(phi) * v) + nrm * rng.choice([-1, 1]) * rng.uniform(1000, 3500)
        R = look_at(Cc, X[:3].mean(0), rng)
        for off in _offsets(rng, thr):
            sets.append(make(X, R, Cc, cam, off))
    return _stack(sets)


def near_collinear(rng, cam, thr, trials=200):
    sets = []
    for trial in range(trials):
        X = _scene(rng)
        d = X[1] - X[0]
        perp = np.cross(d, rng.normal(size=3))
        perp /= np.linalg.norm(perp)
        X[2] = X[0] + rng.uniform(-0.5, 1.5) * d + perp * np.linalg.norm(d) * 10.0 ** rng.uniform(-6, -1)
        Cc = rng.normal(size=3)
        Cc = Cc / np.linalg.norm(Cc) * rng.uniform(1500, 4000)
        R = look_at(Cc, X[:3].mean(0), rng)
        for off in _offsets(rng, thr):
            sets.append(make(X, R, Cc, cam, off))
    return _stack(sets)


def _random_rotation(rng):
    q = rng.normal(size=4)
    a, b, c, d = q / np.linalg.norm(q)
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def _ray(cam, u, v):
    f, cx, cy = cam
    return np.array([(u - cx) / f, (v - cy) / f, 1.0])


def _near_threshold(X, R, Cc, cam, thr, integer, rng, shim):
    """The minimal set of world points X seen from (R, Cc): rounded to the input type, the 4th pixel put inside thr,
    close to it, from where the best exact pose of the rounded set projects the 4th point.  None if that fails."""
    f, cx, cy = cam
    obj = np.round(X) if integer else X
    if integer and np.abs(obj).max() > 32767:
        return None
    obj = obj.astype(np.float32)
    img = project(R, Cc, obj.astype(np.float64), cam)
    if integer:
        img = np.round(img)
    o12, i8 = np.ascontiguousarray(obj.reshape(-1)), np.ascontiguousarray(img.astype(np.float32).reshape(-1))
    Rb, tb, e2 = np.zeros(9), np.zeros(3), C.c_double(0)
    if shim.shim_p3p_best(_p(o12), _p(i8), C.c_double(f), C.c_double(cx), C.c_double(cy), _p(Rb), _p(tb), C.byref(e2)) <= 0:
        return None
    q = Rb.reshape(3, 3) @ obj[3].astype(np.float64) + tb
    if not q[2] > 0:
        return None
    p4 = np.array([f * q[0] / q[2] + cx, f * q[1] / q[2] + cy])
    if integer:
        r = int(np.ceil(thr)) + 1
        g = np.stack(np.meshgrid(np.arange(-r, r + 1), np.arange(-r, r + 1)), -1).reshape(-1, 2) + np.round(p4)
        d = np.linalg.norm(g - p4, axis=1)
        ok = np.flatnonzero((d >= thr - 0.5) & (d < thr))
        if not len(ok):
            return None
        i8[6:] = g[rng.choice(ok)]
    else:
        d = rng.normal(size=2)
        i8[6:] = p4 + d / np.linalg.norm(d) * (thr - rng.uniform(0, 0.2))
    return o12, i8


def _frame_pose(rng):
    """a random camera rotation and a centre within 3 m of the origin"""
    return _random_rotation(rng), rng.uniform(-3000, 3000, 3)


def _to_world(R, Cc, Xc):
    return Xc @ R + Cc               # Xc = R (X - Cc)


def near_camera(rng, cam, thr, n, shim, integer):
    f, cx, cy = cam
    sets = []
    while len(sets) < n:
        R, Cc = _frame_pose(rng)
        tri = [_ray(cam, rng.uniform(0, 2 * cx), rng.uniform(0, 2 * cy)) * rng.uniform(10000, 25000) for _ in range(3)]
        corner = np.array([rng.choice([0, 2 * cx]), rng.choice([0, 2 * cy])])
        u4 = corner + np.sign([cx, cy] - corner) * rng.uniform(0, 0.15, 2) * [2 * cx, 2 * cy]
        X4 = _ray(cam, *u4) * rng.uniform(8, 60)
        s = _near_threshold(_to_world(R, Cc, np.stack(tri + [X4])), R, Cc, cam, thr, integer, rng, shim)
        if s is not None:
            sets.append(s)
    return _stack(sets)


def tiny_triangle(rng, cam, thr, n, shim, integer):
    f, cx, cy = cam
    sets = []
    while len(sets) < n:
        R, Cc = _frame_pose(rng)
        centre = _ray(cam, rng.uniform(0, 2 * cx), rng.uniform(0, 2 * cy)) * rng.uniform(300, 3000)
        side = rng.uniform(5, 50)
        tri = centre + rng.normal(size=(3, 3)) * side / 2
        X4 = _ray(cam, rng.uniform(0, 2 * cx), rng.uniform(0, 2 * cy)) * rng.uniform(300, 6000)
        if not 1000 <= np.linalg.norm(X4 - centre) <= 5000:
            continue
        s = _near_threshold(_to_world(R, Cc, np.vstack([tri, X4])), R, Cc, cam, thr, integer, rng, shim)
        if s is not None:
            sets.append(s)
    return _stack(sets)


def ill_conditioned(rng, cam, thr, n, shim, integer):
    sets = []
    while len(sets) < n:
        e1 = rng.normal(size=3)
        e1 /= np.linalg.norm(e1)
        e2 = np.cross(e1, rng.normal(size=3))
        e2 /= np.linalg.norm(e2)
        sin = np.sqrt(1e-3 * 10.0 ** rng.uniform(-0.5, 0.5))
        cos = np.sqrt(1 - sin * sin) * rng.choice([-1, 1])
        X0 = rng.uniform(-300, 300, 3)
        X = np.stack([X0, X0 + e1 * rng.uniform(300, 1500), X0 + (cos * e1 + sin * e2) * rng.uniform(300, 1500),
                      X0 + rng.uniform(-800, 800, 3)])
        Cc = rng.normal(size=3)
        Cc = Cc / np.linalg.norm(Cc) * rng.uniform(1500, 4000)
        R = look_at(Cc, X[:3].mean(0), rng)
        if not ((X - Cc) @ R.T)[:, 2].min() > 100:
            continue
        s = _near_threshold(X, R, Cc, cam, thr, integer, rng, shim)
        if s is not None:
            sets.append(s)
    return _stack(sets)


NEW_FAMILIES = {"near_camera": near_camera, "tiny_triangle": tiny_triangle, "ill_conditioned": ill_conditioned}
