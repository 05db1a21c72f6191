"""numpy restatement of the reference's score-CNN pre-training data path (train_score.cpp's assembleData), written from
the reference's source types rather than from the device code:

    grid_bounds   stochasticSubSample's float loop (cnn.h:348-374)
    draw          the ThreadRand streams' draw: irand(0, F), the grid, then per hypothesis irand(0, 2) and getRandHyp
    sample        poseGT * Hypothesis(v), calcAngularDistance, the translation error, the label and the 5 deg / 50 mm flag
    diff_map      getDiffMap of the noisy pose (our2cv, cv::projectPoints in double, the float rounding, clamp at 100)

It reuses obj_oracle's MT19937 word source, its Lemire draw and its closed-form 3x3 inverse.  Double arithmetic is
spelled operation by operation on Python floats (IEEE doubles), log is the C library's (math.log)."""
import math

import numpy as np

import obj_oracle as OO

F32 = np.float32
PI_REF = 3.1415926     # types.h:33


def grid_bounds(size):
    """Upper bounds of stochasticSubSample's cells along an axis of `size` pixels (float32 accumulation)."""
    stride = F32(F32(size - 42) / F32(40))
    end = F32(size - 21 + 1)
    out = []
    v = F32(stride + F32(21))
    while v <= end:
        out.append(v)
        v = F32(v + stride)
    return out


def canonical53(w0, w1):
    r = (float(w0) + float(w1) * 4294967296.0) / 18446744073709551616.0
    return math.nextafter(1.0, 0.0) if r >= 1.0 else r


def canonical(words):
    w0 = words()
    w1 = words()
    return canonical53(w0, w1)


def uniform_real(words, a, b):
    return canonical(words) * (b - a) + a


def normal(words, stddev, mean=0.0):
    """A fresh std::normal_distribution<double>: libstdc++'s polar method, y * mult."""
    while True:
        x = 2.0 * canonical(words) - 1.0
        y = 2.0 * canonical(words) - 1.0
        r2 = x * x + y * y
        if not (r2 > 1.0 or r2 == 0.0):
            break
    mult = math.sqrt(-2 * math.log(r2) / r2)
    return y * mult * stddev + mean


def rand_hyp(words, gauss_rot, gauss_trans):
    """getRandHyp as its 6-vector; GCC evaluates the constructor arguments right to left (z, y, x)."""
    tz = normal(words, float(F32(gauss_trans)))
    ty = normal(words, float(F32(gauss_trans)))
    tx = normal(words, float(F32(gauss_trans)))
    az = uniform_real(words, 0.0, 1.0)
    ay = uniform_real(words, 0.0, 1.0)
    ax = uniform_real(words, 0.0, 1.0)
    inv = 1.0 / math.sqrt(ax * ax + ay * ay + az * az)
    ax, ay, az = ax * inv, ay * inv, az * inv
    g = normal(words, float(F32(gauss_rot)))
    k = PI_REF / 180.0
    return np.array([ax * g * k, ay * g * k, az * g * k, tx, ty, tz])


def draw(state, n_frames, width, height, n_images, hyps):
    """One round of assembleData's draw; state [T][625] is advanced in place.  Returns img [n_images], pix
    [n_images][1600][2] (cell y * 40 + x), drift [n_images * hyps], noise [n_images * hyps][6]."""
    T = state.shape[0]
    xb, yb = grid_bounds(width), grid_bounds(height)
    img = np.zeros(n_images, np.int32)
    pix = np.zeros((n_images, 1600, 2), np.int32)
    drift = np.zeros(n_images * hyps, np.int32)
    noise = np.zeros((n_images * hyps, 6))
    streams = [OO._Words(state[t]) for t in range(T)]
    for i in range(n_images):
        w = streams[0]
        img[i] = OO.lemire(w, n_frames)
        for sx in range(len(xb)):
            x0, x1 = (float(xb[sx - 1]) if sx else 21.0), float(xb[sx])
            for sy in range(len(yb)):
                y0, y1 = (float(yb[sy - 1]) if sy else 21.0), float(yb[sy])
                cx = int(uniform_real(w, x0, x1))
                cy = int(uniform_real(w, y0, y1))
                if sx < 40 and sy < 40:
                    pix[i, sy * 40 + sx] = (cx, cy)
        for t in range(T):
            h0, hc = OO.stream_chunk(hyps, T, t)
            for h in range(h0, h0 + hc):
                k = i * hyps + h
                drift[k] = OO.lemire(streams[t], 2)
                noise[k] = rand_hyp(streams[t], 2, 2) if drift[k] == 0 else rand_hyp(streams[t], 10, 100)
    for t in range(T):
        state[t] = streams[t].state()
    return img, pix, drift, noise


def rodrigues_v2m(r):
    """cv::Rodrigues, vector -> matrix: c I + (1 - c) r r^T + s [r]x of the unit axis."""
    r = np.asarray(r, np.float64)
    th = math.sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2])
    if th < 2.220446049250313e-16:
        return np.eye(3)
    c, s = math.cos(th), math.sin(th)
    u = r / th
    K = np.array([[0, -u[2], u[1]], [u[2], 0, -u[0]], [-u[1], u[0], 0]])
    return c * np.eye(3) + (1 - c) * np.outer(u, u) + s * K


def rodrigues_m2v(R):
    """cv::Rodrigues, matrix -> vector, for a rotation matrix away from 180 degrees."""
    rx, ry, rz = R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]
    s = math.sqrt((rx * rx + ry * ry + rz * rz) * 0.25)
    c = min(1.0, max(-1.0, (R[0, 0] + R[1, 1] + R[2, 2] - 1) * 0.5))
    th = math.acos(c)
    if s < 1e-5:
        if c > 0:
            return np.zeros(3)
        # 180 degrees: the axis from the diagonal, signs from the off-diagonal entries
        ax = math.sqrt(max((R[0, 0] + 1) * 0.5, 0.0))
        ay = math.sqrt(max((R[1, 1] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 1] < 0 else 1.0)
        az = math.sqrt(max((R[2, 2] + 1) * 0.5, 0.0)) * (-1.0 if R[0, 2] < 0 else 1.0)
        if abs(ax) < abs(ay) and abs(ax) < abs(az) and (R[1, 2] > 0) != (ay * az > 0):
            az = -az
        return np.array([ax, ay, az]) * (th / math.sqrt(ax * ax + ay * ay + az * az))
    return np.array([rx, ry, rz]) * (th / (2 * s))


def hypothesis_rotation(v):
    """Hypothesis(rodVecAndTrans): the identity for |r| <= 1e-5 (Hypothesis.cpp:91-96)."""
    return rodrigues_v2m(v[:3]) if math.sqrt(v[0] ** 2 + v[1] ** 2 + v[2] ** 2) > 1e-5 else np.eye(3)


def noise_pose(gt_jp, v):
    """poseGT = Hypothesis(info) (rotation through float, centre through float * 1e3), poseNoise = poseGT * Hypothesis(v)
    as the 4x4 product.  Returns (Rg, tg, Rn, tn)."""
    p = np.asarray(gt_jp, np.float64)
    Rg = p[:9].astype(np.float32).astype(np.float64).reshape(3, 3)
    tg = (p[9:12] / 1000.0).astype(np.float32).astype(np.float64) * 1e3
    Rh = hypothesis_rotation(v)
    return Rg, tg, Rg @ Rh, Rg @ np.asarray(v[3:6]) + tg


def sample(gt_jp, v, temperature=10.0):
    """(label, correct, angle in degrees, translation error in mm) of one perturbed pose."""
    Rg, tg, Rn, tn = noise_pose(gt_jp, v)
    Ri = OO.inv_rotation(Rn)
    trace = min(3.0, max(-1.0, float(np.trace(Rg @ Ri))))
    ang = 180 * math.acos((trace - 1.0) / 2.0) / math.pi
    dt = float(np.linalg.norm(tg - tn))
    label = float(-F32(temperature)) * max(ang, dt / 10.0)
    return label, int(ang < 5 and dt < 50), ang, dt


def diff_map(gt_jp, v, coords, pix, f, cx, cy):
    """getDiffMap of the noisy pose: our2cv (rows 1, 2 negated, Rodrigues to a vector), cv::projectPoints in double
    from the matrix rebuilt from that vector, projection rounded to float, float difference to the pixel, norm in
    double, clamp at 100 -> float32 [1600] (cell y * 40 + x)."""
    _, _, Rn, tn = noise_pose(gt_jp, v)
    rm = Rn.copy()
    rm[1:] = -rm[1:]
    U, _, Vt = np.linalg.svd(rm)          # cv::Rodrigues projects its input onto the nearest rotation first
    R = rodrigues_v2m(rodrigues_m2v(U @ Vt))
    t = np.array([tn[0], -tn[1], -tn[2]])
    X = np.asarray(coords, np.float32).astype(np.float64)
    q = X @ R.T + t
    z = np.where(q[:, 2] != 0, 1.0 / np.where(q[:, 2] != 0, q[:, 2], 1.0), 1.0)
    pu = (q[:, 0] * z * f + cx).astype(np.float32)
    pv = (q[:, 1] * z * f + cy).astype(np.float32)
    du = np.asarray(pix[:, 0], np.float32) - pu
    dv = np.asarray(pix[:, 1], np.float32) - pv
    e = np.sqrt(du.astype(np.float64) ** 2 + dv.astype(np.float64) ** 2)
    return np.minimum(e, 100.0).astype(np.float32)


def shuffle_rounds(n, seed, n_rounds):
    """train_score.cpp:381-384 for n_rounds rounds: std::shuffle of a fresh iota(n) per round by one continuing
    std::mt19937(seed) (libstdc++'s two positions per draw while (2^32 - 1) / n >= n)."""
    bg = np.random.MT19937()
    bg._legacy_seeding(seed)
    nxt = lambda: int(bg.random_raw())   # noqa: E731
    out = []
    for _ in range(n_rounds):
        a = list(range(n))
        if 0xffffffff // n >= n:
            i = 1
            if n % 2 == 0:
                j = OO.lemire(nxt, 2)
                a[i], a[j] = a[j], a[i]
                i += 1
            while i != n:
                b0 = i + 1
                b1 = b0 + 1
                x = OO.lemire(nxt, b0 * b1)
                p0, p1 = x // b1, x % b1
                a[i], a[p0] = a[p0], a[i]
                i += 1
                a[i], a[p1] = a[p1], a[i]
                i += 1
        else:
            for i in range(1, n):
                j = OO.lemire(nxt, i + 1)
                a[i], a[j] = a[j], a[i]
        out.append(a)
    return np.array(out, np.int32)
