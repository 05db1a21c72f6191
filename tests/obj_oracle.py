"""numpy restatement of the reference's coordinate-CNN pre-training data path (train_obj.cpp and jp::Dataset), written
from the reference's source types rather than from the device code:

    register_depth   Dataset::getDepth with rawData (dataset.h:180-202), mapDepthToRGB (:93-111)
    obj_coords       Dataset::getObj (dataset.h:226-255): pxToEye (dataset.cpp:37-56), Hypothesis::invTransform
    draw             assembleData's random draw (train_obj.cpp:47-102) over T ThreadRand streams
    mm_to_m          cv::Vec3f /= 1000

The x86 conversions (cvttss2si / cvttsd2si, then the low 16 bits for a short) are spelled out; float arithmetic stays in
float32 and double arithmetic in float64, operation by operation, so nothing is contracted.  The random stream is numpy's
MT19937 with the legacy seeding, which is std::mt19937's seed and state layout (624 words and the position)."""
import numpy as np

F32 = np.float32
INT_MIN = -2147483648


def cam_dict(cam):
    """An RGBDCamera (ctypes) or a dict -> dict of the reference's dP fields."""
    if isinstance(cam, dict):
        return cam
    return dict(focal=cam.focal, x_shift=cam.x_shift, y_shift=cam.y_shift, secondary_focal=cam.secondary_focal,
                raw_x_shift=cam.raw_x_shift, raw_y_shift=cam.raw_y_shift,
                sensor_trans=np.array(list(cam.sensor_trans), np.float64).reshape(4, 4), raw_data=cam.raw_data,
                width=cam.width, height=cam.height)


def cvtt_i32(v):
    """(int) of float32 / float64 values as x86-64 does it: truncation, INT_MIN for NaN and values out of range."""
    v = np.asarray(v)
    w = v.astype(np.float64)
    ok = (w > -2147483649.0) & (w < 2147483648.0)
    out = np.full(v.shape, INT_MIN, np.int64)
    out[ok] = np.trunc(w[ok]).astype(np.int64)
    return out


def low16(v):
    return (np.asarray(v, np.int64) & 0xffff).astype(np.uint16).view(np.int16)


def mm_to_m(v):
    """saturate_cast<float>(float(v) * (1. / 1000)): OpenCV's Vec::operator/=(int)."""
    return (np.asarray(v).astype(np.float32).astype(np.float64) * (1. / 1000)).astype(np.float32)


def inv_rotation(R):
    """cv::Mat::inv of a 3x3 CV_64F matrix: OpenCV's closed form (1 / det3 times the cofactors)."""
    S = R
    d = S[0, 0] * (S[1, 1] * S[2, 2] - S[1, 2] * S[2, 1]) - S[0, 1] * (S[1, 0] * S[2, 2] - S[1, 2] * S[2, 0]) + \
        S[0, 2] * (S[1, 0] * S[2, 1] - S[1, 1] * S[2, 0])
    d = 1. / d
    t = np.empty(9)
    t[0] = (S[1, 1] * S[2, 2] - S[1, 2] * S[2, 1]) * d
    t[1] = (S[0, 2] * S[2, 1] - S[0, 1] * S[2, 2]) * d
    t[2] = (S[0, 1] * S[1, 2] - S[0, 2] * S[1, 1]) * d
    t[3] = (S[1, 2] * S[2, 0] - S[1, 0] * S[2, 2]) * d
    t[4] = (S[0, 0] * S[2, 2] - S[0, 2] * S[2, 0]) * d
    t[5] = (S[0, 2] * S[1, 0] - S[0, 0] * S[1, 2]) * d
    t[6] = (S[1, 0] * S[2, 1] - S[1, 1] * S[2, 0]) * d
    t[7] = (S[0, 1] * S[2, 0] - S[0, 0] * S[2, 1]) * d
    t[8] = (S[0, 0] * S[1, 1] - S[0, 1] * S[1, 0]) * d
    return t.reshape(3, 3)


def inv_rotation_elimination(R):
    """The inverse the API shim's Mat::inv computes (oracle/shim/opencv2/opencv.hpp): Gauss-Jordan elimination with
    partial pivoting.  Real OpenCV uses the closed form above; the reference-built fixture (ref_obj.npz) was made through
    the shim, so it is compared with this one."""
    n = 3
    w = np.zeros((3, 6))
    w[:, :3] = R
    w[:, 3:] = np.eye(3)
    for k in range(n):
        p = k
        for i in range(k + 1, n):
            if abs(w[i, k]) > abs(w[p, k]):
                p = i
        if p != k:
            w[[p, k]] = w[[k, p]]
        d = 1.0 / w[k, k]
        for j in range(6):
            w[k, j] *= d
        for i in range(n):
            if i == k:
                continue
            f = w[i, k]
            if f != 0:
                for j in range(6):
                    w[i, j] -= f * w[k, j]
    return w[:, 3:].copy()


def fixture_depth(F, H, W, salt=0):
    """Deterministic raw depth (integer hashing, no random generator): 500..3999 mm with holes (0), 7-Scenes' invalid
    marker 65535 and values >= 32768."""
    f, y, x = np.meshgrid(np.arange(F, dtype=np.uint64), np.arange(H, dtype=np.uint64), np.arange(W, dtype=np.uint64),
                          indexing="ij")
    h = (x * np.uint64(7919) + y * np.uint64(104729) + f * np.uint64(1299709) + np.uint64(salt) * np.uint64(15485863))
    h = (h * np.uint64(2654435761)) & np.uint64(0xffffffff)
    h2 = ((h ^ (h >> np.uint64(13))) * np.uint64(2246822519)) & np.uint64(0xffffffff)
    d = (np.uint64(500) + h % np.uint64(3500)).astype(np.uint16)
    sel = h2 % np.uint64(100)
    d[sel < 10] = 0
    d[(sel >= 10) & (sel < 13)] = 65535
    d[(sel >= 13) & (sel < 15)] = (np.uint64(32768) + h2[(sel >= 13) & (sel < 15)] % np.uint64(32767)).astype(np.uint16)
    return d


def coded_bgr(F, H, W):
    """BGR bytes that give away (frame, x, y): B = x & 255, G = y & 255, R = 16 frame + (x >> 8) + 4 (y >> 8)."""
    ys, xs = np.mgrid[0:H, 0:W]
    out = np.zeros((F, H, W, 3), np.uint8)
    for f in range(F):
        out[f, ..., 0] = xs & 255
        out[f, ..., 1] = ys & 255
        out[f, ..., 2] = (16 * f + (xs >> 8) + 4 * (ys >> 8)) & 255
    return out


def decode_bgr(px):
    """(frame, x, y) of coded BGR values [..., 3]."""
    b, g, r = (np.asarray(px[..., k]).astype(np.int64) for k in range(3))
    return r // 16, b + 256 * ((r % 16) % 4), g + 256 * ((r % 16) // 4)


def map_depth_to_rgb(cam, x, y, raw):
    """mapDepthToRGB(int x, int y, short depth) for arrays; returns the (int) target columns and rows."""
    c = cam_dict(cam)
    W, H = c["width"], c["height"]
    depth = np.asarray(raw, np.uint16).view(np.int16).astype(np.float64)   # jp::depth_t -> short
    sf = np.float64(F32(c["secondary_focal"])) / depth
    e0 = (x.astype(np.float64) - (W / 2.0 + np.float64(F32(c["raw_x_shift"])))) / sf
    e1 = -((y.astype(np.float64) - (H / 2.0 + np.float64(F32(c["raw_y_shift"])))) / sf)
    e2 = -depth
    S = c["sensor_trans"]
    m0 = 0.0 + S[0, 0] * e0 + S[0, 1] * e1 + S[0, 2] * e2 + S[0, 3] * 1.0
    m1 = 0.0 + S[1, 0] * e0 + S[1, 1] * e1 + S[1, 2] * e2 + S[1, 3] * 1.0
    f = np.float64(F32(c["focal"])) / depth
    cx = np.float64(F32(F32(W) / F32(2)) + F32(c["x_shift"]))
    cy = np.float64(F32(F32(H) / F32(2)) + F32(c["y_shift"]))
    return cvtt_i32(m0 * f + cx + 0.5), cvtt_i32(-(m1 * f) + cy + 0.5)


def register_depth(cam, raw):
    """getDepth of frames raw [F][H][W] uint16 -> (registered depth, dropped target counts [F])."""
    c = cam_dict(cam)
    raw = np.asarray(raw, np.uint16)
    if not c["raw_data"]:
        return raw.copy(), np.zeros(raw.shape[0], np.int32)
    F, H, W = raw.shape
    out = np.zeros_like(raw)
    dropped = np.zeros(F, np.int32)
    xs, ys = np.meshgrid(np.arange(W), np.arange(H), indexing="xy")
    # the reference's loop order: x outer, y inner
    order = np.lexsort((ys.ravel(), xs.ravel()))
    xo, yo = xs.ravel()[order], ys.ravel()[order]
    for f in range(F):
        d = raw[f].ravel()[order]
        nz = d != 0
        xi, yi, di = xo[nz], yo[nz], d[nz]
        nx, ny = map_depth_to_rgb(c, xi, yi, di)
        inside = (nx >= 0) & (ny >= 0) & (nx < W) & (ny < H)
        dropped[f] = int((~inside).sum())
        tgt = (ny[inside] * W + nx[inside])[::-1]
        val = di[inside][::-1]
        u, first = np.unique(tgt, return_index=True)   # first in reverse order = the last write
        out[f].ravel()[u] = val[first]
    return out, dropped


def pose_parts(pose, inv=None):
    """Hypothesis(info) from a jp pose [12] (row-major rotation, translation in mm, as dsac_forward's gt_jp): info_t holds
    the rotation and the centre in metres in float."""
    p = np.asarray(pose, np.float64)
    R = p[:9].astype(np.float32).astype(np.float64)
    c = (p[9:12] / 1000.0).astype(np.float32).astype(np.float64)
    return (inv or inv_rotation)(R.reshape(3, 3)), c * 1e3


def obj_coords(cam, depth, pose, inv=None):
    """getObj of one registered depth frame [H][W] -> int16 [H][W][3] (mm).  inv: the 3x3 inverse (default: OpenCV's)."""
    c = cam_dict(cam)
    H, W = depth.shape
    d = np.asarray(depth, np.uint16)
    ys, xs = np.mgrid[0:H, 0:W]
    cx = F32(F32(W) / F32(2)) + F32(c["x_shift"])
    cy = F32(F32(H) / F32(2)) + F32(c["y_shift"])
    with np.errstate(divide="ignore", invalid="ignore"):   # depth 0 is zeroed below
        fd = F32(c["focal"]) / d.astype(np.float32)
        e0 = low16(cvtt_i32((xs.astype(np.float32) - cx) / fd)).astype(np.float64)
        e1 = low16(cvtt_i32(-((ys.astype(np.float32) - cy) / fd))).astype(np.float64)
    e2 = low16(-d.astype(np.int64)).astype(np.float64)
    Ri, t = pose_parts(pose, inv)
    q = (e0 - t[0], e1 - t[1], e2 - t[2])
    out = np.zeros((H, W, 3), np.int16)
    for r in range(3):
        s = 0.0 + Ri[r, 0] * q[0] + Ri[r, 1] * q[1] + Ri[r, 2] * q[2]
        out[..., r] = low16(cvtt_i32(s))
    out[d == 0] = 0
    return out


def rejected_word_positions(seed, rng, count=1, chunk=1 << 24):
    """Positions (0-based) in std::mt19937(seed)'s output of the first `count` words a Lemire draw over rng values
    rejects (low 32 bits of word * rng below 2^32 mod rng)."""
    bg = np.random.MT19937()
    bg._legacy_seeding(seed)
    thr = (2 ** 32 - rng) % rng
    out, base = [], 0
    while len(out) < count:
        w = bg.random_raw(chunk).astype(np.uint64)
        hit = np.nonzero(((w * np.uint64(rng)) & np.uint64(0xffffffff)) < np.uint64(thr))[0]
        out += [base + int(h) for h in hit[:count - len(out)]]
        base += chunk
    return out


def state_at(seed, pos):
    """[625] std::mt19937(seed) state after `pos` words."""
    bg = np.random.MT19937()
    bg._legacy_seeding(seed)
    left = pos
    while left:
        k = min(left, 1 << 24)
        bg.random_raw(k)
        left -= k
    s = bg.state["state"]
    return np.concatenate([np.asarray(s["key"], np.uint32), np.array([s["pos"]], np.uint32)])


def stream_chunk(n, T, t):
    q, r = divmod(n, T)
    cnt = q + (1 if t < r else 0)
    return t * q + min(t, r), cnt


def rng_init(seed, T):
    """ThreadRand::init(seed): [T][625] uint32 = std::mt19937(seed + t) words and position."""
    st = np.zeros((T, 625), np.uint32)
    for t in range(T):
        bg = np.random.MT19937()
        bg._legacy_seeding((seed + t) & 0xffffffff)
        s = bg.state["state"]
        st[t, :624] = s["key"]
        st[t, 624] = s["pos"]
    return st


class _Words:
    def __init__(self, row):
        self.bg = np.random.MT19937()
        self.bg.state = {"bit_generator": "MT19937", "state": {"key": np.array(row[:624], np.uint32), "pos": int(row[624])}}
        self.buf = np.empty(0, np.uint64)
        self.i = 0

    def __call__(self):
        if self.i == len(self.buf):
            self.buf = self.bg.random_raw(1)   # one at a time keeps the generator's state at the consumed position
            self.i = 0
        w = int(self.buf[self.i])
        self.i += 1
        return w

    def state(self):
        s = self.bg.state["state"]
        return np.concatenate([np.asarray(s["key"], np.uint32), np.array([s["pos"]], np.uint32)])


REJECTED = [0]   # words the Lemire draws below have rejected so far (tests read it to know the path was taken)


def lemire(next_word, rng):
    """uniform_int_distribution over rng values from a 32-bit generator (libstdc++ _S_nd)."""
    product = next_word() * rng
    low = product & 0xffffffff
    if low < rng:
        threshold = (2 ** 32 - rng) % rng
        while low < threshold:
            REJECTED[0] += 1
            product = next_word() * rng
            low = product & 0xffffffff
    return product >> 32


def draw(cam, depth, poses, state, n_images=100, n_patches=512, max_attempts=1 << 20, coords=None):
    """One round of assembleData's draw.  state [T][625] is advanced in place.  Returns img [n], centre [n][2], label
    [n][3] float32 (n = n_images * n_patches) and status [n_images] (8 = exhausted)."""
    c = cam_dict(cam)
    F = depth.shape[0]
    W, H = c["width"], c["height"]
    if coords is None:
        coords = np.stack([obj_coords(c, depth[f], poses[f]) for f in range(F)])
    valid = (coords != 0).any(-1)
    T = state.shape[0]
    n = n_images * n_patches
    img = np.zeros(n, np.int32)
    centre = np.full((n, 2), -1, np.int32)
    label = np.zeros((n, 3), np.float32)
    status = np.zeros(n_images, np.uint32)
    for t in range(T):
        i0, cnt = stream_chunk(n_images, T, t)
        words = _Words(state[t])
        for i in range(i0, i0 + cnt):
            f = lemire(words, F)
            img[i * n_patches:(i + 1) * n_patches] = f
            vf = valid[f]
            for j in range(n_patches):
                found = False
                for _ in range(max_attempts):
                    x = lemire(words, W - 42) + 21
                    y = lemire(words, H - 42) + 21
                    if vf[y, x]:
                        found = True
                        break
                if not found:
                    status[i] = 8
                    break
                k = i * n_patches + j
                centre[k] = (x, y)
                label[k] = mm_to_m(coords[f, y, x])
        state[t] = words.state()
    return img, centre, label, status


def gather_patches(frames, frame_idx, centre, mean=127.0):
    """assembleData's patch copy (train_obj.cpp:83-91) minus the mean, channel-major [n][3][42][42] float32."""
    n = len(frame_idx)
    out = np.zeros((n, 3, 42, 42), np.float32)
    for k in range(n):
        x, y = int(centre[k][0]), int(centre[k][1])
        p = frames[frame_idx[k], y - 21:y + 21, x - 21:x + 21, :].astype(np.float32) - np.float32(mean)
        out[k] = p.transpose(2, 0, 1)
    return out
