"""numpy restatement of the pre-training data paths with a camera per dataset frame (what the reference computes with
each frame's dP in force), on top of the single-camera restatements tests/obj_oracle.py and tests/score_oracle.py:

    frame_cams       one camera, or a sequence of F, as F camera dicts
    register_depth   Dataset::getDepth of every frame with its own camera
    draw             assembleData's draw (train_obj.cpp:47-102) with each frame's getObj labels
    cam_mat          getCamMat() (properties.cpp:308-311) of a dataset camera: what train_score.cpp projects with
    round_maps       getDiffMap of every (image, hypothesis) of a score draw, with one camera or each frame's own

The random streams and the per-pixel arithmetic are obj_oracle's and score_oracle's."""
import numpy as np

import obj_oracle as OO
import score_oracle as SO

F32 = np.float32


def frame_cams(cam, F):
    """[F] camera dicts: F copies of one camera (an RGBDCamera or a dict), or a sequence of F cameras, one per frame."""
    if isinstance(cam, dict) or not hasattr(cam, "__len__"):
        return [OO.cam_dict(cam)] * F
    if len(cam) != F:
        raise ValueError("%d cameras for %d frames" % (len(cam), F))
    return [OO.cam_dict(c) for c in cam]


def register_depth(cam, raw):
    """getDepth of frames raw [F][H][W] uint16, frame f with camera f -> (registered depth, dropped counts [F])."""
    raw = np.asarray(raw, np.uint16)
    cams = frame_cams(cam, raw.shape[0])
    out = np.zeros_like(raw)
    dropped = np.zeros(raw.shape[0], np.int32)
    for f, c in enumerate(cams):
        r, d = OO.register_depth(c, raw[f:f + 1])
        out[f], dropped[f] = r[0], d[0]
    return out, dropped


def draw(cam, depth, poses, state, n_images=100, n_patches=512, max_attempts=1 << 20):
    """One round of assembleData's draw over T streams (state [T][625], advanced in place) on a dataset whose frame f has
    camera f: the frame and centre draws do not depend on the camera, the validity test and the labels are getObj with
    the drawn frame's camera.  Returns img [n], centre [n][2], label [n][3] float32 and status [n_images]."""
    F = depth.shape[0]
    cams = frame_cams(cam, F)
    W, H = cams[0]["width"], cams[0]["height"]
    T = state.shape[0]
    n = n_images * n_patches
    img = np.zeros(n, np.int32)
    centre = np.full((n, 2), -1, np.int32)
    label = np.zeros((n, 3), np.float32)
    status = np.zeros(n_images, np.uint32)
    coords = {}
    for t in range(T):
        i0, cnt = OO.stream_chunk(n_images, T, t)
        words = OO._Words(state[t])
        for i in range(i0, i0 + cnt):
            f = OO.lemire(words, F)
            if f not in coords:
                coords[f] = OO.obj_coords(cams[f], depth[f], poses[f])
            co = coords[f]
            img[i * n_patches:(i + 1) * n_patches] = f
            for j in range(n_patches):
                for _ in range(max_attempts):
                    x = OO.lemire(words, W - 42) + 21
                    y = OO.lemire(words, H - 42) + 21
                    if (co[y, x] != 0).any():
                        break
                else:
                    status[i] = 8
                    break
                centre[i * n_patches + j] = (x, y)
                label[i * n_patches + j] = OO.mm_to_m(co[y, x])
        state[t] = words.state()
    return img, centre, label, status


def cam_mat(cam):
    """getCamMat() of an RGBDCamera or camera dict as float64 (f, cx, cy): the float focal length and
    centerX = imageWidth / 2 + xShift, the INTEGER half width plus the float shift, rounded to float (likewise cy)."""
    c = OO.cam_dict(cam)
    f = F32(c["focal"])
    cx = F32(F32(c["width"] // 2) + F32(c["x_shift"]))
    cy = F32(F32(c["height"] // 2) + F32(c["y_shift"]))
    return float(f), float(cx), float(cy)


def round_maps(img, gt_jp, noise, coords, pix, hyps, cams):
    """score_oracle.diff_map of pose k = i * hyps + h of a score draw: [n_images * hyps][1600].  cams: one (f, cx, cy)
    for every image, or a sequence of dataset cameras, image i then projecting with cam_mat(cams[img[i]])."""
    out = np.zeros((len(img) * hyps, 1600), np.float32)
    for i, fr in enumerate(img):
        f, cx, cy = cams if len(cams) == 3 and np.isscalar(cams[0]) else cam_mat(cams[fr])
        for h in range(hyps):
            k = i * hyps + h
            out[k] = SO.diff_map(gt_jp[fr], noise[k], coords[i], pix[i], f, cx, cy)
    return out
