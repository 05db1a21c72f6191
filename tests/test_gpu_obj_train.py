"""Coordinate-CNN pre-training on the device: registration, getObj, the ThreadRand draw and the patch gather bit for bit
against the numpy restatement (tests/obj_oracle.py); an RGB-D scene through getObj into dsac_forward; and a short
pre-training run."""
import os

import numpy as np
import pytest
import torch

import obj_oracle as OO
from conftest import GOLDEN

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng(engine_mod):
    e = engine_mod.Engine(max_frames=4, n_hyps=256)
    yield e
    e.close()


def seven_scenes_trans():
    from dsac_b200.obj_train import read_sensor_trans
    return read_sensor_trans(os.path.join(GOLDEN, "sensorTrans_7scenes.dat"))


def synthetic_depth(rng, F, H, W, holes=0.1):
    d = rng.integers(500, 4000, (F, H, W)).astype(np.uint16)
    d[rng.random((F, H, W)) < holes] = 0
    d[rng.random((F, H, W)) < 0.03] = 65535
    d[rng.random((F, H, W)) < 0.02] = rng.integers(32768, 65535)
    return d


def random_poses(rng, F):
    from scipy.spatial.transform import Rotation
    P = np.zeros((F, 12))
    for f in range(F):
        P[f, :9] = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix().reshape(9)
        P[f, 9:] = rng.uniform(-2000, 2000, 3)
    return P


def coded_bgr(F, H, W):
    """BGR bytes that give away (frame, x, y): B = x, G = y (mod 256), R = 16 frame + (x >> 8) + 4 (y >> 8)."""
    ys, xs = np.mgrid[0:H, 0:W]
    out = np.zeros((F, H, W, 3), np.uint8)
    for f in range(F):
        out[f, ..., 0] = xs & 255
        out[f, ..., 1] = ys & 255
        out[f, ..., 2] = (16 * f + (xs >> 8) + 4 * (ys >> 8)) & 255
    return out


def scene(engine_mod, eng, F, H, W, rng, trans=None, raw_data=1, **cam_kw):
    from dsac_b200.obj_train import RGBDScene
    cam = engine_mod.default_rgbd_camera(width=W, height=H, raw_data=raw_data,
                                         sensor_trans=np.eye(4) if trans is None else trans, **cam_kw)
    raw = synthetic_depth(rng, F, H, W)
    poses = random_poses(rng, F)
    return RGBDScene(eng, coded_bgr(F, H, W), raw, poses, cam), raw, poses


@pytest.mark.parametrize("W,H,trans,raw_data,xs", [(640, 480, "7scenes", 1, 0.0), (640, 480, "7scenes", 0, 0.0),
                                                   (77, 53, "7scenes", 1, 0.25), (128, 96, "identity", 1, 0.0)])
def test_registration_and_obj_coords_match_oracle(engine_mod, eng, W, H, trans, raw_data, xs):
    rng = np.random.default_rng(W + H + raw_data)
    st = seven_scenes_trans() if trans == "7scenes" else None
    sc, raw, poses = scene(engine_mod, eng, 3, H, W, rng, st, raw_data, x_shift=xs, y_shift=-xs)
    reg, dropped = OO.register_depth(sc.cam, raw)
    assert np.array_equal(sc.depth_u16(), reg)
    assert np.array_equal(sc.dropped.cpu().numpy(), dropped)
    co = sc.scene_coords([2, 0, 1]).cpu().numpy()
    for k, f in enumerate([2, 0, 1]):
        assert np.array_equal(co[k], OO.obj_coords(sc.cam, reg[f], poses[f]))


def test_scene_coords_refuses_frames_outside_the_scene(engine_mod, eng):
    rng = np.random.default_rng(12)
    sc, _, _ = scene(engine_mod, eng, 2, 48, 64, rng)
    for bad in (2, -1, [0, 2], []):
        with pytest.raises(IndexError):
            sc.scene_coords(bad)
    # the entry point itself gives a listed frame outside the scene a zero image instead of reading beyond it
    ids = torch.tensor([1, 7, -3], dtype=torch.int32, device="cuda")
    out = torch.full((3, 48, 64, 3), 5, dtype=torch.int16, device="cuda")
    eng.obj_coords_device(sc.cam, 2, 3, sc.depth.data_ptr(), sc.gt_jp.data_ptr(), out.data_ptr(), d_idx=ids.data_ptr())
    assert torch.equal(out[0], sc.scene_coords(1)) and (out[1:] == 0).all()


def test_out_of_image_targets_are_counted(engine_mod, eng):
    rng = np.random.default_rng(4)
    sc, raw, _ = scene(engine_mod, eng, 2, 96, 128, rng, raw_x_shift=-30.0)
    reg, dropped = OO.register_depth(sc.cam, raw)
    assert (dropped > 0).all()
    assert np.array_equal(sc.dropped.cpu().numpy(), dropped)
    assert (sc.status.cpu().numpy() == engine_mod.ST_DEPTH_DROPPED).all()
    assert np.array_equal(sc.depth_u16(), reg)


def _compare_draw(r, cam, depth, poses, st, n_images, n_patches, max_attempts=1 << 20):
    img, centre, label, status = r.draw(n_images, n_patches)
    oi, oc, ol, os_ = OO.draw(cam, depth, poses, st, n_images, n_patches, max_attempts=max_attempts)
    assert np.array_equal(img.cpu().numpy(), oi)
    assert np.array_equal(centre.cpu().numpy(), oc)
    assert np.array_equal(label.cpu().numpy().view(np.uint32), ol.view(np.uint32))
    assert np.array_equal(status.cpu().numpy().astype(np.uint32), os_)
    assert np.array_equal(r.state.cpu().numpy().view(np.uint32), st)


@pytest.mark.parametrize("T", [1, 3, 16])
def test_draw_matches_oracle_over_two_rounds(engine_mod, eng, T):
    from dsac_b200.obj_train import ObjRound
    rng = np.random.default_rng(T)
    sc, _, poses = scene(engine_mod, eng, 5, 96, 128, rng)
    depth = sc.depth_u16()
    r = ObjRound(sc, seed=1305, n_streams=T)
    st = OO.rng_init(1305, T)
    assert np.array_equal(r.state.cpu().numpy().view(np.uint32), st)
    for _ in range(2):
        _compare_draw(r, sc.cam, depth, poses, st, 19, 70)


def test_full_round_at_640x480(engine_mod, eng):
    from dsac_b200.obj_train import ObjRound
    rng = np.random.default_rng(640)
    sc, _, poses = scene(engine_mod, eng, 4, 480, 640, rng, seven_scenes_trans())
    r = ObjRound(sc, seed=7, n_streams=6)
    st = OO.rng_init(7, 6)
    _compare_draw(r, sc.cam, sc.depth_u16(), poses, st, 100, 512)


def test_patches_at_drawn_centres(engine_mod, eng):
    from oracle import oracle as O
    from dsac_b200.obj_train import ObjRound
    rng = np.random.default_rng(9)
    sc, _, _ = scene(engine_mod, eng, 4, 96, 133, rng)
    r = ObjRound(sc, seed=3, n_streams=2)
    img, centre, _, _ = r.draw(7, 40)
    pt = r.patches().cpu().numpy()
    img, centre = img.cpu().numpy(), centre.cpu().numpy()
    bgr = sc.bgr.cpu().numpy()
    assert np.array_equal(pt.view(np.uint32), OO.gather_patches(bgr, img, centre).view(np.uint32))
    for k in range(0, len(img), 37):
        ref = O.gather_patches(bgr[img[k]], centre[k:k + 1])
        assert np.array_equal(pt[k:k + 1].view(np.uint32), ref.view(np.uint32))
        # the coded bytes give the centre and the frame back
        assert pt[k, 0, 21, 21] + 127 == centre[k, 0] & 255 and pt[k, 1, 21, 21] + 127 == centre[k, 1] & 255
    slots = torch.tensor([5, 0, 279], device="cuda")
    assert np.array_equal(r.patches(slots).cpu().numpy(), pt[[5, 0, 279]])


def test_all_invalid_frame_stops_at_the_attempt_bound(engine_mod, eng):
    from dsac_b200.obj_train import RGBDScene, ObjRound
    cam = engine_mod.default_rgbd_camera(width=64, height=50, raw_data=0)
    depth = np.full((2, 50, 64), 1200, np.uint16)
    depth[1] = 0                                     # frame 1: no valid pixel
    poses = np.tile(np.r_[np.eye(3).reshape(9), 0, 0, 0], (2, 1))
    sc = RGBDScene(eng, coded_bgr(2, 50, 64), depth, poses, cam)
    r = ObjRound(sc, seed=11, n_streams=2, max_attempts=100)
    st = OO.rng_init(11, 2)
    for _ in range(2):
        img, centre, _, status = r.draw(6, 20)
        oi, oc, ol, os_ = OO.draw(cam, depth, poses, st, 6, 20, max_attempts=100)
        assert np.array_equal(img.cpu().numpy(), oi) and np.array_equal(centre.cpu().numpy(), oc)
        assert np.array_equal(status.cpu().numpy().astype(np.uint32), os_)
        assert np.array_equal(r.state.cpu().numpy().view(np.uint32), st)
        bad = oi.reshape(6, 20)[:, 0] == 1
        assert (os_[bad] == engine_mod.ST_OBJ_DRAW_EXHAUSTED).all() and (os_[~bad] == 0).all()
        assert (oc.reshape(6, 20, 2)[bad] == -1).all()
    pt = r.patches()
    assert (pt[torch.as_tensor(np.repeat(bad, 20), device="cuda")] == 0).all()


def test_misuse_is_refused(engine_mod, eng):
    import ctypes as C
    E = engine_mod
    lib = eng.lib
    buf = torch.zeros(1 << 16, dtype=torch.int32, device="cuda")
    p = buf.data_ptr()
    cam = E.default_rgbd_camera(width=42, height=100)
    draw = lambda cam, F, n_img, T, att: lib.dsac_obj_draw_device(   # noqa: E731
        eng.h, C.byref(cam), F, C.c_void_p(p), C.c_void_p(p), n_img, 4, T, att, C.c_void_p(p), C.c_void_p(p),
        C.c_void_p(p), C.c_void_p(p), C.c_void_p(p), None)
    assert draw(cam, 1, 1, 1, 100) == -1                                      # no 42x42 patch centre fits
    ok = E.default_rgbd_camera(width=64, height=64)
    assert draw(ok, 0, 1, 1, 100) == -1 and draw(ok, 1, 1, 0, 100) == -1 and draw(ok, 1, 1, 1, 31) == -1
    assert lib.dsac_obj_rng_init_device(eng.h, 1, 0, C.c_void_p(p), None) == -1
    assert lib.dsac_register_depth_device(eng.h, C.byref(ok), 0, C.c_void_p(p), C.c_void_p(p + 64), None, None, None) == -1
    assert lib.dsac_register_depth_device(eng.h, C.byref(ok), 1, C.c_void_p(p), C.c_void_p(p), None, None, None) == -1
    assert lib.dsac_obj_coords_device(eng.h, C.byref(ok), 1, 0, None, C.c_void_p(p), C.c_void_p(p), C.c_void_p(p), None) == -1
    assert lib.dsac_obj_coords_device(eng.h, C.byref(ok), 0, 1, None, C.c_void_p(p), C.c_void_p(p), C.c_void_p(p), None) == -1
    assert lib.dsac_obj_coords_device(eng.h, C.byref(ok), 2, 3, None, C.c_void_p(p), C.c_void_p(p), C.c_void_p(p), None) == -1
    assert lib.dsac_gather_patches_at_device(eng.h, 1, C.c_void_p(p), 0, 64, 64, C.c_void_p(p), C.c_void_p(p),
                                             C.c_float(127), C.c_void_p(p), None, None) == -1
    assert lib.dsac_shuffle_permutation(0, 1, None) == -1
    torch.cuda.synchronize()


# ------------------------------------------------------------------ a rendered RGB-D scene
def render_room(n, rng, focal=585.0, W=640, H=480, lo=(-2500., -1500., -3500.), hi=(2500., 1500., 2500.), shift=(0, 0, 0)):
    """Depth (mm, uint16) of the walls of a box room seen by a camera with focal `focal` inside it, the jp poses
    (eye = R X + t) and a BGR texture that is a function of the world point."""
    from scipy.spatial.transform import Rotation
    lo, hi, shift = np.array(lo), np.array(hi), np.array(shift, np.float64)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    u = np.stack([(xs - W / 2) / focal, -(ys - H / 2) / focal, -np.ones_like(xs)], -1)
    depth = np.zeros((n, H, W), np.uint16)
    poses = np.zeros((n, 12))
    bgr = np.zeros((n, H, W, 3), np.uint8)
    for f in range(n):
        R = Rotation.from_rotvec(rng.uniform(-0.4, 0.4, 3)).as_matrix()
        c = rng.uniform(-500, 500, 3)
        t = -R @ c
        w = u @ R            # R^T u per pixel
        with np.errstate(divide="ignore"):
            s = np.where(w > 0, (hi - c) / w, (lo - c) / w)
        s = np.where(np.isfinite(s) & (s > 0), s, np.inf).min(-1)
        depth[f] = np.clip(np.round(s), 1, 65000).astype(np.uint16)
        X = c + w * s[..., None] + shift
        bgr[f] = (127.5 + 127 * np.sin(X[..., [0, 1, 2]] / np.array([173., 211., 157.]) +
                                       X[..., [1, 2, 0]] / 997.)).astype(np.uint8)
        poses[f, :9] = R.reshape(9)
        poses[f, 9:] = t - R @ shift
    return depth, poses, bgr


def test_rgbd_scene_through_getobj_into_forward(engine_mod, eng):
    from dsac_b200.obj_train import RGBDScene
    rng = np.random.default_rng(2017)
    depth, poses, bgr = render_room(3, rng)
    cam = engine_mod.default_rgbd_camera(sensor_trans=seven_scenes_trans())
    sc = RGBDScene(eng, bgr, depth, poses, cam)
    co = sc.scene_coords(range(3)).cpu().numpy()
    pix = engine_mod.stochastic_subsample(1305, 640, 480)
    coords = np.stack([co[f][pix[:, 1], pix[:, 0]] for f in range(3)])
    res = eng.forward(coords, pix, poses)
    assert (res.rot_err < 5.0).all() and (res.t_err < 50.0).all(), (res.rot_err, res.t_err)


def test_pretraining_lowers_the_loss(engine_mod, eng):
    from dsac_b200.obj_train import ObjPretrainer, RGBDScene
    from dsac_b200.coord_cnn import CoordPipeline
    torch.manual_seed(0)
    rng = np.random.default_rng(5)
    depth, poses, bgr = render_room(6, rng, lo=(-900., -700., -1200.), hi=(900., 700., 600.), shift=(2000., 0., 0.))
    sc = RGBDScene(eng, bgr, depth, poses, engine_mod.default_rgbd_camera(raw_data=0))
    tr = ObjPretrainer(eng, sc, seed=1305, n_streams=4, n_images=20, n_patches=128)
    loss0, inl0 = tr.evaluate(n_images=6, n_patches=256)
    losses = tr.train(200)
    loss1, inl1 = tr.evaluate(n_images=6, n_patches=256)
    assert len(losses) == 200 and len(tr.log) == 200 and tr.log[-1][0] == 199
    assert np.isfinite(losses).all()
    assert np.mean(losses[-20:]) < 0.5 * np.mean(losses[:20])
    assert loss1 < 0.5 * loss0 and inl1 > inl0, (loss0, loss1, inl0, inl1)
    # the pre-trained network is the pipeline's network
    pipe = CoordPipeline(eng, chunk=1)
    pipe.model.load_state_dict(tr.model.state_dict())


# ------------------------------------------------------------------ Lemire rejections inside the draw
OFFSETS = [1, 2, 3, 4, 5, 6, 7, 9, 11, 21, 31, 33, 62, 63, 64, 65]


@pytest.mark.parametrize("valid_every,max_attempts,n_patches", [(1, 1 << 20, 40), (1, 1 << 20, 3), (1, 1 << 20, 16),
                                                                 (11, 32, 12), (11, 40, 30)])
def test_draw_through_rejected_words(engine_mod, eng, valid_every, max_attempts, n_patches):
    """Streams placed a few words before a word that irand(21, 619) (range 598) or irand(21, 459) (range 438) rejects, so
    that the rejected word falls on an x word, a y word, an image-index word, at every lane of a batch and at the end of
    an image.  valid_every > 1: sparse valid pixels, with the rejected pair near the attempt bound."""
    from dsac_b200.obj_train import ObjRound, RGBDScene
    W, H = 640, 480
    cam = engine_mod.default_rgbd_camera(raw_data=0)
    ys, xs = np.mgrid[0:H, 0:W]
    depth = np.zeros((3, H, W), np.uint16)
    for f in range(3):
        depth[f][((xs * 7 + ys * 13 + f) % valid_every) == 0] = 900 + 100 * f
    poses = np.tile(np.r_[np.eye(3).reshape(9), 0, 0, 0], (3, 1))
    sc = RGBDScene(eng, OO.coded_bgr(3, H, W), depth, poses, cam)
    qx = OO.rejected_word_positions(1305, W - 42, 1)[0]
    qy = OO.rejected_word_positions(1305, H - 42, 1)[0]
    starts = [q - d for q in (qx, qy) for d in OFFSETS]
    T = len(starts)
    st = np.stack([OO.state_at(1305, s) for s in starts])
    r = ObjRound(sc, n_streams=T, max_attempts=max_attempts)
    r.state.copy_(torch.from_numpy(st.view(np.int32)))
    before = OO.REJECTED[0]
    for _ in range(2):
        _compare_draw(r, cam, depth, poses, st, 2 * T + 5, n_patches, max_attempts=max_attempts)
    assert OO.REJECTED[0] > before   # the restated draw did meet rejected words on these streams
