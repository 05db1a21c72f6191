"""Per-frame cameras in the pre-training data paths, on the CPU: the host build of the score path's getCamMat()
conversion against the reference's spelling, and the numpy restatements' per-frame registration, getObj, draw and
error images against frame-by-frame restatements with one camera each."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import camera_oracle as CO
import obj_oracle as OO
import score_oracle as SO
from conftest import GOLDEN, ROOT


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cammatshim") / "libcammat_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "cammat_shim.cpp")])
    return C.CDLL(so)


def seven_scenes_trans():
    from dsac_b200.obj_train import read_sensor_trans
    return read_sensor_trans(os.path.join(GOLDEN, "sensorTrans_7scenes.dat"))


def mixed_cams(engine_mod, W, H, raw_data):
    """Three cameras: the defaults with 7-Scenes' sensorTrans, an off-centre principal point, and another focal length
    with another depth camera."""
    st = seven_scenes_trans()
    return [engine_mod.default_rgbd_camera(width=W, height=H, raw_data=raw_data, sensor_trans=st),
            engine_mod.default_rgbd_camera(width=W, height=H, raw_data=raw_data, sensor_trans=st, x_shift=13.5,
                                           y_shift=-7.25),
            engine_mod.default_rgbd_camera(width=W, height=H, raw_data=raw_data, focal=610.0, secondary_focal=560.0,
                                           raw_x_shift=3.0, raw_y_shift=-2.5, x_shift=-0.75)]


SIZES = [(640, 480), (641, 481), (77, 53), (128, 96), (83, 84)]
SHIFTS = [(0.0, 0.0), (0.5, -0.5), (-3.25, 7.75), (-320.6, -240.4), (1e-3, -1e-3), (-0.3, 0.7)]


@pytest.mark.parametrize("W,H", SIZES)
def test_score_cam_is_getcammat(shim, engine_mod, W, H):
    for xs, ys in SHIFTS:
        for focal in (525.0, 585.3, 1e3 / 3):
            cam = engine_mod.default_rgbd_camera(width=W, height=H, x_shift=xs, y_shift=ys, focal=focal)
            f, cx, cy = C.c_double(), C.c_float(), C.c_float()
            shim.shim_score_cam(C.byref(cam), C.byref(f), C.byref(cx), C.byref(cy))
            rf, rcx, rcy = C.c_float(), C.c_float(), C.c_float()
            shim.shim_ref_getcammat(C.byref(cam), C.byref(rf), C.byref(rcx), C.byref(rcy))
            assert f.value == rf.value and cx.value == rcx.value and cy.value == rcy.value, (W, H, xs, ys)
            assert CO.cam_mat(cam) == (f.value, cx.value, cy.value)
            # getObj's principal point: the same on even sizes, half a pixel further on odd ones (Q27)
            ocx, ocy = C.c_float(), C.c_float()
            shim.shim_ref_getobj_centre(C.byref(cam), C.byref(ocx), C.byref(ocy))
            if W % 2 == 0:
                assert ocx.value == cx.value
            elif abs(xs) < 100:
                assert ocx.value != cx.value and abs(ocx.value - cx.value - 0.5) < 1e-4
            if H % 2 == 0:
                assert ocy.value == cy.value


def test_oracle_frame_cams(engine_mod):
    cam = engine_mod.default_rgbd_camera()
    one = CO.frame_cams(cam, 3)
    assert len(one) == 3 and all(c["focal"] == 525.0 and np.array_equal(c["sensor_trans"], np.eye(4)) for c in one)
    cams = mixed_cams(engine_mod, 640, 480, 1)
    assert [c["focal"] for c in CO.frame_cams(cams, 3)] == [525.0, 525.0, 610.0]
    with pytest.raises(ValueError):
        CO.frame_cams(cams, 4)


@pytest.mark.parametrize("raw_data", [1, 0])
def test_oracle_registration_and_getobj_per_frame(engine_mod, raw_data):
    W, H = 128, 96
    cams = mixed_cams(engine_mod, W, H, raw_data)
    raw = OO.fixture_depth(3, H, W, salt=raw_data)
    reg, dropped = CO.register_depth(cams, raw)
    poses = np.tile(np.r_[np.eye(3).reshape(9), 100.0, -50.0, 20.0], (3, 1))
    for f in range(3):
        r1, d1 = OO.register_depth(cams[f], raw[f:f + 1])
        assert np.array_equal(reg[f], r1[0]) and dropped[f] == d1[0]
    if raw_data:   # the cameras do register differently
        assert not np.array_equal(OO.register_depth(cams[0], raw[2:])[0][0], reg[2])
    co = [OO.obj_coords(cams[f], reg[f], poses[f]) for f in range(3)]
    assert not np.array_equal(co[1], OO.obj_coords(cams[0], reg[1], poses[1]))


@pytest.mark.parametrize("T", [1, 3])
def test_oracle_draw_per_frame(engine_mod, T):
    """The per-frame draw equals the single-camera draw over labels restated frame by frame with each frame's camera
    (the draw consumes the same words), and F identical cameras equal the single camera."""
    W, H = 96, 80
    cams = mixed_cams(engine_mod, W, H, 0)
    depth = OO.fixture_depth(3, H, W, salt=7)
    depth[depth >= 32768] = 0
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(T)
    poses = np.zeros((3, 12))
    for f in range(3):
        poses[f, :9] = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix().reshape(9)
        poses[f, 9:] = rng.uniform(-2000, 2000, 3)
    coords = np.stack([OO.obj_coords(cams[f], depth[f], poses[f]) for f in range(3)])
    st_a, st_b = OO.rng_init(1305, T), OO.rng_init(1305, T)
    for _ in range(2):
        a = CO.draw(cams, depth, poses, st_a, n_images=7, n_patches=9)
        b = OO.draw(cams[0], depth, poses, st_b, n_images=7, n_patches=9, coords=coords)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
        assert np.array_equal(st_a, st_b)
    assert set(np.unique(a[0])) == {0, 1, 2}
    st_c, st_d = OO.rng_init(9, T), OO.rng_init(9, T)
    c = CO.draw([cams[2]] * 3, depth, poses, st_c, n_images=5, n_patches=6)
    d = OO.draw(cams[2], depth, poses, st_d, n_images=5, n_patches=6)
    for x, y in zip(c, d):
        assert np.array_equal(x, y)


def test_oracle_round_maps_per_frame(engine_mod):
    cams = mixed_cams(engine_mod, 641, 480, 1)
    rng = np.random.default_rng(3)
    st = OO.rng_init(5, 2)
    img, pix, _, noise = SO.draw(st, 3, 641, 480, 4, 3)
    gt = np.tile(np.r_[np.eye(3).reshape(9), 0.0, 0.0, 0.0], (3, 1))
    d = rng.uniform(800, 3000, (4, 1600))
    coords = np.stack([(pix[..., 0] - 320) * d / 525, -(pix[..., 1] - 240) * d / 525, -d], -1)
    coords = np.round(coords).astype(np.int16)
    maps = CO.round_maps(img, gt, noise, coords, pix, 3, cams)
    for i in range(4):
        f, cx, cy = CO.cam_mat(cams[img[i]])
        assert cx == float(np.float32(320 + np.float32(cams[img[i]].x_shift)))
        one = CO.round_maps(img[i:i + 1], gt, noise[3 * i:3 * i + 3], coords[i:i + 1], pix[i:i + 1], 3, (f, cx, cy))
        assert np.array_equal(maps[3 * i:3 * i + 3], one)
    # with the config camera of the defaults, the frames of camera 0 agree and the others do not
    cfg = CO.round_maps(img, gt, noise, coords, pix, 3, (525.0, 320.0, 240.0))
    same = np.repeat(img == 0, 3)
    assert same.any() and not same.all()
    assert np.array_equal(maps[same], cfg[same]) and not np.array_equal(maps[~same], cfg[~same])
