"""The numpy restatement of the pre-training data path (tests/obj_oracle.py) against what the reference's own
train_obj.cpp and jp::Dataset computed (tests/golden/ref_obj.npz, frozen by tests/golden/make_ref_obj.py): registered
depth, getObj images, and two consecutive assembleData rounds -- image indices, patch centres, labels -- for 1 and 3
OpenMP threads, plus the batch permutation.  The GPU tests pin the device to the same restatement.

The fixture was computed through the API shim's Mat::inv (Gauss-Jordan), so getObj is restated here with that inverse;
the product uses OpenCV's closed form, which tests/test_obj_train_host.py pins against cv2."""
import hashlib
import os

import numpy as np
import pytest

import obj_oracle as OO
from conftest import GOLDEN

FIX = os.path.join(GOLDEN, "ref_obj.npz")
CASES = ["small_identity", "small_7scenes", "small_raw0", "vga_7scenes"]


@pytest.fixture(scope="module")
def ref():
    return np.load(FIX)


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def case_inputs(ref, name):
    fo, xs, ys, sfl, rxs, rys, raw_data, W, H = ref[name + "/camera"]
    W, H = int(W), int(H)
    cam = dict(focal=fo, x_shift=xs, y_shift=ys, secondary_focal=sfl, raw_x_shift=rxs, raw_y_shift=rys,
               sensor_trans=ref[name + "/sensor_trans"], raw_data=int(raw_data), width=W, height=H)
    F = ref[name + "/rotation"].shape[0]
    raw = OO.fixture_depth(F, H, W, salt=len(name))
    raw[np.unpackbits(ref[name + "/zeroed"])[:F * H * W].reshape(F, H, W).astype(bool)] = 0
    poses = np.concatenate([ref[name + "/rotation"].astype(np.float64),
                            ref[name + "/center"].astype(np.float64) * 1000.0], 1)
    return cam, raw, poses


@pytest.mark.parametrize("name", CASES)
def test_registration_and_getobj_equal_the_reference(ref, name):
    cam, raw, poses = case_inputs(ref, name)
    reg, dropped = OO.register_depth(cam, raw)
    assert (dropped == 0).all()
    assert np.array_equal(reg[:, :4], ref[name + "/depth_rows"])
    for f in range(raw.shape[0]):
        assert np.array_equal(digest(reg[f]), ref[name + "/depth_sha"][f]), f
        co = OO.obj_coords(cam, reg[f], poses[f], inv=OO.inv_rotation_elimination)
        assert np.array_equal(co[:2], ref[name + "/coords_rows"][f]), f
        assert np.array_equal(digest(co), ref[name + "/coords_sha"][f]), f


@pytest.mark.parametrize("name", CASES)
def test_draw_equals_the_reference_over_two_rounds(ref, name):
    cam, raw, poses = case_inputs(ref, name)
    reg, _ = OO.register_depth(cam, raw)
    coords = np.stack([OO.obj_coords(cam, reg[f], poses[f], inv=OO.inv_rotation_elimination) for f in range(len(reg))])
    n_img, n_pat, seed = int(ref["n_images"]), int(ref["n_patches"]), int(ref["seed"])
    threads = sorted({int(k.split("/")[1][1:]) for k in ref.files if k.startswith(name + "/T")})
    assert threads
    for T in threads:
        st = OO.rng_init(seed, T)
        for rnd in range(2):
            key = "%s/T%d/round%d" % (name, T, rnd)
            img, centre, label, status = OO.draw(cam, reg, poses, st, n_img, n_pat, coords=coords)
            assert (status == 0).all()
            assert np.array_equal(img, ref[key + "/img"]), key
            assert np.array_equal(centre, ref[key + "/centre"]), key
            assert np.array_equal(label.view(np.uint32), ref[key + "/label"].view(np.uint32)), key


def test_permutation_equals_the_reference(ref, engine_mod):
    perm = engine_mod.shuffle_permutation(51200, 5489)
    assert np.array_equal(perm[:64], ref["permutation_head"])
    assert np.array_equal(digest(perm.astype(np.int32)), ref["permutation_sha"])
