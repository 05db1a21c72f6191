"""Coordinate-CNN pre-training data path on the CPU: the host build of objtrain.cuh's arithmetic against the numpy
restatement (tests/obj_oracle.py), against gcc's own conversions and libstdc++'s distributions, the shuffle against a
restatement of libstdc++'s std::shuffle, and the trainer's loss and optimiser against numpy."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import obj_oracle as OO
from conftest import GOLDEN, ROOT


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("objshim") / "libobj_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "obj_shim.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _cam(engine_mod, **kw):
    return engine_mod.default_rgbd_camera(**kw)


def seven_scenes_trans():
    from dsac_b200.obj_train import read_sensor_trans
    return read_sensor_trans(os.path.join(GOLDEN, "sensorTrans_7scenes.dat"))


def synthetic_depth(rng, F, H, W):
    """Depth with holes (0), 7-Scenes' invalid marker 65535, values >= 32768 and ordinary 500..4000 mm."""
    d = rng.integers(500, 4000, (F, H, W)).astype(np.uint16)
    d[rng.random((F, H, W)) < 0.1] = 0
    d[rng.random((F, H, W)) < 0.03] = 65535
    d[rng.random((F, H, W)) < 0.03] = rng.integers(32768, 65535)
    return d


def random_poses(rng, F):
    from scipy.spatial.transform import Rotation
    P = np.zeros((F, 12))
    for f in range(F):
        P[f, :9] = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix().reshape(9)
        P[f, 9:] = rng.uniform(-2000, 2000, 3)
    return P


def test_conversions_match_gcc(shim):
    v = np.array([0.0, -0.0, 0.4, -0.4, -0.99, 1.5, -1.5, 32767.9, 32768.0, -32769.5, 65535.2, 65536.0, 1e5, -1e5,
                  2147483647.0, 2147483648.0, -2147483648.0, -2147483649.0, 3e9, -3e9, 1e20, np.inf, -np.inf, np.nan])
    rng = np.random.default_rng(3)
    v = np.concatenate([v, rng.uniform(-1e6, 1e6, 5000), rng.uniform(-4e9, 4e9, 5000)])
    n = len(v)
    d2i, f2i = np.zeros(n, np.int32), np.zeros(n, np.int32)
    arrs = [np.zeros(n, np.int16) for _ in range(4)]
    shim.shim_cvt(n, _p(v), _p(d2i), _p(f2i), *[_p(a) for a in arrs])
    d2s_ref, f2s_ref, d2s, f2s = arrs
    assert np.array_equal(d2s, d2s_ref)
    assert np.array_equal(f2s, f2s_ref)
    assert np.array_equal(d2i, OO.cvtt_i32(v))
    assert np.array_equal(f2i, OO.cvtt_i32(v.astype(np.float32)))


def test_mm_to_m_all_int16(shim):
    v = np.arange(-32768, 32768, dtype=np.int16)
    out = np.zeros(v.size, np.float32)
    shim.shim_mm_to_m(v.size, _p(v), _p(out))
    assert np.array_equal(out.view(np.uint32), OO.mm_to_m(v).view(np.uint32))
    # over int16 inputs the double product rounded to float happens to equal the float quotient v / 1000.f everywhere
    assert np.array_equal(out, v.astype(np.float32) / np.float32(1000))


def test_inv_rotation_is_opencv_closed_form(shim):
    rng = np.random.default_rng(5)
    for i in range(300):
        R = random_poses(rng, 1)[0, :9].reshape(3, 3) if i % 2 else rng.standard_normal((3, 3))
        out = np.zeros(9)
        shim.shim_inv_rotation(_p(np.ascontiguousarray(R)), _p(out))
        assert np.array_equal(out, OO.inv_rotation(R).reshape(9))
    cv2 = pytest.importorskip("cv2")
    for i in range(300):
        R = rng.standard_normal((3, 3))
        assert np.array_equal(cv2.invert(R)[1], OO.inv_rotation(R))


@pytest.mark.parametrize("W,H,trans", [(128, 96, "identity"), (128, 96, "7scenes"), (77, 53, "7scenes")])
def test_obj_coords_and_registration_match_oracle(shim, engine_mod, W, H, trans):
    rng = np.random.default_rng(W * H)
    st = np.eye(4) if trans == "identity" else seven_scenes_trans()
    for raw_data in (0, 1):
        cam = _cam(engine_mod, width=W, height=H, raw_data=raw_data, sensor_trans=st, x_shift=0.25 if W % 2 else 0.0)
        raw = synthetic_depth(rng, 3, H, W)
        reg, dropped = OO.register_depth(cam, raw)
        poses = random_poses(rng, 3)
        for f in range(3):
            out = np.zeros((H, W), np.uint16)
            nd = shim.shim_register_depth(C.byref(cam), _p(np.ascontiguousarray(raw[f])), _p(out))
            assert np.array_equal(out, reg[f])
            assert nd == dropped[f]
            co = np.zeros((H, W, 3), np.int16)
            shim.shim_obj_coords(C.byref(cam), _p(np.ascontiguousarray(reg[f])), _p(np.ascontiguousarray(poses[f])), _p(co))
            assert np.array_equal(co, OO.obj_coords(cam, reg[f], poses[f]))
    cam = _cam(engine_mod, width=W, height=H, raw_x_shift=-30.0, sensor_trans=st)
    raw = synthetic_depth(rng, 1, H, W)
    reg, dropped = OO.register_depth(cam, raw)
    out = np.zeros((H, W), np.uint16)
    assert shim.shim_register_depth(C.byref(cam), _p(np.ascontiguousarray(raw[0])), _p(out)) == dropped[0] > 0
    assert np.array_equal(out, reg[0])


def test_registration_wrap_and_truncation_quirks(engine_mod):
    cam = _cam(engine_mod, width=64, height=48)
    # a depth >= 32768 arrives as a negative short; with an identity sensorTrans the sign cancels in the projection
    nx, ny = OO.map_depth_to_rgb(cam, np.array([10]), np.array([10]), np.array([40000, 1000], np.uint16))
    assert nx[0] == nx[1] and ny[0] == ny[1]
    # identity transform and equal focals: a target in (-1, 0) truncates to column 0
    cam2 = _cam(engine_mod, width=64, height=48, secondary_focal=525.0)
    nx, ny = OO.map_depth_to_rgb(cam2, np.array([0]), np.array([5]), np.array([1000], np.uint16))
    assert nx[0] == 0
    # 65535 (7-Scenes' invalid depth) is nonzero, so getObj gives it coordinates: (short)-65535 = 1
    co = OO.obj_coords(cam, np.full((48, 64), 65535, np.uint16), np.r_[np.eye(3).reshape(9), 0, 0, 0])
    assert (co[..., 2] == 1).all()


@pytest.mark.parametrize("rng_", [1, 2, 40, 598, 438, 5, 100, (1 << 30) + 1, (1 << 31) - 1])
def test_lemire_draw_matches_libstdcxx(shim, rng_):
    n = 4000
    mine, theirs = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    same = shim.shim_lemire_vs_std(C.c_uint32(1305), C.c_uint32(rng_), n, _p(mine), _p(theirs))
    assert same == 1 and np.array_equal(mine, theirs)


def _std_shuffle(n, seed):
    """libstdc++'s std::shuffle (bits/stl_algo.h) with a 32-bit engine: two swap positions per draw while
    (2^32 - 1) / n >= n, from uniform_int_distribution<unsigned long>(0, b0 * b1 - 1)."""
    bg = np.random.MT19937()
    bg._legacy_seeding(seed)
    nxt = lambda: int(bg.random_raw())   # noqa: E731
    a = list(range(n))
    urng = 0xffffffff
    if urng // n >= n:
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
        return np.array(a)
    for i in range(1, n):
        j = OO.lemire(nxt, i + 1)
        a[i], a[j] = a[j], a[i]
    return np.array(a)


@pytest.mark.parametrize("n,seed", [(51200, 5489), (7, 1), (10, 5489), (70000, 3)])
def test_shuffle_permutation_matches_libstdcxx(engine_mod, n, seed):
    assert np.array_equal(engine_mod.shuffle_permutation(n, seed), _std_shuffle(n, seed))


def test_l1_criterion_matches_numpy():
    from dsac_b200.obj_train import l1_criterion
    rng = np.random.default_rng(0)
    pred = rng.normal(size=(64, 3))
    gt = rng.normal(size=(64, 3))
    p = torch.tensor(pred, requires_grad=True)
    loss = l1_criterion(p, torch.tensor(gt))
    loss.backward()
    d = np.linalg.norm(pred - gt, axis=1)
    assert abs(float(loss) - d.mean()) < 1e-12
    assert np.allclose(p.grad.numpy(), (pred - gt) / d[:, None] / 64, rtol=1e-12, atol=0)
    # zero distance: the reference's 0 / 0 -- a NaN gradient on that row only
    gt[3] = pred[3]
    p = torch.tensor(pred, requires_grad=True)
    l1_criterion(p, torch.tensor(gt)).backward()
    assert torch.isnan(p.grad[3]).all() and torch.isfinite(p.grad[torch.arange(64) != 3]).all()


def test_torch7_adam_matches_numpy():
    from dsac_b200.obj_train import Torch7Adam
    rng = np.random.default_rng(1)
    x0 = rng.normal(size=50)
    grads = rng.normal(size=(20, 50))
    x = torch.tensor(x0.copy(), requires_grad=True)
    opt = Torch7Adam([x], lr=1e-2)
    for g in grads:
        x.grad = torch.tensor(g)
        opt.step()
    xr, m, v = x0.copy(), np.zeros(50), np.zeros(50)
    for t, g in enumerate(grads, 1):
        m = 0.9 * m + 0.1 * g
        v = 0.999 * v + 0.001 * g * g
        xr -= 1e-2 * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) * m / (np.sqrt(v) + 1e-8)
    assert np.allclose(x.detach().numpy(), xr, rtol=1e-12, atol=1e-15)
    # and it is not torch.optim.Adam, whose eps enters after the bias correction
    y = torch.tensor(x0.copy(), requires_grad=True)
    o2 = torch.optim.Adam([y], lr=1e-2, eps=1e-1)
    z = torch.tensor(x0.copy(), requires_grad=True)
    o3 = Torch7Adam([z], lr=1e-2, eps=1e-1)
    for g in grads[:3]:
        y.grad = torch.tensor(g); z.grad = torch.tensor(g)
        o2.step(); o3.step()
    assert not torch.allclose(y, z)


def test_oracle_draw_consumes_like_a_reference_round(engine_mod):
    """The restated draw on a tiny all-valid scene: every pair is accepted, so a round of n images x p patches uses
    exactly n * (1 + 2p) words per stream (no Lemire rejection at these ranges in this prefix), and a second round
    continues the stream."""
    cam = _cam(engine_mod, width=50, height=45, raw_data=0)
    depth = np.full((2, 45, 50), 1000, np.uint16)
    poses = np.tile(np.r_[np.eye(3).reshape(9), 0, 0, 0], (2, 1))
    st = OO.rng_init(1305, 1)
    img, centre, label, status = OO.draw(cam, depth, poses, st, n_images=3, n_patches=5)
    assert (status == 0).all() and (centre[:, 0] >= 21).all() and (centre[:, 0] <= 50 - 22).all()
    assert (centre[:, 1] >= 21).all() and (centre[:, 1] <= 45 - 22).all()
    bg = np.random.MT19937()
    bg._legacy_seeding(1305)
    bg.random_raw(3 * (1 + 2 * 5))
    assert np.array_equal(st[0, :624], bg.state["state"]["key"]) and st[0, 624] == bg.state["state"]["pos"]
