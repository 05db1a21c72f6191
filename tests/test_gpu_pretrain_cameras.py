"""Per-frame cameras in the pre-training data paths on the device (dsac_set_dataset_cameras): registration, getObj, the
patch draw and the score CNN's error images with a dataset camera table, bit for bit against single-camera calls and
against the numpy restatements (tests/obj_oracle.py, tests/score_oracle.py); validation; independence from the forward's
cameras; and the Python trainers on a scene that mixes cameras."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import camera_oracle as CO
import obj_oracle as OO
from conftest import GOLDEN

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng(engine_mod):
    e = engine_mod.Engine(max_frames=4, n_hyps=64)
    yield e
    e.close()


@pytest.fixture(autouse=True)
def _no_table(eng):
    eng.set_dataset_cameras(None)
    yield
    eng.set_dataset_cameras(None)


def seven_scenes_trans():
    from dsac_b200.obj_train import read_sensor_trans
    return read_sensor_trans(os.path.join(GOLDEN, "sensorTrans_7scenes.dat"))


def mixed_cams(E, W, H, raw_data):
    """7-Scenes' defaults and sensorTrans; an off-centre principal point; another focal length and depth camera."""
    st = seven_scenes_trans()
    return [E.default_rgbd_camera(width=W, height=H, raw_data=raw_data, sensor_trans=st),
            E.default_rgbd_camera(width=W, height=H, raw_data=raw_data, sensor_trans=st, x_shift=13.5, y_shift=-7.25),
            E.default_rgbd_camera(width=W, height=H, raw_data=raw_data, focal=610.0, secondary_focal=560.0,
                                  raw_x_shift=3.0, raw_y_shift=-2.5, x_shift=-0.75)]


def synthetic_depth(rng, F, H, W):
    d = rng.integers(500, 4000, (F, H, W)).astype(np.uint16)
    d[rng.random((F, H, W)) < 0.1] = 0
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


def dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def u16(t):
    return t.cpu().numpy().view(np.uint16)


def register(eng, cam, raw_d, F, H, W):
    out = torch.empty((F, H, W), dtype=torch.int16, device="cuda")
    dropped = torch.zeros(F, dtype=torch.int32, device="cuda")
    status = torch.zeros(F, dtype=torch.int32, device="cuda")
    eng.register_depth_device(cam, F, raw_d.data_ptr(), out.data_ptr(), dropped.data_ptr(), status.data_ptr())
    return out, dropped, status


def obj_coords(eng, cam, n_frames, depth_d, poses_d, idx):
    ids = torch.tensor(idx, dtype=torch.int32, device="cuda")
    H, W = depth_d.shape[1], depth_d.shape[2]
    out = torch.empty((len(idx), H, W, 3), dtype=torch.int16, device="cuda")
    eng.obj_coords_device(cam, n_frames, len(idx), depth_d.data_ptr(), poses_d.data_ptr(), out.data_ptr(),
                          d_idx=ids.data_ptr())
    return out


def draw(eng, cam, F, depth_d, poses_d, state, n_images, n_patches):
    n = n_images * n_patches
    img = torch.empty(n, dtype=torch.int32, device="cuda")
    centre = torch.empty((n, 2), dtype=torch.int32, device="cuda")
    label = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    status = torch.empty(n_images, dtype=torch.int32, device="cuda")
    eng.obj_draw_device(cam, F, depth_d.data_ptr(), poses_d.data_ptr(), n_images, n_patches, state.shape[0], 1 << 20,
                        state.data_ptr(), img.data_ptr(), centre.data_ptr(), label.data_ptr(), status.data_ptr())
    return img, centre, label, status


def rng_state(eng, seed, T):
    st = torch.empty((T, 625), dtype=torch.int32, device="cuda")
    eng.obj_rng_init_device(seed, T, st.data_ptr())
    return st


class ScoreInputs:
    """One score draw over F frames of a W x H dataset and coordinates back-projected from a plausible depth, so the
    error images are mostly below the clamp."""

    def __init__(self, eng, F, W, H, n_images=6, hyps=8, seed=3):
        rng = np.random.default_rng(seed)
        self.n_images, self.hyps = n_images, hyps
        st = rng_state(eng, 1305, 2)
        self.img = torch.empty(n_images, dtype=torch.int32, device="cuda")
        self.pix = torch.empty((n_images, 1600, 2), dtype=torch.int32, device="cuda")
        self.drift = torch.empty(n_images * hyps, dtype=torch.int32, device="cuda")
        self.noise = torch.empty((n_images * hyps, 6), dtype=torch.float64, device="cuda")
        eng.score_draw_device(F, W, H, n_images, hyps, 2, st.data_ptr(), self.img.data_ptr(), self.pix.data_ptr(),
                              self.drift.data_ptr(), self.noise.data_ptr())
        pix = self.pix.cpu().numpy()
        d = rng.uniform(800, 3000, (n_images, 1600))
        co = np.stack([(pix[..., 0] - W / 2) * d / 525, -(pix[..., 1] - H / 2) * d / 525, -d], -1)
        self.coords = dev(np.round(co).astype(np.int16), torch.int16)
        gt = np.zeros((F, 12))
        gt[:, [0, 4, 8]] = 1.0
        gt[:, 9:] = rng.uniform(-20, 20, (F, 3))
        self.gt = dev(gt, torch.float64)

    def maps(self, eng, img=None):
        n = self.n_images * self.hyps
        img = self.img if img is None else img
        maps = torch.full((n, 1600), -1.0, dtype=torch.float32, device="cuda")
        labels = torch.full((n,), -1.0, dtype=torch.float64, device="cuda")
        correct = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        eng.score_maps_device(self.n_images, self.hyps, img.data_ptr(), self.gt.data_ptr(), self.coords.data_ptr(),
                              self.pix.data_ptr(), self.noise.data_ptr(), 10.0, maps.data_ptr(), labels.data_ptr(),
                              correct.data_ptr())
        torch.cuda.synchronize()
        return maps.cpu().numpy(), labels.cpu().numpy(), correct.cpu().numpy()


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


# ------------------------------------------------------------------ 1. a table of identical cameras
def test_identical_table_equals_single_camera(engine_mod, eng):
    E = engine_mod
    rng = np.random.default_rng(1)
    F, W, H = 4, 128, 96
    cam = E.default_rgbd_camera(width=W, height=H, sensor_trans=seven_scenes_trans(), x_shift=0.25, y_shift=-1.5)
    raw = dev(synthetic_depth(rng, F, H, W).view(np.int16), torch.int16)
    poses = dev(random_poses(rng, F), torch.float64)
    one = register(eng, cam, raw, F, H, W)
    eng.set_dataset_cameras([cam] * F)
    tab = register(eng, None, raw, F, H, W)
    for a, b in zip(one, tab):
        assert torch.equal(a, b)
    idx = [3, 0, 2, 1, 2]
    assert torch.equal(obj_coords(eng, cam, F, one[0], poses, idx), obj_coords(eng, None, F, one[0], poses, idx))
    s1, s2 = rng_state(eng, 77, 3), rng_state(eng, 77, 3)
    for _ in range(2):
        a = draw(eng, cam, F, one[0], poses, s1, 7, 50)
        b = draw(eng, None, F, one[0], poses, s2, 7, 50)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        assert torch.equal(s1, s2)
    # the score path: 640 x 480 defaults give getCamMat() = (525, 320, 240), the config's camera
    sc = E.default_rgbd_camera()
    inp = ScoreInputs(eng, F, 640, 480)
    eng.set_dataset_cameras(None)
    ref = inp.maps(eng)
    eng.set_dataset_cameras([sc] * F)
    for x, y in zip(ref, inp.maps(eng)):
        assert same_bits(x, y)


# ------------------------------------------------------------------ 2. mixed tables: registration and getObj
@pytest.mark.parametrize("raw_data", [1, 0])
def test_mixed_registration_and_getobj(engine_mod, eng, raw_data):
    E = engine_mod
    rng = np.random.default_rng(10 + raw_data)
    W, H = 77, 53
    cams3 = mixed_cams(E, W, H, raw_data)
    cams = [cams3[k] for k in (0, 1, 2, 1)]
    F = len(cams)
    raw_np = synthetic_depth(rng, F, H, W)
    raw = dev(raw_np.view(np.int16), torch.int16)
    poses_np = random_poses(rng, F)
    poses = dev(poses_np, torch.float64)
    eng.set_dataset_cameras(cams)
    dep, dropped, _ = register(eng, None, raw, F, H, W)
    co = obj_coords(eng, None, F, dep, poses, list(range(F)))
    reg, o_dropped = CO.register_depth(cams, raw_np)
    assert np.array_equal(u16(dep), reg) and np.array_equal(dropped.cpu().numpy(), o_dropped)
    for f in range(F):
        d1, dr1, _ = register(eng, cams[f], raw[f:f + 1].contiguous(), 1, H, W)
        assert torch.equal(dep[f], d1[0]) and int(dropped[f]) == int(dr1[0])
        c1 = obj_coords(eng, cams[f], 1, dep[f:f + 1].contiguous(), poses[f:f + 1].contiguous(), [0])
        assert torch.equal(co[f], c1[0])
        assert np.array_equal(co[f].cpu().numpy(), OO.obj_coords(cams[f], reg[f], poses_np[f]))
    if raw_data:   # the frames did register with different cameras
        assert not np.array_equal(OO.register_depth(cams[0], raw_np[2:3])[0][0], reg[2])
    assert not np.array_equal(co[1].cpu().numpy(), OO.obj_coords(cams[0], reg[1], poses_np[1]))
    # a listed frame outside the dataset still gives a zero image
    out = obj_coords(eng, None, F, dep, poses, [1, F, -2])
    assert torch.equal(out[0], co[1]) and (out[1:] == 0).all()


# ------------------------------------------------------------------ 3. the draw on a mixed dataset
@pytest.mark.parametrize("T", [1, 3, 16])
def test_mixed_draw_matches_oracle(engine_mod, eng, T):
    from dsac_b200.obj_train import ObjRound, RGBDScene
    E = engine_mod
    rng = np.random.default_rng(100 + T)
    W, H = 128, 96
    cams3 = mixed_cams(E, W, H, 1)
    cams = [cams3[k] for k in (2, 0, 1, 2, 1)]
    F = len(cams)
    raw = synthetic_depth(rng, F, H, W)
    poses = random_poses(rng, F)
    sc = RGBDScene(eng, OO.coded_bgr(F, H, W), raw, poses, cams)
    depth = sc.depth_u16()
    assert np.array_equal(depth, CO.register_depth(cams, raw)[0])
    r = ObjRound(sc, seed=1305, n_streams=T)
    st = OO.rng_init(1305, T)
    for _ in range(2):
        img, centre, label, status = r.draw(19, 40)
        oi, oc, ol, os_ = CO.draw(cams, depth, poses, st, 19, 40)
        assert np.array_equal(img.cpu().numpy(), oi) and np.array_equal(centre.cpu().numpy(), oc)
        assert np.array_equal(label.cpu().numpy().view(np.uint32), ol.view(np.uint32))
        assert np.array_equal(status.cpu().numpy().astype(np.uint32), os_)
        assert np.array_equal(r.state.cpu().numpy().view(np.uint32), st)
    assert len(np.unique(oi)) > 2


# ------------------------------------------------------------------ 4. score maps on a mixed dataset
@pytest.mark.parametrize("W", [640, 641])
def test_mixed_score_maps(engine_mod, eng, W):
    E = engine_mod
    H = 480
    cams3 = mixed_cams(E, W, H, 1)
    which = [0, 1, 2, 2, 1]
    cams = [cams3[k] for k in which]
    F = len(cams)
    inp = ScoreInputs(eng, F, W, H, n_images=9, hyps=8)
    img = inp.img.cpu().numpy()
    assert len({which[f] for f in img}) == 3
    eng.set_dataset_cameras(cams)
    maps, labels, correct = inp.maps(eng)
    for k in range(3):
        f, cx, cy = CO.cam_mat(cams3[k])
        e1 = E.Engine(max_frames=1, n_hyps=64, focal=f, cx=cx, cy=cy)
        m1, l1, c1 = inp.maps(e1)
        e1.close()
        sel = np.repeat([which[fr] == k for fr in img], inp.hyps)
        assert sel.any()
        assert same_bits(maps[sel], m1[sel]) and same_bits(labels[sel], l1[sel]) and same_bits(correct[sel], c1[sel])
    if W % 2:   # getCamMat's integer half width, not getObj's width / 2.f
        assert CO.cam_mat(cams3[0])[1] == 320.0
    ref = CO.round_maps(img, inp.gt.cpu().numpy(), inp.noise.cpu().numpy(), inp.coords.cpu().numpy(),
                        inp.pix.cpu().numpy(), inp.hyps, cams)
    assert np.abs(maps - ref).max() <= 2e-3 and (maps < 100).mean() > 0.2
    # an image whose frame lies outside the table: NaN map and label, correct 0, the others unchanged
    bad = inp.img.clone()
    bad[1], bad[4] = F, -1
    m2, l2, c2 = inp.maps(eng, bad)
    hit = np.repeat(np.isin(np.arange(inp.n_images), [1, 4]), inp.hyps)
    assert np.isnan(m2[hit]).all() and np.isnan(l2[hit]).all() and (c2[hit] == 0).all()
    assert same_bits(m2[~hit], maps[~hit]) and same_bits(l2[~hit], labels[~hit])


# ------------------------------------------------------------------ 5. validation
def test_validation(engine_mod, eng):
    E = engine_mod
    lib = eng.lib
    W, H = 64, 48
    good = mixed_cams(E, W, H, 1) + [E.default_rgbd_camera(width=W, height=H)]
    F = len(good)
    rng = np.random.default_rng(5)
    raw = dev(synthetic_depth(rng, F, H, W).view(np.int16), torch.int16)
    poses = dev(random_poses(rng, F), torch.float64)
    eng.set_dataset_cameras(good)
    want = register(eng, None, raw, F, H, W)[0]
    want_co = obj_coords(eng, None, F, want, poses, list(range(F)))

    def bad(**kw):
        c = E.default_rgbd_camera(width=W, height=H)
        for k, v in kw.items():
            if k == "sensor_trans_5":
                c.sensor_trans[5] = v
            else:
                setattr(c, k, v)
        return c

    nan, inf = float("nan"), float("inf")
    cases = [dict(focal=nan), dict(focal=0.0), dict(focal=-525.0), dict(focal=inf), dict(secondary_focal=0.0),
             dict(secondary_focal=nan), dict(x_shift=inf), dict(y_shift=nan), dict(raw_x_shift=-inf),
             dict(raw_y_shift=nan), dict(sensor_trans_5=nan), dict(width=W + 1), dict(height=H - 1),
             dict(raw_data=0), dict(width=0, height=0)]
    for kw in cases:
        cams = list(good)
        cams[2] = bad(**kw)
        table = E.camera_table(cams)
        assert lib.dsac_set_dataset_cameras(eng.h, F, C.cast(table, C.c_void_p), None) == -1, kw
        assert "camera 2" in lib.dsac_last_error(eng.h).decode(), kw
    # a secondary focal length is not needed without registration
    nr = [E.default_rgbd_camera(width=W, height=H, raw_data=0, secondary_focal=0.0)] * 2
    assert lib.dsac_set_dataset_cameras(eng.h, 2, C.cast(E.camera_table(nr), C.c_void_p), None) == 0
    eng.set_dataset_cameras(good)
    assert lib.dsac_set_dataset_cameras(eng.h, 0, C.cast(E.camera_table(good), C.c_void_p), None) == -1
    with pytest.raises(RuntimeError):
        eng.set_dataset_cameras(good[:2] + [bad(focal=nan)])
    # the engine kept the table in force
    assert torch.equal(register(eng, None, raw, F, H, W)[0], want)
    assert torch.equal(obj_coords(eng, None, F, want, poses, list(range(F))), want_co)
    # n_frames must match the table
    with pytest.raises(RuntimeError, match="cover"):
        register(eng, None, raw[:3].contiguous(), 3, H, W)
    with pytest.raises(RuntimeError, match="cover"):
        obj_coords(eng, None, 3, want, poses, [0])
    with pytest.raises(RuntimeError, match="cover"):
        draw(eng, None, 3, want, poses, rng_state(eng, 1, 1), 1, 4)
    # NULL clears the table: cam = NULL is refused again, and the score path is back on the config camera
    eng.set_dataset_cameras(None)
    inp = ScoreInputs(eng, F, 640, 480, n_images=3, hyps=4)
    no_table = inp.maps(eng)
    eng.set_dataset_cameras([E.default_rgbd_camera(focal=600.0)] * F)
    assert not same_bits(inp.maps(eng)[0], no_table[0])
    eng.set_dataset_cameras(None)
    for x, y in zip(inp.maps(eng), no_table):
        assert same_bits(x, y)
    for call in (lambda: register(eng, None, raw, F, H, W), lambda: obj_coords(eng, None, F, want, poses, [0]),
                 lambda: draw(eng, None, F, want, poses, rng_state(eng, 1, 1), 1, 4)):
        with pytest.raises(RuntimeError, match="no dataset cameras"):
            call()
    torch.cuda.synchronize()


# ------------------------------------------------------------------ 6. independence from the forward's cameras
def test_tables_are_independent(engine_mod, eng):
    E = engine_mod
    coords, pix, _, gt_jp = E.synth_frames(2, rho=0.6)
    a = eng.forward(coords, pix, gt_jp, want_diffmaps=True)
    eng.set_dataset_cameras(mixed_cams(E, 640, 480, 1))
    b = eng.forward(coords, pix, gt_jp, want_diffmaps=True)
    for k in ("hyp_pose", "scores", "diffmaps", "ref_pose", "loss", "status"):
        assert same_bits(getattr(a, k), getattr(b, k)), k
    # dsac_set_cameras leaves the pre-training outputs alone
    rng = np.random.default_rng(6)
    F, W, H = 3, 640, 480
    cams = mixed_cams(E, W, H, 1)
    raw = dev(synthetic_depth(rng, F, H, W).view(np.int16), torch.int16)
    poses = dev(random_poses(rng, F), torch.float64)
    inp = ScoreInputs(eng, F, W, H, n_images=4, hyps=4)

    def outputs():
        dep = register(eng, None, raw, F, H, W)[0]
        co = obj_coords(eng, None, F, dep, poses, [2, 1, 0])
        d = draw(eng, None, F, dep, poses, rng_state(eng, 9, 2), 3, 20)
        return [dep, co, *d], inp.maps(eng)

    eng.set_dataset_cameras(cams)
    t1, s1 = outputs()
    eng.set_cameras(np.array([[700.0, 300.0, 250.0], [500.0, 330.0, 230.0]]))
    t2, s2 = outputs()
    eng.set_cameras(None)
    for x, y in zip(t1, t2):
        assert torch.equal(x, y)
    for x, y in zip(s1, s2):
        assert same_bits(x, y)


# ------------------------------------------------------------------ 7. Python
class StubCoords(torch.nn.Module):
    """A coordinate "network" for coded frames (obj_oracle.coded_bgr): the patch centre's (x, y) at 2 m depth, metres."""

    def forward(self, patches):
        c = (patches[:, :, 21, 21] + 127.0).round()
        x = c[:, 0] + 256 * ((c[:, 2] % 16) % 4)
        y = c[:, 1] + 256 * ((c[:, 2] % 16) // 4)
        return torch.stack([(x - 320) * 2000 / 525, -(y - 240) * 2000 / 525, torch.full_like(x, -2000.0)], 1) / 1000


def test_pretrainers_on_a_mixed_scene(engine_mod, eng):
    from dsac_b200.coord_cnn import CoordPipeline
    from dsac_b200.obj_train import ObjPretrainer, RGBDScene
    from dsac_b200.score_train import ScorePretrainer
    E = engine_mod
    torch.manual_seed(0)
    rng = np.random.default_rng(7)
    W, H = 640, 480
    cams = [c for c in mixed_cams(E, W, H, 1) for _ in range(2)]
    F = len(cams)
    poses = np.zeros((F, 12))   # cameras near the origin, so that the stub's points lie in front of every noisy pose
    poses[:, [0, 4, 8]] = 1.0
    poses[:, 9:] = rng.uniform(-50, 50, (F, 3))
    sc = RGBDScene(eng, OO.coded_bgr(F, H, W), synthetic_depth(rng, F, H, W), poses, cams)
    assert sc.cam is None and len(sc.cams) == F
    tr = ObjPretrainer(eng, sc, n_streams=4, n_images=8, n_patches=64)
    losses = tr.train(12)
    assert len(losses) == 12 and np.isfinite(losses).all()
    pipe = CoordPipeline(eng)
    pipe.model = StubCoords()
    st = ScorePretrainer(eng, sc.bgr, sc.gt_jp, pipe, n_streams=4, n_images=8, hyps_per_image=16, cameras=sc.cams)
    losses = st.train(6)
    assert len(losses) == 6 and np.isfinite(losses).all()
    # the round's error images are those of the frames' own cameras
    maps, _, _ = st.round.draw(4, 16)
    r = st.round
    ref = CO.round_maps(r.img.cpu().numpy(), r.gt_jp.cpu().numpy(), r.noise.cpu().numpy(), r.coords.cpu().numpy(),
                        r.pix.cpu().numpy(), 16, cams)
    assert np.abs(maps.cpu().numpy().reshape(-1, 1600) - ref).max() <= 2e-3
    # cameras=None clears the table: the config camera again
    from dsac_b200.score_train import ScoreRound
    ScoreRound(eng, sc.bgr, sc.gt_jp, pipe).draw(2, 4)
    assert eng._dataset_cameras is None


def test_two_scenes_share_one_engine(engine_mod, eng):
    from dsac_b200.obj_train import ObjRound, RGBDScene
    E = engine_mod
    W, H = 96, 80
    cams3 = mixed_cams(E, W, H, 1)
    rng = np.random.default_rng(8)
    data = []
    for order in ((0, 1, 2), (2, 2, 1, 0)):
        F = len(order)
        data.append(([cams3[k] for k in order], OO.coded_bgr(F, H, W), synthetic_depth(rng, F, H, W),
                     random_poses(rng, F)))
    shared = [RGBDScene(eng, d[1], d[2], d[3], d[0]) for d in data]
    own_engines = [E.Engine(max_frames=1, n_hyps=64) for _ in data]
    own = [RGBDScene(e, d[1], d[2], d[3], d[0]) for e, d in zip(own_engines, data)]
    rs = [ObjRound(s, seed=5, n_streams=3) for s in shared]
    ro = [ObjRound(s, seed=5, n_streams=3) for s in own]
    for k in range(2):
        assert torch.equal(shared[k].depth, own[k].depth)
    for _ in range(2):
        for k in (0, 1):
            a, b = rs[k].draw(6, 30), ro[k].draw(6, 30)
            for x, y in zip(a, b):
                assert torch.equal(x, y)
            ids = list(range(shared[k].n_frames))[::-1]
            assert torch.equal(shared[k].scene_coords(ids), own[k].scene_coords(ids))
    for e in own_engines:
        e.close()
