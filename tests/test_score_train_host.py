"""Score-CNN pre-training data path on the CPU: the host build of scoretrain.cuh's draws and pose arithmetic against the
numpy restatement (tests/score_oracle.py) and against libstdc++'s own distributions and gcc's argument order, the
per-round shuffles against a continuing std::mt19937, and the trainer's loss, lr schedule and selectBest against numpy."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import obj_oracle as OO
import score_oracle as SO
from conftest import ROOT


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("scoreshim") / "libscore_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "score_shim.cpp")])
    lib = C.CDLL(so)
    lib.shim_normal_vs_std.argtypes = [C.c_uint32, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
    lib.shim_uniform_vs_std.argtypes = [C.c_uint32, C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
    lib.shim_rand_hyp_vs_ref.argtypes = [C.c_uint32, C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_void_p]
    lib.shim_score_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.mark.parametrize("seed", [1305, 1306, 7, 2 ** 32 - 1])
@pytest.mark.parametrize("stddev", [2.0, 10.0, 100.0])
def test_normal_draw_matches_libstdcxx(shim, seed, stddev):
    n = 5000
    mine, theirs = np.zeros(n), np.zeros(n)
    assert shim.shim_normal_vs_std(seed, stddev, n, _p(mine), _p(theirs)) == 1
    assert np.array_equal(_bits(mine), _bits(theirs))


@pytest.mark.parametrize("lo,hi", [(0.0, 1.0), (21.0, 35.95), (456.25, 471.2)])
def test_uniform_real_matches_libstdcxx(shim, lo, hi):
    n = 5000
    mine, theirs = np.zeros(n), np.zeros(n)
    assert shim.shim_uniform_vs_std(1305, lo, hi, n, _p(mine), _p(theirs)) == 1
    assert np.array_equal(_bits(mine), _bits(theirs))


@pytest.mark.parametrize("rot,trans", [(2.0, 2.0), (10.0, 100.0)])
def test_rand_hyp_matches_reference_spelling(shim, rot, trans):
    """getRandHyp as gcc compiles the reference's spelling (the draws as constructor arguments): z before y before x.
    The restatement draws in the same order, from the same words."""
    n = 2000
    for seed in (1305, 1306, 99):
        mine, theirs = np.zeros((n, 6)), np.zeros((n, 6))
        assert shim.shim_rand_hyp_vs_ref(seed, rot, trans, n, _p(mine), _p(theirs)) == 1
        assert np.array_equal(_bits(mine), _bits(theirs))
        bg = np.random.MT19937()
        bg._legacy_seeding(seed)
        words = lambda: int(bg.random_raw())   # noqa: E731
        ora = np.stack([SO.rand_hyp(words, rot, trans) for _ in range(n)])
        assert np.array_equal(_bits(ora), _bits(mine))
        # the axis lies in the positive octant; the angle's sign flips all three components together
        s = np.sign(mine[:, :3])
        assert ((s == s[:, :1]) | (s == 0)).all() and (s[:, 0] < 0).any() and (s[:, 0] > 0).any()


@pytest.mark.parametrize("size", [43, 50, 96, 128, 480, 640, 641, 1000, 1920])
def test_grid_bounds_match_restatement(shim, size):
    out = np.zeros(4096, np.float32)
    n = shim.shim_grid_bounds(size, _p(out))
    ref = SO.grid_bounds(size)
    assert n == len(ref) and np.array_equal(out[:n], np.array(ref, np.float32))


CASES = [  # (T, n_frames, width, height, n_images, hyps)
    (1, 5, 128, 96, 3, 4),
    (3, 4, 128, 96, 3, 5),      # hyps not divisible by T
    (16, 7, 640, 480, 2, 5),    # T > hyps: streams 5.. draw nothing
    (3, 9, 640, 480, 2, 16),
]


@pytest.mark.parametrize("T,F,W,H,n_images,hyps", CASES)
def test_draw_matches_restatement(shim, T, F, W, H, n_images, hyps):
    st_o = OO.rng_init(1305, T)
    st_s = st_o.copy()
    for _ in range(2):   # two consecutive rounds continue the streams
        img, pix, drift, noise = SO.draw(st_o, F, W, H, n_images, hyps)
        o = [np.zeros(n_images, np.int32), np.zeros((n_images, 1600, 2), np.int32), np.zeros(n_images * hyps, np.int32),
             np.zeros((n_images * hyps, 6))]
        shim.shim_score_draw(_p(st_s), T, F, W, H, n_images, hyps, *[_p(a) for a in o])
        assert np.array_equal(o[0], img) and np.array_equal(o[1], pix) and np.array_equal(o[2], drift)
        assert np.array_equal(_bits(o[3]), _bits(noise))
        assert np.array_equal(st_s, st_o)
    assert set(np.unique(drift)) <= {0, 1}
    if T > hyps:
        assert np.array_equal(st_o[hyps:], OO.rng_init(1305, T)[hyps:])


def _random_pose(rng):
    from scipy.spatial.transform import Rotation
    p = np.zeros(12)
    p[:9] = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix().reshape(9)
    p[9:] = rng.uniform(-2000, 2000, 3)
    return p


def _check_sample(shim, rng, gt, v, f=525.0, cx=320.0, cy=240.0):
    """shim_score_sample against the restatement: the label within 1e-9, and the error image of the projection rows
    (the fp32 arithmetic K2 applies) within 2e-3 px of getDiffMap's double arithmetic on a scene in front of the noisy
    camera.  Returns (flag, restated flag, angle, translation error)."""
    P = np.zeros(12, np.float32)
    lab, cor = np.zeros(1), np.zeros(1, np.int32)
    shim.shim_score_sample(_p(gt), _p(v), f, 10.0, _p(P), _p(lab), _p(cor))
    r_lab, r_cor, ang, dt = SO.sample(gt, v)
    assert abs(lab[0] - r_lab) <= 1e-9 * max(1.0, abs(r_lab))
    Rg, tg, Rn, tn = SO.noise_pose(gt, v)
    pix = np.stack(np.meshgrid(np.linspace(30, 610, 40), np.linspace(30, 450, 40)), -1).reshape(1600, 2).astype(np.int32)
    d = rng.uniform(500, 4000, 1600)
    cam = np.stack([(pix[:, 0] - cx) * d / f, (pix[:, 1] - cy) * d / f, d], 1) + rng.normal(0, 20, (1600, 3))
    cam_jp = cam * np.array([1, -1, -1])            # the jp camera frame (our2cv flips y and z)
    X = np.round((cam_jp - tn) @ Rn).clip(-32768, 32767)   # scene = Rn^T (cam - tn)
    ref = SO.diff_map(gt, v, X, pix, f, cx, cy)
    Pm = P.astype(np.float64).reshape(3, 4)
    q = np.c_[X.astype(np.float32).astype(np.float64), np.ones(1600)] @ Pm.T
    e = np.hypot((pix[:, 0] - cx) * q[:, 2] - q[:, 0], (pix[:, 1] - cy) * q[:, 2] - q[:, 1]) / np.abs(q[:, 2])
    assert np.abs(np.minimum(e, 100) - ref).max() < 2e-3
    assert (ref < 100).mean() > 0.2
    return int(cor[0]), r_cor, ang, dt


def test_sample_matches_restatement(shim):
    rng = np.random.default_rng(4)
    st = OO.rng_init(77, 1)
    _, _, drift, noise = SO.draw(st, 1, 640, 480, 4, 64)
    n_flag = 0
    for k in range(len(noise)):
        v = noise[k].copy()
        if k == 5:
            v[:3] = 1e-6     # |r| <= 1e-5: the identity rotation
        cor, r_cor, ang, dt = _check_sample(shim, rng, _random_pose(rng), v)
        if abs(ang - 5) > 1e-6 and abs(dt - 50) > 1e-6:
            assert cor == r_cor
            n_flag += r_cor
    assert n_flag > 0 and (drift == 0).any() and (drift == 1).any()


def test_sample_near_identity_rotation(shim):
    """A ground-truth rotation near the identity and a small noise rotation: the noisy pose's rotation is near the
    identity, so our2cv's row flip puts it near 180 degrees, where the axis amplifies the float rounding of poseGT's
    rotation unless the matrix is first projected onto the nearest rotation (as cv::Rodrigues does)."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(8)
    for k in range(60):
        gt = np.zeros(12)
        r = rng.normal(size=3)
        gt[:9] = Rotation.from_rotvec(r / np.linalg.norm(r) * 10.0 ** rng.uniform(-7, -2)).as_matrix().reshape(9)
        if k == 0:
            gt[:9] = np.eye(3).reshape(9)
        gt[9:] = rng.uniform(-500, 500, 3)
        v = np.zeros(6)
        a = rng.normal(size=3)
        v[:3] = a / np.linalg.norm(a) * (0.0 if k == 1 else 10.0 ** rng.uniform(-5, -2))
        v[3:] = rng.normal(0, 2, 3)
        _check_sample(shim, rng, gt, v)


@pytest.mark.parametrize("n,seed", [(1600, 5489), (7, 1), (70000, 3)])
def test_shuffle_permutations_continue_one_generator(engine_mod, n, seed):
    ref = SO.shuffle_rounds(n, seed, 3)
    assert np.array_equal(engine_mod.shuffle_permutations(n, seed, 0, 3), ref)
    assert np.array_equal(engine_mod.shuffle_permutations(n, seed, 2, 1), ref[2:])
    assert np.array_equal(engine_mod.shuffle_permutations(n, seed)[0], engine_mod.shuffle_permutation(n, seed))
    assert not np.array_equal(ref[0], ref[1])
    with pytest.raises(ValueError):
        engine_mod.shuffle_permutations(0, seed)
    with pytest.raises(ValueError):
        engine_mod.shuffle_permutations(n, seed, -1, 1)


class _Lin(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.full((1600,), 1e-3, dtype=torch.float64))

    def forward(self, x):
        return (x.reshape(x.shape[0], -1).double() @ self.w).reshape(-1, 1).float()


def test_step_loss_and_lr_schedule_match_numpy():
    """ScorePretrainer.step: AbsCriterion (mean |pred - label|) of the network on maps - 45 against float32 labels, one
    Torch7Adam update, the learning rate halved after every lr_interval updates."""
    from dsac_b200.score_train import ScorePretrainer
    from dsac_b200.obj_train import Torch7Adam
    tr = ScorePretrainer.__new__(ScorePretrainer)
    tr.model = _Lin()
    tr.opt = Torch7Adam(tr.model.parameters(), lr=1e-4)
    tr.updates, tr.log, tr.lr_interval = 0, [], 3
    rng = np.random.default_rng(5)
    for u in range(7):
        maps = torch.tensor(rng.uniform(0, 100, (64, 1, 40, 40)), dtype=torch.float32)
        labels = torch.tensor(-rng.uniform(0, 500, 64), dtype=torch.float64)
        w = tr.model.w.detach().numpy().copy()
        pred = ((maps.numpy().reshape(64, -1) - np.float32(45)).astype(np.float64) @ w).astype(np.float32)
        ref = np.abs(pred - labels.numpy().astype(np.float32)).mean()
        assert abs(tr.step(maps, labels) - ref) < 1e-5 * max(1.0, ref)
        assert tr.opt.param_groups[0]["lr"] == 1e-4 * 0.5 ** ((u + 1) // 3)
    assert [k for k, _ in tr.log] == list(range(7))


def test_select_best_first_maximum_wins():
    from dsac_b200.score_train import select_best
    labels = torch.tensor([-60.0, -10.0, -49.0, -70.0])
    assert select_best(torch.tensor([0.1, 0.5, 0.5, 0.2]), labels) == 1    # tie: the first maximum, label -10
    assert select_best(torch.tensor([0.9, 0.5, 0.5, 0.2]), labels) == 0    # -60 is not above -50
    assert select_best(torch.tensor([0.1, 0.2, 0.3, 0.2]), labels) == 1    # -49 is above -50
    assert select_best(torch.tensor([0.1, 0.2, 0.3, 0.9]), labels) == 0
