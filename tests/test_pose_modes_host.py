"""Pose modes (dsac_pose_modes_device) on the host: the nearness test and the ranking key of dsac_b200/csrc/modes.cuh,
compiled for the host, against scipy; and a numpy restatement of the call's selection and merge (select, merge), checked
on hand-built pools with known answers.  tests/test_gpu_pose_modes.py checks the engine against the same restatement."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ST_BAD_PRIOR = 128


# ---------------------------------------------------------------------------------------------- the numpy restatement

def rotations(poses):
    """Row-major rotation matrices [k][9] of cv poses [k][6]."""
    poses = np.asarray(poses, np.float64).reshape(-1, 6)
    return Rotation.from_rotvec(poses[:, :3]).as_matrix().reshape(-1, 9)


def angle(Ra, Rb):
    """theta of M = Ra Rb^T with v and c as so3_log forms them (modes.cuh, mode_angle)."""
    A, B = np.asarray(Ra).reshape(3, 3), np.asarray(Rb).reshape(3, 3)
    M = (A @ B.T).reshape(9)
    v = 0.5 * np.array([M[7] - M[5], M[2] - M[6], M[3] - M[1]])
    s = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    c = 0.5 * (M[0] + M[4] + M[8] - 1.0)
    return math.atan2(s, c)


def dist(ta, tb):
    d = np.asarray(ta, np.float64) - np.asarray(tb, np.float64)
    return math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])


def near(Ra, ta, Rb, tb, rot, trans):
    return dist(ta, tb) <= trans and angle(Ra, Rb) <= rot


def occupied(img_idx, status, prior_k):
    """Step 1: img_idx[h][0] >= 0, or a prior slot of a frame without DSAC_ST_BAD_PRIOR."""
    img_idx = np.asarray(img_idx).reshape(-1, 4)
    H = len(img_idx)
    occ = img_idx[:, 0] >= 0
    if prior_k and not (int(status) & ST_BAD_PRIOR):
        occ[H - prior_k:] = True
    return occ


def ranking(scores, occ):
    """Step 2: occupied slots by score descending, ties to the lower slot, NaN after every score."""
    slots = [h for h in range(len(occ)) if occ[h]]
    return sorted(slots, key=lambda h: (1, 0.0, h) if math.isnan(scores[h]) else (0, -scores[h], h))


def select(hyp_pose, img_idx, scores, sf, status, prior_k, M, rot, trans):
    """Steps 1-3 of one frame: (seed slots, their mass, their member counts, owner of every slot or -1)."""
    H = len(scores)
    R = rotations(hyp_pose)
    t = np.asarray(hyp_pose, np.float64).reshape(H, 6)[:, 3:]
    seeds, mass, members = [], [], []
    owner = np.full(H, -1)
    for h in ranking(scores, occupied(img_idx, status, prior_k)):
        for s, g in enumerate(seeds):
            if near(R[h], t[h], R[g], t[g], rot, trans):
                owner[h] = s
                break
        else:
            if len(seeds) < M:
                owner[h] = len(seeds)
                seeds.append(h)
                mass.append(0.0)
                members.append(0)
        if owner[h] >= 0:
            mass[owner[h]] += float(sf[h])
            members[owner[h]] += 1
    return seeds, mass, members, owner


def merge(ref_poses, mass, members, rot, trans):
    """Step 5 over the refined seed poses [k][6]: (indices of the surviving seeds in seed order, their mass, members)."""
    k = len(mass)
    R = rotations(ref_poses) if k else np.zeros((0, 9))
    t = np.asarray(ref_poses, np.float64).reshape(k, 6)[:, 3:]
    alive, mass, members = [], list(mass), list(members)
    for s in range(k):
        for a in alive:
            if near(R[s], t[s], R[a], t[a], rot, trans):
                mass[a] += mass[s]
                members[a] += members[s]
                break
        else:
            alive.append(s)
    return alive, [mass[a] for a in alive], [members[a] for a in alive]


# ---------------------------------------------------------------------------------------------- the host build

@pytest.fixture(scope="module")
def shim():
    so = os.path.join(tempfile.mkdtemp(prefix="modes_shim_"), "libmodes_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "modes_shim.cpp")])
    lib = C.CDLL(so)
    lib.shim_mode_angle.restype = C.c_double
    lib.shim_mode_dist.restype = C.c_double
    lib.shim_mode_near.argtypes = [C.c_void_p] * 4 + [C.c_double, C.c_double]
    lib.shim_mode_rank_key.restype = C.c_ulonglong
    lib.shim_mode_rank_key.argtypes = [C.c_int, C.c_double]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f64(a):
    return np.ascontiguousarray(a, np.float64)


@pytest.mark.parametrize("target", [None, 0.0, 1e-9, 1e-7, 1e-6, np.pi - 1e-6, np.pi - 1e-8, np.pi])
def test_angle_matches_scipy(shim, target):
    rng = np.random.default_rng(17 if target is None else int(target * 1e6) + 3)
    for _ in range(200):
        a = Rotation.random(random_state=rng.integers(1 << 30))
        if target is None:
            b = Rotation.random(random_state=rng.integers(1 << 30))
        else:
            axis = rng.normal(size=3)
            axis /= np.linalg.norm(axis)
            b = Rotation.from_rotvec(target * axis) * a
        Ra, Rb = _f64(a.as_matrix()), _f64(b.as_matrix())
        ref = (Rotation.from_matrix(Ra) * Rotation.from_matrix(Rb).inv()).magnitude()
        got = shim.shim_mode_angle(_p(Ra), _p(Rb))
        assert abs(got - ref) <= 1e-12, (target, got, ref)
        assert got == angle(Ra, Rb) or abs(got - angle(Ra, Rb)) <= 4e-16 * max(1.0, got)


def test_near_is_both_radii(shim):
    rng = np.random.default_rng(5)
    for _ in range(500):
        pa, pb = rng.normal(size=6) * [1, 1, 1, 300, 300, 300], rng.normal(size=6) * [1, 1, 1, 300, 300, 300]
        Ra, Rb = _f64(rotations(pa)[0]), _f64(rotations(pb)[0])
        th = shim.shim_mode_angle(_p(Ra), _p(Rb))
        d = shim.shim_mode_dist(_p(_f64(pa[3:])), _p(_f64(pb[3:])))
        assert abs(d - np.linalg.norm(pa[3:] - pb[3:])) <= 1e-12 * d
        for rot, trans in [(th * 1.01, d * 1.01), (th * 0.99, d * 1.01), (th * 1.01, d * 0.99), (th, d)]:
            got = shim.shim_mode_near(_p(Ra), _p(_f64(pa[3:])), _p(Rb), _p(_f64(pb[3:])), rot, trans)
            assert got == int(rot >= th and trans >= d)
    nan = _f64([np.nan, 0, 0])
    assert shim.shim_mode_near(_p(_f64(np.eye(3))), _p(nan), _p(_f64(np.eye(3))), _p(_f64(np.zeros(3))), 1.0, 1e9) == 0


def test_rank_key_orders_as_the_restatement(shim):
    """Sorting by (key descending, slot ascending) is ranking(): NaN after -inf, -0 ties +0, empty slots last."""
    rng = np.random.default_rng(23)
    specials = [np.nan, -np.inf, np.inf, 0.0, -0.0, 5e-324, -5e-324, 1.0, 1.0, -1.0, 1e308, -1e308]
    for trial in range(50):
        H = 64
        scores = rng.choice(specials + list(rng.normal(size=8) * 10.0 ** rng.integers(-3, 4, size=8)), size=H)
        occ = rng.random(H) < 0.8
        keys = [int(shim.shim_mode_rank_key(int(occ[h]), float(scores[h]))) for h in range(H)]
        order = sorted(range(H), key=lambda h: (-keys[h], h))
        n_occ = int(occ.sum())
        assert order[:n_occ] == ranking(scores, occ)
        assert all(keys[h] == 0 for h in order[n_occ:]) and all(keys[h] > 0 for h in order[:n_occ])


# ---------------------------------------------------------------------------------------------- hand-built pools

def _pool(poses, scores, sf=None, empty=()):
    H = len(poses)
    img_idx = np.tile(np.arange(4, dtype=np.int32), (H, 1))
    for h in empty:
        img_idx[h] = -1
    sf = np.full(H, 1.0 / H) if sf is None else np.asarray(sf, np.float64)
    return np.asarray(poses, np.float64), img_idx, np.asarray(scores, np.float64), sf


def _at(deg, x_mm, axis=(0.0, 0.0, 1.0)):
    """A cv pose rotated deg about axis, translated x_mm along x, 3 m in front."""
    return np.concatenate([np.radians(deg) * np.asarray(axis), [x_mm, 0.0, 3000.0]])


ROT, TRANS = np.radians(5.0), 50.0


def test_ties_go_to_the_lower_slot():
    poses, img, sc, sf = _pool([_at(0, 0), _at(40, 0), _at(80, 0)], [2.0, 2.0, 2.0])
    seeds, mass, members, owner = select(poses, img, sc, sf, 0, 0, 2, ROT, TRANS)
    assert seeds == [0, 1] and members == [1, 1] and list(owner) == [0, 1, -1]


def test_nan_and_minus_inf_scores_rank_last():
    poses, img, sc, sf = _pool([_at(0, 0), _at(40, 0), _at(80, 0), _at(120, 0)], [np.nan, -np.inf, 1.0, np.nan])
    assert ranking(sc, np.ones(4, bool)) == [2, 1, 0, 3]
    seeds, _, _, _ = select(poses, img, sc, sf, 0, 0, 4, ROT, TRANS)
    assert seeds == [2, 1, 0, 3]


def test_empty_and_prior_slots():
    """Slots 1 and 3 are empty (img_idx -1); slot 3 is also the prior slot of a k = 1 pass, which counts unless the frame
    has DSAC_ST_BAD_PRIOR."""
    poses, img, sc, sf = _pool([_at(0, 0), _at(40, 0), _at(80, 0), _at(120, 0)], [1.0, 9.0, 2.0, 5.0], empty=(1, 3))
    assert select(poses, img, sc, sf, 0, 0, 4, ROT, TRANS)[0] == [2, 0]
    assert select(poses, img, sc, sf, 0, 1, 4, ROT, TRANS)[0] == [3, 2, 0]
    assert select(poses, img, sc, sf, ST_BAD_PRIOR, 1, 4, ROT, TRANS)[0] == [2, 0]
    # a bad-prior frame's slots are all empty: no seeds at all
    img[:] = -1
    assert select(poses, img, sc, sf, ST_BAD_PRIOR | 1, 1, 4, ROT, TRANS)[0] == []


def test_M_reached_with_slots_left_over():
    """Slots near an existing seed still join it once M seeds exist; the others join nothing and add no mass."""
    poses, img, sc, sf = _pool([_at(0, 0), _at(40, 0), _at(80, 0), _at(1, 10), _at(41, 0)], [5, 4, 3, 2, 1],
                               sf=[0.1, 0.2, 0.3, 0.15, 0.25])
    seeds, mass, members, owner = select(poses, img, sc, sf, 0, 0, 2, ROT, TRANS)
    assert seeds == [0, 1] and list(owner) == [0, 1, -1, 0, 1] and members == [2, 2]
    assert mass == [0.1 + 0.15, 0.2 + 0.25]


def test_chain_is_not_transitive():
    """c is near b but not a; b joins a; c becomes its own seed."""
    poses, img, sc, sf = _pool([_at(0, 0), _at(0, 40), _at(0, 80)], [3, 2, 1])
    seeds, mass, members, owner = select(poses, img, sc, sf, 0, 0, 4, ROT, TRANS)
    assert seeds == [0, 2] and list(owner) == [0, 0, 1] and members == [2, 1]
    # with c also near a (a larger radius) all three are one seed
    assert select(poses, img, sc, sf, 0, 0, 4, ROT, 100.0)[0] == [0]


def test_first_near_seed_in_seed_order_wins():
    """d is near seeds 0 and 1 (seeds 0 and 1 are not near each other): it joins seed 0, the earlier."""
    poses, img, sc, sf = _pool([_at(0, 0), _at(0, 60), _at(0, 30)], [3, 2, 1])
    seeds, _, members, owner = select(poses, img, sc, sf, 0, 0, 4, ROT, TRANS)
    assert seeds == [0, 1] and list(owner) == [0, 1, 0] and members == [2, 1]


def test_merge_moves_mass_in_seed_order():
    """Seeds 1 and 3 refine onto seed 0's pose, seed 2 onto nothing: 2 modes, seed 0 with everyone's mass but seed 2's."""
    ref = [_at(0, 0), _at(0.5, 5), _at(60, 0), _at(1, -10)]
    alive, mass, members = merge(ref, [0.4, 0.1, 0.3, 0.05], [3, 1, 2, 1], ROT, TRANS)
    assert alive == [0, 2] and members == [5, 2]
    assert mass == [((0.4 + 0.1) + 0.05), 0.3]
    # a merge goes to the first near survivor, and a dropped seed absorbs nothing
    ref = [_at(0, 0), _at(0, 80), _at(0, 40), _at(0, 60)]
    alive, mass, members = merge(ref, [1.0, 2.0, 4.0, 8.0], [1, 1, 1, 1], ROT, TRANS)
    assert alive == [0, 1] and mass == [5.0, 10.0] and members == [2, 2]
    assert merge([], [], [], ROT, TRANS) == ([], [], [])
