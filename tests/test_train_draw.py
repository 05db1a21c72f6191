"""k_dsac_draw's arithmetic (dsac_b200/csrc/train.cuh) compiled for the host against the libstdc++ calls of the engine's
former host draw: std::mt19937 + discard + std::uniform_real_distribution<double> + the cumulative pick."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def draw_shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("draw_shim") / "libdraw_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "host_shim", "draw_shim.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _sf_batch(rng, n, H):
    """Softmax-like vectors with many entries below the draw's 1e-8 cut, some exactly at it, and all-zero rows."""
    x = rng.standard_normal((n, H)) * rng.uniform(0.5, 20, (n, 1))
    p = np.exp(x - x.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    p[rng.random((n, H)) < 0.05] = 1e-8
    p[rng.random((n, H)) < 0.05] = 0.99e-8
    p[:5] = 0.0
    return np.ascontiguousarray(p)


def _run(shim, sf, seeds, endpos, random_draw):
    n, H = sf.shape
    out = [np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(2 * n, np.uint32), np.zeros(2 * n, np.uint32)]
    shim.shim_draw_cases(n, H, _p(sf), _p(seeds), _p(endpos), random_draw, *[_p(a) for a in out])
    return out


def test_draw_matches_libstdcxx_on_random_softmax(draw_shim):
    rng = np.random.default_rng(5)
    n, H = 100_000, 64
    sf = _sf_batch(rng, n, H)
    seeds = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    endpos = rng.integers(0, 3000, n).astype(np.uint64)
    pp, ps, wp, ws = _run(draw_shim, sf, seeds, endpos, 1)
    assert np.array_equal(wp, ws)
    assert np.array_equal(pp, ps)
    assert len(np.unique(pp)) > H // 2
    pp, ps, _, _ = _run(draw_shim, sf, seeds, endpos, 0)
    assert np.array_equal(pp, ps)


def test_draw_words_at_state_boundaries(draw_shim):
    """endpos on, just before and just after multiples of 624: the two words come from different regenerations."""
    rng = np.random.default_rng(6)
    ks = np.arange(0, 40)
    endpos = np.concatenate([624 * ks + d for d in (-2, -1, 0, 1)])
    endpos = endpos[endpos >= 0].astype(np.uint64)
    endpos = np.concatenate([endpos, np.array([6400, 6400 + 623, 123_456, 624 * 1000 - 1], np.uint64)])
    n, H = len(endpos), 256
    sf = _sf_batch(rng, n, H)
    seeds = (1305 + np.arange(n)).astype(np.uint32)
    pp, ps, wp, ws = _run(draw_shim, sf, seeds, endpos, 1)
    assert np.array_equal(wp, ws)
    assert np.array_equal(pp, ps)


def test_draw_u_next_to_prob_sum(draw_shim):
    """Words whose canonical value rounds to 1 (replaced by the largest double below 1) or lies just below it: u next to
    probSum, where the cumulative sums may never exceed u and the last eligible hypothesis is drawn."""
    rng = np.random.default_rng(7)
    H = 32
    cases = [(0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFF800, 0xFFFFFFFF), (0xFFFFF7FF, 0xFFFFFFFF), (0, 0xFFFFFFFF), (0, 0), (1, 0),
             (0x12345678, 0x80000000)]
    last_seen = False
    for i in range(2000):
        sf = _sf_batch(rng, 1, H)[0] if i >= 5 else np.full(H, 1.0 / H)
        for w0, w1 in cases:
            up, us, pp, ps = C.c_double(), C.c_double(), C.c_int32(), C.c_int32()
            draw_shim.shim_draw_words(H, _p(sf), C.c_uint32(w0), C.c_uint32(w1), C.byref(up), C.byref(us), C.byref(pp), C.byref(ps))
            assert up.value == us.value and pp.value == ps.value, (i, w0, w1)
            elig = np.nonzero(sf >= 1e-8)[0]
            if len(elig) and w0 == w1 == 0xFFFFFFFF and pp.value == elig[-1]:
                last_seen = True
    assert last_seen
