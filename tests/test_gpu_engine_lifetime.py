"""Lifetime of the engine's buffers that grow on use (engine.cu: DevMem::reserve): they are sized by the first call that
needs them, re-allocated only when a later call needs more, and then reused.

  - the Kabsch block stays the Kabsch block across a hooked backward, which grows the seam's gradient buffer, in both
    pipelines (a block's growth frees only that block);
  - every growable buffer, grown twice in one engine's life (a small call, then a larger one), gives the small call's
    results again, bit for bit, when the small call is repeated."""
import numpy as np
import pytest
import torch

import obj_oracle as OO

pytestmark = pytest.mark.gpu

N = 1600


class _W:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}


def _fwd_hook(dm, n, Hh, sc, stream):
    return 0   # k_score has already written the closed-form scores


def _bwd_hook(dm, sg, n, Hh, out, stream):
    """The analytic adjoint of the closed-form soft-inlier score (test_gpu_configs.py: test_score_seam_adjoint_hook)."""
    with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
        d = torch.as_tensor(_W(dm, (n, Hh, N), "<f4"), device="cuda").double()
        g = torch.as_tensor(_W(sg, (n, Hh), "<f8"), device="cuda")
        o = torch.as_tensor(_W(out, (n, Hh, N), "<f8"), device="cuda")
        s = torch.sigmoid(0.5 * (10.0 - d))
        o.copy_(g[:, :, None] * (-0.1 * 0.5) * s * (1 - s))
    return 0


def _hooked(E, **kw):
    eng = E.Engine(**kw)
    eng.set_score_hook(_fwd_hook)
    eng.set_score_backward_hook(_bwd_hook)
    return eng


def _frames(E, n):
    coords, pix, _, gt_jp = E.synth_frames(n)
    return coords, pix, gt_jp


def _point_sets(O, n, m, seed):
    rng = np.random.default_rng(seed)
    a = rng.normal(0, 100, (n, m, 3))
    R0 = np.stack([O.rodrigues(rng.uniform(-1, 1, 3)) for _ in range(n)])
    b = np.einsum("nij,nmj->nmi", R0, a) + rng.normal(0, 50, (n, 1, 3)) + rng.normal(0, 1.0, (n, m, 3))
    return a, b


def _check_kabsch(O, a, b, R, t):
    for i in range(a.shape[0]):
        Ro, to = O.kabsch(a[i], b[i])
        assert np.abs(R[i] - Ro).max() <= 1e-9
        assert np.abs(t[i] - to).max() <= 1e-7


def _assert_same(x, y):
    """Every array of two result objects, bit for bit."""
    arrays = {k: v for k, v in vars(x).items() if isinstance(v, np.ndarray)}
    assert arrays
    for k, v in arrays.items():
        assert np.array_equal(v.view(np.uint8), getattr(y, k).view(np.uint8)), k


@pytest.mark.parametrize("pipeline", ["soft_argmax", "dsac"])
def test_kabsch_block_survives_the_seam_backward(engine_mod, oracle, pipeline):
    E, O = engine_mod, oracle
    nf, H = 2, 64
    coords, pix, gt_jp = _frames(E, nf)
    a, b = _point_sets(O, 64, 7, seed=3)
    eng = _hooked(E, max_frames=nf, n_hyps=H)
    R1, t1 = eng.kabsch(a, b)
    if pipeline == "soft_argmax":
        eng.forward(coords, pix, gt_jp)
        g1 = eng.backward(coords, pix, gt_jp, full=False)   # sizes the seam's gradient buffer
    else:
        eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
        g1 = eng.backward_dsac(nf)
    R2, t2 = eng.kabsch(a, b)
    assert np.array_equal(R1, R2) and np.array_equal(t1, t2)
    _check_kabsch(O, a, b, R2, t2)
    # ... and the Kabsch call left the seam's buffer alone
    if pipeline == "soft_argmax":
        eng.forward(coords, pix, gt_jp)
        _assert_same(g1, eng.backward(coords, pix, gt_jp, full=False))
    else:
        eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
        _assert_same(g1, eng.backward_dsac(nf))
    eng.close()


def test_dsac_variant_buffers_grow_and_are_reused(engine_mod):
    """The refine-all buffers, the per-hypothesis inlier maps and the backward's buffer pool."""
    E = engine_mod
    coords, pix, gt_jp = _frames(E, 3)
    eng = E.Engine(max_frames=3, n_hyps=24)

    def step(n):
        fw = eng.forward_dsac(coords[:n], pix[:n], gt_jp[:n], random_draw=False, want_inlier_maps=True)
        return fw, eng.backward_dsac(n)

    small = step(1)
    large = step(3)
    again = step(1)
    for x, y in zip(small, again):
        _assert_same(x, y)
    assert np.array_equal(small[0].inlier_maps[0], large[0].inlier_maps[0])   # frames are independent
    assert (small[0].inlier_maps != 0).any()
    eng.close()


def test_hooked_backward_buffers_grow_and_are_reused(engine_mod):
    """The seam's gradient buffer and the soft-argmax backward's scratch block."""
    E = engine_mod
    coords, pix, gt_jp = _frames(E, 3)
    eng = _hooked(E, max_frames=3, n_hyps=32)

    def step(n):
        eng.forward(coords[:n], pix[:n], gt_jp[:n])
        return eng.backward(coords[:n], pix[:n], gt_jp[:n], full=False)

    small = step(1)
    large = step(3)
    again = step(1)
    _assert_same(small, again)
    # frame 0 of the larger call: the same frame, its k_dscore sums split over a different number of CTAs
    assert np.allclose(small.score_grads[0], large.score_grads[0], rtol=1e-12, atol=0)
    scale = np.abs(small.dloss_dobj).max()
    assert scale > 0
    assert np.abs(small.dloss_dobj[0] - large.dloss_dobj[0]).max() <= 1e-9 * scale
    eng.close()


def test_kabsch_block_grows_and_is_reused(engine_mod, oracle):
    E, O = engine_mod, oracle
    eng = E.Engine(max_frames=1)
    a1, b1 = _point_sets(O, 8, 5, seed=11)
    a2, b2 = _point_sets(O, 96, 9, seed=12)
    R1, t1 = eng.kabsch(a1, b1)
    R2, t2 = eng.kabsch(a2, b2)
    R3, t3 = eng.kabsch(a1, b1)
    assert np.array_equal(R1, R3) and np.array_equal(t1, t3)
    _check_kabsch(O, a1, b1, R3, t3)
    _check_kabsch(O, a2, b2, R2, t2)
    eng.close()


def test_depth_registration_keys_grow_and_are_reused(engine_mod):
    E = engine_mod
    W, Hh = 64, 48
    cam = E.default_rgbd_camera(width=W, height=Hh, raw_data=1, sensor_trans=np.eye(4))
    rng = np.random.default_rng(5)
    raw = rng.integers(500, 4000, (3, Hh, W)).astype(np.uint16)
    raw[rng.random(raw.shape) < 0.1] = 0
    eng = E.Engine(max_frames=1)

    def register(n):
        d_raw = torch.from_numpy(raw[:n].view(np.int16).copy()).cuda()
        depth = torch.empty_like(d_raw)
        dropped = torch.zeros(n, dtype=torch.int32, device="cuda")
        eng.register_depth_device(cam, n, d_raw.data_ptr(), depth.data_ptr(), dropped.data_ptr())
        torch.cuda.synchronize()
        return depth.cpu().numpy().view(np.uint16), dropped.cpu().numpy()

    small = register(1)
    large = register(3)
    again = register(1)
    assert np.array_equal(small[0], again[0]) and np.array_equal(small[1], again[1])
    reg, dropped = OO.register_depth(cam, raw)
    assert np.array_equal(large[0], reg) and np.array_equal(large[1], dropped)
    assert np.array_equal(small[0], reg[:1])
    eng.close()
