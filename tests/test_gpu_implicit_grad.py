"""Implicit-function scene-coordinate derivatives on the GPU (dsac_set_coord_derivatives(DSAC_DERIV_IMPLICIT)): the
central mode stays bit-identical, the implicit quantities match the host build of ift.cuh (tests/host_shim/ift_shim.cpp)
evaluated at the engine's own poses and fitted sets, and everything else is unchanged."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600


@pytest.fixture(scope="module")
def shim():
    so = os.path.join(tempfile.mkdtemp(prefix="ift_shim_"), "libift_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_shim", "ift_shim.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _rel(a, b, floor=1e-300):
    return np.abs(a - b).max() / max(floor, np.abs(b).max())


def _bw_fields(bw):
    return {k: v.copy() for k, v in vars(bw).items() if isinstance(v, np.ndarray)}


def test_mode_setter_contract(engine_mod):
    E = engine_mod
    eng = E.Engine(max_frames=1, n_hyps=8)
    with pytest.raises(ValueError):
        eng.set_coord_derivatives("forward")
    assert eng.lib.dsac_set_coord_derivatives(eng.h, 2) != 0
    eng.set_coord_derivatives("implicit")
    eng.set_coord_derivatives("central")


@pytest.mark.parametrize("H", [64, 256])
def test_central_mode_unchanged_after_switching(engine_mod, H):
    E = engine_mod
    nf = 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    ref, sw = E.Engine(max_frames=nf, n_hyps=H), E.Engine(max_frames=nf, n_hyps=H)
    for eng in (ref, sw):
        eng.forward(coords, pix, gt_jp)
    sw.set_coord_derivatives("implicit")
    sw.backward(coords, pix, gt_jp)
    sw.set_coord_derivatives("central")
    a, b = _bw_fields(ref.backward(coords, pix, gt_jp)), _bw_fields(sw.backward(coords, pix, gt_jp))
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    for eng in (ref, sw):
        eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    sw.set_coord_derivatives("implicit")
    sw.backward_dsac(nf)
    sw.set_coord_derivatives("central")
    a, b = _bw_fields(ref.backward_dsac(nf)), _bw_fields(sw.backward_dsac(nf))
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def _ift_at(shim, pose, coords, pix, cells, cam):
    Y = np.ascontiguousarray(coords[cells], np.float64)
    e = np.concatenate([pix[cells].astype(np.float64), np.zeros((len(cells), 1))], 1)
    D = np.zeros((len(cells), 6, 3))
    ok = shim.shim_ift_fit_deriv(len(cells), _p(Y), _p(np.ascontiguousarray(e)), _p(np.ascontiguousarray(pose, np.float64)),
                                 C.c_double(cam[0]), C.c_double(cam[1]), C.c_double(cam[2]), 0, _p(D))
    return bool(ok), D


@pytest.mark.parametrize("H", [64, 256])
def test_softam_implicit_matches_host_ift(engine_mod, shim, H):
    E = engine_mod
    nf = 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    fwd = eng.forward(coords, pix, gt_jp)
    central = eng.backward(coords, pix, gt_jp)
    eng.set_coord_derivatives("implicit")
    bw = eng.backward(coords, pix, gt_jp)
    bw2 = eng.backward(coords, pix, gt_jp)
    cam = (eng.cfg.focal, eng.cfg.cx, eng.cfg.cy)
    for k, v in _bw_fields(bw).items():   # a repeated backward gives the same bits
        assert np.array_equal(v, getattr(bw2, k)), k
    assert np.array_equal(bw.dref_dhyp, central.dref_dhyp)
    assert np.array_equal(bw.score_grads, central.score_grads)
    assert np.array_equal(bw.dloss_dref, central.dloss_dref)
    for f in range(nf):
        D = bw.dref_dobj[f].reshape(6, N, 3)
        cells = np.nonzero(np.abs(D).sum((0, 2)) > 0)[0]
        assert 50 <= len(cells) <= eng.cfg.inlier_count
        ok, Dh = _ift_at(shim, fwd.ref_pose[f], coords[f].reshape(N, 3), pix[f].reshape(N, 2), cells, cam)
        assert ok
        assert _rel(D[:, cells, :].transpose(1, 0, 2), Dh) <= 1e-9
        # path I's refinement part is dLossMax . dRefineObj over the same cells
        assert np.isfinite(bw.dloss_dobj[f]).all() and np.abs(bw.dloss_dobj[f]).max() > 0
        # dPNP by the IFT of the P3P equations at the engine's hypotheses
        for h in range(0, H, max(1, H // 16)):
            idx = fwd.img_idx[f, h]
            if (idx < 0).any():
                assert not bw.dpnp[f, h].any()
                continue
            c3 = coords[f].reshape(N, 3)[idx[:3]].astype(np.float64)
            uv = pix[f].reshape(N, 2)[idx[:3]].astype(np.float64)
            out = np.zeros(72)
            shim.shim_ift_dpnp_p3p(_p(np.ascontiguousarray(fwd.hyp_pose[f, h])), _p(np.ascontiguousarray(c3)),
                                   _p(np.ascontiguousarray(uv)), C.c_double(cam[0]), C.c_double(cam[1]), C.c_double(cam[2]), _p(out))
            assert np.abs(bw.dpnp[f, h].reshape(72) - out).max() <= 1e-9 * max(1e-300, np.abs(out).max()), (f, h)
    # dPNP differs from the central differences by their truncation error only
    assert _rel(bw.dpnp, central.dpnp) <= 1e-2


def test_sub_sample_one_accepted_only_in_implicit_mode(engine_mod):
    E = engine_mod
    coords, pix, gt_cv, gt_jp = E.synth_frames(1)
    eng = E.Engine(max_frames=1, n_hyps=64, sub_sample=1.0)
    eng.forward(coords, pix, gt_jp)
    with pytest.raises(RuntimeError):
        eng.backward(coords, pix, gt_jp)
    eng.set_coord_derivatives("implicit")
    a = eng.backward(coords, pix, gt_jp)
    b = E.Engine(max_frames=1, n_hyps=64)
    b.forward(coords, pix, gt_jp)
    b.set_coord_derivatives("implicit")
    assert np.array_equal(a.dloss_dobj, b.backward(coords, pix, gt_jp).dloss_dobj)   # sub_sample does not enter


@pytest.mark.parametrize("random_draw", [False, True])
def test_dsac_implicit(engine_mod, random_draw):
    E = engine_mod
    nf = 3
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=64)
    eng.forward_dsac(coords, pix, gt_jp, random_draw=random_draw)
    central = eng.backward_dsac(nf)
    eng.set_coord_derivatives("implicit")
    bw = eng.backward_dsac(nf)
    bw2 = eng.backward_dsac(nf)
    for k, v in _bw_fields(bw).items():
        assert np.array_equal(v, getattr(bw2, k)), k
    assert np.array_equal(bw.n_selected, central.n_selected)
    assert np.array_equal(bw.n_refine_jobs, 18 * bw.n_selected)
    assert np.array_equal(bw.score_grads, central.score_grads)
    for f in range(nf):
        assert np.isfinite(bw.path1[f]).all() and np.isfinite(bw.path2[f]).all()
        assert (np.abs(bw.path1[f]).sum(1) > 0).sum() > (np.abs(central.path1[f]).sum(1) > 0).sum()   # dense
        # path II changes through dPNP only, by the central differences' truncation error
        assert _rel(bw.path2[f], central.path2[f]) <= 1e-2


def test_autograd_derivatives_matches_entry_point(engine_mod):
    import torch
    from dsac_b200 import autograd as A
    E = engine_mod
    nf = 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    pred = torch.from_numpy(coords.astype(np.float32) / np.float32(1000)).cuda().requires_grad_()
    pix_t = torch.from_numpy(np.ascontiguousarray(pix)).cuda()
    gt_t = torch.from_numpy(np.ascontiguousarray(gt_jp)).cuda()
    eng = E.Engine(max_frames=nf, n_hyps=64)
    grads = {}
    for mode in ("central", "implicit", "central"):
        pred.grad = None
        A.softam_loss(eng, pred, pix_t, gt_t, derivatives=mode).sum().backward()
        grads.setdefault(mode, []).append(pred.grad.clone())
    assert torch.equal(grads["central"][0], grads["central"][1])
    assert not torch.equal(grads["central"][0], grads["implicit"][0])
    # the same through the device entry point
    eng2 = E.Engine(max_frames=nf, n_hyps=64)
    eng2.set_coord_derivatives("implicit")
    pred.grad = None
    A.softam_loss(eng2, pred, pix_t, gt_t).sum().backward()
    assert torch.equal(pred.grad, grads["implicit"][0])


# ---------------------------------------------------------------- against the oracle's recorded sets and chains
def _perm_cfg(O, **kw):
    return O.default_config(**kw)


@pytest.mark.parametrize("H", [1, 64])
def test_softam_recorded_set_and_chain_match_oracle(engine_mod, oracle, shim, H):
    """S of the recording replay is the oracle's (tests/host_shim/ift_oracle.cpp); the gradient the caller consumes,
    dloss_dobj, is the oracle's chain with the implicit parts evaluated at the oracle's S and pose."""
    import ift_oracle as I
    E, O = engine_mod, oracle
    nf = 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    fwd = eng.forward(coords, pix, gt_jp)
    central = eng.backward(coords, pix, gt_jp)
    eng.set_coord_derivatives("implicit")
    bw = eng.backward(coords, pix, gt_jp)
    cam = (eng.cfg.focal, eng.cfg.cx, eng.cfg.cy)
    for f in range(nf):
        cfg = O.default_config(seed=1305 + f, n_hyps=H)
        ofw = O.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
        obw = O.backward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw)
        pose, S, _ = I.refine_record(cfg, coords[f], pix[f], ofw.pixel_idxs, ofw.n_perm_steps, ofw.avg)
        assert np.array_equal(pose, ofw.ref)
        c3, p2 = coords[f].reshape(N, 3), pix[f].reshape(N, 2)
        D = bw.dref_dobj[f].reshape(6, N, 3)
        assert np.array_equal(np.sort(np.nonzero(np.abs(D).sum((0, 2)) > 0)[0]), np.sort(S))   # the recorded set
        ok, Dh = _ift_at(shim, pose, c3, p2, S, cam)
        assert ok
        assert _rel(D[:, S, :].transpose(1, 0, 2), Dh) <= 1e-8
        dL = obw.dloss_dref
        expect = np.zeros((N, 3))
        expect[S] = np.einsum("k,ikj->ij", dL, Dh)   # dLossMax . dRefineObj
        if H == 1:
            # sf = 1, path II vanishes: dloss_dobj = dL . dRefineObj + (dL . dRefineHyp) . dPNP on the support cells
            idx = ofw.img_idx[0]
            out = np.zeros(72)
            assert shim.shim_ift_dpnp_p3p(_p(np.concatenate([ofw.hyp_rvec[0], ofw.hyp_tvec[0]])),
                                          _p(np.ascontiguousarray(c3[idx[:3]], np.float64)),
                                          _p(np.ascontiguousarray(p2[idx[:3]], np.float64)), C.c_double(cam[0]),
                                          C.c_double(cam[1]), C.c_double(cam[2]), _p(out))
            w = dL @ obw.dref_dhyp.reshape(6, 6)
            sp = w @ out.reshape(6, 12)
            for q in range(4):
                expect[idx[q]] += sp[q * 3:q * 3 + 3]
            assert _rel(bw.dloss_dobj[f], expect) <= 1e-6
        else:
            # on cells no hypothesis uses, only dRefineObj differs from central mode; k_dscore adds dPNP's terms at the
            # support cells' x-major columns too (quirk Q4), so those are excluded as well
            free = np.ones(N, bool)
            used = fwd.img_idx[f].reshape(-1)
            used = used[used >= 0]
            free[used] = False
            free[(used % 40) * 40 + used // 40] = False
            dc = np.einsum("k,kcj->cj", dL, central.dref_dobj[f].reshape(6, N, 3))
            got = bw.dloss_dobj[f] - central.dloss_dobj[f]
            assert np.abs((got - (expect - dc))[free]).max() <= 1e-7 * np.abs(expect).max()


@pytest.mark.parametrize("random_draw", [False, True])
def test_dsac_path1_matches_oracle_chain(engine_mod, oracle, shim, random_draw):
    """With skip larger than any cell count the oracle's central path I holds the 9 minimal-set pairs only; implicit
    path I adds sf_h dLossMax_h . dRefine_h over each selected hypothesis' recorded set, support cells excluded."""
    import ift_oracle as I
    E, O = engine_mod, oracle
    nf, H = 2, 48
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H, sub_sample=0.0005)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=random_draw)
    eng.set_coord_derivatives("implicit")
    bw = eng.backward_dsac(nf)
    cam = (eng.cfg.focal, eng.cfg.cx, eng.cfg.cy)
    for f in range(nf):
        cfg = O.default_config(seed=1305 + f, n_hyps=H, sub_sample=0.0005)
        perm = O.refine_permutations(cfg.ref_steps)
        ofw = O.ForwardDsac(cfg)
        ofw.hyp_rvec[:] = fw.hyp_pose[f][:, :3]; ofw.hyp_tvec[:] = fw.hyp_pose[f][:, 3:]
        ofw.img_idx[:] = fw.img_idx[f]; ofw.sf[:] = fw.sf[f]; ofw.ref_pose[:] = fw.ref_pose[f]; ofw.losses[:] = fw.losses[f]
        obw = O.backward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw)
        assert obw.n_selected == bw.n_selected[f] >= 1
        assert obw.n_refine_jobs == bw.n_refine_jobs[f] == 18 * obw.n_selected
        c3, p2 = coords[f].reshape(N, 3), pix[f].reshape(N, 2)
        gt6 = np.concatenate([O.rodrigues_inv(gt_jp[f, :9]), gt_jp[f, 9:]])
        expect = obw.path1.reshape(N, 3).copy()
        for h in range(H):
            if not fw.sf[f, h] > 1e-4 or fw.img_idx[f, h, 0] < 0:
                continue
            pose, S, _ = I.refine_record(cfg, c3, p2, perm, cfg.ref_steps, fw.hyp_pose[f, h])
            assert np.abs(pose - fw.ref_pose[f, h]).max() <= 1e-9 * max(1.0, np.abs(pose).max())
            if len(S) == 0:
                continue
            ok, Dh = _ift_at(shim, fw.ref_pose[f, h], c3, p2, S, cam)
            if not ok:
                continue
            dl = O.dloss_max(O.jp6(fw.ref_pose[f, h, :3], fw.ref_pose[f, h, 3:]), gt6)
            contrib = fw.sf[f, h] * np.einsum("k,ikj->ij", dl, Dh)
            keep = ~np.isin(S, fw.img_idx[f, h])
            expect[S[keep]] += contrib[keep]
        assert _rel(bw.path1[f], expect) <= 1e-5
        assert np.median(np.abs(bw.path1[f] - expect)) <= 1e-9 * np.abs(expect).max()
        assert _rel(bw.path2[f], obw.path2) <= 1e-2   # path II: central dPNP in the oracle, implicit here


def test_dsac_seeded_implicit_equals_loss_backward(engine_mod, oracle):
    """dsac_backward_dsac_pose_device in implicit mode with seed_h = sf_h dLossMax_h and grad_sf = losses: the loss
    backward's implicit-mode path I, jobs and score gradients."""
    import torch
    E, O = engine_mod, oracle
    nf, H = 3, 48
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    eng.set_coord_derivatives("implicit")
    bw = eng.backward_dsac(nf)
    seed = np.zeros((nf, H, 6))
    for f in range(nf):
        gt6 = np.concatenate([O.rodrigues_inv(gt_jp[f, :9]), gt_jp[f, 9:]])
        for h in range(H):
            seed[f, h] = fw.sf[f, h] * O.dloss_max(O.jp6(fw.ref_pose[f, h, :3], fw.ref_pose[f, h, 3:]), gt6)
    outs = {k: torch.zeros((nf, N, 3), dtype=torch.float64, device="cuda") for k in ("path1", "path2")}
    outs["n_refine_jobs"] = torch.zeros(nf, dtype=torch.int32, device="cuda")
    ds = torch.from_numpy(seed).cuda()
    dg = torch.from_numpy(np.ascontiguousarray(fw.losses)).cuda()
    eng.backward_dsac_pose_device(nf, ds.data_ptr(), dg.data_ptr(), None, 0.0, torch.cuda.current_stream().cuda_stream,
                                  **{k: v.data_ptr() for k, v in outs.items()})
    torch.cuda.synchronize()
    assert np.array_equal(outs["n_refine_jobs"].cpu().numpy(), bw.n_refine_jobs)
    p1 = outs["path1"].cpu().numpy()
    assert np.abs(p1 - bw.path1).max() <= 1e-9 * np.abs(bw.path1).max()
    assert np.abs(outs["path2"].cpu().numpy() - bw.path2).max() <= 1e-12 * np.abs(bw.path2).max()


def test_softam_pose_seeded_implicit_equals_loss_backward(engine_mod):
    import torch
    E = engine_mod
    nf, H = 3, 64
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    eng.forward(coords, pix, gt_jp)
    eng.set_coord_derivatives("implicit")
    bw = eng.backward(coords, pix, gt_jp)
    dobj = torch.zeros((nf, N, 3), dtype=torch.float64, device="cuda")
    seed = torch.from_numpy(np.ascontiguousarray(bw.dloss_dref)).cuda()
    eng.backward_pose_device(nf, seed.data_ptr(), dobj.data_ptr(), None, 0.0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(dobj.cpu().numpy(), bw.dloss_dobj)


# ---------------------------------------------------------------- per-frame cameras and RGB-D
@pytest.mark.parametrize("rgbd,cams", [(False, True), (True, False), (True, True)])
def test_cameras_and_rgbd_instantiations(engine_mod, shim, rgbd, cams):
    """k_refine_ift_cam / _rgbd / _rgbd_cam, the recording replays with the camera table and depth, and k_dkabsch_ift:
    dref_dobj and dPNP against the host build at the engine's poses, central mode unchanged after switching."""
    import torch
    import rgbd_oracle as R
    E = engine_mod
    nf, H = 3, 64
    cam_tab = np.array([[525.0, 320.0, 240.0], [900.0, 300.5, 250.0], [2500.0, 330.0, 200.0]]) if cams else None
    coords, pix, depth, _, gt_jp = R.synth(nf, seed=91, holes=0.15 if rgbd else 0.0, cams=cam_tab)
    engs = []
    keep = []
    for _ in range(2):
        eng = E.Engine(max_frames=nf, n_hyps=H)
        if cams:
            eng.set_cameras(cam_tab)
        if rgbd:
            d = torch.from_numpy(np.ascontiguousarray(depth, np.float32)).cuda()
            eng.set_cell_depth_device(nf, d.data_ptr())
            torch.cuda.synchronize()
            keep.append(d)
        engs.append(eng)
    ref, eng = engs
    fwd = eng.forward(coords, pix, gt_jp)
    ref.forward(coords, pix, gt_jp)
    eng.set_coord_derivatives("implicit")
    bw = eng.backward(coords, pix, gt_jp)
    bw2 = eng.backward(coords, pix, gt_jp)
    for k, v in _bw_fields(bw).items():
        assert np.array_equal(v, getattr(bw2, k)), k
    eng.set_coord_derivatives("central")
    a, b = _bw_fields(ref.backward(coords, pix, gt_jp)), _bw_fields(eng.backward(coords, pix, gt_jp))
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    for f in range(nf):
        cam = tuple(cam_tab[f]) if cams else (525.0, 320.0, 240.0)
        c3 = coords[f].reshape(N, 3).astype(np.float64)
        D = bw.dref_dobj[f].reshape(6, N, 3)
        cells = np.nonzero(np.abs(D).sum((0, 2)) > 0)[0]
        assert 50 <= len(cells) <= eng.cfg.inlier_count
        if rgbd:
            ey, _ = R.eye(pix[f], depth[f], *cam)
            assert np.isfinite(ey[cells]).all()
            e = np.ascontiguousarray(ey[cells])
        else:
            e = np.ascontiguousarray(np.concatenate([pix[f].reshape(N, 2)[cells].astype(np.float64), np.zeros((len(cells), 1))], 1))
        Dh = np.zeros((len(cells), 6, 3))
        assert shim.shim_ift_fit_deriv(len(cells), _p(np.ascontiguousarray(c3[cells])), _p(e),
                                       _p(np.ascontiguousarray(fwd.ref_pose[f])), C.c_double(cam[0]), C.c_double(cam[1]),
                                       C.c_double(cam[2]), int(rgbd), _p(Dh))
        assert _rel(D[:, cells, :].transpose(1, 0, 2), Dh) <= 1e-8
        for h in range(0, H, 8):
            idx = fwd.img_idx[f, h]
            if (idx < 0).any():
                assert not bw.dpnp[f, h].any()
                continue
            out = np.zeros(72)
            if rgbd:
                shim.shim_ift_dpnp_kabsch(_p(np.ascontiguousarray(c3[idx[:3]])), _p(np.ascontiguousarray(ey[idx[:3]])), _p(out))
            else:
                shim.shim_ift_dpnp_p3p(_p(np.ascontiguousarray(fwd.hyp_pose[f, h])), _p(np.ascontiguousarray(c3[idx[:3]])),
                                       _p(np.ascontiguousarray(pix[f].reshape(N, 2)[idx[:3]].astype(np.float64))),
                                       C.c_double(cam[0]), C.c_double(cam[1]), C.c_double(cam[2]), _p(out))
            assert np.abs(bw.dpnp[f, h].reshape(72) - out).max() <= 1e-9 * max(1e-300, np.abs(out).max()), (f, h)
    # the DSAC variant on the same settings: deterministic, finite, 18 jobs per selected hypothesis
    eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    eng.set_coord_derivatives("implicit")
    d1, d2 = eng.backward_dsac(nf), eng.backward_dsac(nf)
    for k, v in _bw_fields(d1).items():
        assert np.array_equal(v, getattr(d2, k)), k
    assert np.array_equal(d1.n_refine_jobs, 18 * d1.n_selected)
    assert np.isfinite(d1.dloss_dobj).all() and np.abs(d1.path1).max() > 0
    del keep


def test_autograd_pose_outputs_with_derivatives(engine_mod):
    import torch
    from dsac_b200 import autograd as A
    E = engine_mod
    nf = 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    pred = torch.from_numpy(coords.astype(np.float32) / np.float32(1000)).cuda().requires_grad_()
    pix_t = torch.from_numpy(np.ascontiguousarray(pix)).cuda()
    res = {}
    for mode in ("implicit", "central"):
        eng = E.Engine(max_frames=nf, n_hyps=64)
        pred.grad = None
        A.softam_pose(eng, pred, pix_t, derivatives=mode).sum().backward()
        g1 = pred.grad.clone()
        pred.grad = None
        sf, ref = A.dsac_hypotheses(eng, pred, pix_t, derivatives=mode)
        (ref.sum() + sf.sum()).backward()
        res[mode] = (g1, pred.grad.clone())
    for a, b in zip(res["implicit"], res["central"]):
        assert torch.isfinite(a).all() and not torch.equal(a, b)
