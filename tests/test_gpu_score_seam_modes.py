"""The score seam (dsac_set_score_hook + dsac_set_score_backward_hook) with scores that differ from the engine's own, in
every mode the engine has: both pipelines, RGB-D, guided sampling, per-frame cameras and implicit derivatives.

1. A scorer with a float64 reference.  The forward hook writes alpha' sum_i sigmoid(beta' (thr2d - d_hi)) in float64 from
   the device's fp32 error matrix, with alpha' = 0.3 and beta' = 1.5, while the engine keeps its defaults (alpha 0.1,
   beta 0.5); the backward hook writes its analytic adjoint -alpha' beta' s (1 - s) g.  So the oracle run with alpha = 0.3,
   beta = 1.5 is a float64 reference for the whole hooked pass, and an engine that ignored what the hook wrote, read it
   at the wrong frame, or dropped the hook's adjoint, is off by a factor, not by rounding.
2. Scores only an external scorer produces: +-1e3, exact ties, one score 700 above the rest, sf on both sides of the DSAC
   variant's 1e-4 selection threshold; and the backward's linearity in the hook's adjoint.
3. Plumbing: every frame scored exactly once by the hook (800 frames, host chunks), errors from inside the backward, and
   the misuse errors of the DSAC variant's backward.

Tolerances (test_gpu_params.py's with beta' in place of beta; de = the frame's largest difference between the error
matrix the hook saw and the oracle's float64 reprojection errors at the engine's hypothesis poses):
  scores ................................. (1e-5 + beta' de) max|score| (the hook sums in fp64: no 2^-25 floor)
  sf ..................................... max(1e-4, 2 ds), ds the frame's largest score difference
  soft-argmax pose ....................... 1e-3 + sum_h |d sf_h| |pose_h|
  refined pose ........................... 1e-6 rad, 1e-3 mm
  gradients through the hook's adjoint ... 5 beta' de of max (the adjoint sees the fp32 errors, the engine's closed form
                                           the exact ones: |d(s (1 - s))/de| <= beta' s (1 - s); test_gpu_configs.py's
                                           5e-3 at beta = 0.5, de = 2e-3), plus 1e-3 where the fp32-score error of the
                                           forward also enters (soft-argmax dLoss/dObj, test_gpu_params.py's band)
  fp64 factors (dpnp, path I, DSAC score gradients fed the engine's sf) as in test_gpu_params.py

Run with -s to see the measured maxima per case."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import guided_oracle as G
import rgbd_oracle as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600
A1, B1, THR = 0.3, 1.5, 10.0            # the hooked scorer's alpha', beta' and the engine's default thr2d


class _W:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}


def _stream(s):
    return torch.cuda.ExternalStream(s) if s else torch.cuda.default_stream()


def _rel(a, b, floor=1e-300):
    return float(np.abs(a - b).max() / max(floor, np.abs(b).max()))


def _score_np(dm):
    """The scorer in float64 numpy, [.., H, N] fp32 errors -> [.., H]."""
    return A1 * (1.0 / (1.0 + np.exp(-B1 * (THR - dm.astype(np.float64))))).sum(-1)


class Scorer:
    """The hooked scorer.  Frames are scored one at a time (the same torch reduction whatever the batch), on the stream
    the engine passes.  fixed: [n][H] scores to write instead (part 2); scale: c of the backward hook's c * adjoint;
    keep: host copies of the error matrices the hook saw, by frame; fail_backward: the backward hook returns 1."""

    def __init__(self, eng, keep=True, fixed=None, scale=1.0):
        self.eng, self.keep, self.fixed, self.scale = eng, keep, fixed, scale
        self.calls, self.seen, self.written, self.fail_backward = [], {}, {}, False
        eng.set_score_hook(self.forward)
        eng.set_score_backward_hook(self.backward)

    def _frame0(self, dm, sc, n, H):
        v = self.eng.device_view()
        f_dm, r_dm = divmod(dm - v.diffmaps, H * N * 4)
        f_sc, r_sc = divmod(sc - v.scores, H * 8)
        self.calls.append((n, H, f_dm, f_sc))
        assert r_dm == 0 and r_sc == 0 and f_dm == f_sc, (f_dm, f_sc)
        return f_dm

    def forward(self, dm, n, H, sc, stream):
        try:
            return self._forward(dm, n, H, sc, stream)
        except Exception as ex:   # an exception cannot cross the C callback: the engine sees the nonzero return and raises
            print("score hook:", repr(ex))
            return 1

    def _forward(self, dm, n, H, sc, stream):
        f0 = self._frame0(dm, sc, n, H)
        with torch.cuda.stream(_stream(stream)):
            d = torch.as_tensor(_W(dm, (n, H, N), "<f4"), device="cuda")
            s = torch.as_tensor(_W(sc, (n, H), "<f8"), device="cuda")
            if self.fixed is not None:
                s.copy_(torch.from_numpy(np.ascontiguousarray(self.fixed[f0:f0 + n])).cuda())
            else:
                for f in range(n):
                    s[f].copy_(A1 * torch.sigmoid(B1 * (THR - d[f].double())).sum(1))
            if self.keep:
                dh, sh = d.cpu().numpy(), s.cpu().numpy()
                for f in range(n):
                    self.seen[f0 + f], self.written[f0 + f] = dh[f].copy(), sh[f].copy()
        return 0

    def backward(self, dm, sg, n, H, out, stream):
        if self.fail_backward:
            return 1
        with torch.cuda.stream(_stream(stream)):
            d = torch.as_tensor(_W(dm, (n, H, N), "<f4"), device="cuda")
            g = torch.as_tensor(_W(sg, (n, H), "<f8"), device="cuda")
            o = torch.as_tensor(_W(out, (n, H, N), "<f8"), device="cuda")
            for f in range(n):
                s = torch.sigmoid(B1 * (THR - d[f].double()))
                o[f].copy_(g[f][:, None] * (-A1 * B1 * self.scale) * s * (1 - s))
        return 0

    def frames_scored(self):
        covered = sorted(f for n, H, f0, _ in self.calls for f in range(f0, f0 + n))
        return covered


def _hooked(E, **kw):
    eng = E.Engine(**kw)
    return eng, Scorer(eng)


def _cfg(O, H, T=1, seed=1305, cam=(525.0, 320.0, 240.0), **kw):
    return O.default_config(seed=seed, n_hyps=H, n_streams=T, alpha=A1, beta=B1, f=cam[0], cx=cam[1], cy=cam[2], **kw)


def _exact_dm(O, coords, pix, hyp_pose, cam=(525.0, 320.0, 240.0)):
    """The oracle's reprojection errors [H][N] at the given hypothesis poses."""
    return np.stack([O.diff_map(coords, pix, p[:3], p[3:], *cam) for p in hyp_pose])


def _gt6(O, gt_jp):
    return np.concatenate([O.rodrigues_inv(gt_jp[:9]), gt_jp[9:]])


def _score_tol(de, smax):
    return (1e-5 + B1 * de) * smax


class Maxima(dict):
    def put(self, k, v):
        self[k] = max(self.get(k, 0.0), float(v))

    def show(self, name):
        print("%-24s maxima:" % name, " ".join("%s %.3g" % kv for kv in sorted(self.items())))


def _check_softam_forward(O, name, res, sc, ora, coords, pix, frames, mx, cams=None):
    """Hooked soft-argmax forward against the oracle's forward (one per frame in `frames`); returns de per frame."""
    de_all = {}
    for f, o in zip(frames, ora):
        cam = cams[f] if cams is not None else (525.0, 320.0, 240.0)
        assert np.array_equal(o.img_idx, res.img_idx[f]), (name, f)
        # what the engine kept is what the hook wrote, and what the hook wrote is the scorer of what it saw
        assert np.array_equal(res.scores[f], sc.written[f]), (name, f)
        assert _rel(sc.written[f], _score_np(sc.seen[f])) <= 1e-12, (name, f)
        de = float(np.abs(sc.seen[f] - _exact_dm(O, coords[f], pix[f], res.hyp_pose[f], cam)).max())
        de_all[f] = de
        mx.put("de", de)
        smax = np.abs(o.scores).max()
        ds = float(np.abs(o.scores - res.scores[f]).max())
        mx.put("score/tol", ds / _score_tol(de, smax))
        assert ds <= _score_tol(de, smax), (name, f, ds, de)
        assert np.abs(O.softmax(res.scores[f]) - res.sf[f]).max() <= 1e-12
        dsf = np.abs(o.sf - res.sf[f])
        mx.put("sf", dsf.max())
        assert dsf.max() <= max(1e-4, 2 * ds), (name, f, dsf.max(), ds)
        davg = np.abs(o.avg - res.avg_pose[f]).max()
        mx.put("avg", davg)
        assert davg <= 1e-3 + (dsf[:, None] * np.abs(res.hyp_pose[f])).sum(0).max(), (name, f, davg)
        mx.put("ref_r", np.abs(o.ref[:3] - res.ref_pose[f][:3]).max())
        mx.put("ref_t", np.abs(o.ref[3:] - res.ref_pose[f][3:]).max())
        assert np.abs(o.ref[:3] - res.ref_pose[f][:3]).max() <= 1e-6 and np.abs(o.ref[3:] - res.ref_pose[f][3:]).max() <= 1e-3, (name, f)
    return de_all


def _check_softam_backward(O, name, bw, obws, gt_jp, fwd, frames, de, mx):
    for f, obw in zip(frames, obws):
        want_dref = O.dloss_max(O.jp6(fwd.ref_pose[f][:3], fwd.ref_pose[f][3:]), _gt6(O, gt_jp[f]))
        m = dict(dloss_dref=_rel(bw.dloss_dref[f], want_dref), dpnp=_rel(bw.dpnp[f], obw.dpnp),
                 score_grads=_rel(bw.score_grads[f], obw.score_grads, floor=1e-6),
                 dloss_dobj=_rel(bw.dloss_dobj[f], obw.dloss_dobj, floor=1e-6))
        for k, v in m.items():
            mx.put(k, v)
        tol = 1e-3 + 5 * B1 * de[f]
        mx.put("dloss_dobj/tol", m["dloss_dobj"] / tol)
        assert m["dloss_dref"] <= 1e-9 and m["dpnp"] <= 1e-7, (name, f, m)
        assert m["score_grads"] <= 1e-4, (name, f, m)
        assert m["dloss_dobj"] <= tol, (name, f, m, tol)
        assert np.abs(bw.dloss_dobj[f]).max() > 0


def _dsac_state(O, cfg, fw, f):
    """The oracle's DSAC forward record filled with the ENGINE's forward state (test_gpu_params.py)."""
    ofw = O.ForwardDsac(cfg)
    ofw.hyp_rvec[:] = fw.hyp_pose[f][:, :3]; ofw.hyp_tvec[:] = fw.hyp_pose[f][:, 3:]
    ofw.img_idx[:] = fw.img_idx[f]; ofw.sf[:] = fw.sf[f]; ofw.ref_pose[:] = fw.ref_pose[f]; ofw.losses[:] = fw.losses[f]
    return ofw


def _check_dsac_forward(O, name, res, sc, ora, coords, pix, frames, mx, cams=None):
    for f, o in zip(frames, ora):
        cam = cams[f] if cams is not None else (525.0, 320.0, 240.0)
        assert np.array_equal(o.img_idx, res.img_idx[f]) and o.hyp_idx == res.hyp_idx[f], (name, f, o.hyp_idx, res.hyp_idx[f])
        assert _rel(sc.written[f], _score_np(sc.seen[f])) <= 1e-12
        assert np.abs(O.softmax(sc.written[f]) - res.sf[f]).max() <= 1e-12, (name, f)   # the softmax of the hook's scores
        exact = _exact_dm(O, coords[f], pix[f], res.hyp_pose[f], cam)
        de = float(np.abs(sc.seen[f] - exact).max())
        o_scores = np.array([O.soft_inlier_score(row, THR, A1, B1) for row in exact])
        ds = float(np.abs(o_scores - sc.written[f]).max())
        mx.put("de", de)
        mx.put("score/tol", ds / _score_tol(de, np.abs(o_scores).max()))
        assert ds <= _score_tol(de, np.abs(o_scores).max()), (name, f, ds, de)
        mx.put("sf", np.abs(o.sf - res.sf[f]).max())
        assert np.abs(o.sf - res.sf[f]).max() <= max(1e-4, 2 * ds), (name, f)
        assert np.abs(o.ref_pose[:, :3] - res.ref_pose[f][:, :3]).max() <= 1e-8
        assert np.abs(o.ref_pose[:, 3:] - res.ref_pose[f][:, 3:]).max() <= 1e-5
        assert np.abs(o.losses - res.losses[f]).max() <= 1e-6 * max(1.0, np.abs(o.losses).max())
        mx.put("expected_loss", abs(o.expected_loss - res.expected_loss[f]) / max(1.0, abs(o.expected_loss)))
        assert abs(o.expected_loss - res.expected_loss[f]) <= 1e-3 * max(1.0, abs(o.expected_loss)), (name, f)


def _check_dsac_backward(O, name, bw, orb, sc, fw, coords, pix, frames, mx, cams=None):
    for f, obw in zip(frames, orb):
        cam = cams[f] if cams is not None else (525.0, 320.0, 240.0)
        de = float(np.abs(sc.seen[f] - _exact_dm(O, coords[f], pix[f], fw.hyp_pose[f], cam)).max())
        assert obw.n_selected == bw.n_selected[f] and obw.n_selected >= 1, (name, f)
        assert obw.n_refine_jobs == bw.n_refine_jobs[f], (name, f)
        m = dict(score_grads=_rel(bw.score_grads[f], obw.score_grads, floor=1e-12), path1=_rel(bw.path1[f], obw.path1),
                 path2=_rel(bw.path2[f], obw.path2), dloss_dobj=_rel(bw.dloss_dobj[f], obw.dloss_dobj))
        for k, v in m.items():
            mx.put(k, v)
        tol = 1e-6 + 5 * B1 * de
        mx.put("path2/tol", m["path2"] / tol)
        assert m["score_grads"] <= 1e-9 and m["path1"] <= 1e-5, (name, f, m)
        assert m["path2"] <= tol and m["dloss_dobj"] <= tol, (name, f, m, tol)
        assert np.abs(obw.path2).max() > 0


# ------------------------------------------------------------------------------------------------ 1(a) soft-argmax
@pytest.mark.parametrize("H,T,tile,nf", [(1, 1, 0, 2), (37, 1, 0, 2), (64, 1, 0, 2), (64, 3, 8, 3)],
                         ids=["H1", "H37", "H64", "H64_T3_tile8"])
def test_softam_hooked_matches_oracle(engine_mod, oracle, H, T, tile, nf):
    E, O = engine_mod, oracle
    coords, pix, _, gt_jp = E.synth_frames(nf, n_streams=T)
    eng, sc = _hooked(E, max_frames=nf, n_hyps=H, n_streams=T, hyps_per_cta=tile)
    res = eng.forward(coords, pix, gt_jp)
    bw = eng.backward(coords, pix, gt_jp)
    eng.close()
    assert sc.frames_scored() == list(range(nf))
    ora, orb = [], []
    for f in range(nf):
        cfg = _cfg(O, H, T, seed=1305 + f * T)
        ofw = O.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
        ora.append(ofw)
        orb.append(O.backward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw))
    mx = Maxima()
    de = _check_softam_forward(O, "softam H%d" % H, res, sc, ora, coords, pix, range(nf), mx)
    _check_softam_backward(O, "softam H%d" % H, bw, orb, gt_jp, res, range(nf), de, mx)
    mx.show("softam H%d T%d tile%d" % (H, T, tile))


# ------------------------------------------------------------------------------------------------ 1(b) DSAC variant
@pytest.mark.parametrize("random_draw", [0, 1])
def test_dsac_hooked_matches_oracle(engine_mod, oracle, random_draw):
    E, O = engine_mod, oracle
    nf, H = 2, 32
    coords, pix, _, gt_jp = E.synth_frames(nf)
    eng, sc = _hooked(E, max_frames=nf, n_hyps=H)
    res = eng.forward_dsac(coords, pix, gt_jp, random_draw=bool(random_draw))
    ora = [O.forward_dsac(_cfg(O, H, seed=1305 + f), coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], bool(random_draw))
           for f in range(nf)]
    mx = Maxima()
    _check_dsac_forward(O, "dsac", res, sc, ora, coords, pix, range(nf), mx)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    bw = eng.backward_dsac(nf)
    eng.close()
    orb = [O.backward_dsac(_cfg(O, H, seed=1305 + f), coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:],
                           _dsac_state(O, _cfg(O, H, seed=1305 + f), fw, f)) for f in range(nf)]
    _check_dsac_backward(O, "dsac", bw, orb, sc, fw, coords, pix, range(nf), mx)
    mx.show("dsac draw=%d" % random_draw)


# ------------------------------------------------------------------------------------------------ 1(c) RGB-D
def _set_depth(eng, depth):
    d = torch.from_numpy(np.ascontiguousarray(depth, np.float32)).cuda()
    eng.set_cell_depth_device(len(depth), d.data_ptr())
    torch.cuda.synchronize()
    return d


def test_rgbd_hooked_matches_oracle(engine_mod, oracle):
    """Depth holes everywhere; frame 2 has 3 cells with depth (DSAC_ST_NO_DEPTH) in the forward passes.  The backward
    passes run over the frames with depth."""
    E, O = engine_mod, oracle
    n, H = 3, 32
    coords, pix, depth, _, gt_jp = R.synth(n, seed=83, holes=0.1)
    depth[2, 3:] = np.nan
    mx = Maxima()
    eng, sc = _hooked(E, max_frames=n, n_hyps=H)
    d = _set_depth(eng, depth)
    res = eng.forward(coords, pix, gt_jp)
    assert res.status[2] & E.ST_NO_DEPTH and not res.status[0] & E.ST_NO_DEPTH and not res.status[1] & E.ST_NO_DEPTH
    eyes = [R.eye(pix[f], depth[f])[0] for f in range(2)]
    ora = [R.forward(O, _cfg(O, H), f, coords[f], pix[f], eyes[f], None, gt_jp[f, :9], gt_jp[f, 9:])[0] for f in range(2)]
    ok = [f for f in range(2) if ora[f].n_fragile == 0]     # the oracle's fragile frames are skipped (test_gpu_rgbd.py)
    assert ok
    _check_softam_forward(O, "rgbd", res, sc, [ora[f] for f in ok], coords, pix, ok, mx)
    dres = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    assert dres.status[2] & E.ST_NO_DEPTH
    dora = [R.forward_dsac(O, _cfg(O, H), f, coords[f], pix[f], eyes[f], gt_jp[f, :9], gt_jp[f, 9:], True) for f in range(2)]
    _check_dsac_forward(O, "rgbd dsac", dres, sc, dora, coords, pix, range(2), mx)
    eng.close()
    del d

    eng, sc = _hooked(E, max_frames=2, n_hyps=H)
    d = _set_depth(eng, depth[:2])
    res = eng.forward(coords[:2], pix[:2], gt_jp[:2])
    bw = eng.backward(coords[:2], pix[:2], gt_jp[:2])
    orb = [R.backward(O, _cfg(O, H), coords[f], pix[f], eyes[f], gt_jp[f, :9], gt_jp[f, 9:], ora[f]) for f in ok]
    de = _check_softam_forward(O, "rgbd", res, sc, [ora[f] for f in ok], coords, pix, ok, mx)
    _check_softam_backward(O, "rgbd", bw, orb, gt_jp, res, ok, de, mx)
    fw = eng.forward_dsac(coords[:2], pix[:2], gt_jp[:2], random_draw=False)
    bwd = eng.backward_dsac(2)
    orbd = [R.backward_dsac(O, _cfg(O, H), coords[f], pix[f], eyes[f], gt_jp[f, :9], gt_jp[f, 9:], _dsac_state(O, _cfg(O, H), fw, f))
            for f in range(2)]
    _check_dsac_backward(O, "rgbd dsac", bwd, orbd, sc, fw, coords, pix, range(2), mx)
    eng.close()
    del d
    mx.show("rgbd")


# ------------------------------------------------------------------------------------------------ 1(d) guided sampling
def test_guided_hooked_matches_oracle(engine_mod, oracle):
    E, O = engine_mod, oracle
    n, H = 2, 32
    coords, pix, _, gt_jp = E.synth_frames(n)
    logits = np.random.default_rng(8).standard_normal((n, N)).astype(np.float32)
    eng, sc = _hooked(E, max_frames=n, n_hyps=H)
    dl = torch.from_numpy(logits).cuda()
    eng.set_sampling_logits_device(n, dl.data_ptr())
    torch.cuda.synchronize()
    cums = [G.table(logits[f])[2] for f in range(n)]
    mx = Maxima()
    res = eng.forward(coords, pix, gt_jp)
    bw = eng.backward(coords, pix, gt_jp)
    ora = [G.forward(O, _cfg(O, H), cums[f], f, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])[0] for f in range(n)]
    orb = [O.backward(_cfg(O, H), coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ora[f]) for f in range(n)]
    de = _check_softam_forward(O, "guided", res, sc, ora, coords, pix, range(n), mx)
    _check_softam_backward(O, "guided", bw, orb, gt_jp, res, range(n), de, mx)
    dres = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    dora = [G.forward_dsac(O, _cfg(O, H), cums[f], f, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], True) for f in range(n)]
    _check_dsac_forward(O, "guided dsac", dres, sc, dora, coords, pix, range(n), mx)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    bwd = eng.backward_dsac(n)
    orbd = [O.backward_dsac(_cfg(O, H), coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], _dsac_state(O, _cfg(O, H), fw, f))
            for f in range(n)]
    _check_dsac_backward(O, "guided dsac", bwd, orbd, sc, fw, coords, pix, range(n), mx)
    eng.close()
    del dl
    mx.show("guided")


# ------------------------------------------------------------------------------------------------ 1(e) mixed cameras
CAMS = [(525.0, 320.0, 240.0), (585.0, 324.5, 236.25), (1800.0, 511.5, 400.0)]
FWD = ("img_idx", "cand_idx", "n_candidates", "hyp_pose", "scores", "sf", "avg_pose", "ref_pose", "inlier_map", "loss",
       "status", "diffmaps")
BWD = ("dloss_dobj", "dloss_dref", "dref_dhyp", "score_grads", "dpnp")
DSAC_FWD = ("hyp_pose", "img_idx", "sf", "entropy", "ref_pose", "losses", "steps_done", "expected_loss", "hyp_idx",
            "rot_err", "t_err", "correct", "status")
DSAC_BWD = ("dloss_dobj", "path1", "path2", "score_grads", "n_selected", "n_refine_jobs")


def _close(got, g, want, names):
    """Frame g of a batch backward against a one-frame backward: k_dscore splits a frame's sum over a number of CTAs that
    depends on the batch, so to 1e-12 of max rather than bit for bit."""
    for k in names:
        a, b = getattr(got, k)[g], getattr(want, k)[0]
        assert np.abs(a - b).max() <= 1e-12 * max(1e-300, np.abs(b).max()), (k, g)


def test_mixed_cameras_hooked_equal_per_camera_engines(engine_mod):
    E = engine_mod
    nf, H = 3, 64
    cam = np.array(CAMS, np.float64)
    parts = [E.synth_frames(1, frame0=g, focal=cam[g, 0], cx=cam[g, 1], cy=cam[g, 2]) for g in range(nf)]
    coords, pix, _, gt_jp = (np.concatenate([p[k] for p in parts]) for k in range(4))
    eng, sc = _hooked(E, max_frames=nf, n_hyps=H)
    eng.set_cameras(cam)
    res = eng.forward(coords, pix, gt_jp, want_diffmaps=True)
    bw = eng.backward(coords, pix, gt_jp, full=False)
    dres = eng.forward_dsac(coords, pix, gt_jp, random_draw=True)
    bwd = eng.backward_dsac(nf)
    eng.close()
    assert (res.status == 0).all()
    for g in range(nf):
        one, s1 = _hooked(E, max_frames=1, n_hyps=H, focal=cam[g, 0], cx=cam[g, 1], cy=cam[g, 2])
        sl = slice(g, g + 1)
        r1 = one.forward(coords[sl], pix[sl], gt_jp[sl], frame0=g, want_diffmaps=True)
        for k in FWD:
            assert np.array_equal(getattr(res, k)[g], getattr(r1, k)[0]), (k, g)
        assert _rel(res.scores[g], _score_np(res.diffmaps[g])) <= 1e-12
        _close(bw, g, one.backward(coords[sl], pix[sl], gt_jp[sl], full=False), ("dloss_dobj", "dloss_dref", "score_grads"))
        d1 = one.forward_dsac(coords[sl], pix[sl], gt_jp[sl], random_draw=True, frame0=g)
        for k in DSAC_FWD:
            assert np.array_equal(getattr(dres, k)[g], getattr(d1, k)[0]), (k, g)
        b1 = one.backward_dsac(1)
        assert bwd.n_selected[g] == b1.n_selected[0] and bwd.n_refine_jobs[g] == b1.n_refine_jobs[0]
        _close(bwd, g, b1, ("dloss_dobj", "path1", "path2", "score_grads"))
        one.close()


# ------------------------------------------------------------------------------------------------ 1(f) implicit derivatives
@pytest.mark.parametrize("rgbd", [False, True], ids=["rgb", "rgbd"])
def test_implicit_hooked_equals_unhooked_engine_at_the_scorers_parameters(engine_mod, oracle, rgbd):
    """The hooked implicit backward against the unhooked implicit backward of an engine built with alpha', beta'."""
    E, O = engine_mod, oracle
    n, H = 2, 32
    if rgbd:
        coords, pix, depth, _, gt_jp = R.synth(n, seed=87, holes=0.1)
    else:
        coords, pix, _, gt_jp = E.synth_frames(n)
    eng, sc = _hooked(E, max_frames=n, n_hyps=H)
    ref = E.Engine(max_frames=n, n_hyps=H, alpha=A1, beta=B1)
    keep = [_set_depth(e, depth) for e in (eng, ref)] if rgbd else []
    for e in (eng, ref):
        e.set_coord_derivatives("implicit")
    mx = Maxima()
    got_f, want_f = eng.forward(coords, pix, gt_jp), ref.forward(coords, pix, gt_jp)
    got, want = eng.backward(coords, pix, gt_jp), ref.backward(coords, pix, gt_jp)
    for f in range(n):
        assert np.array_equal(got_f.img_idx[f], want_f.img_idx[f]) and np.array_equal(got_f.hyp_pose[f], want_f.hyp_pose[f])
        de = float(np.abs(sc.seen[f] - _exact_dm(O, coords[f], pix[f], got_f.hyp_pose[f])).max())
        mx.put("de", de)
        assert np.array_equal(got.dpnp[f], want.dpnp[f]), f                 # the sampled hypotheses alone
        tol = 1e-3 + 5 * B1 * de
        m = dict(score_grads=_rel(got.score_grads[f], want.score_grads[f], floor=1e-6),
                 dref_dobj=_rel(got.dref_dobj[f], want.dref_dobj[f], floor=1e-3),
                 dloss_dobj=_rel(got.dloss_dobj[f], want.dloss_dobj[f], floor=1e-6))
        for k, v in m.items():
            mx.put(k, v)
        assert m["score_grads"] <= 1e-4 and m["dref_dobj"] <= tol and m["dloss_dobj"] <= tol, (f, m, tol)
        assert np.abs(got.dloss_dobj[f]).max() > 0
    got_d = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    want_d = ref.forward_dsac(coords, pix, gt_jp, random_draw=False)
    gb, wb = eng.backward_dsac(n), ref.backward_dsac(n)
    for f in range(n):
        de = float(np.abs(sc.seen[f] - _exact_dm(O, coords[f], pix[f], got_d.hyp_pose[f])).max())
        assert np.abs(got_d.sf[f] - want_d.sf[f]).max() <= 1e-4
        assert gb.n_selected[f] == wb.n_selected[f] and gb.n_refine_jobs[f] == wb.n_refine_jobs[f], f
        tol = 1e-3 + 5 * B1 * de
        # path II against the frame's whole dLoss/dObj: in an RGB-D pass it is a small part of it, and the hook's share,
        # dScore/dHyp summed over 1600 cells at a hypothesis close to the score's optimum, cancels to a small vector whose
        # relative error is far above that of its terms (22 % of path II's own max, 6e-16 of dLoss/dObj, measured on an H100)
        scale = np.abs(wb.dloss_dobj[f]).max()
        m = dict(dsac_path1=_rel(gb.path1[f], wb.path1[f]), dsac_path2=np.abs(gb.path2[f] - wb.path2[f]).max() / scale,
                 dsac_dloss_dobj=_rel(gb.dloss_dobj[f], wb.dloss_dobj[f]))
        for k, v in m.items():
            mx.put(k, v)
        assert m["dsac_path1"] <= 1e-3 and m["dsac_path2"] <= tol and m["dsac_dloss_dobj"] <= tol, (f, m, tol)
        assert np.abs(gb.path2[f]).max() > 0
    eng.close()
    ref.close()
    del keep
    mx.show("implicit %s" % ("rgbd" if rgbd else "rgb"))


# ------------------------------------------------------------------------------------------------ 1(g) seeded pose backward
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_seeded_pose_backward_under_hooks_equals_the_loss_backward(engine_mod, oracle):
    """Soft-argmax: dsac_backward_pose_device seeded with dLoss/dRef = the hooked loss backward, bit for bit.  DSAC variant:
    dsac_backward_dsac_pose_device (what dsac_hypotheses' autograd calls) with the expected-loss seeds sf_h dLossMax_h and
    dOuter/dsf = the losses = dsac_backward_dsac: the same selection, jobs and score gradients, dLoss/dObj to 1e-12."""
    E, O = engine_mod, oracle
    nf, H = 3, 48
    coords, pix, _, gt_jp = E.synth_frames(nf, frame0=2)
    a, _ = _hooked(E, max_frames=nf, n_hyps=H)
    a.forward(coords, pix, gt_jp, frame0=2)
    bw = a.backward(coords, pix, gt_jp, full=False)
    a.close()
    b, _ = _hooked(E, max_frames=nf, n_hyps=H)
    st = torch.cuda.current_stream().cuda_stream
    dc, dp = _dev(coords), _dev(pix)
    b.forward_device(nf, dc.data_ptr(), dp.data_ptr(), 0, None, 2, st)
    dobj = torch.full((nf, N, 3), np.nan, dtype=torch.float64, device="cuda")
    seed = _dev(bw.dloss_dref)
    b.backward_pose_device(nf, seed.data_ptr(), dobj.data_ptr(), None, 0.0, st)
    torch.cuda.synchronize()
    assert np.array_equal(dobj.cpu().numpy(), bw.dloss_dobj) and np.abs(bw.dloss_dobj).max() > 0

    b.close()
    nf, H = 4, 48
    coords, pix, _, gt_jp = E.synth_frames(nf, frame0=3)
    b, _ = _hooked(E, max_frames=nf, n_hyps=H)
    fw = b.forward_dsac(coords, pix, gt_jp, random_draw=True, frame0=3)
    bwd = b.backward_dsac(nf)
    ref6 = torch.full((nf, H, 6), np.nan, dtype=torch.float64, device="cuda")
    b.refined_jp6_device(nf, ref6.data_ptr(), st)
    torch.cuda.synchronize()
    ref6 = ref6.cpu().numpy()
    seeds = np.stack([[fw.sf[f, h] * O.dloss_max(ref6[f, h], _gt6(O, gt_jp[f])) for h in range(H)] for f in range(nf)])
    outs = {"dloss_dobj": torch.full((nf, N, 3), np.nan, dtype=torch.float64, device="cuda"),
            "score_grads": torch.full((nf, H), np.nan, dtype=torch.float64, device="cuda"),
            "n_selected": torch.full((nf,), -1, dtype=torch.int32, device="cuda"),
            "n_refine_jobs": torch.full((nf,), -1, dtype=torch.int32, device="cuda")}
    assert np.isfinite(seeds).all() and np.isfinite(bwd.dloss_dobj).all()
    ds, dg = _dev(seeds), _dev(fw.losses)
    b.backward_dsac_pose_device(nf, ds.data_ptr(), dg.data_ptr(), None, 0.0, st, **{k: v.data_ptr() for k, v in outs.items()})
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in outs.items()}
    b.close()
    assert np.array_equal(got["n_selected"], bwd.n_selected) and bwd.n_selected.min() >= 1
    assert np.array_equal(got["n_refine_jobs"], bwd.n_refine_jobs)
    assert np.array_equal(got["score_grads"], bwd.score_grads)
    assert np.abs(got["dloss_dobj"] - bwd.dloss_dobj).max() <= 1e-12 * np.abs(bwd.dloss_dobj).max()


# ------------------------------------------------------------------------------------------------ 2. scores only a scorer writes
@pytest.fixture(scope="module")
def draw_shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("draw_shim") / "libdraw_shim.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "host_shim", "draw_shim.cpp")])
    return C.CDLL(so)


def _threshold_scores(H):
    """log-probabilities: 6 hypotheses at sf = 1e-4 (1 + 1e-9), 6 at 1e-4 (1 - 1e-9), the rest share what is left."""
    p = np.empty(H)
    p[:6], p[6:12] = 1e-4 * (1 + 1e-9), 1e-4 * (1 - 1e-9)
    p[12:] = (1.0 - p[:12].sum()) / (H - 12)
    return np.log(p)


def _fixed_scores(kind, nf, H):
    rng = np.random.default_rng(["uniform", "equal", "spike", "threshold"].index(kind) + 17)
    if kind == "uniform":
        return rng.uniform(-1e3, 1e3, (nf, H))
    if kind == "equal":
        return np.full((nf, H), 5.0)
    if kind == "spike":
        s = rng.normal(0, 3, (nf, H))
        s[np.arange(nf), rng.integers(0, H, nf)] = s.max(1) + 700.0
        return s
    return np.stack([np.roll(_threshold_scores(H), 5 * f) for f in range(nf)])


@pytest.mark.parametrize("kind", ["uniform", "equal", "spike", "threshold"])
def test_scores_only_an_external_scorer_writes(engine_mod, oracle, draw_shim, kind):
    E, O = engine_mod, oracle
    nf, H = 2, 64
    coords, pix, _, gt_jp = E.synth_frames(nf)
    scores = _fixed_scores(kind, nf, H)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    sc = Scorer(eng, fixed=scores)
    res = eng.forward(coords, pix, gt_jp)
    perm = O.refine_permutations(eng.cfg.ref_steps)
    for f in range(nf):
        assert np.array_equal(res.scores[f], scores[f])
        sf = O.softmax(scores[f])
        assert np.abs(res.sf[f] - sf).max() <= 1e-12 * max(1.0, sf.max()), (kind, f)
        assert abs(res.entropy[f] - O.entropy(sf)) <= 1e-10 * max(1.0, O.entropy(sf)), (kind, f)
        avg = (sf[:, None] * res.hyp_pose[f]).sum(0)
        assert np.abs(res.avg_pose[f] - avg).max() <= 1e-9 * max(1.0, np.abs(avg).max()), (kind, f)
        cfg = O.default_config(seed=1305 + f, n_hyps=H)
        rep = O.refine(cfg, perm, eng.cfg.ref_steps, coords[f], pix[f], res.avg_pose[f])
        got = O.jp6(res.ref_pose[f][:3], res.ref_pose[f][3:])
        assert np.abs(rep[:3] - got[:3]).max() <= 1e-8 and np.abs(rep[3:] - got[3:]).max() <= 1e-5, (kind, f, rep, got)
        if kind == "equal":
            assert np.all(res.sf[f] == 1.0 / H) or np.abs(res.sf[f] - 1.0 / H).max() <= 1e-15
        if kind == "threshold":
            assert (res.sf[f] > 1e-4).sum() == H - 6 and (sf > 1e-4).sum() == H - 6
    # the DSAC variant: the draw from the same sf, and the backward's selection sf > 1e-4
    for random_draw in (1, 0):
        fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=bool(random_draw))
        bw = eng.backward_dsac(nf)
        for f in range(nf):
            sf = O.softmax(scores[f])
            assert np.abs(fw.sf[f] - sf).max() <= 1e-12 * max(1.0, sf.max())
            o = O.forward_dsac(O.default_config(seed=1305 + f, n_hyps=H), coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], bool(random_draw))
            assert np.array_equal(o.img_idx, fw.img_idx[f])
            pp, ps = np.zeros(1, np.int32), np.zeros(1, np.int32)
            w = np.zeros(2, np.uint32), np.zeros(2, np.uint32)
            seeds, endpos = np.array([1305 + f], np.uint32), np.array([o.stream0_endpos], np.uint64)
            sfa = np.ascontiguousarray(fw.sf[f])
            draw_shim.shim_draw_cases(1, H, sfa.ctypes.data_as(C.c_void_p), seeds.ctypes.data_as(C.c_void_p),
                                      endpos.ctypes.data_as(C.c_void_p), random_draw, pp.ctypes.data_as(C.c_void_p),
                                      ps.ctypes.data_as(C.c_void_p), w[0].ctypes.data_as(C.c_void_p), w[1].ctypes.data_as(C.c_void_p))
            assert fw.hyp_idx[f] == ps[0], (kind, random_draw, f, fw.hyp_idx[f], ps[0])
            assert bw.n_selected[f] == int((fw.sf[f] > 1e-4).sum()) == int((sf > 1e-4).sum()), (kind, f)
    eng.close()
    assert sc.frames_scored() == [0, 0, 0, 1, 1, 1]   # one soft-argmax and two DSAC-variant forwards


@pytest.mark.parametrize("pipeline", ["softam", "dsac"])
def test_backward_is_linear_in_the_hooks_adjoint(engine_mod, pipeline):
    """c * adjoint for c in {0, 1, 2}: path II doubles (to 1e-12 relative), path I and the score gradients (upstream of
    the hook) are bit-identical."""
    E = engine_mod
    nf, H = 2, 48
    coords, pix, _, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    sc = Scorer(eng, keep=False)
    out = {}
    for c in (0.0, 1.0, 2.0):
        sc.scale = c
        if pipeline == "softam":
            eng.forward(coords, pix, gt_jp)
            out[c] = eng.backward(coords, pix, gt_jp, full=False)
        else:
            eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
            out[c] = eng.backward_dsac(nf)
    eng.close()
    assert np.array_equal(out[1.0].score_grads, out[2.0].score_grads) and np.array_equal(out[0.0].score_grads, out[1.0].score_grads)
    if pipeline == "softam":
        p1 = out[0.0].dloss_dobj
        p2, p2x2 = out[1.0].dloss_dobj - p1, out[2.0].dloss_dobj - p1
    else:
        assert np.array_equal(out[1.0].path1, out[2.0].path1) and np.array_equal(out[0.0].path1, out[1.0].path1)
        assert np.abs(out[0.0].path2).max() == 0
        p2, p2x2 = out[1.0].path2, out[2.0].path2
    assert np.abs(p2).max() > 0
    # relative to the larger of the two paths: the soft-argmax path II is a difference of two sums that both hold path I
    d = np.abs(p2x2 - 2 * p2).max() / max(np.abs(2 * p2).max(), np.abs(out[0.0].path1 if pipeline == "dsac" else p1).max())
    print("linearity %s: %.3g" % (pipeline, d))
    assert d <= 1e-12


# ------------------------------------------------------------------------------------------------ 3. plumbing
@pytest.mark.parametrize("chunks", [None, "3"], ids=["one_pass", "host_chunks"])
def test_hook_scores_every_frame_once(engine_mod, monkeypatch, chunks):
    """800 frames: with hooks the engine runs neither the two lanes nor the tail split (engine.cu: forward_split), and the
    host path may cut the batch into chunks (DSAC_PIPE_CHUNKS).  Every frame is scored once, at its own offsets; the
    integer outputs are an unhooked engine's; the scores and sf are those of an unhooked engine at alpha', beta'."""
    E = engine_mod
    nf, H, T = 800, 16, 4
    if chunks:
        monkeypatch.setenv("DSAC_PIPE_CHUNKS", chunks)
    coords, pix, _, gt_jp = E.synth_frames(nf, n_streams=T)
    eng = E.Engine(max_frames=nf, n_hyps=H, n_streams=T)
    sc = Scorer(eng, keep=False)
    got = eng.forward(coords, pix, gt_jp)
    eng.close()
    ref = E.Engine(max_frames=nf, n_hyps=H, n_streams=T, alpha=A1, beta=B1)
    want = ref.forward(coords, pix, gt_jp)
    ref.close()
    print("hook calls (n, H, first frame):", [c[:3] for c in sc.calls])
    assert sc.frames_scored() == list(range(nf))
    if chunks:
        assert len(sc.calls) > 1
    for k in ("img_idx", "cand_idx", "n_candidates", "hyp_pose"):
        assert np.array_equal(getattr(got, k), getattr(want, k)), k
    smax = np.abs(want.scores).max(1)
    ds = np.abs(got.scores - want.scores).max(1)
    assert (ds <= A1 * N * 2.0 ** -25 + 1e-5 * smax).all(), ds.max()   # the closed form's fp32 sum against the hook's fp64 one
    assert (np.abs(got.sf - want.sf).max(1) <= np.maximum(1e-4, 2 * ds)).all()


def test_hook_error_inside_the_dsac_backward(engine_mod):
    E = engine_mod
    nf, H = 2, 32
    coords, pix, _, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    sc = Scorer(eng, keep=False)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    want = eng.backward_dsac(nf)
    sc.fail_backward = True
    with pytest.raises(RuntimeError, match="score backward hook returned 1"):
        eng.backward_dsac(nf)
    sc.fail_backward = False
    fw2 = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    got = eng.backward_dsac(nf)
    for k in ("sf", "ref_pose", "hyp_idx", "expected_loss"):
        assert np.array_equal(getattr(fw, k), getattr(fw2, k)), k
    for k in DSAC_BWD:
        assert np.array_equal(getattr(want, k), getattr(got, k)), k
    eng.close()


def test_dsac_backward_misuse(engine_mod):
    """One hook without the other is an error in the DSAC variant's backward too; a score hook needs write_diffmaps=1."""
    E = engine_mod
    nf, H = 1, 16
    coords, pix, _, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    sc = Scorer(eng, keep=False)
    eng.set_score_backward_hook(None)
    eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    with pytest.raises(RuntimeError, match="both hooks"):
        eng.backward_dsac(nf)
    eng.set_score_hook(None)
    eng.set_score_backward_hook(sc.backward)
    eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    with pytest.raises(RuntimeError, match="both hooks"):
        eng.backward_dsac(nf)
    eng.close()
    eng = E.Engine(max_frames=nf, n_hyps=H, write_diffmaps=0)
    with pytest.raises(RuntimeError, match="write_diffmaps=1"):
        eng.set_score_hook(lambda *a: 0)
    eng.set_score_backward_hook(lambda *a: 0)
    eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    with pytest.raises(RuntimeError, match="both hooks"):
        eng.backward_dsac(nf)
    eng.close()
