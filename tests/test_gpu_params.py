"""The CUDA engine against the oracle away from the default configuration: other cameras, inlier thresholds, inlier
counts, refinement steps, score parameters, hypothesis counts that are not multiples of 8 (up to DSAC_MAX_HYPS = 1024),
explicit score tiles, both backward passes, the argument limits at creation, and the reference's own outputs at
non-default parameters (tests/golden/ref_params.npz, written by tests/golden/make_ref_params.py).

Every one of these parameters reaches the kernels as a run-time value (k_score: cx, cy, thr, beta log2 e, alpha;
k_refine: f, cx, cy, thr, inlier_count, ref_steps; the sampler's filters: f, cx, cy, thr; the backward: sub_sample,
alpha, beta, grad_clamp), so a kernel that silently used a default would pass every test at the default configuration.

Tolerances, and where they come from (test_gpu_forward.py's, scaled where a parameter scales the error):
  sampled indices, candidate indices and counts, inlier maps,
  refinement steps and permutation counts, status ............. bit-exact
  hypothesis poses (fp64 P3P) ................................. 1e-9 rad, 1e-6 mm
  diffmap entries (fp32 projection) ........................... 2e-3 px x max(1, f / 525): the fp32 error of the projection
                                                                 scales with the f-scaled rows of P
  scores ...................................................... alpha N 2^-25 + (1e-5 + beta de) max|score|: the 2^-25
        floor under every sigmoid (at most alpha N 2^-25 on a score), 1e-5 relative for the fp32 sigmoid sum, and the
        frame's largest diffmap difference de through the sigmoid, |d sigma / d e| <= beta sigma (test_host_params.py)
  softmax of the engine's own scores .......................... 1e-12
  softmax against the oracle .................................. max(1e-4, 2 ds): d sf_h = sf_h (ds_h - sum_j sf_j ds_j),
                                                                 so |d sf| <= 2 max|ds| for the frame's score error ds
  soft-argmax pose ............................................ 1e-3 rad-or-mm + sum_h |d sf_h| |pose_h| (linear in sf)
  refined pose ................................................ 1e-6 rad, 1e-3 mm
  loss, rotation / translation error .......................... 1e-4, 1e-4 deg, 1e-2 mm, `correct` equal
  soft-argmax backward ........................................ test_gpu_backward.py's: 1e-9 (dLossMax, against the oracle's
                                                                 at the engine's refined pose), 1e-7 (dRefine, dPNP), 1e-4
                                                                 (score gradients), 1e-3 (dLoss/dObj) of max
  DSAC-variant forward / backward ............................. test_gpu_forward.py's / test_gpu_backward.py's
  scheduling-only settings (hyps_per_cta) ..................... bit-identical, diffmaps included

Run with -s to see the measured maxima per case.
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1600


def _threads():
    try:
        return max(1, len(os.sched_getaffinity(0)))
    except Exception:
        return os.cpu_count() or 1


def _rel(a, b, floor=1e-300):
    return np.abs(a - b).max() / max(floor, np.abs(b).max())


def _cam(kw):
    return kw.get("focal", 525.0), kw.get("cx", 320.0), kw.get("cy", 240.0)


def _oracle_cfg(O, kw, seed):
    """The oracle's configuration for the engine's keyword arguments (the oracle names the focal length f)."""
    okw = {("f" if k == "focal" else k): v for k, v in kw.items() if k not in ("max_frames", "hyps_per_cta", "write_diffmaps")}
    return O.default_config(seed=seed, **okw)


def _frames(E, nf, kw, frame0=0):
    f, cx, cy = _cam(kw)
    return E.synth_frames(nf, frame0=frame0, n_streams=kw.get("n_streams", 1), focal=f, cx=cx, cy=cy)


def _oracle_forward(O, kw, coords, pix, gt_jp, frame0=0):
    T = kw.get("n_streams", 1)

    def one(f):
        cfg = _oracle_cfg(O, kw, 1305 + (frame0 + f) * T)
        return O.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
    with ThreadPoolExecutor(max_workers=min(coords.shape[0], _threads())) as ex:
        return list(ex.map(one, range(coords.shape[0])))


def _check_forward(E, O, kw, nf, name, frame0=0):
    """Engine vs oracle on nf frames at the configuration kw; returns the measured maxima."""
    coords, pix, gt_cv, gt_jp = _frames(E, nf, kw, frame0)
    eng = E.Engine(max_frames=nf, **kw)
    res = eng.forward(coords, pix, gt_jp, frame0=frame0, want_diffmaps=True)
    eng.close()
    ora = _oracle_forward(O, kw, coords, pix, gt_jp, frame0)
    f_len = _cam(kw)[0]
    alpha, beta = kw.get("alpha", 0.1), kw.get("beta", 0.5)
    ref_steps = kw.get("ref_steps", 8)
    mx = dict(rvec=0.0, tvec=0.0, dm=0.0, score=0.0, sf=0.0, avg=0.0, ref_r=0.0, ref_t=0.0, loss=0.0)
    for f, o in enumerate(ora):
        assert o.n_fragile == 0 and o.status == 0, (name, f)
        bad = np.flatnonzero((o.img_idx != res.img_idx[f]).any(1))
        if len(bad):
            h = bad[0]
            print("%s frame %d: first differing hypothesis %d: oracle %s (candidate %d), engine %s (candidate %d)"
                  % (name, f, h, o.img_idx[h], o.cand_idx[h], res.img_idx[f][h], res.cand_idx[f][h]))
        # integer work: bit-exact
        assert np.array_equal(o.img_idx, res.img_idx[f]), (name, f)
        assert np.array_equal(o.cand_idx, res.cand_idx[f]), (name, f)
        assert o.n_candidates == res.n_candidates[f], (name, f)
        assert np.array_equal(o.inlier_map, res.inlier_map[f]), (name, f)
        assert o.ref_steps_done == res.ref_steps_done[f] and o.n_perm_steps == res.n_perm_steps[f], (name, f)
        assert res.status[f] == (E.ST_REFINE_ABORTED if o.ref_steps_done < ref_steps else 0), (name, f, res.status[f])
        # hypotheses
        mx["rvec"] = max(mx["rvec"], np.abs(o.hyp_rvec - res.hyp_pose[f][:, :3]).max())
        mx["tvec"] = max(mx["tvec"], np.abs(o.hyp_tvec - res.hyp_pose[f][:, 3:]).max())
        assert np.abs(o.hyp_rvec - res.hyp_pose[f][:, :3]).max() <= 1e-9 and np.abs(o.hyp_tvec - res.hyp_pose[f][:, 3:]).max() <= 1e-6
        # error matrix
        de = float(np.abs(o.diffmaps - res.diffmaps[f]).max())
        mx["dm"] = max(mx["dm"], de)
        assert de <= 2e-3 * max(1.0, f_len / 525.0), (name, f, de)
        assert res.diffmaps[f].max() <= 100.0 and res.diffmaps[f].min() >= 0.0
        # scores, softmax, soft-argmax
        smax = np.abs(o.scores).max()
        ds = float(np.abs(o.scores - res.scores[f]).max())
        tol_s = alpha * N * 2.0 ** -25 + (1e-5 + beta * de) * smax
        mx["score"] = max(mx["score"], ds / tol_s)
        assert ds <= tol_s, (name, f, ds, tol_s)
        assert np.abs(O.softmax(res.scores[f]) - res.sf[f]).max() <= 1e-12
        dsf = np.abs(o.sf - res.sf[f])
        mx["sf"] = max(mx["sf"], dsf.max())
        assert dsf.max() <= max(1e-4, 2 * ds), (name, f, dsf.max(), ds)
        avg_from_gpu_sf = (res.sf[f][:, None] * res.hyp_pose[f]).sum(0)
        assert np.abs(avg_from_gpu_sf - res.avg_pose[f]).max() <= 1e-9 * max(1.0, np.abs(avg_from_gpu_sf).max())
        davg = np.abs(o.avg - res.avg_pose[f]).max()
        mx["avg"] = max(mx["avg"], davg)
        assert davg <= 1e-3 + (dsf[:, None] * np.abs(res.hyp_pose[f])).sum(0).max(), (name, f, davg)
        # refinement and evaluation
        mx["ref_r"] = max(mx["ref_r"], np.abs(o.ref[:3] - res.ref_pose[f][:3]).max())
        mx["ref_t"] = max(mx["ref_t"], np.abs(o.ref[3:] - res.ref_pose[f][3:]).max())
        assert np.abs(o.ref[:3] - res.ref_pose[f][:3]).max() <= 1e-6 and np.abs(o.ref[3:] - res.ref_pose[f][3:]).max() <= 1e-3, (name, f)
        mx["loss"] = max(mx["loss"], abs(o.loss - res.loss[f]))
        assert abs(o.loss - res.loss[f]) <= 1e-4 and abs(o.rot_err - res.rot_err[f]) <= 1e-4
        assert abs(o.t_err - res.t_err[f]) <= 1e-2 and o.correct == res.correct[f], (name, f)
    print("%-14s maxima: hyp %.2g rad %.2g mm | diffmap %.2g px | score %.2g of tol | sf %.2g | avg %.2g | ref %.2g rad %.2g mm | loss %.2g"
          % (name, mx["rvec"], mx["tvec"], mx["dm"], mx["score"], mx["sf"], mx["avg"], mx["ref_r"], mx["ref_t"], mx["loss"]))
    return res, ora


# ------------------------------------------------------------------------------------------------ (a) parameter grid
GRID = [
    ("thr3", dict(thr2d=3)),
    ("thr20", dict(thr2d=20)),
    ("inliers128", dict(inlier_count=128)),                 # K4_MAX_INLIERS: two selected points per k_refine thread
    ("inliers50", dict(inlier_count=50)),                   # the "< 50" stop at its boundary
    ("steps0", dict(ref_steps=0)),
    ("steps1", dict(ref_steps=1)),
    ("steps16", dict(ref_steps=16)),                        # DSAC_MAX_REF_STEPS
    ("score_a.3_b1.5", dict(alpha=0.3, beta=1.5)),
    ("score_a.05_b2", dict(alpha=0.05, beta=2.0)),
    ("cam585", dict(focal=585.0)),
    ("cam1500", dict(focal=1500.0)),                        # a near-double root of the P3P quartic (frame 1, candidate 25360)
    ("cam_off", dict(cx=330.5, cy=235.25)),
    ("cam1000_off", dict(focal=1000.0, cx=480.0, cy=360.0)),   # 640 x 480 inside a 960 x 720 sampling grid, off-centre
    ("combined", dict(thr2d=3, inlier_count=60, ref_steps=12, alpha=0.05, beta=2.0, n_hyps=37, n_streams=3)),
]


@pytest.mark.parametrize("name,kw", GRID, ids=[g[0] for g in GRID])
def test_forward_across_parameters(engine_mod, oracle, name, kw):
    kw = dict(kw)
    kw.setdefault("n_hyps", 128)
    res, ora = _check_forward(engine_mod, oracle, kw, 3 if name == "combined" else 2, name)
    if name == "inliers128":
        assert (res.inlier_map.max(1) > 0).all()
    if name == "steps16":
        assert res.ref_steps_done.max() == 16


def test_forward_below_the_inlier_minimum_aborts_every_refinement(engine_mod, oracle):
    """inlier_count = 49 < 50: every refinement stops at step 0 (cnn_softam.h:1136), so the refined pose is the soft-argmax
    pose, as in the oracle."""
    E = engine_mod
    res, ora = _check_forward(E, oracle, dict(inlier_count=49, n_hyps=64), 2, "inliers49")
    for f, o in enumerate(ora):
        assert o.ref_steps_done == 0 and res.ref_steps_done[f] == 0
        assert res.status[f] == E.ST_REFINE_ABORTED
        assert np.array_equal(res.ref_pose[f], res.avg_pose[f])
        assert np.array_equal(o.ref, o.avg)


# ------------------------------------------------------------------------------------------------ (b) hypothesis counts
HT = [(H, T) for H in (3, 37, 100, 257, 1000, 1024) for T in (1, 7) if T <= H and (T == 1 or H % T != 0)]


@pytest.mark.parametrize("H,T", HT, ids=["H%d_T%d" % ht for ht in HT])
def test_forward_at_odd_hypothesis_counts(engine_mod, oracle, H, T):
    """Tail tiles, partial groups of 8 hypotheses in k_score (score_group8<FULL = false>) and DSAC_MAX_HYPS."""
    _check_forward(engine_mod, oracle, dict(n_hyps=H, n_streams=T), 1 if H >= 257 else 2, "H%d_T%d" % (H, T), frame0=3)


# ------------------------------------------------------------------------------------------------ (c) score tiles
@pytest.mark.parametrize("n", [1, 40])
def test_score_tile_is_scheduling_only(engine_mod, n):
    """Tiles are multiples of 8 hypotheses, so a hypothesis always sits at the same lane position of its group of 8: its
    warp reduction and the fixed-order cross-warp sum do not depend on the tile.  Every output, diffmaps included, must be
    bit-identical for hyps_per_cta in {0 (automatic), 8, 24, 64, 256}; H = 1003 leaves a partial group in the last tile."""
    E = engine_mod
    H = 1003
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    keys = ("img_idx", "cand_idx", "n_candidates", "hyp_pose", "scores", "sf", "entropy", "avg_pose", "ref_pose", "inlier_map",
            "ref_steps_done", "n_perm_steps", "loss", "status", "diffmaps")
    out = {}
    for tile in (0, 8, 24, 64, 256):
        eng = E.Engine(max_frames=n, n_hyps=H, hyps_per_cta=tile)
        out[tile] = eng.forward(coords, pix, gt_jp, want_diffmaps=True)
        eng.close()
    for tile in (8, 24, 64, 256):
        for k in keys:
            assert np.array_equal(getattr(out[0], k), getattr(out[tile], k)), (tile, k)
    assert (out[0].scores > 0).all()


# ------------------------------------------------------------------------------------------------ (d) soft-argmax backward
# dRefineObj takes every skip-th pixel that was an inlier in some refinement step (cnn_softam.h:866-920): skip = 200 needs
# more than 200 such pixels, hence inlier_count x ref_steps = 128 x 4 (64 x 3 could never reach 200)
BW = dict(thr2d=5, inlier_count=128, ref_steps=4, sub_sample=0.005, alpha=0.3, beta=1.5, grad_clamp=0.02, focal=1500.0, n_hyps=64)


def _gt6(O, gt_jp):
    return np.concatenate([O.rodrigues_inv(gt_jp[:9]), gt_jp[9:]])   # poseGT.getRodVecAndTrans()


@pytest.mark.parametrize("fix_q4", [0, 1])
def test_backward_across_parameters(engine_mod, oracle, fix_q4):
    """sub_sample = 0.005: skip = 200, at most 8 dRefineObj pixels per frame; alpha, beta and a grad_clamp small enough
    that score gradients reach it; the 1500 px camera.  The synthetic inliers' noise is scaled to 25 mm x 525 / 1500, so
    that it is as many pixels as at the default camera (at 25 mm thr2d = 5 leaves fewer than 50 inliers and every
    refinement stops at step 0)."""
    E, O = engine_mod, oracle
    kw = dict(BW, fix_q4=fix_q4)
    nf = 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, focal=kw["focal"], sigma=25.0 * 525.0 / kw["focal"])
    eng = E.Engine(max_frames=nf, **kw)
    fwd = eng.forward(coords, pix, gt_jp)
    bw = eng.backward(coords, pix, gt_jp)
    eng.close()

    def one(f):
        cfg = _oracle_cfg(O, kw, 1305 + f)
        ofw = O.forward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:])
        return ofw, O.backward(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw)
    with ThreadPoolExecutor(max_workers=nf) as ex:
        ora = list(ex.map(one, range(nf)))
    worst, clamped = 0.0, 0
    for f, (ofw, obw) in enumerate(ora):
        assert np.array_equal(ofw.img_idx, fwd.img_idx[f]) and np.array_equal(ofw.inlier_map, fwd.inlier_map[f])
        assert ofw.ref_steps_done == fwd.ref_steps_done[f] == kw["ref_steps"]
        # dLossMax is closed-form: the oracle's at the ENGINE's refined pose (the refined poses themselves are compared by
        # the forward tests), so the comparison does not inherit the fp32-score difference of the two refinement starts
        want_dref = O.dloss_max(O.jp6(fwd.ref_pose[f][:3], fwd.ref_pose[f][3:]), _gt6(O, gt_jp[f]))
        m = dict(dloss_dref=_rel(bw.dloss_dref[f], want_dref), dref_dhyp=_rel(bw.dref_dhyp[f], obw.dref_dhyp, floor=1e-3),
                 dref_dobj=_rel(bw.dref_dobj[f], obw.dref_dobj, floor=1e-3), dpnp=_rel(bw.dpnp[f], obw.dpnp),
                 score_grads=_rel(bw.score_grads[f], obw.score_grads, floor=1e-6), dloss_dobj=_rel(bw.dloss_dobj[f], obw.dloss_dobj, floor=1e-6))
        print("backward fix_q4=%d frame %d:" % (fix_q4, f), {k: float("%.3g" % v) for k, v in m.items()})
        assert m["dloss_dref"] <= 1e-9
        assert m["dref_dhyp"] <= 1e-7 and m["dref_dobj"] <= 1e-7
        cols = np.flatnonzero(np.abs(obw.dref_dobj).sum(0))
        assert 0 < len(cols) <= 8 * 3                        # at least one gradient pixel, at most 8, of 3 channels each
        assert (np.abs(bw.dref_dobj[f]).sum(0) > 0).sum() == len(cols)
        assert m["dpnp"] <= 1e-7 and m["score_grads"] <= 1e-4
        clamped += int((np.abs(obw.score_grads) > kw["grad_clamp"]).sum())
        worst = max(worst, m["dloss_dobj"])
        assert m["dloss_dobj"] <= 1e-3
        assert np.abs(bw.dloss_dobj[f]).max() > 0
    print("backward fix_q4=%d: dLoss/dObj %.3g of max, %d score gradients beyond the clamp" % (fix_q4, worst, clamped))
    assert clamped > 0


def test_backward_rejects_too_many_gradient_pixels(engine_mod, oracle):
    """sub_sample = 0.02 -> skip = 50 -> up to 32 dRefineObj pixels, more than the soft-argmax backward's 16: DSAC_ERR_ARG.
    The engine stays usable: the same forward again, the same refusal, and the DSAC variant's backward (which has no such
    cap) on the same engine against the oracle."""
    E, O = engine_mod, oracle
    kw = dict(sub_sample=0.02, n_hyps=16)
    coords, pix, gt_cv, gt_jp = _frames(E, 1, kw)
    eng = E.Engine(max_frames=1, **kw)
    a = eng.forward(coords, pix, gt_jp)
    with pytest.raises(RuntimeError, match="sub_sample"):
        eng.backward(coords, pix, gt_jp)
    b = eng.forward(coords, pix, gt_jp)
    for k in ("img_idx", "scores", "ref_pose", "inlier_map"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    with pytest.raises(RuntimeError, match="sub_sample"):
        eng.backward(coords, pix, gt_jp)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    bw = eng.backward_dsac(1)
    eng.close()
    ofw = _dsac_oracle_state(O, kw, fw, 0, 1305)
    obw = O.backward_dsac(_oracle_cfg(O, kw, 1305), coords[0], pix[0], gt_jp[0, :9], gt_jp[0, 9:], ofw)
    assert obw.n_selected == bw.n_selected[0] and obw.n_refine_jobs == bw.n_refine_jobs[0]
    assert _rel(bw.dloss_dobj[0], obw.dloss_dobj) <= 1e-5


# ------------------------------------------------------------------------------------------------ (e) DSAC variant
def _dsac_oracle_state(O, kw, fw, f, seed):
    """The oracle's DSAC forward record filled with the ENGINE's forward state (test_gpu_backward.py)."""
    ofw = O.ForwardDsac(_oracle_cfg(O, kw, seed))
    ofw.hyp_rvec[:] = fw.hyp_pose[f][:, :3]; ofw.hyp_tvec[:] = fw.hyp_pose[f][:, 3:]
    ofw.img_idx[:] = fw.img_idx[f]; ofw.sf[:] = fw.sf[f]; ofw.ref_pose[:] = fw.ref_pose[f]; ofw.losses[:] = fw.losses[f]
    return ofw


DSAC = [
    ("subsample.05", dict(sub_sample=0.05, n_hyps=32), 2, True),        # skip 20: ~5x the refine jobs per hypothesis
    ("cam1000_off", dict(focal=1000.0, cx=480.0, cy=360.0, n_hyps=32, n_streams=3), 2, True),
    ("thr5", dict(thr2d=5, n_hyps=32), 2, True),
    ("H1024", dict(n_hyps=1024, n_streams=7), 1, True),                # DSAC_MAX_HYPS: k_dsac_scan / k_dsac_combine full size
]


@pytest.mark.parametrize("name,kw,nf,with_backward", DSAC, ids=[d[0] for d in DSAC])
def test_dsac_variant_across_parameters(engine_mod, oracle, name, kw, nf, with_backward):
    E, O = engine_mod, oracle
    T = kw.get("n_streams", 1)
    coords, pix, gt_cv, gt_jp = _frames(E, nf, kw)
    eng = E.Engine(max_frames=nf, **kw)
    res = eng.forward_dsac(coords, pix, gt_jp, random_draw=True, want_inlier_maps=True)

    def one(f):
        cfg = _oracle_cfg(O, kw, 1305 + f * T)
        return O.forward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], True)
    with ThreadPoolExecutor(max_workers=min(nf, _threads())) as ex:
        ora = list(ex.map(one, range(nf)))
    for f, o in enumerate(ora):
        assert np.array_equal(o.img_idx, res.img_idx[f]) and o.hyp_idx == res.hyp_idx[f], (name, f)
        assert np.array_equal(o.steps_done, res.steps_done[f]) and np.array_equal(o.inlier_maps, res.inlier_maps[f]), (name, f)
        assert np.abs(o.ref_pose[:, :3] - res.ref_pose[f][:, :3]).max() <= 1e-8
        assert np.abs(o.ref_pose[:, 3:] - res.ref_pose[f][:, 3:]).max() <= 1e-5
        assert np.abs(o.losses - res.losses[f]).max() <= 1e-6 * max(1.0, np.abs(o.losses).max())
        assert np.abs(o.sf - res.sf[f]).max() <= 1e-4
        assert abs(o.expected_loss - res.expected_loss[f]) <= 1e-3 * max(1.0, abs(o.expected_loss))
        assert abs(o.rot_err - res.rot_err[f]) <= 1e-6 and abs(o.t_err - res.t_err[f]) <= 1e-4 and o.correct == res.correct[f]
    if not with_backward:
        eng.close()
        return
    # backward, the oracle fed the engine's forward state (same selection, every factor fp64)
    fw = eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
    bw = eng.backward_dsac(nf)
    eng.close()

    def oneb(f):
        ofw = _dsac_oracle_state(O, kw, fw, f, 1305 + f * T)
        return O.backward_dsac(_oracle_cfg(O, kw, 1305 + f * T), coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], ofw)
    with ThreadPoolExecutor(max_workers=min(nf, _threads())) as ex:
        orb = list(ex.map(oneb, range(nf)))
    worst = 0.0
    for f, obw in enumerate(orb):
        assert obw.n_selected == bw.n_selected[f] and obw.n_selected >= 1
        assert obw.n_refine_jobs == bw.n_refine_jobs[f] and obw.n_refine_jobs >= 18 * obw.n_selected
        assert _rel(bw.score_grads[f], obw.score_grads, floor=1e-12) <= 1e-9
        assert _rel(bw.path1[f], obw.path1) <= 1e-5
        assert np.median(np.abs(bw.path1[f] - obw.path1)) <= 1e-10 * np.abs(obw.path1).max()
        assert _rel(bw.path2[f], obw.path2) <= 1e-6
        d = _rel(bw.dloss_dobj[f], obw.dloss_dobj)
        worst = max(worst, d)
        assert d <= 1e-5
    print("dsac %-12s backward: %s selected, %s refine jobs, dLoss/dObj %.3g of max"
          % (name, list(bw.n_selected), list(bw.n_refine_jobs), worst))
    if name == "H1024":
        assert bw.n_selected[0] >= 50


# ------------------------------------------------------------------------------------------------ (f) argument limits
@pytest.mark.parametrize("kw", [dict(n_hyps=0), dict(n_hyps=1025), dict(inlier_count=0), dict(inlier_count=129),
                                dict(ref_steps=-1), dict(ref_steps=17), dict(n_hyps=4, n_streams=5)],
                         ids=["hyps0", "hyps1025", "inliers0", "inliers129", "steps-1", "steps17", "streams>hyps"])
def test_out_of_range_arguments_are_rejected(engine_mod, kw):
    with pytest.raises(RuntimeError, match="out of range"):
        engine_mod.Engine(max_frames=1, **kw)


def test_largest_arguments_are_accepted_and_run(engine_mod, oracle):
    _check_forward(engine_mod, oracle, dict(n_hyps=1024, inlier_count=128, ref_steps=16), 1, "largest")


# ------------------------------------------------------------------------------------------------ (g) the reference's own outputs
def test_engine_matches_the_reference_at_non_default_parameters(engine_mod):
    """The engine against outputs of the reference's own code at non-default parameters and cameras (frozen in
    tests/golden/ref_params.npz), with test_engine_matches_the_reference_fixtures' and the DSAC-variant forward tests'
    tolerances; the diffmap and score tolerances are scaled as above (de = the largest difference on the stored rows)."""
    import hashlib
    E = engine_mod
    z = np.load(os.path.join(ROOT, "tests", "golden", "ref_params.npz"))
    names = sorted({k.split("/")[0] for k in z.files})
    assert len(names) >= 8
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a, np.int32).tobytes()).hexdigest()   # noqa: E731
    for name in names:
        g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}
        H, T, fr = int(g["H"]), int(g["T"]), int(g["frame"])
        f_len, cx, cy = (float(v) for v in g["camera"])
        kw = dict(n_hyps=H, n_streams=T, focal=f_len, cx=cx, cy=cy, thr2d=int(g["thr2d"]), inlier_count=int(g["inlier_count"]),
                  ref_steps=int(g["ref_steps"]), sub_sample=float(g["sub_sample"]), alpha=float(g["alpha"]), beta=float(g["beta"]))
        gt = np.concatenate([g["gt_R"].reshape(9), g["gt_t"].reshape(3)])[None]
        eng = E.Engine(max_frames=1, **kw)
        if str(g["kind"]) == "dsac_forward":
            r = eng.forward_dsac(g["coords"][None], g["pix"][None], gt, random_draw=True, frame0=fr, want_inlier_maps=True)
            eng.close()
            assert np.array_equal(r.img_idx[0], g["img_idx"]) and r.hyp_idx[0] == int(g["hyp_idx"]), name
            assert sha(r.inlier_maps[0]) == str(g["inlier_maps_sha256"]), name
            assert np.abs(r.ref_pose[0][:, :3] - g["ref_pose"][:, :3]).max() <= 1e-8
            assert np.abs(r.ref_pose[0][:, 3:] - g["ref_pose"][:, 3:]).max() <= 1e-5
            assert np.abs(r.losses[0] - g["losses"]).max() <= 1e-6 * max(1.0, np.abs(g["losses"]).max())
            assert np.abs(r.sf[0] - g["sf"]).max() <= 1e-4
            assert abs(r.expected_loss[0] - float(g["expected_loss"])) <= 1e-3 * max(1.0, abs(float(g["expected_loss"])))
            assert r.correct[0] == int(g["correct"]), name
            continue
        r = eng.forward(g["coords"][None], g["pix"][None], gt, frame0=fr, want_diffmaps=True)
        eng.close()
        assert np.array_equal(r.img_idx[0], g["img_idx"]), name
        assert sha(r.inlier_map[0]) == str(g["inlier_map_sha256"]) and r.n_perm_steps[0] == int(g["n_perm_steps"]), name
        assert np.abs(r.hyp_pose[0][:, :3] - g["hyp_rvec"]).max() <= 1e-9 and np.abs(r.hyp_pose[0][:, 3:] - g["hyp_tvec"]).max() <= 1e-6
        de = float(np.abs(r.diffmaps[0][:: max(1, H // 8)] - g["diffmap_rows"]).max())
        assert de <= 2e-3 * max(1.0, f_len / 525.0), name
        tol_s = kw["alpha"] * N * 2.0 ** -25 + (1e-5 + kw["beta"] * de) * np.abs(g["scores"]).max()
        assert np.abs(r.scores[0] - g["scores"]).max() <= tol_s, name
        assert np.abs(r.sf[0] - g["sf"]).max() <= 1e-4 and abs(r.entropy[0] - float(g["entropy"])) <= 1e-3, name
        assert np.abs(r.ref_pose[0][:3] - g["ref"][:3]).max() <= 1e-6 and np.abs(r.ref_pose[0][3:] - g["ref"][3:]).max() <= 1e-3, name
        assert abs(r.loss[0] - float(g["loss"])) <= 1e-4 and r.correct[0] == int(g["correct"]), name
