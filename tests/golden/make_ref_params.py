"""Freeze outputs of the REFERENCE'S OWN code (oracle/_ref) at non-default parameters and cameras: inlier threshold,
inlier count, refinement steps, sub-sampling of the dRefineObj pixels, alpha / beta, hypothesis counts that are not
multiples of 8, several sampler streams, and two cameras besides the default one.

    DSAC_REFERENCE=<reference>/core python tests/golden/make_ref_params.py        ->  tests/golden/ref_params.npz

Consumers: tests/test_oracle_params.py (oracle vs fixtures, CPU) and tests/test_gpu_params.py (CUDA engine vs fixtures).
Every case stores its inputs.  The reference samples its pixel grid from the 640 x 480 image whatever the camera, so for
a principal point off the image centre the scene coordinates are generated here, for that grid and camera, with the
synthetic generator's recipe (depth 500..3500 mm, half inliers with 25 mm noise, half uniform outliers).  Large arrays
are stored as SHA-256 digests (inlier map, full diffmaps, refinement permutations, the DSAC variant's inlier maps),
samples with their indices beside them (dRefine/dObj columns, dPNP hypotheses), and every (H/8)-th diffmap row in full.
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from dsac_b200 import synth as E  # noqa: E402   (host-only build of the engine's frame generator)
from oracle import oracle as O  # noqa: E402
from oracle import ref as R  # noqa: E402

DEFAULT_CAM = (525.0, 320.0, 240.0)
# (name, kind, H, T, frame, camera, parameters); kind "forward" also freezes the backward factors
CASES = [
    ("fwd_thr3", "forward", 64, 1, 0, DEFAULT_CAM, dict(thr2d=3)),
    ("fwd_combined", "forward", 37, 3, 2, DEFAULT_CAM, dict(thr2d=3, inlier_count=60, ref_steps=12, alpha=0.05, beta=2.0)),
    ("fwd_inliers128", "forward", 64, 1, 1, DEFAULT_CAM, dict(inlier_count=128)),
    ("fwd_thr20_steps16", "forward", 100, 7, 4, DEFAULT_CAM, dict(thr2d=20, ref_steps=16)),
    ("fwd_score_subsample", "forward", 48, 1, 5, DEFAULT_CAM, dict(alpha=0.3, beta=1.5, sub_sample=0.005, ref_steps=3)),
    ("fwd_cam585", "forward", 64, 1, 6, (585.0, 320.0, 240.0), dict(thr2d=5)),
    ("fwd_cam_off", "forward", 64, 2, 7, (525.0, 330.5, 235.25), dict()),
    ("dsac_cam585_thr5", "dsac_forward", 32, 1, 3, (585.0, 320.0, 240.0), dict(thr2d=5)),
]
PARAMS = dict(thr2d=10, inlier_count=100, ref_steps=8, sub_sample=0.01, alpha=0.1, beta=0.5)


def sample(n, k, seed):
    return np.sort(np.random.default_rng(seed).choice(n, min(n, k), replace=False)).astype(np.int16)


def digest(a, dtype=np.int32):
    return hashlib.sha256(np.ascontiguousarray(a, dtype).tobytes()).hexdigest()


def frame(g, T, cam):
    """One synthetic frame on the reference's pixel grid for camera cam = (f, cx, cy)."""
    f, cx, cy = cam
    coords, pix, gt_cv, gt_jp = E.synth_frames(1, frame0=g, n_streams=T, focal=f)   # grid of the 640 x 480 image
    if (cx, cy) != (320.0, 240.0):
        rng = np.random.default_rng(20170721 + g)
        Rm = O.rodrigues(gt_cv[0, :3])
        u, v = pix[0, :, 0].astype(np.float64), pix[0, :, 1].astype(np.float64)
        d = rng.uniform(500, 3500, E.N)
        Xc = np.stack([(u - cx) * d / f, (v - cy) * d / f, d], 1) - gt_cv[0, 3:]
        Y = Xc @ Rm + rng.normal(0, 25.0, (E.N, 3))          # R^T (X_cam - t) per cell
        out = rng.uniform(size=E.N) >= 0.5
        Y[out] = rng.uniform(-2000, 2000, (int(out.sum()), 3))
        coords = np.clip(np.rint(Y), -32768, 32767).astype(np.int16)[None]
    return coords[0], pix[0], gt_jp[0]


def main():
    if not R.available():
        raise SystemExit("DSAC_REFERENCE must name the core/ directory of a checkout of the reference")
    out = {}
    cols = sample(E.N * 3, 64, 20170721)
    for name, kind, H, T, g, cam, kw in CASES:
        p = dict(PARAMS, **kw)
        coords, pix, gt_jp = frame(g, T, cam)
        R.set_camera(*cam)
        cfg = R.config(n_hyps=H, n_threads=T, frame=g, **p)
        rec = dict(kind=kind, H=H, T=T, frame=g, camera=np.array(cam), coords=coords, pix=pix, gt_R=gt_jp[:9].reshape(3, 3),
                   gt_t=gt_jp[9:], **p)
        if kind == "forward":
            fw = R.forward(cfg, coords, gt_jp[:9], gt_jp[9:])
            assert np.array_equal(fw.pix, pix) and np.array_equal(fw.est_obj, coords)
            fa = R.factors(cfg)
            dpnp_hyps = sample(H, 8, g)
            rec.update(img_idx=fw.img_idx, hyp_rvec=fw.hyp_rvec, hyp_tvec=fw.hyp_tvec, scores=fw.scores, sf=fw.sf, entropy=fw.entropy,
                       avg=fw.avg, ref=fw.ref, inlier_map_sha256=digest(fw.inlier_map), n_perm_steps=fw.n_perm_steps, loss=fw.loss,
                       rot_err=fw.rot_err, t_err=fw.t_err, correct=fw.correct, diffmaps_sha256=digest(fw.diffmaps, np.float32),
                       diffmap_rows=fw.diffmaps[:: max(1, H // 8)], pixel_idxs_sha256=digest(fw.pixel_idxs),
                       dloss_dref=fa["dloss_dref"], dref_dhyp=fa["dref_dhyp"], dref_dobj_cols=cols, dref_dobj=fa["dref_dobj"][:, cols],
                       dref_dobj_absmax=np.abs(fa["dref_dobj"]).max(), dpnp_hyps=dpnp_hyps, dpnp=fa["dpnp"][dpnp_hyps],
                       dpnp_absmax=np.abs(fa["dpnp"]).max())
            print(name, "loss %.6f" % fw.loss, "correct", fw.correct, "perm steps", fw.n_perm_steps, flush=True)
        else:
            r = R.forward_dsac(cfg, coords, gt_jp[:9], gt_jp[9:], True)
            rec.update(img_idx=r.img_idx, hyp_idx=r.hyp_idx, correct=r.correct, inlier_maps_sha256=digest(r.inlier_maps),
                       hyp_rvec=r.hyp_rvec, hyp_tvec=r.hyp_tvec, sf=r.sf, ref_pose=r.ref_pose, losses=r.losses,
                       expected_loss=r.expected_loss, rot_err=r.rot_err, t_err=r.t_err)
            print(name, "expected loss %.6f" % r.expected_loss, "hyp", r.hyp_idx, flush=True)
        for k, v in rec.items():
            out[name + "/" + k] = np.asarray(v)
    R.set_camera(*DEFAULT_CAM)
    path = os.path.join(ROOT, "tests", "golden", "ref_params.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
