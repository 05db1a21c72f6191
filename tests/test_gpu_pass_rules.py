"""Which consumers of a forward pass accept it, and what they report when they do not.

Every consumer of the pass the engine holds -- the soft-argmax backward, the DSAC backward, the refined poses, pose
uncertainty, pose modes and the sampling log-probability -- is called after a soft-argmax pass, after a DSAC pass and
on an engine that ran neither, with each of the four per-frame settings (cameras, sampling logits, cell depth, pose
priors) set or cleared between the pass and the call.  The expected outcome restates each consumer's rule: the pipeline
it needs, and the settings whose change makes the held pass stale for it."""
import numpy as np
import pytest
import torch

import rgbd_oracle as R

pytestmark = pytest.mark.gpu
N = 1600
NF, H = 2, 64
SETTINGS = ("cameras", "logits", "depth", "priors")
PASSES = ("softam", "dsac", "none")
CONSUMERS = ("backward", "backward_dsac", "refined_jp6", "pose_uncertainty", "pose_modes", "sampling_log_prob")
# a change between the pass and the call: None, or (setting, "set" | "clear"); "clear" means the pass ran with it
CHANGES = [None] + [(s, a) for s in SETTINGS for a in ("set", "clear")]

CHANGED = {   # the refined-pose consumers' text for a setting changed after the pass
    "cameras": "the cameras were changed (dsac_set_cameras) after the forward pass",
    "depth": "the cell depth was changed (dsac_set_cell_depth_device) after the forward pass",
    "priors": "the pose priors were changed (dsac_set_pose_priors_device) after the forward pass",
}
CHANGED_LOGP = {   # the sampling log-probability's
    "logits": "the sampling logits were changed after the last pass",
    "depth": "the cell depth was changed after the last pass",
    "priors": "the pose priors were changed after the last pass",
}


def expected(consumer, kind, change):
    """None if the call is accepted, else a substring of the error it reports."""
    setting, action = change if change else (None, None)
    if consumer == "sampling_log_prob":
        who = "dsac_sampling_log_prob_device"
        guided = kind != "none" and setting == "logits" and action == "clear"
        if not guided:
            return who + ": the last forward pass was not guided"
        return None if setting not in CHANGED_LOGP else who + ": " + CHANGED_LOGP[setting]
    stale = CHANGED.get(setting)
    if consumer == "backward":
        if kind != "softam":
            return "dsac_backward must follow a dsac_forward over the same %d frames" % NF
        return None if stale is None else "dsac_backward: " + stale
    if consumer == "backward_dsac":
        if kind != "dsac":
            return "dsac_backward_dsac must follow a dsac_forward_dsac over the same %d frames" % NF
        return None if stale is None else "dsac_backward_dsac: " + stale
    who = {"refined_jp6": "dsac_refined_jp6_device", "pose_uncertainty": "dsac_pose_uncertainty_device",
           "pose_modes": "dsac_pose_modes_device"}[consumer]
    if stale is not None:   # these report a stale setting before a missing pass
        return who + ": " + stale
    return None if kind != "none" else who + " must follow a forward pass over the same %d frames" % NF


@pytest.fixture(scope="module")
def frames(engine_mod):
    coords, pix, depth, gt_cv, gt_jp = R.synth(NF, seed=11)
    dev = torch.device("cuda")
    rng = np.random.default_rng(3)
    priors = np.repeat(gt_cv[:, None, :], 2, axis=1) + rng.normal(0, 0.01, (NF, 2, 6))
    return {
        "coords": torch.from_numpy(coords).to(dev), "pix": torch.from_numpy(pix).to(dev),
        "gt": torch.from_numpy(gt_jp).to(dev), "depth": torch.from_numpy(depth).to(dev),
        "logits": torch.from_numpy(rng.normal(0, 1, (NF, N)).astype(np.float32)).to(dev),
        "priors": torch.from_numpy(priors).to(dev),
        "cams": np.array([[525.0, 320.0, 240.0], [600.0, 310.0, 250.0]]),
    }


def apply(eng, fr, setting, on):
    if setting == "cameras":
        eng.set_cameras(fr["cams"] if on else None)
    elif setting == "logits":
        eng.set_sampling_logits_device(NF, fr["logits"].data_ptr() if on else None)
    elif setting == "depth":
        eng.set_cell_depth_device(NF, fr["depth"].data_ptr() if on else None)
    else:
        eng.set_pose_priors_device(NF, 2, fr["priors"].data_ptr() if on else None)


def consume(eng, consumer):
    dev = torch.device("cuda")
    f64 = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    i32 = lambda *s: torch.zeros(s, dtype=torch.int32, device=dev)
    keep = []

    def ptrs(d):
        keep.extend(d.values())
        return {k: v.data_ptr() for k, v in d.items()}

    if consumer == "backward":
        eng.backward_device(NF, d_dloss_dobj=ptrs({"o": f64(NF, N, 3)})["o"])
    elif consumer == "backward_dsac":
        eng.backward_dsac_device(NF, **ptrs({"dloss_dobj": f64(NF, N, 3)}))
    elif consumer == "refined_jp6":
        eng.refined_jp6_device(NF, ptrs({"o": f64(NF, H, 6)})["o"])
    elif consumer == "pose_uncertainty":
        eng.pose_uncertainty_device(NF, **ptrs({"cov_jp6": f64(NF * H, 36), "cov_xi": f64(NF * H, 36), "sigma2": f64(NF * H),
                                                "n_fit": i32(NF * H), "support": i32(NF * H), "ok": i32(NF * H)}))
    elif consumer == "pose_modes":
        M = 4
        eng.pose_modes_device(NF, M, 0.1, 100.0, **ptrs({
            "n_modes": i32(NF), "pose": f64(NF, M, 6), "cov_xi": f64(NF, M, 36), "score": f64(NF, M), "mass": f64(NF, M),
            "sigma2": f64(NF, M), "hyp": i32(NF, M), "members": i32(NF, M), "steps_done": i32(NF, M), "n_fit": i32(NF, M),
            "support": i32(NF, M), "ok": i32(NF, M)}))
    else:
        eng.sampling_log_prob_device(NF, ptrs({"o": f64(NF)})["o"])
    torch.cuda.synchronize()


@pytest.mark.parametrize("consumer", CONSUMERS)
@pytest.mark.parametrize("kind", PASSES)
def test_pass_rules(engine_mod, frames, consumer, kind):
    E = engine_mod
    fr = frames
    outcomes = []
    for change in CHANGES:
        eng = E.Engine(max_frames=NF, n_hyps=H)
        try:
            if change and change[1] == "clear":
                apply(eng, fr, change[0], True)
            if kind == "softam":
                eng.forward_device(NF, fr["coords"].data_ptr(), fr["pix"].data_ptr(), 0, fr["gt"].data_ptr())
            elif kind == "dsac":
                eng.forward_dsac_device(NF, fr["coords"].data_ptr(), fr["pix"].data_ptr(), 0, fr["gt"].data_ptr())
            torch.cuda.synchronize()
            if change:
                apply(eng, fr, change[0], change[1] == "set")
            want = expected(consumer, kind, change)
            try:
                consume(eng, consumer)
                got = None
            except RuntimeError as ex:
                got = str(ex)
            ok = got is None if want is None else (got is not None and want in got)
            outcomes.append((change, want, got, ok))
        finally:
            eng.close()
    bad = [o for o in outcomes if not o[3]]
    assert not bad, "\n".join("%s: want %r, got %r" % (c, w, g) for c, w, g, _ in bad)
