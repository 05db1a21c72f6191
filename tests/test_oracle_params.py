"""Pins the oracle to the REFERENCE'S OWN CODE at non-default parameters and cameras: the cases of
tests/golden/ref_params.npz (written by tests/golden/make_ref_params.py from oracle/_ref) -- inlier threshold, inlier
count, refinement steps, dRefineObj sub-sampling, alpha / beta, odd hypothesis counts, several sampler streams, a longer
focal length and an off-centre principal point, for processImage, the backward factors and the DSAC variant.

Tolerances as in tests/test_oracle_vs_ref.py: integer work (sampled indices, inlier maps, permutations, step counts) and
the diffmaps bit-exact; poses, scores, softmax, losses and all gradient factors 1e-12 relative.
"""
import os

import numpy as np
import pytest

from test_oracle_vs_ref import check_forward, rel, rel_sampled, same

PARAMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_params.npz")


def _cases():
    z = np.load(PARAMS)
    names = sorted({k.split("/")[0] for k in z.files})
    return {n: {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(n + "/")} for n in names}


CASES = _cases()


def _config(O, r):
    H, T, g = int(r["H"]), int(r["T"]), int(r["frame"])
    f, cx, cy = (float(v) for v in r["camera"])
    return O.default_config(seed=1305 + g * T, n_hyps=H, n_streams=T, f=f, cx=cx, cy=cy, thr2d=int(r["thr2d"]),
                            inlier_count=int(r["inlier_count"]), ref_steps=int(r["ref_steps"]), sub_sample=float(r["sub_sample"]),
                            alpha=float(r["alpha"]), beta=float(r["beta"]))


def test_the_cases_cover_the_parameters():
    rs = CASES.values()
    assert len(CASES) >= 8
    assert {int(r["thr2d"]) for r in rs} >= {3, 5, 10, 20}
    assert {int(r["inlier_count"]) for r in rs} >= {60, 100, 128}
    assert {int(r["ref_steps"]) for r in rs} >= {3, 8, 12, 16}
    assert any(int(r["H"]) % 8 for r in rs) and any(int(r["T"]) > 1 for r in rs)
    assert len({tuple(r["camera"]) for r in rs}) >= 3
    assert any(str(r["kind"]) == "dsac_forward" for r in rs)
    # dRefine/dObj is exactly zero where every perturbed refinement ends where the unperturbed one does (fwd_thr3)
    assert sum(float(r["dref_dobj_absmax"]) > 0 for r in rs if str(r["kind"]) == "forward") >= 5


@pytest.mark.parametrize("name", [n for n, r in CASES.items() if str(r["kind"]) == "forward"])
def test_forward_and_factors_equal_the_references(oracle, name):
    O = oracle
    r = CASES[name]
    H = int(r["H"])
    cfg = _config(O, r)
    o = O.forward(cfg, r["coords"], r["pix"], r["gt_R"], r["gt_t"])
    assert o.n_fragile == 0
    check_forward(o, r, H)
    assert same(o.diffmaps, r, "diffmaps", np.float32)
    assert same(o.pixel_idxs, r, "pixel_idxs")
    ob = O.backward(cfg, r["coords"], r["pix"], r["gt_R"], r["gt_t"], o)
    assert rel(ob.dloss_dref, r["dloss_dref"]) <= 1e-12
    assert rel(ob.dref_dhyp, r["dref_dhyp"]) <= 1e-12
    dobj = np.asarray(ob.dref_dobj).reshape(6, -1)
    cols = r["dref_dobj_cols"]
    assert rel_sampled(dobj, np.ravel_multi_index(np.ix_(np.arange(6), cols), dobj.shape), r["dref_dobj"], r["dref_dobj_absmax"]) <= 1e-12
    dpnp = np.asarray(ob.dpnp).reshape(H, 6, 12)
    assert abs(np.abs(dpnp).max() - float(r["dpnp_absmax"])) <= 1e-12 * float(r["dpnp_absmax"])
    assert np.abs(dpnp[r["dpnp_hyps"]] - r["dpnp"]).max() <= 1e-12 * float(r["dpnp_absmax"])


@pytest.mark.parametrize("name", [n for n, r in CASES.items() if str(r["kind"]) == "dsac_forward"])
def test_dsac_variant_forward_equals_the_references(oracle, name):
    O = oracle
    r = CASES[name]
    o = O.forward_dsac(_config(O, r), r["coords"], r["pix"], r["gt_R"], r["gt_t"], True)
    assert same(o.img_idx, r, "img_idx") and o.hyp_idx == int(r["hyp_idx"]) and o.correct == int(r["correct"])
    assert same(o.inlier_maps, r, "inlier_maps")
    assert rel(o.hyp_rvec, r["hyp_rvec"]) <= 1e-12 and rel(o.hyp_tvec, r["hyp_tvec"]) <= 1e-12
    assert np.abs(o.sf - r["sf"]).max() <= 1e-12 and rel(o.ref_pose, r["ref_pose"]) <= 1e-12
    assert np.abs(o.losses - r["losses"]).max() <= 1e-9 and abs(o.expected_loss - float(r["expected_loss"])) <= 1e-10
    assert abs(o.rot_err - float(r["rot_err"])) <= 1e-9 and abs(o.t_err - float(r["t_err"])) <= 1e-9
