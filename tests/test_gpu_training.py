"""Training from PyTorch: the device-side backward entry points, the DSAC variant's device forward / backward and the
autograd losses of dsac_b200/autograd.py, against the host entry points and the oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_backward_device_equals_host_backward(engine_mod):
    """dsac_backward_device after dsac_forward_device on a non-default stream: the same dLoss/dObj as dsac_backward."""
    import torch
    E = engine_mod
    nf = 4
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, frame0=3)
    eng = E.Engine(max_frames=nf, n_hyps=64)
    s = torch.cuda.Stream()
    dc, dp, dg = _dev(coords), _dev(pix), _dev(gt_jp)
    out = torch.full((nf, E.N, 3), np.nan, dtype=torch.float64, device="cuda")
    with torch.cuda.stream(s):
        eng.forward_device(nf, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 3, s.cuda_stream)
        eng.backward_device(nf, d_dloss_dobj=out.data_ptr(), stream=s.cuda_stream)
    s.synchronize()
    ref = E.Engine(max_frames=nf, n_hyps=64)
    ref.forward(coords, pix, gt_jp, frame0=3)
    bw = ref.backward(coords, pix, gt_jp, full=False)
    assert np.array_equal(out.cpu().numpy(), bw.dloss_dobj)
    assert np.abs(bw.dloss_dobj).max() > 0


@pytest.mark.parametrize("T", [1, 4])
def test_dsac_forward_device_matches_oracle(engine_mod, oracle, T):
    """Device draw (k_dsac_draw) over 32 frames from frame0 = 5: drawn hypothesis, minimal sets, refinement steps and
    inlier maps (support cells zeroed on the device) equal the oracle's forward_dsac."""
    import torch
    E, O = engine_mod, oracle
    nf, H, frame0 = 32, 32, 5
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, frame0=frame0, n_streams=T)
    eng = E.Engine(max_frames=nf, n_hyps=H, n_streams=T)
    dc, dp, dg = _dev(coords), _dev(pix), _dev(gt_jp)
    hyp_idx = torch.empty(nf, dtype=torch.int32, device="cuda")
    img_idx = torch.empty((nf, H, 4), dtype=torch.int32, device="cuda")
    steps = torch.empty((nf, H), dtype=torch.int32, device="cuda")
    imaps = torch.empty((nf, H, E.N), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    eng.forward_dsac_device(nf, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), True, frame0, stream, hyp_idx=hyp_idx.data_ptr(),
                            img_idx=img_idx.data_ptr(), steps_done=steps.data_ptr(), inlier_maps=imaps.data_ptr())
    torch.cuda.synchronize()
    hyp_idx, img_idx, steps, imaps = (t.cpu().numpy() for t in (hyp_idx, img_idx, steps, imaps))
    drawn_not_max = 0
    for f in range(nf):
        cfg = O.default_config(seed=1305 + (frame0 + f) * T, n_hyps=H, n_streams=T)
        o = O.forward_dsac(cfg, coords[f], pix[f], gt_jp[f, :9], gt_jp[f, 9:], True)
        assert np.array_equal(o.img_idx, img_idx[f])
        assert o.hyp_idx == hyp_idx[f], f
        assert np.array_equal(o.steps_done, steps[f])
        assert np.array_equal(o.inlier_maps, imaps[f])
        drawn_not_max += int(o.hyp_idx != int(np.argmax(o.sf)))
    assert drawn_not_max > 0   # the draw is random, not the arg-max


def test_dsac_device_round_equals_host_round(engine_mod):
    """dsac_forward_dsac_device + dsac_backward_dsac_device against the host entry points on the same inputs."""
    import torch
    E = engine_mod
    nf, H = 6, 48
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, frame0=2)
    host = E.Engine(max_frames=nf, n_hyps=H)
    fw = host.forward_dsac(coords, pix, gt_jp, random_draw=True, frame0=2)
    bw = host.backward_dsac(nf)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    dc, dp, dg = _dev(coords), _dev(pix), _dev(gt_jp)
    exp = torch.empty(nf, dtype=torch.float64, device="cuda")
    pick = torch.empty(nf, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    outs = {"dloss_dobj": torch.empty((nf, E.N, 3), dtype=torch.float64, device="cuda"),
            "score_grads": torch.empty((nf, H), dtype=torch.float64, device="cuda"),
            "n_selected": torch.empty(nf, dtype=torch.int32, device="cuda"),
            "n_refine_jobs": torch.empty(nf, dtype=torch.int32, device="cuda")}
    with torch.cuda.stream(s):
        eng.forward_dsac_device(nf, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), True, 2, s.cuda_stream,
                                expected_loss=exp.data_ptr(), hyp_idx=pick.data_ptr())
        eng.backward_dsac_device(nf, stream=s.cuda_stream, **{k: v.data_ptr() for k, v in outs.items()})
    s.synchronize()
    assert np.array_equal(pick.cpu().numpy(), fw.hyp_idx)
    assert np.array_equal(exp.cpu().numpy(), fw.expected_loss)
    assert np.array_equal(outs["n_selected"].cpu().numpy(), bw.n_selected) and bw.n_selected.min() >= 1
    assert np.array_equal(outs["n_refine_jobs"].cpu().numpy(), bw.n_refine_jobs)
    assert np.array_equal(outs["score_grads"].cpu().numpy(), bw.score_grads)
    d = outs["dloss_dobj"].cpu().numpy()
    assert np.abs(d - bw.dloss_dobj).max() <= 1e-5 * np.abs(bw.dloss_dobj).max()
    assert np.abs(bw.dloss_dobj).max() > 0


def _prediction(coords, seed=0, noise_mm=0.0):
    import torch
    rng = np.random.default_rng(seed)
    p = coords.astype(np.float32) / np.float32(1000) + (rng.normal(0, noise_mm, coords.shape) / 1000).astype(np.float32)
    return torch.from_numpy(p).cuda()


@pytest.mark.parametrize("variant", ["softam", "dsac"])
@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_autograd_hand_off(engine_mod, variant, reduction):
    """prediction.grad = float32(g * clip(dLoss/dObj, +-0.1)) with dLoss/dObj from the host entry points on the coordinates
    the loss rounded the prediction to; the loss equals the host forward's."""
    import torch
    from dsac_b200.autograd import dsac_expected_loss, softam_loss
    E = engine_mod
    nf, H, frame0 = 16, 64, 7
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf, frame0=frame0)
    pred = _prediction(coords, seed=1, noise_mm=3.0).requires_grad_(True)
    eng = E.Engine(max_frames=nf, n_hyps=H)
    dpix, dgt = _dev(pix), _dev(gt_jp)
    fn = softam_loss if variant == "softam" else dsac_expected_loss
    loss = fn(eng, pred, dpix, dgt, frame0=frame0)
    (loss.sum() if reduction == "sum" else loss.mean()).backward()
    torch.cuda.synchronize()
    q = torch.empty((nf, E.N, 3), dtype=torch.int16, device="cuda")
    eng.coords_from_prediction_device(nf, pred.detach().data_ptr(), q.data_ptr())
    torch.cuda.synchronize()
    qc = q.cpu().numpy()
    ref = E.Engine(max_frames=nf, n_hyps=H)
    if variant == "softam":
        fw = ref.forward(qc, pix, gt_jp, frame0=frame0)
        want_loss = fw.loss
        dobj = ref.backward(qc, pix, gt_jp, full=False).dloss_dobj
    else:
        fw = ref.forward_dsac(qc, pix, gt_jp, random_draw=True, frame0=frame0)
        want_loss = fw.expected_loss
        dobj = ref.backward_dsac(nf).dloss_dobj
    assert np.array_equal(loss.detach().cpu().numpy(), want_loss)
    g = 1.0 if reduction == "sum" else 1.0 / nf
    want = (g * np.clip(dobj, -0.1, 0.1)).astype(np.float32)
    got = pred.grad.cpu().numpy()
    if variant == "softam":
        assert np.array_equal(got, want)
    else:   # the DSAC variant's dLoss/dObj tolerance of test_gpu_backward.py
        assert np.abs(got - want).max() <= 1e-5 * max(1e-12, np.abs(want).max())
        assert np.mean(got == want) > 0.99
    assert np.abs(got).max() > 0


def test_autograd_misuse_raises(engine_mod):
    import torch
    from dsac_b200.autograd import dsac_expected_loss, softam_loss
    E = engine_mod
    nf = 2
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    eng = E.Engine(max_frames=nf, n_hyps=16)
    pred = _prediction(coords).requires_grad_(True)
    dpix, dgt = _dev(pix), _dev(gt_jp)
    for fn in (softam_loss, dsac_expected_loss):
        loss = fn(eng, pred, dpix, dgt)
        fn(eng, pred.detach(), dpix, dgt)          # a second pass on the same engine
        with pytest.raises(RuntimeError, match="another forward pass"):
            loss.sum().backward()
        with pytest.raises(ValueError, match="ground-truth"):
            fn(eng, pred, dpix, None)
        with pytest.raises(ValueError, match="is on cpu"):
            fn(eng, pred, torch.from_numpy(pix), dgt)


def test_sgd_on_a_per_cell_offset_lowers_the_softam_loss(engine_mod):
    """A learnable per-cell offset added to noisy predictions of fixed frames, trained with SGD through softam_loss."""
    import torch
    from dsac_b200.autograd import softam_loss
    E = engine_mod
    nf = 16
    coords, pix, gt_cv, gt_jp = E.synth_frames(nf)
    base = _prediction(coords, seed=2, noise_mm=20.0)
    eng = E.Engine(max_frames=nf, n_hyps=64)
    dpix, dgt = _dev(pix), _dev(gt_jp)
    offset = torch.zeros((1, E.N, 3), dtype=torch.float32, device="cuda", requires_grad=True)
    opt = torch.optim.SGD([offset], lr=SGD_LR)
    losses = []
    for _ in range(SGD_STEPS):
        opt.zero_grad()
        loss = softam_loss(eng, base + offset, dpix, dgt).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    with torch.no_grad():
        final = float(softam_loss(eng, base + offset, dpix, dgt).mean())
    assert final < losses[0], (losses, final)


SGD_LR, SGD_STEPS = 0.3, 3
