"""The engine's losses and refined poses as differentiable PyTorch functions, for training the coordinate CNN end to end.

    loss = softam_loss(engine, prediction, pix, gt_jp)              # soft-argmax pipeline, [n]
    loss = dsac_expected_loss(engine, prediction, pix, gt_jp)       # DSAC / RANSAC variant, [n]
    loss.sum().backward()                                           # prediction.grad

    pose = softam_pose(engine, prediction, pix)                     # refined jp 6-vector per frame, [n][6]
    sf, ref = dsac_hypotheses(engine, prediction, pix)              # softmax [n][H], refined jp 6-vectors [n][H][6]
    my_loss(pose).backward()                                        # prediction.grad, no ground truth needed
    unc = pose_uncertainty(engine, n)                               # covariances and support of the last pass's poses
    modes = pose_modes(engine, n, 4, 0.17, 100.0)                   # up to 4 distinct refined poses per frame
    loss = rig_softam_loss(engine, prediction, pix, ext, C, gt_rig)  # one loss per rig of C cameras, [n / C]
    pose = rig_softam_pose(engine, prediction, pix, ext, C)          # refined jp 6-vector per rig, [n / C][6]
    modes = rig_pose_modes(engine, n, C, 4, 0.17, 100.0)             # up to 4 distinct refined poses per rig

`prediction` is the coordinate CNN's output: float32 [n][1600][3] scene coordinates in metres on the engine's device,
cell y*40+x.  It is the only input that receives a gradient.  The gradient is the one the reference hands to
model:backward (lua/train_obj_softam.lua:101-105): dLoss/dObj clamped to +-clamp, scaled by the incoming gradient, per
millimetre of the int16 grid, straight through the rounding to millimetres (DESIGN.md quirk Q12).

The pose outputs are jp 6-vectors [rodrigues(R); t in mm], the vector the reference's refine() and dLossMax work on.
Their backward is the reference's chain with the incoming gradient in place of dLossMax (INTEGRATION.md, "Pose-valued
outputs"): it inherits the reference's finite differences and quirks, and the clamp applies to the total dLoss/dObj,
since the incoming gradient is already inside it.

`cameras` (float64 [n][3] = focal, cx, cy of every frame; a host array or CPU tensor) gives each frame of the batch its
own camera: it is applied with Engine.set_cameras before the forward, on the current stream, and stays in force on the
engine.  None leaves the engine's setting alone.  Changing the cameras between a loss and its backward() makes that
backward() raise.

`sampling_logits` (float32 [n][1600] on the engine's device, cell y*40+x) draws the pass's minimal sets from
softmax(logits) instead of uniformly (guided sampling, INTEGRATION.md): the engine reads a detached copy, applied before
the forward on the current stream, and the setting stays in force on the engine; None leaves it alone.
sampling_log_prob(engine, logits) is then the log-probability of that draw, float64 [n], differentiable with respect to
the logits, for a REINFORCE-style gradient:

    loss = softam_loss(engine, pred, pix, gt_jp, frame0=g0, sampling_logits=logits)
    logp = sampling_log_prob(engine, logits)
    (loss + (loss.detach() - baseline) * logp).sum().backward()

`cell_depth` (float32 [n][1600] on the engine's device, depth in mm at each cell's grid pixel; cell_depth() gathers it
from registered depth maps) makes the pass an RGB-D pass (INTEGRATION.md, "RGB-D localisation"): hypotheses and
refinement are Kabsch fits of scene to eye coordinates.  Like sampling_logits, the engine reads a detached copy applied on
the current stream, and None leaves the setting alone.  The gradient goes to `prediction` only: depth is not differentiated.

`pose_priors` = (poses, info, gate) puts k caller poses per frame into the hypothesis pool (INTEGRATION.md, "Pose
priors"): poses float64 [n][k][6] cv poses, info float64 [n][k][6][6] information matrices or None (no gate), gate the
chi^2 bound of the gate.  Like cell_depth, the engine reads a detached copy applied on the current stream, and None
leaves the setting alone.  The priors are constants: no gradient flows to them.

`derivatives` ("central" or "implicit") selects the scene-coordinate derivatives of the backward (INTEGRATION.md,
"Implicit-function gradients"): it is applied to the engine right before the backward call and stays in force there;
None leaves the engine's setting alone.

Everything stays on the device, on torch.cuda.current_stream().  The engine holds one pass: a forward on the same engine
between a loss and its backward() makes that backward() raise.
"""
import torch

from . import engine as _E


def _check_inputs(engine, prediction, pix, gt_jp, need_gt=True):
    dev = torch.device("cuda", engine.cfg.device)
    if gt_jp is None and need_gt:
        raise ValueError("the loss needs the ground-truth poses gt_jp [n][12]")
    n = prediction.shape[0] if prediction.dim() == 3 else -1
    if prediction.dtype != torch.float32 or tuple(prediction.shape[1:]) != (_E.N, 3) or prediction.dim() != 3:
        raise ValueError("prediction must be float32 [n][%d][3], got %s %s" % (_E.N, prediction.dtype, tuple(prediction.shape)))
    if not 1 <= n <= engine.cfg.max_frames:
        raise ValueError("%d frames, the engine holds 1..%d" % (n, engine.cfg.max_frames))
    for name, t in (("prediction", prediction), ("pix", pix), ("gt_jp", gt_jp)):
        if t is not None and t.device != dev:
            raise ValueError("%s is on %s, the engine on %s" % (name, t.device, dev))
    if pix.dtype != torch.int32 or pix.numel() not in (_E.N * 2, n * _E.N * 2):
        raise ValueError("pix must be int32 [N][2] (shared) or [n][N][2]")
    if gt_jp is not None and (gt_jp.dtype != torch.float64 or gt_jp.numel() != n * 12):
        raise ValueError("gt_jp must be float64 [n][12]")
    return n, pix.contiguous(), gt_jp.contiguous() if gt_jp is not None else None, (1 if pix.numel() == _E.N * 2 else 0)


def _set_cameras(engine, prediction, cameras):
    if cameras is not None:
        engine.set_cameras(cameras, torch.cuda.current_stream(prediction.device).cuda_stream)


def _set_sampling(engine, prediction, logits):
    if logits is None:
        return
    n = prediction.shape[0]
    if logits.dtype != torch.float32 or tuple(logits.shape) != (n, _E.N) or logits.device != prediction.device:
        raise ValueError("sampling_logits must be float32 [%d][%d] on %s, got %s %s on %s"
                         % (n, _E.N, prediction.device, logits.dtype, tuple(logits.shape), logits.device))
    copy = logits.detach().contiguous()
    stream = torch.cuda.current_stream(prediction.device)
    engine.set_sampling_logits_device(n, copy.data_ptr(), stream.cuda_stream)
    copy.record_stream(stream)
    # the pass that follows is sampled with this tensor as it is now (sampling_log_prob checks identity and version)
    engine._sampling_key = (id(logits), logits._version, engine.passes + 1)


def _set_depth(engine, prediction, depth, n_cameras=None):
    # n_cameras: the rig passes' setting (set_rig_cell_depth_device) rather than the ordinary passes'
    if depth is None:
        return
    n = prediction.shape[0]
    if depth.dtype != torch.float32 or tuple(depth.shape) != (n, _E.N) or depth.device != prediction.device:
        raise ValueError("cell_depth must be float32 [%d][%d] on %s, got %s %s on %s"
                         % (n, _E.N, prediction.device, depth.dtype, tuple(depth.shape), depth.device))
    copy = depth.detach().contiguous()
    stream = torch.cuda.current_stream(prediction.device)
    if n_cameras is None:
        engine.set_cell_depth_device(n, copy.data_ptr(), stream.cuda_stream)
    else:
        engine.set_rig_cell_depth_device(n, int(n_cameras), copy.data_ptr(), stream.cuda_stream)
    copy.record_stream(stream)


def cell_depth(depth, pix):
    """Per-cell depth float32 [n][1600] (mm) for cell_depth=: the registered uint16 depth maps `depth` [n][H][W] (mm, on
    the RGB camera, e.g. dsac_register_depth_device's output) at the cells' grid pixels `pix` (int32 [1600][2] shared or
    [n][1600][2], (x, y)).  0 and 65535 (7-Scenes' invalid value, DESIGN.md Q13) are missing depth (NaN), as are pixels
    outside the map."""
    if depth.dim() != 3 or depth.dtype.is_floating_point or depth.dtype == torch.bool:
        raise ValueError("depth must be uint16 [n][H][W], got %s %s" % (depth.dtype, tuple(depth.shape)))
    n, Hh, W = depth.shape
    p = pix.reshape(-1, _E.N, 2).to(torch.int64).expand(n, _E.N, 2)
    x, y = p[..., 0], p[..., 1]
    inside = (x >= 0) & (x < W) & (y >= 0) & (y < Hh)
    flat = depth.reshape(n, -1).to(torch.int64) & 0xffff   # (int16 storage holds the uint16 values too)
    d = torch.gather(flat, 1, (y.clamp(0, Hh - 1) * W + x.clamp(0, W - 1)))
    out = d.to(torch.float32)
    bad = ~inside | (d == 0) | (d == 65535)
    return torch.where(bad, torch.full_like(out, float("nan")), out)


def _coords(engine, prediction, stream):
    n = prediction.shape[0]
    coords = torch.empty((n, _E.N, 3), dtype=torch.int16, device=prediction.device)
    engine.coords_from_prediction_device(n, prediction.data_ptr(), coords.data_ptr(), stream)
    return coords


def _grad_input(ctx, grad_loss):
    if ctx.engine.passes != ctx.pass_id:
        raise RuntimeError("the engine ran another forward pass after this loss was computed: its backward() would "
                           "differentiate that pass; call backward() before the next forward, or use a second engine")
    g = grad_loss.detach().to(torch.float64).contiguous()
    return g, torch.empty((ctx.n, _E.N, 3), dtype=torch.float32, device=g.device)


class _SoftamLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, prediction, engine, pix, gt_jp, frame0, clamp, derivatives):
        n, pix, gt_jp, shared = _check_inputs(engine, prediction, pix, gt_jp)
        stream = torch.cuda.current_stream(prediction.device).cuda_stream
        pred = prediction.detach().contiguous()
        coords = _coords(engine, pred, stream)
        engine.forward_device(n, coords.data_ptr(), pix.data_ptr(), shared, gt_jp.data_ptr(), frame0, stream)
        loss = torch.empty(n, dtype=torch.float64, device=prediction.device)
        engine.fetch_device(n, stream, loss=loss.data_ptr())
        ctx.engine, ctx.pass_id, ctx.n, ctx.clamp = engine, engine.passes, n, clamp
        ctx.derivatives = derivatives
        ctx.keep = (coords, pix, gt_jp)   # the engine's backward reads the pass's inputs
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        g, grad = _grad_input(ctx, grad_loss)
        _apply_deriv(ctx)
        ctx.engine.backward_device(ctx.n, g.data_ptr(), None, grad.data_ptr(), ctx.clamp, torch.cuda.current_stream(g.device).cuda_stream)
        return grad, None, None, None, None, None, None


class _DsacExpectedLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, prediction, engine, pix, gt_jp, frame0, random_draw, clamp, derivatives):
        n, pix, gt_jp, shared = _check_inputs(engine, prediction, pix, gt_jp)
        stream = torch.cuda.current_stream(prediction.device).cuda_stream
        coords = _coords(engine, prediction.detach().contiguous(), stream)
        loss = torch.empty(n, dtype=torch.float64, device=prediction.device)
        engine.forward_dsac_device(n, coords.data_ptr(), pix.data_ptr(), shared, gt_jp.data_ptr(), random_draw, frame0, stream,
                                   expected_loss=loss.data_ptr())
        ctx.engine, ctx.pass_id, ctx.n, ctx.clamp = engine, engine.passes, n, clamp
        ctx.derivatives = derivatives
        ctx.keep = (coords, pix, gt_jp)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        g, grad = _grad_input(ctx, grad_loss)
        _apply_deriv(ctx)
        ctx.engine.backward_dsac_device(ctx.n, g.data_ptr(), grad.data_ptr(), ctx.clamp, torch.cuda.current_stream(g.device).cuda_stream)
        return grad, None, None, None, None, None, None, None


class _SoftamPose(torch.autograd.Function):
    @staticmethod
    def forward(ctx, prediction, engine, pix, frame0, clamp, derivatives):
        n, pix, _, shared = _check_inputs(engine, prediction, pix, None, need_gt=False)
        stream = torch.cuda.current_stream(prediction.device).cuda_stream
        coords = _coords(engine, prediction.detach().contiguous(), stream)
        engine.forward_device(n, coords.data_ptr(), pix.data_ptr(), shared, None, frame0, stream)
        pose = torch.empty((n, 6), dtype=torch.float64, device=prediction.device)
        engine.refined_jp6_device(n, pose.data_ptr(), stream)
        ctx.engine, ctx.pass_id, ctx.n, ctx.clamp = engine, engine.passes, n, clamp
        ctx.derivatives = derivatives
        ctx.keep = (coords, pix)
        return pose

    @staticmethod
    def backward(ctx, grad_pose):
        seed, grad = _grad_input(ctx, grad_pose)
        _apply_deriv(ctx)
        ctx.engine.backward_pose_device(ctx.n, seed.data_ptr(), None, grad.data_ptr(), ctx.clamp,
                                        torch.cuda.current_stream(seed.device).cuda_stream)
        return grad, None, None, None, None, None


class _DsacHypotheses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, prediction, engine, pix, frame0, random_draw, clamp, derivatives):
        n, pix, _, shared = _check_inputs(engine, prediction, pix, None, need_gt=False)
        stream = torch.cuda.current_stream(prediction.device).cuda_stream
        coords = _coords(engine, prediction.detach().contiguous(), stream)
        H = engine.cfg.n_hyps
        sf = torch.empty((n, H), dtype=torch.float64, device=prediction.device)
        engine.forward_dsac_device(n, coords.data_ptr(), pix.data_ptr(), shared, None, random_draw, frame0, stream,
                                   sf=sf.data_ptr())
        ref = torch.empty((n, H, 6), dtype=torch.float64, device=prediction.device)
        engine.refined_jp6_device(n, ref.data_ptr(), stream)
        ctx.engine, ctx.pass_id, ctx.n, ctx.clamp = engine, engine.passes, n, clamp
        ctx.derivatives = derivatives
        ctx.keep = (coords, pix)
        ctx.set_materialize_grads(False)   # an unused output skips its path of the backward
        return sf, ref

    @staticmethod
    def backward(ctx, grad_sf, grad_ref):
        seeds = [g for g in (grad_sf, grad_ref) if g is not None]
        if not seeds:
            return None, None, None, None, None, None, None
        _, grad = _grad_input(ctx, seeds[0])
        ptr = [g.detach().to(torch.float64).contiguous() if g is not None else None for g in (grad_sf, grad_ref)]
        _apply_deriv(ctx)
        ctx.engine.backward_dsac_pose_device(ctx.n, ptr[1].data_ptr() if ptr[1] is not None else None,
                                             ptr[0].data_ptr() if ptr[0] is not None else None, grad.data_ptr(), ctx.clamp,
                                             torch.cuda.current_stream(grad.device).cuda_stream)
        return grad, None, None, None, None, None, None


def _deriv(derivatives):
    if derivatives not in (None, "central", "implicit"):
        raise ValueError("derivatives must be None, 'central' or 'implicit', got %r" % (derivatives,))
    return derivatives


def _set_priors(engine, prediction, priors):
    if priors is None:
        return
    poses, info, gate = priors
    n = prediction.shape[0]
    if poses.dtype != torch.float64 or poses.dim() != 3 or poses.shape[0] != n or poses.shape[2] != 6 \
            or poses.device != prediction.device:
        raise ValueError("pose_priors poses must be float64 [%d][k][6] on %s, got %s %s on %s"
                         % (n, prediction.device, poses.dtype, tuple(poses.shape), poses.device))
    k = poses.shape[1]
    if info is not None and (info.dtype != torch.float64 or tuple(info.shape) != (n, k, 6, 6) or info.device != prediction.device):
        raise ValueError("pose_priors info must be float64 [%d][%d][6][6] on %s, got %s %s on %s"
                         % (n, k, prediction.device, info.dtype, tuple(info.shape), info.device))
    pc = poses.detach().contiguous()
    ic = info.detach().contiguous() if info is not None else None
    stream = torch.cuda.current_stream(prediction.device)
    engine.set_pose_priors_device(n, k, pc.data_ptr(), ic.data_ptr() if ic is not None else None, float(gate), stream.cuda_stream)
    pc.record_stream(stream)
    if ic is not None:
        ic.record_stream(stream)


def _apply_deriv(ctx):
    # the engine reads the setting when the backward starts; None leaves it as it is
    if ctx.derivatives is not None:
        ctx.engine.set_coord_derivatives(ctx.derivatives)


def softam_loss(engine, prediction, pix, gt_jp, frame0=0, clamp=0.1, cameras=None, sampling_logits=None, cell_depth=None,
                derivatives=None, pose_priors=None):
    """Per-frame loss of the soft-argmax pipeline (train_ransac_softam.cpp) on `prediction`, float64 [n]; differentiable
    with respect to `prediction`.  frame0: global index of the first frame (keys the sampler streams)."""
    _set_cameras(engine, prediction, cameras)
    _set_sampling(engine, prediction, sampling_logits)
    _set_depth(engine, prediction, cell_depth)
    _set_priors(engine, prediction, pose_priors)
    return _SoftamLoss.apply(prediction, engine, pix, gt_jp, int(frame0), float(clamp), _deriv(derivatives))


def dsac_expected_loss(engine, prediction, pix, gt_jp, frame0=0, random_draw=True, clamp=0.1, cameras=None,
                       sampling_logits=None, cell_depth=None, derivatives=None, pose_priors=None):
    """Per-frame expected loss of the DSAC / RANSAC variant (train_ransac.cpp) on `prediction`, float64 [n];
    differentiable with respect to `prediction`."""
    _set_cameras(engine, prediction, cameras)
    _set_sampling(engine, prediction, sampling_logits)
    _set_depth(engine, prediction, cell_depth)
    _set_priors(engine, prediction, pose_priors)
    return _DsacExpectedLoss.apply(prediction, engine, pix, gt_jp, int(frame0), bool(random_draw), float(clamp), _deriv(derivatives))


def softam_pose(engine, prediction, pix, frame0=0, clamp=0.1, cameras=None, sampling_logits=None, cell_depth=None,
                derivatives=None, pose_priors=None):
    """Refined pose of every frame of the soft-argmax pipeline as a jp 6-vector [rodrigues(R); t in mm], float64 [n][6];
    differentiable with respect to `prediction`.  Needs no ground truth."""
    _set_cameras(engine, prediction, cameras)
    _set_sampling(engine, prediction, sampling_logits)
    _set_depth(engine, prediction, cell_depth)
    _set_priors(engine, prediction, pose_priors)
    return _SoftamPose.apply(prediction, engine, pix, int(frame0), float(clamp), _deriv(derivatives))


def dsac_hypotheses(engine, prediction, pix, frame0=0, random_draw=True, clamp=0.1, cameras=None, sampling_logits=None,
                    cell_depth=None, derivatives=None, pose_priors=None):
    """(sf [n][H], refined jp 6-vectors [n][H][6]) of the DSAC / RANSAC variant, both float64 and differentiable with
    respect to `prediction`.  The gradient through the poses covers the hypotheses with sf > 1e-4 whose incoming
    gradient is nonzero; an output that receives no gradient costs nothing in the backward."""
    _set_cameras(engine, prediction, cameras)
    _set_sampling(engine, prediction, sampling_logits)
    _set_depth(engine, prediction, cell_depth)
    _set_priors(engine, prediction, pose_priors)
    return _DsacHypotheses.apply(prediction, engine, pix, int(frame0), bool(random_draw), float(clamp), _deriv(derivatives))


def pose_uncertainty(engine, n):
    """Uncertainty of the refined poses of the engine's last pass over n frames (INTEGRATION.md, "Pose uncertainty"), a
    dict of device tensors on torch.cuda.current_stream(): after softam_pose / softam_loss, one entry per frame
    (cov_jp6 and cov_xi float64 [n][6][6], sigma2 float64 [n], n_fit, support and ok int32 [n]); after dsac_hypotheses /
    dsac_expected_loss, one per hypothesis ([n][H][6][6], [n][H]).  cov_xi is the Gauss-Newton covariance of the last
    refinement step's fit, in the chart R = exp([w]x) R*, t = t* + tau (w rad, tau mm); cov_jp6 the same in the jp
    6-vector of the pose outputs.  These outputs are not differentiable: they carry no autograd history.  The shapes follow
    the pass the engine holds (Engine.last_pass), which is the pass the engine reads: a forward it refused leaves both as
    they were."""
    dev = torch.device("cuda", engine.cfg.device)
    lead = (n,) if engine.last_pass(n) == "softam" else (n, engine.cfg.n_hyps)
    out = {k: torch.empty(lead + (6, 6), dtype=torch.float64, device=dev) for k in ("cov_jp6", "cov_xi")}
    out["sigma2"] = torch.empty(lead, dtype=torch.float64, device=dev)
    for k in ("n_fit", "support", "ok"):
        out[k] = torch.empty(lead, dtype=torch.int32, device=dev)
    engine.pose_uncertainty_device(n, torch.cuda.current_stream(dev).cuda_stream, **{k: v.data_ptr() for k, v in out.items()})
    return out


def pose_modes(engine, n, max_modes, rot_rad, trans_mm):
    """The distinct refined poses of each frame's hypothesis pool after the engine's last pass over n frames, of either
    pipeline (INTEGRATION.md, "Pose modes"), a dict of device tensors on torch.cuda.current_stream(): n_modes int32 [n];
    hyp, members, steps_done, n_fit, support and ok int32 [n][M]; score, mass and sigma2 float64 [n][M]; pose float64
    [n][M][6] (cv poses, as the priors of pose_priors= take them); cov_xi float64 [n][M][6][6], M = max_modes.  Modes
    0 .. n_modes - 1 are in seed order (the best-scored first); later entries have hyp -1 and zeros.  Two poses are near
    iff their rotations differ by at most rot_rad and their translations by at most trans_mm.  These outputs carry no
    autograd history."""
    dev = torch.device("cuda", engine.cfg.device)
    M = int(max_modes)
    out = {"n_modes": torch.empty((n,), dtype=torch.int32, device=dev),
           "pose": torch.empty((n, M, 6), dtype=torch.float64, device=dev),
           "cov_xi": torch.empty((n, M, 6, 6), dtype=torch.float64, device=dev)}
    for k in ("score", "mass", "sigma2"):
        out[k] = torch.empty((n, M), dtype=torch.float64, device=dev)
    for k in ("hyp", "members", "steps_done", "n_fit", "support", "ok"):
        out[k] = torch.empty((n, M), dtype=torch.int32, device=dev)
    engine.pose_modes_device(n, M, rot_rad, trans_mm, torch.cuda.current_stream(dev).cuda_stream,
                             **{k: v.data_ptr() for k, v in out.items()})
    return out


def _set_rig_priors(engine, prediction, n_cameras, priors):
    if priors is None:
        return
    poses, info, gate = priors
    C = int(n_cameras)
    R = prediction.shape[0] // C
    if poses.dtype != torch.float64 or poses.dim() != 3 or poses.shape[0] != R or poses.shape[2] != 6 \
            or poses.device != prediction.device:
        raise ValueError("rig_priors poses must be float64 [%d][k][6] on %s, got %s %s on %s"
                         % (R, prediction.device, poses.dtype, tuple(poses.shape), poses.device))
    k = poses.shape[1]
    if info is not None and (info.dtype != torch.float64 or tuple(info.shape) != (R, k, 6, 6) or info.device != prediction.device):
        raise ValueError("rig_priors info must be float64 [%d][%d][6][6] on %s, got %s %s on %s"
                         % (R, k, prediction.device, info.dtype, tuple(info.shape), info.device))
    pc = poses.detach().contiguous()
    ic = info.detach().contiguous() if info is not None else None
    stream = torch.cuda.current_stream(prediction.device)
    engine.set_rig_pose_priors_device(prediction.shape[0], C, k, pc.data_ptr(), ic.data_ptr() if ic is not None else None,
                                      float(gate), stream.cuda_stream)
    pc.record_stream(stream)
    if ic is not None:
        ic.record_stream(stream)


def rig_pose_uncertainty(engine, n, n_cameras):
    """Covariance of each refined rig pose of the engine's last rig pass over n frames of n_cameras cameras (INTEGRATION.md,
    "Rig tracking"), a dict of device tensors on torch.cuda.current_stream(), one entry per rig (R = n / n_cameras):
    cov_jp6 and cov_xi float64 [R][6][6], sigma2 float64 [R], n_fit, support and ok int32 [R], as pose_uncertainty's in the
    rig chart.  inv(cov_xi + Q) is an information matrix for rig_priors=.  These outputs carry no autograd history."""
    dev = torch.device("cuda", engine.cfg.device)
    R = n // int(n_cameras)
    out = {k: torch.empty((R, 6, 6), dtype=torch.float64, device=dev) for k in ("cov_jp6", "cov_xi")}
    out["sigma2"] = torch.empty((R,), dtype=torch.float64, device=dev)
    for k in ("n_fit", "support", "ok"):
        out[k] = torch.empty((R,), dtype=torch.int32, device=dev)
    engine.rig_pose_uncertainty_device(n, int(n_cameras), torch.cuda.current_stream(dev).cuda_stream,
                                       **{k: v.data_ptr() for k, v in out.items()})
    return out


def rig_pose_modes(engine, n, n_cameras, max_modes, rot_rad, trans_mm):
    """The distinct refined rig poses of each rig's pool after the engine's last rig pass over n frames of n_cameras
    cameras (INTEGRATION.md, "Rig pose modes"), a dict of device tensors on torch.cuda.current_stream() shaped as
    pose_modes shapes them, one row per rig (R = n / n_cameras): n_modes int32 [R]; hyp, members, steps_done, n_fit,
    support and ok int32 [R][M]; score, mass and sigma2 float64 [R][M]; pose float64 [R][M][6] (cv rig poses, as the
    poses of rig_priors= take them); cov_xi float64 [R][M][6][6] in the rig chart, M = max_modes.  hyp is the pool slot
    c * n_hyps + h of the mode's seed (an index into rig_pose's rig_hyp, scores and sf), -1 for an unused entry.  These
    outputs carry no autograd history."""
    dev = torch.device("cuda", engine.cfg.device)
    R, M = n // int(n_cameras), int(max_modes)
    out = {"n_modes": torch.empty((R,), dtype=torch.int32, device=dev),
           "pose": torch.empty((R, M, 6), dtype=torch.float64, device=dev),
           "cov_xi": torch.empty((R, M, 6, 6), dtype=torch.float64, device=dev)}
    for k in ("score", "mass", "sigma2"):
        out[k] = torch.empty((R, M), dtype=torch.float64, device=dev)
    for k in ("hyp", "members", "steps_done", "n_fit", "support", "ok"):
        out[k] = torch.empty((R, M), dtype=torch.int32, device=dev)
    engine.rig_pose_modes_device(n, int(n_cameras), M, rot_rad, trans_mm, torch.cuda.current_stream(dev).cuda_stream,
                                 **{k: v.data_ptr() for k, v in out.items()})
    return out


def _check_rig(engine, prediction, pix, cam_from_rig, n_cameras, gt_jp):
    C = int(n_cameras)
    n, pix, _, shared = _check_inputs(engine, prediction, pix, None, need_gt=False)
    dev = prediction.device
    if not 1 <= C <= _E.MAX_RIG_CAMERAS or n % C:
        raise ValueError("n_cameras %d must be in [1, %d] and divide the %d frames" % (C, _E.MAX_RIG_CAMERAS, n))
    R = n // C
    if cam_from_rig.dtype != torch.float64 or cam_from_rig.numel() != n * 6 or cam_from_rig.device != dev:
        raise ValueError("cam_from_rig must be float64 [%d][6] on %s" % (n, dev))
    if gt_jp is not None and (gt_jp.dtype != torch.float64 or gt_jp.numel() != R * 12 or gt_jp.device != dev):
        raise ValueError("gt_jp must be float64 [%d][12] on %s" % (R, dev))
    return C, n, R, pix, shared


class _RigSoftam(torch.autograd.Function):
    """The rig pass with the loss per rig (gt_jp given) or the refined rig jp 6-vector (gt_jp None) as its output."""

    @staticmethod
    def forward(ctx, prediction, engine, pix, cam_from_rig, n_cameras, gt_jp, frame0, clamp):
        C, n, R, pix, shared = _check_rig(engine, prediction, pix, cam_from_rig, n_cameras, gt_jp)
        dev = prediction.device
        stream = torch.cuda.current_stream(dev).cuda_stream
        coords = _coords(engine, prediction.detach().contiguous(), stream)
        ext = cam_from_rig.detach().contiguous()
        gt = gt_jp.detach().contiguous() if gt_jp is not None else None
        if gt is not None:
            out = torch.empty((R,), dtype=torch.float64, device=dev)
            engine.forward_rig_device(n, C, coords.data_ptr(), pix.data_ptr(), ext.data_ptr(), shared, gt.data_ptr(), frame0, stream,
                                      loss=out.data_ptr())
        else:
            out = torch.empty((R, 6), dtype=torch.float64, device=dev)
            engine.forward_rig_device(n, C, coords.data_ptr(), pix.data_ptr(), ext.data_ptr(), shared, None, frame0, stream)
            engine.rig_refined_jp6_device(n, out.data_ptr(), stream)
        ctx.engine, ctx.pass_id, ctx.n, ctx.clamp, ctx.loss = engine, engine.passes, n, clamp, gt is not None
        ctx.keep = (coords, pix, ext, gt)   # the rig backward reads the pass's inputs
        return out

    @staticmethod
    def backward(ctx, grad_out):
        g, grad = _grad_input(ctx, grad_out)
        stream = torch.cuda.current_stream(g.device).cuda_stream
        if ctx.loss:
            ctx.engine.backward_rig_device(ctx.n, g.data_ptr(), None, grad.data_ptr(), ctx.clamp, stream)
        else:
            ctx.engine.backward_rig_pose_device(ctx.n, g.data_ptr(), None, grad.data_ptr(), ctx.clamp, stream)
        return grad, None, None, None, None, None, None, None


def rig_softam_loss(engine, prediction, pix, cam_from_rig, n_cameras, gt_jp, frame0=0, clamp=0.1, cameras=None,
                    sampling_logits=None, rig_priors=None, cell_depth=None):
    """Per-rig loss of the rig pass (rig_pose's rig layout; INTEGRATION.md, "Rig gradients"): dLossMax's loss of each refined
    rig pose against gt_jp float64 [R][12], float64 [R]; differentiable with respect to `prediction` through every camera's
    scene coordinates, by the implicit-function derivatives whatever the engine's set_coord_derivatives.  clamp, cameras
    and sampling_logits as in softam_loss; with sampling_logits, sampling_log_prob gives the REINFORCE term of the rigs.
    rig_priors and cell_depth as in rig_pose; the priors and the depth are constants of the gradient."""
    if gt_jp is None:
        raise ValueError("the loss needs the rig ground-truth poses gt_jp [R][12]")
    _check_rig(engine, prediction, pix, cam_from_rig, n_cameras, gt_jp)
    _set_cameras(engine, prediction, cameras)
    _set_sampling(engine, prediction, sampling_logits)
    _set_rig_priors(engine, prediction, n_cameras, rig_priors)
    _set_depth(engine, prediction, cell_depth, n_cameras)
    return _RigSoftam.apply(prediction, engine, pix, cam_from_rig, int(n_cameras), gt_jp, int(frame0), float(clamp))


def rig_softam_pose(engine, prediction, pix, cam_from_rig, n_cameras, frame0=0, clamp=0.1, cameras=None, sampling_logits=None,
                    rig_priors=None, cell_depth=None):
    """Refined pose of every rig as a jp 6-vector [rodrigues(R); t in mm] of the rig frame, float64 [R][6]; differentiable
    with respect to `prediction` as rig_softam_loss.  Needs no ground truth."""
    _check_rig(engine, prediction, pix, cam_from_rig, n_cameras, None)
    _set_cameras(engine, prediction, cameras)
    _set_sampling(engine, prediction, sampling_logits)
    _set_rig_priors(engine, prediction, n_cameras, rig_priors)
    _set_depth(engine, prediction, cell_depth, n_cameras)
    return _RigSoftam.apply(prediction, engine, pix, cam_from_rig, int(n_cameras), None, int(frame0), float(clamp))


def rig_pose(engine, prediction, pix, cam_from_rig, n_cameras, frame0=0, cameras=None, sampling_logits=None, gt_jp=None,
             rig_priors=None, cell_depth=None):
    """One pose per multi-camera rig (INTEGRATION.md, "Multi-camera rigs"): the n frames of `prediction` are R = n / C rigs
    of C = n_cameras cameras, frame r C + c camera c of rig r, whose extrinsic cam_from_rig[r C + c] (float64 [n][6], a cv
    pose: X_cam = R_c X_rig + t_c) is known.  cameras and sampling_logits as in softam_pose, per frame; gt_jp float64
    [R][12] (the jp pose of the rig frame) adds loss, rot_err, t_err and correct.  A dict of device tensors on
    torch.cuda.current_stream(), without autograd history: hyp_pose [n][H][6]; rig_hyp [R][C H][6], scores and sf
    [R][C H]; entropy [R]; avg_pose and ref_pose [R][6] (cv poses of the rig); inlier_map int32 [n][1600]; steps_done int32,
    status int32 [R]; and with gt_jp loss, rot_err, t_err float64 and correct int32 [R].
    rig_priors = (poses float64 [R][k][6] cv rig poses, info float64 [R][k][6][6] or None, gate) puts k rig poses per rig
    into every camera's hypotheses (INTEGRATION.md, "Rig tracking"); sticky like pose_priors=: None leaves the engine's
    setting as it is, and Engine.set_rig_pose_priors_device(n, n_cameras, 0, None) clears it.
    cell_depth float32 [n][1600] (mm per cell of every camera frame, as cell_depth() gathers it) makes the rigs RGB-D:
    Kabsch hypotheses per camera and a Kabsch refinement of the rig pose over every camera's cells with depth
    (INTEGRATION.md, "RGB-D rigs"); sticky like rig_priors=, and Engine.set_rig_cell_depth_device(n, n_cameras, None)
    clears it."""
    C, n, R, pix, shared = _check_rig(engine, prediction, pix, cam_from_rig, n_cameras, gt_jp)
    dev, H = prediction.device, engine.cfg.n_hyps
    _set_cameras(engine, prediction, cameras)
    _set_sampling(engine, prediction, sampling_logits)
    _set_rig_priors(engine, prediction, C, rig_priors)
    _set_depth(engine, prediction, cell_depth, C)
    stream = torch.cuda.current_stream(dev).cuda_stream
    coords = _coords(engine, prediction.detach().contiguous(), stream)
    ext = cam_from_rig.detach().contiguous()
    gt = gt_jp.detach().contiguous() if gt_jp is not None else None
    f64 = dict(dtype=torch.float64, device=dev)
    i32 = dict(dtype=torch.int32, device=dev)
    out = {"hyp_pose": torch.empty((n, H, 6), **f64), "rig_hyp": torch.empty((R, C * H, 6), **f64),
           "scores": torch.empty((R, C * H), **f64), "sf": torch.empty((R, C * H), **f64), "entropy": torch.empty((R,), **f64),
           "avg_pose": torch.empty((R, 6), **f64), "ref_pose": torch.empty((R, 6), **f64),
           "inlier_map": torch.empty((n, _E.N), **i32), "steps_done": torch.empty((R,), **i32), "status": torch.empty((R,), **i32)}
    if gt is not None:
        out.update(loss=torch.empty((R,), **f64), rot_err=torch.empty((R,), **f64), t_err=torch.empty((R,), **f64),
                   correct=torch.empty((R,), **i32))
    engine.forward_rig_device(n, C, coords.data_ptr(), pix.data_ptr(), ext.data_ptr(), shared, gt.data_ptr() if gt is not None else None,
                              int(frame0), stream, **{k: v.data_ptr() for k, v in out.items()})
    engine._rig_inputs = (coords, pix, ext, gt)   # rig_pose_uncertainty reads the pass's inputs: alive until the next rig_pose
    return out


class _SamplingLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, engine):
        n = logits.shape[0]
        stream = torch.cuda.current_stream(logits.device).cuda_stream
        logp = torch.empty(n, dtype=torch.float64, device=logits.device)
        engine.sampling_log_prob_device(n, logp.data_ptr(), stream)
        ctx.engine, ctx.pass_id, ctx.n = engine, engine.passes, n
        return logp

    @staticmethod
    def backward(ctx, grad_logp):
        if ctx.engine.passes != ctx.pass_id:
            raise RuntimeError("the engine ran another forward pass after this log-probability was computed")
        g = grad_logp.detach().to(torch.float64).contiguous()
        grad = torch.empty((ctx.n, _E.N), dtype=torch.float32, device=g.device)
        ctx.engine.sampling_log_prob_backward_device(ctx.n, g.data_ptr(), grad.data_ptr(), torch.cuda.current_stream(g.device).cuda_stream)
        return grad, None


def sampling_log_prob(engine, logits):
    """Log-probability of the minimal sets the engine's last pass drew, float64 [n]: per frame the sum over every
    candidate up to each stream's last accepted one (accepted and rejected alike) of the log-probability of its four
    cells in draw order.  Differentiable with respect to `logits`, which must be the tensor that pass was sampled with
    (sampling_logits=), unmodified since."""
    key = getattr(engine, "_sampling_key", None)
    if key is None or key[0] != id(logits) or key[1] != logits._version or key[2] != engine.passes:
        raise RuntimeError("the engine's last pass was not sampled with this logits tensor as it is now "
                           "(pass it as sampling_logits= to the forward, and do not modify it in between)")
    return _SamplingLogProb.apply(logits, engine)
