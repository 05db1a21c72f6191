"""Pre-training of the coordinate CNN from RGB-D frames (the reference's train_obj.cpp with lua/train_obj.lua and
MyL1Criterion.lua), with the data path on the device:

    RGBDScene      BGR frames, raw depth and ground-truth poses in HBM; depth registered once (Dataset::getDepth)
    ObjRound       assembleData: the ThreadRand streams' draw of images and patch centres, labels from getObj
    l1_criterion   MyL1Criterion: batch mean of ||pred - gt||_2, gradient (pred - gt) / dist / count
    Torch7Adam     optim.adam as torch7 writes it
    ObjPretrainer  the reference's schedule: fixed permutation, batches of 64, lr 1e-4 halved every 50 000 updates

The network is coord_cnn.build_model(), so a pre-trained model loads into CoordPipeline (and from there into softam_loss
and the other end-to-end paths) unchanged.  PNG decoding stays with the caller (INTEGRATION.md)."""
import numpy as np
import torch

from . import coord_cnn
from . import engine as E

DEFAULT_THREADRAND_SEED = 1305   # ThreadRand::init's default (thread_rand.h)
DEFAULT_PERM_SEED = 5489         # train_obj.cpp:208: a default-constructed std::mt19937
INLIER_THRESHOLD_M = 0.1         # rT3D = 100 mm (train_obj.cpp:219)


def _dev(a, dtype, device):
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=dtype).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a)).to(device=device, dtype=dtype).contiguous()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def read_sensor_trans(path):
    """sensorTrans.dat (jp::read of a cv::Mat_<double>: int32 rows, int32 cols, row-major doubles) -> [4][4]."""
    b = open(path, "rb").read()
    rows, cols = np.frombuffer(b[:8], np.int32)
    return np.frombuffer(b[8:8 + 8 * rows * cols], np.float64).reshape(rows, cols).copy()


class RGBDScene:
    """A training set in device memory: bgr [F][H][W][3] uint8, raw depth [F][H][W] uint16 (as the depth PNGs hold it),
    gt_jp [F][12] (the jp pose as dsac_forward takes it: row-major rotation, translation in mm) and its camera: one
    RGBDCamera for every frame, or a sequence of F, one per frame (frames with their own intrinsics), all with the frame
    size as width / height and the same raw_data.  The depth is registered to the RGB camera once, here (with raw_data = 0
    it is used as given).

    cam is the single camera (None with per-frame cameras); cams is the per-frame table (None with one camera).  A scene
    with per-frame cameras installs its table on the engine (Engine.use_dataset_cameras) before each of its calls if
    another one is installed, so several scenes can share an engine."""

    def __init__(self, engine, bgr, raw_depth, gt_jp, cam=None, device="cuda"):
        self.engine, self.device = engine, device
        raw = raw_depth.cpu().numpy() if isinstance(raw_depth, torch.Tensor) else np.asarray(raw_depth)
        raw = np.ascontiguousarray(raw.astype(np.uint16)).view(np.int16)   # the bits; torch has no uint16 arithmetic
        self.n_frames, self.height, self.width = raw.shape
        if cam is None or isinstance(cam, E.RGBDCamera):
            self.cam = cam if cam is not None else E.default_rgbd_camera()
            self.cams = None
            shapes = [(self.cam.width, self.cam.height)]
        else:
            self.cam = None
            self.cams = E.camera_table(list(cam))
            if len(self.cams) != self.n_frames:
                raise ValueError("%d cameras for %d frames" % (len(self.cams), self.n_frames))
            shapes = {(c.width, c.height) for c in self.cams}
        for w, h in shapes:
            if (self.width, self.height) != (w, h):
                raise ValueError("frames are %dx%d, a camera %dx%d" % (self.width, self.height, w, h))
        self.bgr = _dev(bgr, torch.uint8, device)
        if tuple(self.bgr.shape) != (self.n_frames, self.height, self.width, 3):
            raise ValueError("bgr must be [F][H][W][3] uint8 like the depth")
        self.gt_jp = _dev(gt_jp, torch.float64, device).reshape(self.n_frames, 12)
        self.raw_depth = _dev(raw, torch.int16, device)
        self.depth = torch.empty_like(self.raw_depth)
        self.dropped = torch.zeros(self.n_frames, dtype=torch.int32, device=device)
        self.status = torch.zeros(self.n_frames, dtype=torch.int32, device=device)
        engine.register_depth_device(self.camera_arg(), self.n_frames, self.raw_depth.data_ptr(), self.depth.data_ptr(),
                                     self.dropped.data_ptr(), self.status.data_ptr(), stream=_stream())

    def camera_arg(self):
        """The `cam` argument of the engine's data-path calls on this scene: its camera, or None (the dataset camera
        table) after installing its per-frame table on the engine where another one is installed."""
        if self.cams is None:
            return self.cam
        self.engine.use_dataset_cameras(self.cams, stream=_stream())
        return None

    def depth_u16(self):
        """The registered depth as a host uint16 array."""
        return self.depth.cpu().numpy().view(np.uint16)

    def scene_coords(self, idx):
        """getObj: int16 scene coordinates (mm) [H][W][3] of frame idx (an int) or [n][H][W][3] of a list of frames."""
        one = np.isscalar(idx)
        ids = [int(i) for i in ([idx] if one else list(idx))]
        if not ids or min(ids) < 0 or max(ids) >= self.n_frames:
            raise IndexError("frame indices must lie in [0, %d)" % self.n_frames)
        ids = torch.as_tensor(ids, dtype=torch.int32, device=self.device)
        out = torch.empty((len(ids), self.height, self.width, 3), dtype=torch.int16, device=self.device)
        self.engine.obj_coords_device(self.camera_arg(), self.n_frames, len(ids), self.depth.data_ptr(), self.gt_jp.data_ptr(),
                                      out.data_ptr(),
                                      d_idx=ids.data_ptr(), stream=_stream())
        return out[0] if one else out


class ObjRound:
    """assembleData's rounds on a scene.  state: [n_streams][625] int32 holding the uint32 words of the OpenMP threads'
    std::mt19937 engines and their positions; every draw continues from it, as ThreadRand's generators do across the
    reference's rounds, and a trainer may save and restore it."""

    def __init__(self, scene, seed=DEFAULT_THREADRAND_SEED, n_streams=1, max_attempts=1 << 20):
        self.scene, self.n_streams, self.max_attempts = scene, n_streams, max_attempts
        self.state = torch.empty((n_streams, E.OBJ_STATE_WORDS), dtype=torch.int32, device=scene.device)
        scene.engine.obj_rng_init_device(seed, n_streams, self.state.data_ptr(), stream=_stream())
        self.img = self.centre = self.label = self.status = None

    def draw(self, n_images=100, n_patches=512):
        """One round: img [n] int32 frame of each patch, centre [n][2] int32 (x, y), label [n][3] float32 metres,
        status [n_images] (E.ST_OBJ_DRAW_EXHAUSTED) with n = n_images * n_patches, in the reference's data order."""
        s, dev = self.scene, self.scene.device
        n = n_images * n_patches
        self.img = torch.empty(n, dtype=torch.int32, device=dev)
        self.centre = torch.empty((n, 2), dtype=torch.int32, device=dev)
        self.label = torch.empty((n, 3), dtype=torch.float32, device=dev)
        self.status = torch.empty(n_images, dtype=torch.int32, device=dev)
        s.engine.obj_draw_device(s.camera_arg(), s.n_frames, s.depth.data_ptr(), s.gt_jp.data_ptr(), n_images, n_patches,
                                 self.n_streams, self.max_attempts, self.state.data_ptr(), self.img.data_ptr(),
                                 self.centre.data_ptr(), self.label.data_ptr(), self.status.data_ptr(), stream=_stream())
        return self.img, self.centre, self.label, self.status

    def patches(self, slots=None, out=None):
        """The 3x42x42 patches (minus 127) of the last draw's patches `slots` (a device index tensor; None: all)."""
        s = self.scene
        img, centre = (self.img, self.centre) if slots is None else (self.img[slots], self.centre[slots])
        img, centre = img.contiguous(), centre.contiguous()
        n = img.numel()
        if out is None:
            out = torch.empty((n, 3, coord_cnn.PATCH, coord_cnn.PATCH), dtype=torch.float32, device=s.device)
        s.engine.gather_patches_at_device(n, s.bgr.data_ptr(), s.n_frames, s.width, s.height, img.data_ptr(),
                                          centre.data_ptr(), out.data_ptr(), mean=coord_cnn.MEAN, stream=_stream())
        return out


class _L1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, gt):
        diff = pred - gt
        dist = diff.norm(dim=1, keepdim=True)
        ctx.save_for_backward(diff, dist)
        return dist.mean()

    @staticmethod
    def backward(ctx, g):
        diff, dist = ctx.saved_tensors
        return g * (diff / dist / diff.shape[0]), None


def l1_criterion(pred, gt):
    """MyL1Criterion: mean over the batch of ||pred - gt||_2; its gradient is (pred - gt) / dist / count, exactly the
    reference's.  Where pred == gt the distance is 0 and that row's gradient is 0 / 0 = NaN, as in torch7 (the subgradient
    would be 0); no gradient flows to gt."""
    return _L1.apply(pred, gt)


def inlier_ratio(pred, labels, threshold=INLIER_THRESHOLD_M):
    """getInliers (train_obj.cpp:111-122): the fraction of predictions within `threshold` (metres) of their label."""
    return float(((pred - labels).norm(dim=1) < threshold).float().mean())


class Torch7Adam(torch.optim.Optimizer):
    """optim.adam as torch7 writes it:  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  denom = sqrt(v) + eps;
    x -= lr sqrt(1 - b2^t) / (1 - b1^t) * m / denom.  Unlike torch.optim.Adam, eps is added to the uncorrected sqrt(v)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["t"] = 0
                    st["m"] = torch.zeros_like(p)
                    st["v"] = torch.zeros_like(p)
                st["t"] += 1
                t = st["t"]
                st["m"].mul_(b1).add_(p.grad, alpha=1 - b1)
                st["v"].mul_(b2).addcmul_(p.grad, p.grad, value=1 - b2)
                denom = st["v"].sqrt().add_(group["eps"])
                step = group["lr"] * (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
                p.addcdiv_(st["m"], denom, value=-step)
        return loss


class ObjPretrainer:
    """train_obj.cpp's loop: each round draws n_images x n_patches patches, then takes batches of `batch` in the order of
    one fixed permutation (std::shuffle of iota(n_images * n_patches) by std::mt19937(perm_seed)), one Torch7Adam update
    per batch on l1_criterion; the learning rate halves after every lr_interval updates.  log: (update, loss) per update,
    as training_loss_*.txt holds it."""

    def __init__(self, engine, scene, model=None, seed=DEFAULT_THREADRAND_SEED, n_streams=1, n_images=100, n_patches=512,
                 batch=64, lr=1e-4, lr_interval=50000, perm_seed=DEFAULT_PERM_SEED, max_attempts=1 << 20):
        self.scene, self.n_images, self.n_patches, self.batch, self.lr_interval = scene, n_images, n_patches, batch, lr_interval
        self.model = (model if model is not None else coord_cnn.build_model()).to(scene.device).train()
        self.opt = Torch7Adam(self.model.parameters(), lr=lr)
        self.round = ObjRound(scene, seed=seed, n_streams=n_streams, max_attempts=max_attempts)
        self.perm = torch.from_numpy(E.shuffle_permutation(n_images * n_patches, perm_seed).astype(np.int64)).to(scene.device)
        self.updates = 0
        self.log = []

    def step(self, patches, labels):
        """One update: forward, MyL1Criterion, backward, Adam; the lr halving as train_obj.lua:259-262 does it."""
        self.opt.zero_grad(set_to_none=True)
        loss = l1_criterion(self.model(patches), labels)
        loss.backward()
        self.opt.step()
        self.updates += 1
        if self.updates % self.lr_interval == 0:
            for g in self.opt.param_groups:
                g["lr"] *= 0.5
        v = float(loss.detach())
        self.log.append((self.updates - 1, v))
        return v

    def train(self, n_updates):
        """Runs n_updates updates, drawing a new round whenever the previous one is used up (rounds of
        n_images * n_patches // batch updates).  Returns the losses of these updates."""
        per_round = self.n_images * self.n_patches // self.batch
        out = []
        while len(out) < n_updates:
            _, _, label, _ = self.round.draw(self.n_images, self.n_patches)
            for b in range(per_round):
                if len(out) == n_updates:
                    break
                slots = self.perm[b * self.batch:(b + 1) * self.batch]
                out.append(self.step(self.round.patches(slots), label[slots]))
        return out

    @torch.no_grad()
    def evaluate(self, n_images=10, n_patches=512, seed=DEFAULT_THREADRAND_SEED + 1000):
        """Mean loss and inlier ratio (getInliers at 100 mm) over a fresh draw, in evaluation mode."""
        self.model.eval()
        r = ObjRound(self.scene, seed=seed, max_attempts=self.round.max_attempts)
        _, _, label, _ = r.draw(n_images, n_patches)
        preds = []
        for i in range(0, label.shape[0], 1024):
            preds.append(self.model(r.patches(torch.arange(i, min(i + 1024, label.shape[0]), device=self.scene.device))))
        pred = torch.cat(preds)
        self.model.train()
        return float(l1_criterion(pred, label)), inlier_ratio(pred, label)
