"""Pre-training of the score CNN on perturbed ground-truth poses (the reference's train_score.cpp with
lua/train_score.lua), with the data path on the device:

    ScoreRound       assembleData: the ThreadRand streams' draw of frames, sampling grids, drift levels and getRandHyp
                     vectors; the coordinate CNN on the drawn grids; the 40x40 reprojection-error images and the labels
    ScorePretrainer  the reference's schedule: 100 images x 16 hypotheses per round, a fresh shuffle per round from one
                     continuing std::mt19937, batches of 64, nn.AbsCriterion, optim.adam with lr 1e-4 halved every 5000
                     updates

The network is score_cnn.build_model(), so the result loads into the score seam unchanged:
ScoreCNN().model.load_state_dict(trainer.model.state_dict()).  The coordinate CNN comes in as a coord_cnn.CoordPipeline
(e.g. after obj_train.ObjPretrainer) and is used as it is."""
import numpy as np
import torch
import torch.nn.functional as Fn

from . import engine as E
from . import score_cnn
from .obj_train import DEFAULT_PERM_SEED, DEFAULT_THREADRAND_SEED, Torch7Adam, _dev, _stream

TEMPERATURE = 10.0     # objTemperature (train_score.cpp:268)


def select_best(pred, labels, temperature=TEMPERATURE):
    """selectBest (train_score.cpp:123-149): 1 if the label of the highest prediction (the first maximum) is above
    -temperature * 5, else 0."""
    best = int(torch.argmax(pred.reshape(-1)))   # torch.argmax returns the first maximal index
    return 1 if float(labels.reshape(-1)[best]) > -temperature * 5 else 0


class ScoreRound:
    """assembleData's rounds on a scene: bgr [F][H][W][3] uint8 and gt_jp [F][12] (the jp pose as dsac_forward takes it:
    row-major rotation, translation in mm) on the device, e.g. an obj_train.RGBDScene's .bgr and .gt_jp.  pipe is a
    coord_cnn.CoordPipeline.  state: [n_streams][625] int32 holding the uint32 words and positions of the OpenMP threads'
    std::mt19937 engines; every draw continues from it, as ThreadRand's generators do across the reference's rounds.
    cameras: None projects the error images with the engine's config camera; a sequence of F RGBDCamera (e.g. an
    RGBDScene's .cams) projects image i with frame img[i]'s camera as getCamMat() gives it, installed on the engine as its
    dataset camera table before each draw's error images."""

    def __init__(self, engine, bgr, gt_jp, pipe, seed=DEFAULT_THREADRAND_SEED, n_streams=1, cameras=None):
        self.engine, self.pipe, self.n_streams = engine, pipe, n_streams
        self.bgr = bgr
        self.device = bgr.device
        self.n_frames, self.height, self.width = bgr.shape[0], bgr.shape[1], bgr.shape[2]
        if tuple(bgr.shape) != (self.n_frames, self.height, self.width, 3) or bgr.dtype != torch.uint8:
            raise ValueError("bgr must be [F][H][W][3] uint8")
        self.gt_jp = _dev(gt_jp, torch.float64, self.device).reshape(self.n_frames, 12)
        self.cameras = None if cameras is None else E.camera_table(list(cameras))
        if self.cameras is not None and len(self.cameras) != self.n_frames:
            raise ValueError("%d cameras for %d frames" % (len(self.cameras), self.n_frames))
        self.state = torch.empty((n_streams, E.OBJ_STATE_WORDS), dtype=torch.int32, device=self.device)
        engine.obj_rng_init_device(seed, n_streams, self.state.data_ptr(), stream=_stream())
        self.img = self.pix = self.drift = self.noise = self.coords = None

    def draw(self, n_images=100, hyps_per_image=16, temperature=TEMPERATURE):
        """One round: maps [n][1][40][40] float32, labels [n] float64 and correct [n] int32 (1: below 5 deg and 50 mm),
        n = n_images * hyps_per_image, in the reference's data order (image-major)."""
        dev, e = self.device, self.engine
        n = n_images * hyps_per_image
        self.img = torch.empty(n_images, dtype=torch.int32, device=dev)
        self.pix = torch.empty((n_images, E.N, 2), dtype=torch.int32, device=dev)
        self.drift = torch.empty(n, dtype=torch.int32, device=dev)
        self.noise = torch.empty((n, 6), dtype=torch.float64, device=dev)
        e.score_draw_device(self.n_frames, self.width, self.height, n_images, hyps_per_image, self.n_streams,
                            self.state.data_ptr(), self.img.data_ptr(), self.pix.data_ptr(), self.drift.data_ptr(),
                            self.noise.data_ptr(), stream=_stream())
        self.coords = self.pipe(self.bgr.index_select(0, self.img.long()), self.pix)
        maps = torch.empty((n, 1, E.GRID, E.GRID), dtype=torch.float32, device=dev)
        labels = torch.empty(n, dtype=torch.float64, device=dev)
        correct = torch.empty(n, dtype=torch.int32, device=dev)
        e.use_dataset_cameras(self.cameras, stream=_stream())
        e.score_maps_device(n_images, hyps_per_image, self.img.data_ptr(), self.gt_jp.data_ptr(), self.coords.data_ptr(),
                            self.pix.data_ptr(), self.noise.data_ptr(), temperature, maps.data_ptr(), labels.data_ptr(),
                            correct.data_ptr(), stream=_stream())
        return maps, labels, correct


class ScorePretrainer:
    """train_score.cpp's loop: each round draws n_images x hyps_per_image error images, shuffles them with the round's
    permutation of one continuing std::mt19937(perm_seed) and takes batches of `batch`, one Torch7Adam update per batch
    on nn.AbsCriterion (the mean absolute error) of the network's output on maps - 45 against the labels in float32; the
    learning rate halves after every lr_interval updates.  log: (update, loss) per update, as
    score_training_loss_*.txt holds it.  cameras: as ScoreRound's (None: the engine's config camera)."""

    def __init__(self, engine, bgr, gt_jp, pipe, model=None, seed=DEFAULT_THREADRAND_SEED, n_streams=1, n_images=100,
                 hyps_per_image=16, batch=64, lr=1e-4, lr_interval=5000, temperature=TEMPERATURE,
                 perm_seed=DEFAULT_PERM_SEED, cameras=None):
        self.engine, self.bgr, self.gt_jp, self.pipe, self.cameras = engine, bgr, gt_jp, pipe, cameras
        self.n_images, self.hyps, self.batch, self.lr_interval = n_images, hyps_per_image, batch, lr_interval
        self.temperature, self.perm_seed = temperature, perm_seed
        self.model = (model if model is not None else score_cnn.build_model()).to(bgr.device).train()
        self.opt = Torch7Adam(self.model.parameters(), lr=lr)
        self.round = ScoreRound(engine, bgr, gt_jp, pipe, seed=seed, n_streams=n_streams, cameras=cameras)
        self.rounds = 0
        self.updates = 0
        self.log = []

    def step(self, maps, labels):
        """One update: forward on maps - 45, AbsCriterion against the float32 labels, backward, Adam; the lr halving as
        train_score.lua:201-204 does it."""
        self.opt.zero_grad(set_to_none=True)
        loss = Fn.l1_loss(self.model(maps - score_cnn.MEAN).reshape(-1), labels.float())
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
        n_images * hyps_per_image // batch updates).  Returns the losses of these updates."""
        n = self.n_images * self.hyps
        out = []
        while len(out) < n_updates:
            maps, labels, _ = self.round.draw(self.n_images, self.hyps, self.temperature)
            perm = torch.from_numpy(E.shuffle_permutations(n, self.perm_seed, self.rounds, 1)[0].astype(np.int64))
            perm = perm.to(maps.device)
            self.rounds += 1
            for b in range(n // self.batch):
                if len(out) == n_updates:
                    break
                slots = perm[b * self.batch:(b + 1) * self.batch]
                out.append(self.step(maps[slots], labels[slots]))
        return out

    @torch.no_grad()
    def evaluate(self, n_images=100, hyps_per_image=64, seed=DEFAULT_THREADRAND_SEED + 1000):
        """The reference's (compiled-out) validation pass on a fresh draw: batches of `batch` in data order, mean of the
        per-batch losses and the ratio of batches whose selectBest is correct.  Evaluation mode."""
        r = ScoreRound(self.engine, self.bgr, self.gt_jp, self.pipe, seed=seed, cameras=self.cameras)
        maps, labels, _ = r.draw(n_images, hyps_per_image, self.temperature)
        self.model.eval()
        losses, best = [], []
        for b in range(maps.shape[0] // self.batch):
            x, y = maps[b * self.batch:(b + 1) * self.batch], labels[b * self.batch:(b + 1) * self.batch]
            pred = self.model(x - score_cnn.MEAN).reshape(-1)
            losses.append(float(Fn.l1_loss(pred, y.float())))
            best.append(select_best(pred, y, self.temperature))
        self.model.train()
        return float(np.mean(losses)), float(np.mean(best))
