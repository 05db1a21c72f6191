"""Times one round of the score-CNN pre-training data path on the device: the draw (frames, grids, drift levels and
getRandHyp vectors), the coordinate CNN on the drawn grids (coord_cnn.build_model(), library convolutions), the error
images and labels, and one pre-training update (batch 64).  CUDA events around each step, median of --reps after
--warmup.  Frames are synthetic (coded BGR); the timings do not depend on their content.

    python tools/score_round.py [--frames 16] [--images 100] [--hyps 16] [--reps 5] [--json out.json]
                                [--cameras none|identical|mixed] [--mixed-cameras] [--dump out.npz]

--cameras: the engine's config camera (none), a dataset camera table of F identical cameras (whose getCamMat() is the
config's), or a table mixing three cameras (the defaults, an off-centre principal point, another focal length);
--mixed-cameras is --cameras mixed.  --dump writes one draw's outputs and error images to an .npz.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from dsac_b200 import engine as E              # noqa: E402
from dsac_b200.coord_cnn import CoordPipeline   # noqa: E402
from dsac_b200.score_train import ScorePretrainer, ScoreRound   # noqa: E402
import obj_oracle as OO                        # noqa: E402


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--hyps", type=int, default=16)
    ap.add_argument("--streams", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default="")
    ap.add_argument("--cameras", choices=["none", "identical", "mixed"], default="none")
    ap.add_argument("--mixed-cameras", action="store_const", const="mixed", dest="cameras")
    ap.add_argument("--dump", default="")
    a = ap.parse_args()
    eng = E.Engine(max_frames=4, n_hyps=64)
    rng = np.random.default_rng(0)
    gt = np.zeros((a.frames, 12))
    gt[:, [0, 4, 8]] = 1.0
    gt[:, 9:] = rng.uniform(-500, 500, (a.frames, 3))
    bgr = torch.from_numpy(OO.coded_bgr(a.frames, 480, 640)).cuda()
    pipe = CoordPipeline(eng)
    cam = E.default_rgbd_camera()
    three = [cam, E.default_rgbd_camera(x_shift=13.5, y_shift=-7.25), E.default_rgbd_camera(focal=610.0, x_shift=-0.75)]
    cams = {"none": None, "identical": [cam] * a.frames, "mixed": [three[f % 3] for f in range(a.frames)]}[a.cameras]
    r = ScoreRound(eng, bgr, torch.from_numpy(gt).cuda(), pipe, n_streams=a.streams, cameras=cams)
    n_img, H = a.images, a.hyps
    first = r.draw(n_img, H)   # allocates img / pix / drift / noise / coords
    if a.dump:
        np.savez(a.dump, maps=first[0].cpu().numpy(), labels=first[1].cpu().numpy(), correct=first[2].cpu().numpy(),
                 img=r.img.cpu().numpy(), pix=r.pix.cpu().numpy(), drift=r.drift.cpu().numpy(),
                 noise=r.noise.cpu().numpy(), coords=r.coords.cpu().numpy(), state=r.state.cpu().numpy())
    st = torch.cuda.current_stream().cuda_stream
    maps = torch.empty((n_img * H, 1, 40, 40), dtype=torch.float32, device="cuda")
    labels = torch.empty(n_img * H, dtype=torch.float64, device="cuda")

    def draw():
        eng.score_draw_device(r.n_frames, r.width, r.height, n_img, H, r.n_streams, r.state.data_ptr(), r.img.data_ptr(),
                              r.pix.data_ptr(), r.drift.data_ptr(), r.noise.data_ptr(), stream=st)

    def coords():
        pipe(bgr.index_select(0, r.img.long()), r.pix)

    def score_maps():
        eng.score_maps_device(n_img, H, r.img.data_ptr(), r.gt_jp.data_ptr(), r.coords.data_ptr(), r.pix.data_ptr(),
                              r.noise.data_ptr(), 10.0, maps.data_ptr(), labels.data_ptr(), stream=st)

    tr = ScorePretrainer(eng, bgr, torch.from_numpy(gt).cuda(), pipe, n_images=n_img, hyps_per_image=H, cameras=cams)
    x, y = maps[:64].clone(), labels[:64].clone()
    out = {
        "draw_ms": timed(draw, a.reps, a.warmup),
        "coord_cnn_ms": timed(coords, a.reps, a.warmup),
        "maps_ms": timed(score_maps, a.reps, a.warmup),
        "update_ms": timed(lambda: tr.step(x, y), a.reps, a.warmup),
        "images": n_img, "hyps_per_image": H, "streams": a.streams, "cameras": a.cameras,
        "device": torch.cuda.get_device_name(0),
    }
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh)


if __name__ == "__main__":
    main()
