"""Times the coordinate-CNN pre-training data path on the device against the numpy restatement (tests/obj_oracle.py) on
the same synthetic data:  registration of F frames, one draw + gather round (n_images x n_patches), one pre-training
update (batch 64).  CUDA events around each device step (median of --reps after --warmup); wall clock for the CPU side.

    python tools/obj_round.py [--frames 64] [--reps 5] [--json out.json] [--cameras none|identical|mixed]
                              [--mixed-cameras] [--dump out.npz]

--cameras: one camera (none: no dataset camera table), a table of F identical cameras, or a table mixing three cameras
(7-Scenes' defaults, an off-centre principal point, another RGB and depth focal length); --mixed-cameras is
--cameras mixed.  --dump writes the registered depth and the first draw (device outputs and stream state) to an .npz.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from dsac_b200 import engine as E          # noqa: E402
from dsac_b200.obj_train import ObjPretrainer, ObjRound, RGBDScene, read_sensor_trans   # noqa: E402
import camera_oracle as CO                 # noqa: E402
import obj_oracle as OO                    # noqa: E402


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
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--patches", type=int, default=512)
    ap.add_argument("--streams", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cpu-frames", type=int, default=4, help="frames the CPU restatement registers (time scaled to --frames)")
    ap.add_argument("--json", default=None)
    ap.add_argument("--cameras", choices=["none", "identical", "mixed"], default="none")
    ap.add_argument("--mixed-cameras", action="store_const", const="mixed", dest="cameras")
    ap.add_argument("--dump", default=None)
    ap.add_argument("--skip-cpu", action="store_true", help="time the device only, not the numpy restatement")
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    F, H, W = a.frames, 480, 640
    raw = rng.integers(500, 4000, (F, H, W)).astype(np.uint16)
    raw[rng.random((F, H, W)) < 0.1] = 0
    poses = np.tile(np.r_[np.eye(3).reshape(9), 0.0, 0.0, 0.0], (F, 1))
    bgr = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    eng = E.Engine(max_frames=1, n_hyps=64)
    trans = read_sensor_trans(os.path.join(ROOT, "tests", "golden", "sensorTrans_7scenes.dat"))
    cam = E.default_rgbd_camera(sensor_trans=trans)
    three = [cam, E.default_rgbd_camera(sensor_trans=trans, x_shift=13.5, y_shift=-7.25),
             E.default_rgbd_camera(sensor_trans=trans, focal=610.0, secondary_focal=560.0, x_shift=-0.75)]
    cams = {"none": cam, "identical": [cam] * F, "mixed": [three[f % 3] for f in range(F)]}[a.cameras]
    sc = RGBDScene(eng, bgr, raw, poses, cams)
    st = torch.cuda.current_stream().cuda_stream
    out = {"frames": F, "images": a.images, "patches": a.patches, "streams": a.streams, "cameras": a.cameras,
           "gpu": torch.cuda.get_device_name()}
    out["register_ms"] = timed(lambda: eng.register_depth_device(sc.camera_arg(), F, sc.raw_depth.data_ptr(),
                                                                 sc.depth.data_ptr(), stream=st), a.reps, a.warmup)
    r = ObjRound(sc, n_streams=a.streams)
    if a.dump:
        d = r.draw(a.images, a.patches)
        np.savez(a.dump, depth=sc.depth_u16(), state=r.state.cpu().numpy(), **{k: v.cpu().numpy() for k, v in
                                                                                zip(("img", "centre", "label", "status"), d)})
        r = ObjRound(sc, n_streams=a.streams)
    out["draw_ms"] = timed(lambda: r.draw(a.images, a.patches), a.reps, a.warmup)
    out["gather_ms"] = timed(lambda: r.patches(), a.reps, a.warmup)
    tr = ObjPretrainer(eng, sc, n_streams=a.streams, n_images=a.images, n_patches=a.patches)
    tr.round.draw(a.images, a.patches)
    slots = tr.perm[:64]
    pt, lb = tr.round.patches(slots), tr.round.label[slots]
    out["update_ms"] = timed(lambda: tr.step(pt, lb), a.reps, a.warmup)
    if a.skip_cpu:
        eng.close()
        print(json.dumps(out))
        return
    # the CPU restatement on the same data
    t0 = time.perf_counter()
    fcams = CO.frame_cams(cams, F)
    reg, _ = CO.register_depth(fcams[:a.cpu_frames], raw[:a.cpu_frames])
    out["cpu_register_ms"] = (time.perf_counter() - t0) * 1e3 * F / a.cpu_frames
    depth = sc.depth_u16()
    t0 = time.perf_counter()
    coords = np.stack([OO.obj_coords(fcams[f], depth[f], poses[f]) for f in range(F)])
    out["cpu_getobj_all_frames_ms"] = (time.perf_counter() - t0) * 1e3
    state = OO.rng_init(1305, a.streams)
    t0 = time.perf_counter()
    OO.draw(cam, depth, poses, state, a.images, a.patches, coords=coords)
    out["cpu_draw_ms"] = (time.perf_counter() - t0) * 1e3
    img, centre = r.img.cpu().numpy(), r.centre.cpu().numpy()
    t0 = time.perf_counter()
    OO.gather_patches(bgr, img, centre)
    out["cpu_gather_ms"] = (time.perf_counter() - t0) * 1e3
    eng.close()
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
