"""Times RGB-D rigs (dsac_set_rig_cell_depth_device): 256 rigs of 4 cameras at H = 256, and of 8 cameras at H = 128 (a
rig's pool C H may not exceed 1024).  For each it reports the median RGB-D rig pass (dsac_forward_rig_device), its
backward (dsac_backward_rig_pose_device), its covariance call (dsac_rig_pose_uncertainty_device) and the RGB rig pass on
the same frames, host clock around each call and a device synchronise, median of --reps after --warmup calls, the RGB
and RGB-D passes alternating; then, in a separate profiled run (torch.profiler), the device time of every kernel of one
RGB-D pass, backward and covariance call, k_refine_rig_rgbd and its recording replay among them.  Prints one JSON line
with the card's name and power limit, read in the same call.

    python tools/rig_rgbd_probe.py [--reps 10] [--warmup 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N = 1600


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def scene(R, C, seed=0):
    """R RGB-D rigs of C ring cameras: every cell has depth U(1500, 4000) mm; 60 % of each camera's cells are the eye point
    of the rig's pose (0.5 px noise), the rest random scene points.  (coords, pix, depth, ext)."""
    import numpy as np
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    f, cx, cy = 525.0, 320.0, 240.0
    gx, gy = np.meshgrid(np.arange(40) * 16 + 8, np.arange(40) * 12 + 6)
    pix1 = np.stack([gx.ravel(), gy.ravel()], 1).astype(np.int32)
    ext1 = np.zeros((C, 6))
    for c in range(C):
        a = 2 * np.pi * c / C
        ext1[c, :3] = Rotation.from_euler("y", a).as_rotvec()
        ext1[c, 3:] = [80.0 * np.sin(a), 0.0, 80.0 * np.cos(a)]
    n = R * C
    coords = np.empty((n, N, 3), np.int16)
    depth = rng.uniform(1500.0, 4000.0, size=(n, N)).astype(np.float32)
    for r in range(R):
        rot = Rotation.from_euler("xyz", rng.normal(scale=0.2, size=3))
        t = rng.normal(scale=300.0, size=3) + [0.0, 0.0, 1500.0]
        for c in range(C):
            fr = r * C + c
            Rc = Rotation.from_rotvec(ext1[c, :3])
            cam_R, cam_t = Rc * rot, Rc.apply(t) + ext1[c, 3:]
            d = depth[fr].astype(np.float64)
            u = pix1[:, 0] + rng.normal(scale=0.5, size=N)
            v = pix1[:, 1] + rng.normal(scale=0.5, size=N)
            X = cam_R.inv().apply(np.stack([(u - cx) / f * d, (v - cy) / f * d, d], 1) - cam_t)
            out = rng.uniform(size=N) >= 0.6
            X[out] = rng.uniform(-4000.0, 4000.0, size=(out.sum(), 3))
            coords[fr] = np.clip(np.round(X), -32767, 32767).astype(np.int16)
    return coords, np.tile(pix1[None], (n, 1, 1)), depth, np.tile(ext1, (R, 1))


def run(R, C, H, reps, warmup, out_dir):
    import numpy as np
    import torch
    import dsac_b200.engine as E
    n = R * C
    coords, pix, depth, ext = scene(R, C)
    dev = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()
    dc, dp, de, dd = dev(coords, np.int16), dev(pix, np.int32), dev(ext, np.float64), dev(depth, np.float32)
    eng = E.Engine(max_frames=n, n_hyps=H)
    f64 = dict(dtype=torch.float64, device="cuda")
    ref, st = torch.zeros((R, 6), **f64), torch.zeros(R, dtype=torch.int32, device="cuda")
    seed = torch.ones((R, 6), **f64)
    dpred = torch.zeros((n, N, 3), dtype=torch.float32, device="cuda")
    cov = torch.zeros((R, 6, 6), **f64)

    def rig_pass(rgbd):
        eng.set_rig_cell_depth_device(n, C, dd.data_ptr() if rgbd else None)
        eng.forward_rig_device(n, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr(), ref_pose=ref.data_ptr(), status=st.data_ptr())

    calls = {
        "rgb_pass": lambda: rig_pass(False),
        "rgbd_pass": lambda: rig_pass(True),
        "rgbd_backward": lambda: eng.backward_rig_pose_device(n, seed.data_ptr(), None, dpred.data_ptr()),
        "rgbd_covariance": lambda: eng.rig_pose_uncertainty_device(n, C, cov_xi=cov.data_ptr()),
    }
    times = {k: [] for k in calls}
    for i in range(warmup + reps):
        for k, fn in calls.items():   # (the backward and the covariance follow the RGB-D pass)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if i >= warmup:
                times[k].append(time.perf_counter() - t0)
    res = {k + "_ms": round(1e3 * float(np.median(v)), 3) for k, v in times.items()}
    status = st.cpu().numpy()
    res["rigs_refined"] = int(((status & (2 | 256)) == 0).sum())
    from torch.profiler import ProfilerActivity, profile
    rig_pass(True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rig_pass(True)
        calls["rgbd_backward"]()
        calls["rgbd_covariance"]()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            kern[ev.key] = round(t / 1e3, 3)
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "rig_rgbd_C%d.pt.trace.json" % C))
    res["kernels_ms"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:16])
    res["k_refine_rig_rgbd_ms"] = round(sum(v for k, v in kern.items() if "k_refine_rig_rgbd" in k and "rec" not in k), 3)
    res["k_refine_rig_rgbd_rec_ms"] = round(sum(v for k, v in kern.items() if "k_refine_rig_rgbd_rec" in k), 3)
    eng.close()
    return {"R": R, "C": C, "H": H, **res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    out = {"card": card(), "cases": [run(256, 4, 256, a.reps, a.warmup, a.out), run(256, 8, 128, a.reps, a.warmup, a.out)]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
