"""Times rig tracking on a synthetic rig trajectory: 256 rigs of 4 cameras (1024 frames), H = 256.  Reports the median rig
pass (dsac_forward_rig_device) with no priors, with k = 1 ungated rig priors and with k = 1 gated ones (prior = the
previous step's refined rig pose, information inv(cov_xi + Q) from dsac_rig_pose_uncertainty_device, chi^2 16.81), the
sampler candidates per frame of each, and the median rig_pose_uncertainty call with its kernel split from torch.profiler
(a separate, profiled run).  Host clock around each call and a device synchronise, median of --reps after --warmup calls;
the three pass kinds alternate.  Prints one JSON line with the card's name and power limit, read in the same call.

    python tools/rig_track_probe.py [--reps 10] [--warmup 3] [--out DIR]
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


def ring(C):
    import numpy as np
    from scipy.spatial.transform import Rotation
    ext = np.zeros((C, 6))
    for c in range(C):
        a = 2 * np.pi * c / C
        ext[c, :3] = Rotation.from_euler("y", a).as_rotvec()
        ext[c, 3:] = [80.0 * np.sin(a), 0.0, 80.0 * np.cos(a)]
    return ext


def scene(R, C, step, rng):
    """Scene coordinates of R rigs of C ring cameras at step `step` of a trajectory (the rig moves 50 mm and turns 1 degree
    per step): 60 % of each camera's cells at the rig's pose (0.5 px noise), the rest random."""
    import numpy as np
    from scipy.spatial.transform import Rotation
    f, cx, cy = 525.0, 320.0, 240.0
    gx, gy = np.meshgrid(np.arange(40) * 16 + 8, np.arange(40) * 12 + 6)
    pix = np.stack([gx.ravel(), gy.ravel()], 1).astype(np.int32)
    ext = ring(C)
    coords = np.empty((R * C, N, 3), np.int16)
    poses = np.empty((R, 6))
    for r in range(R):
        base = np.random.default_rng(r)
        rot = Rotation.from_euler("xyz", base.normal(scale=0.2, size=3)) * Rotation.from_euler("y", np.radians(step))
        t = base.normal(scale=300.0, size=3) + [50.0 * step, 0.0, 1500.0]
        poses[r] = np.concatenate([rot.as_rotvec(), t])
        for c in range(C):
            Rc = Rotation.from_rotvec(ext[c, :3])
            cam_R, cam_t = Rc * rot, Rc.apply(t) + ext[c, 3:]
            d = rng.uniform(1500.0, 4000.0, size=N)
            u = pix[:, 0] + rng.normal(scale=0.5, size=N)
            v = pix[:, 1] + rng.normal(scale=0.5, size=N)
            Xc = np.stack([(u - cx) / f * d, (v - cy) / f * d, d], 1)
            X = cam_R.inv().apply(Xc - cam_t)
            out = rng.uniform(size=N) >= 0.6
            X[out] = rng.uniform(-4000.0, 4000.0, size=(out.sum(), 3))
            coords[r * C + c] = np.clip(np.round(X), -32767, 32767).astype(np.int16)
    return coords, pix, np.tile(ext, (R, 1)), poses


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table")
    a = ap.parse_args()
    import numpy as np
    import torch
    import dsac_b200.engine as E
    from dsac_b200 import autograd as A
    E.load()
    name = card()
    R, C, H = 256, 4, 256
    n = R * C
    rng = np.random.default_rng(0)
    coords, pix, ext, poses = scene(R, C, 0, rng)
    coords1, _, _, _ = scene(R, C, 1, rng)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    dc0, dc1, dp, de = dev(coords), dev(coords1), dev(pix), dev(ext)
    eng = E.Engine(max_frames=n, n_hyps=H)
    f64 = dict(dtype=torch.float64, device="cuda")
    ref = torch.empty((R, 6), **f64)
    status = torch.empty((R,), dtype=torch.int32, device="cuda")
    hyp = torch.empty((n, H, 6), **f64)
    # step 0 without priors gives the priors of step 1: the refined rig poses and their covariance
    # pix is one grid shared by every frame: pix_shared = 1
    eng.forward_rig_device(n, C, dc0.data_ptr(), dp.data_ptr(), de.data_ptr(), 1, None, 0, ref_pose=ref.data_ptr())
    unc = A.rig_pose_uncertainty(eng, n, C)
    torch.cuda.synchronize()
    Q = torch.diag(torch.tensor([1e-3] * 3 + [100.0 ** 2] * 3, **f64))
    info = torch.linalg.inv(unc["cov_xi"] + Q)[:, None].contiguous()
    prior = ref[:, None].clone()
    ok_frac = float(unc["ok"].float().mean())

    def rig_pass(kind):
        if kind == "none":
            eng.set_rig_pose_priors_device(n, C, 0, None)
        elif kind == "ungated":
            eng.set_rig_pose_priors_device(n, C, 1, prior.data_ptr())
        else:
            eng.set_rig_pose_priors_device(n, C, 1, prior.data_ptr(), info.data_ptr(), 16.81)
        torch.cuda.synchronize()
        t = time.perf_counter()
        eng.forward_rig_device(n, C, dc1.data_ptr(), dp.data_ptr(), de.data_ptr(), 1, None, n,
                               ref_pose=ref.data_ptr(), status=status.data_ptr(), hyp_pose=hyp.data_ptr())
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3

    kinds = ("none", "ungated", "gated")
    times = {k: [] for k in kinds}
    cands = {}
    for i in range(a.warmup + a.reps):
        for k in kinds:
            ms = rig_pass(k)
            if i >= a.warmup:
                times[k].append(ms)
            if i == 0:
                res = eng.fetch(n)   # the frames' sampler counts of this pass (n_candidates)
                cands[k] = float(np.mean(res.n_candidates))

    def unc_call():
        torch.cuda.synchronize()
        t = time.perf_counter()
        A.rig_pose_uncertainty(eng, n, C)
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3

    rig_pass("gated")
    for _ in range(a.warmup):
        unc_call()
    unc_ms = [unc_call() for _ in range(a.reps)]
    split = {}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            A.rig_pose_uncertainty(eng, n, C)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", 0.0)
        if t > 0 and ev.key.startswith(("dsac::k_", "Memcpy", "Memset")):
            split[ev.key[:60]] = round(t / 1e3 / a.reps, 4)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "rig_track_profile.txt"), "w") as fh:
            fh.write(prof.key_averages().table(sort_by="device_time_total", row_limit=20))
    eng.close()
    print(json.dumps({"card": name, "rigs": R, "cameras": C, "hyps": H,
                      "rig_pass_ms_median": {k: round(float(np.median(v)), 3) for k, v in times.items()},
                      "candidates_per_frame": {k: round(v, 1) for k, v in cands.items()},
                      "rig_pose_uncertainty_ms_median": round(float(np.median(unc_ms)), 3),
                      "rig_pose_uncertainty_kernel_ms": split, "covariance_ok_fraction": ok_frac}), flush=True)


if __name__ == "__main__":
    main()
