"""Times dsac_forward_rig_device on the GPU against the ordinary pass over the same frames: --rigs rigs of --cameras
cameras with --hyps hypotheses per frame (the pool holds cameras x hyps), synthetic frames, one ring of extrinsics.  CUDA
events around each call on the current stream, the two passes alternating, median of --reps after --warmup calls of each.
Then the two-cluster rig of tests/test_gpu_rig.py (camera 0: 40 % of its cells from a pose 1 m and 30 degrees away, 30 %
from the true one; the other cameras see the true pose) over --cluster-seeds seeds: rotation and translation error of the
rig's pose against camera 0 alone.  Prints JSON lines with the card's name, power limit and SM clock.  --profile: instead,
the rig pass's kernel split from torch.profiler (a run of its own).

    python tools/rig_probe.py --rigs 256 --cameras 4 --hyps 256 --reps 10 [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rigs", type=int, default=256)
    ap.add_argument("--cameras", type=int, default=4)
    ap.add_argument("--hyps", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cluster-seeds", type=int, default=16)
    ap.add_argument("--profile", action="store_true", help="the rig pass's kernels with torch.profiler instead of the timings")
    a = ap.parse_args()
    import numpy as np
    import torch
    import dsac_b200.engine as E
    from test_gpu_rig import _compose, _dev, _jp, _ring, _two_cluster_rig
    E.load()
    C, R, H = a.cameras, a.rigs, a.hyps
    n = R * C
    coords, pix, gt_cv, gt_jp = E.synth_frames(n)
    ext = np.tile(_ring(C), (R, 1))
    dc, dp, de = _dev(coords, np.int16), _dev(pix, np.int32), _dev(ext, np.float64)
    ref = torch.zeros((R, 6), dtype=torch.float64, device="cuda")
    eng = E.Engine(max_frames=n, n_hyps=H)
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream

    def rig():
        eng.forward_rig_device(n, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr(), 0, None, 0, s, ref_pose=ref.data_ptr())

    def ordinary():
        eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, None, 0, s)

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for _ in range(a.warmup):
            rig()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                rig()
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and ev.device_time_total > 0:
                split[ev.key] = split.get(ev.key, 0.0) + ev.device_time_total / a.reps / 1000.0
        top = sorted(split.items(), key=lambda kv: -kv[1])
        print(json.dumps({"card": card(), "rigs": R, "cameras": C, "hyps": H, "ms_per_pass_by_kernel": {k[:80]: round(v, 4) for k, v in top}}))
        return

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        fn()
        t1.record(stream)
        t1.synchronize()
        return t0.elapsed_time(t1)

    for _ in range(a.warmup):
        timed(rig)
        timed(ordinary)
    tr, to = [], []
    for _ in range(a.reps):
        tr.append(timed(rig))
        to.append(timed(ordinary))
    print(json.dumps({"card": card(), "rigs": R, "cameras": C, "frames": n, "hyps": H, "pool": C * H,
                      "rig_ms_median": round(float(np.median(tr)), 3), "rig_ms_min": round(float(np.min(tr)), 3),
                      "ordinary_ms_median": round(float(np.median(to)), 3), "ordinary_ms_min": round(float(np.min(to)), 3)}))
    eng.close()

    # accuracy on the two-cluster rigs: rig pose against camera 0 alone (its camera pose lifted back to the rig frame)
    from scipy.spatial.transform import Rotation
    eng = E.Engine(max_frames=C, n_hyps=H, n_streams=2)
    errs = {"rig": [], "camera0": []}
    for seed in range(a.cluster_seeds):
        cc, pp, ee, true, wrong = _two_cluster_rig(E, C, seed=100 + seed)
        d = [_dev(cc, np.int16), _dev(pp, np.int32), _dev(ee, np.float64)]
        out = torch.zeros((1, 6), dtype=torch.float64, device="cuda")
        eng.forward_rig_device(C, C, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), 0, None, 0, s, ref_pose=out.data_ptr())
        one = eng.forward(cc[:1], pp[:1])
        torch.cuda.synchronize()
        cam_true = _compose(ee[0], true)
        for name, pose, want in (("rig", out.cpu().numpy()[0], true), ("camera0", one.ref_pose[0], cam_true)):
            dr = Rotation.from_rotvec(pose[:3]) * Rotation.from_rotvec(want[:3]).inv()
            # translation error of the camera centre (mm), as the evaluation measures it
            c_est = -Rotation.from_rotvec(pose[:3]).inv().apply(pose[3:])
            c_want = -Rotation.from_rotvec(want[:3]).inv().apply(want[3:])
            errs[name].append((np.degrees(dr.magnitude()), float(np.linalg.norm(c_est - c_want))))
    eng.close()
    summary = {}
    for name, v in errs.items():
        v = np.array(v)
        summary[name] = {"rot_deg_median": round(float(np.median(v[:, 0])), 3), "t_mm_median": round(float(np.median(v[:, 1])), 2),
                         "correct": int(((v[:, 0] < 5) & (v[:, 1] < 50)).sum()), "of": len(v)}
    print(json.dumps({"card": card(), "two_cluster_rigs": a.cluster_seeds, "cameras": C, "hyps": H, **summary}))


if __name__ == "__main__":
    main()
