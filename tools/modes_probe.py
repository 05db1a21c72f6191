"""Times dsac_pose_modes_device on the GPU: after a soft-argmax forward of --softam-frames frames and after a DSAC-variant
forward of --dsac-frames frames (H = --hyps), on synthetic frames and on two-cluster frames (40 % of the cells consistent
with one pose, 30 % with another 30 degrees and 1 m away, tests/test_gpu_pose_modes.py), for each M of --modes.  CUDA
events around each call on the engine's stream, median of --reps after --warmup calls.  Prints one JSON line per case
with the card's name and power limit.  --profile: instead, the call's kernel split from torch.profiler (a run of its own).

    python tools/modes_probe.py --softam-frames 1024 --dsac-frames 64 --reps 20 [--profile]
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--softam-frames", type=int, default=1024)
    ap.add_argument("--dsac-frames", type=int, default=64)
    ap.add_argument("--hyps", type=int, default=256)
    ap.add_argument("--modes", default="1,4,16")
    ap.add_argument("--rot-deg", type=float, default=10.0)
    ap.add_argument("--trans-mm", type=float, default=100.0)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="the call's kernels with torch.profiler instead of the timings")
    a = ap.parse_args()
    import math
    import numpy as np
    import torch
    import dsac_b200.engine as E
    from dsac_b200 import autograd as A
    from test_gpu_pose_modes import _two_cluster_frames
    E.load()
    gpu = card()
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream
    rot = math.radians(a.rot_deg)

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        fn()
        t1.record(stream)
        t1.synchronize()
        return t0.elapsed_time(t1)

    for pipeline, n in (("softam", a.softam_frames), ("dsac", a.dsac_frames)):
        for frames in ("synthetic", "two-cluster"):
            if frames == "synthetic":
                coords, pix, _, _ = E.synth_frames(n)
            else:
                coords, pix, _, _ = _two_cluster_frames(n, 41)
            dc, dp = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (coords, pix))
            eng = E.Engine(max_frames=n, n_hyps=a.hyps)
            if pipeline == "softam":
                eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, None, 0, s)
            else:
                eng.forward_dsac_device(n, dc.data_ptr(), dp.data_ptr(), 0, None, True, 0, s)
            for M in (int(m) for m in a.modes.split(",")):
                out = A.pose_modes(eng, n, M, rot, a.trans_mm)
                ptrs = {k: v.data_ptr() for k, v in out.items()}

                def call():
                    eng.pose_modes_device(n, M, rot, a.trans_mm, s, **ptrs)

                for _ in range(a.warmup):
                    call()
                torch.cuda.synchronize()
                rec = {"pipeline": pipeline, "frames": frames, "n": n, "hyps": a.hyps, "M": M, "rot_deg": a.rot_deg,
                       "trans_mm": a.trans_mm, "gpu": gpu, "reps": a.reps,
                       "n_modes_mean": float(out["n_modes"].float().mean())}
                if a.profile:
                    from torch.profiler import ProfilerActivity, profile
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for _ in range(a.reps):
                            call()
                        torch.cuda.synchronize()
                    kernels = {}
                    for ev in prof.key_averages():
                        if any(w in ev.key for w in ("mode", "refine", "uncertainty")):
                            us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                            kernels[ev.key.split("(")[0]] = us / 1e3 / a.reps
                    rec["kernel_ms_per_call"] = kernels
                else:
                    t = [timed(call) for _ in range(a.reps)]
                    rec["call_ms_median"] = float(np.median(t))
                    rec["call_ms_min"] = float(np.min(t))
                print(json.dumps(rec), flush=True)
            eng.close()


if __name__ == "__main__":
    main()
