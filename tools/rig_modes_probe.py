"""Times dsac_rig_pose_modes_device on the GPU: after a rig pass of --rigs rigs of --cameras cameras (H = --hyps), on
synthetic rigs (test_gpu_rig_limits.py's consistent ring rigs) and on two-cluster rigs (every camera sees 40 % of its cells
from one rig pose and 30 % from another 30 degrees and 1 m away, tests/test_gpu_rig_pose_modes.py), for each M of --modes.
CUDA events around each call on the engine's stream, median of --reps after --warmup calls; the rig pass and
rig_pose_uncertainty are timed beside it for scale.  Prints one JSON line per case with the card's name and power limit.
--profile: instead, the call's kernel split from torch.profiler (a run of its own).

    python tools/rig_modes_probe.py --rigs 256 --cameras 4 --hyps 256 --reps 20 [--profile]
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
    ap.add_argument("--rigs", type=int, default=256)
    ap.add_argument("--cameras", type=int, default=4)
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
    from test_gpu_rig_limits import _scene
    from test_gpu_rig_pose_modes import _two_cluster_rigs
    E.load()
    gpu = card()
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream
    rot = math.radians(a.rot_deg)
    C, R = a.cameras, a.rigs
    n = R * C

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        fn()
        t1.record(stream)
        t1.synchronize()
        return t0.elapsed_time(t1)

    def median(fn):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        return float(np.median([timed(fn) for _ in range(a.reps)]))

    for frames in ("synthetic", "two-cluster"):
        if frames == "synthetic":   # 8 distinct rigs repeated (the scene builder is slow in Python)
            coords, pix, ext, _ = (np.tile(x, (R // 8,) + (1,) * (x.ndim - 1)) for x in _scene(E, C, 8, seed=1))
        else:
            coords, pix, ext, _, _ = (np.tile(x, (R // 8,) + (1,) * (x.ndim - 1)) for x in _two_cluster_rigs(E, C, 8, seed=2))
        dc, dp, de = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (coords, pix, ext))
        eng = E.Engine(max_frames=n, n_hyps=a.hyps)

        def rig_pass():
            eng.forward_rig_device(n, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr(), 0, None, 0, s)

        rig_pass()
        base = {"frames": frames, "rigs": R, "cameras": C, "hyps": a.hyps, "rot_deg": a.rot_deg, "trans_mm": a.trans_mm,
                "gpu": gpu, "reps": a.reps}
        if not a.profile:
            unc = A.rig_pose_uncertainty(eng, n, C)
            uptr = {k: v.data_ptr() for k, v in unc.items()}
            rec = dict(base, rig_pass_ms_median=median(rig_pass),
                       rig_pose_uncertainty_ms_median=median(lambda: eng.rig_pose_uncertainty_device(n, C, s, **uptr)))
            print(json.dumps(rec), flush=True)
        for M in (int(m) for m in a.modes.split(",")):
            out = A.rig_pose_modes(eng, n, C, M, rot, a.trans_mm)
            ptrs = {k: v.data_ptr() for k, v in out.items()}

            def call():
                eng.rig_pose_modes_device(n, C, M, rot, a.trans_mm, s, **ptrs)

            for _ in range(a.warmup):
                call()
            torch.cuda.synchronize()
            rec = dict(base, M=M, n_modes_mean=float(out["n_modes"].float().mean()))
            if a.profile:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(a.reps):
                        call()
                    torch.cuda.synchronize()
                kernels = {}
                for ev in prof.key_averages():
                    if any(w in ev.key for w in ("mode", "refine", "uncertainty", "Memcpy")):
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
