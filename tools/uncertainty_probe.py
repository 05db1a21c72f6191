"""Times dsac_pose_uncertainty_device on the GPU: after a soft-argmax forward of --softam-frames frames and after a
DSAC-variant forward of --dsac-frames frames (H = --hyps), CUDA events around each call on the engine's stream, median of
--reps after --warmup calls.  The forward pass itself is timed the same way for scale.  Prints one JSON line per pipeline
with the card's name and power limit.

    python tools/uncertainty_probe.py --softam-frames 1024 --dsac-frames 64 --reps 20
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--softam-frames", type=int, default=1024)
    ap.add_argument("--dsac-frames", type=int, default=64)
    ap.add_argument("--hyps", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="also time the call's kernels with torch.profiler")
    a = ap.parse_args()
    import numpy as np
    import torch
    import dsac_b200.engine as E
    from dsac_b200 import autograd as A
    E.load()
    gpu = card()
    stream = torch.cuda.current_stream()

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        fn()
        t1.record(stream)
        t1.synchronize()
        return t0.elapsed_time(t1)

    for pipeline, n in (("softam", a.softam_frames), ("dsac", a.dsac_frames)):
        coords, pix, gt_cv, gt_jp = E.synth_frames(n)
        dc, dp, dg = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (coords, pix, gt_jp))
        eng = E.Engine(max_frames=n, n_hyps=a.hyps)
        s = stream.cuda_stream
        if pipeline == "softam":
            def fwd():
                eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 0, s)
        else:
            def fwd():
                eng.forward_dsac_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), True, 0, s)
        fwd()
        out = A.pose_uncertainty(eng, n)
        ptrs = {k: v.data_ptr() for k, v in out.items()}

        def call():
            eng.pose_uncertainty_device(n, s, **ptrs)

        for _ in range(a.warmup):
            call()
        t_call = [timed(call) for _ in range(a.reps)]
        for _ in range(a.warmup):
            fwd()
        t_fwd = [timed(fwd) for _ in range(a.reps)]
        call()
        torch.cuda.synchronize()
        kernels = {}
        if a.profile:   # kernel times of --reps calls, in a run of their own after the timed ones
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    call()
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                if "refine" in ev.key or "uncertainty" in ev.key:
                    us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    kernels[ev.key.split("(")[0]] = us / 1e3 / a.reps
        ok = out["ok"].reshape(-1)
        print(json.dumps({"pipeline": pipeline, "frames": n, "hyps": a.hyps, "jobs": int(ok.numel()), "gpu": gpu,
                          "call_ms_median": float(np.median(t_call)), "call_ms_min": float(np.min(t_call)),
                          "forward_ms_median": float(np.median(t_fwd)), "ok_fraction": float(ok.float().mean()),
                          "n_fit_median": float(out["n_fit"].reshape(-1).float().median()),
                          "support_median": float(out["support"].reshape(-1).float().median()), "reps": a.reps,
                          "kernel_ms_per_call": kernels}), flush=True)


if __name__ == "__main__":
    main()
