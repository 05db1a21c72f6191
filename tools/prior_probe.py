"""Times the config-4 step (1024 frames x 256 hypotheses, synthetic trajectory frames, sample + score + soft-argmax +
refinement on device inputs) with pose priors: none, k = 1 ungated, and k = 1 gated at chi^2 --gate around the previous
frame's refined pose with Lambda = inv(cov_xi + Q) (INTEGRATION.md, "Pose priors").  Per setting: the median of --reps
CUDA-event-timed steps after --warmup, candidates per frame, and the sampler's split from dsac_sampler_profile in a profiled
pass of its own.  Prints one JSON line per setting with the card's name and power limit.

    python tools/prior_probe.py --frames 1024 --hyps 256 --reps 20
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
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--hyps", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gate", type=float, default=16.81, help="chi^2 bound (16.81: chi^2_6 at 99 %%)")
    ap.add_argument("--q-rot", type=float, default=0.02, help="motion noise Q: rotation sigma (rad)")
    ap.add_argument("--q-t", type=float, default=20.0, help="motion noise Q: translation sigma (mm)")
    a = ap.parse_args()
    import numpy as np
    import torch
    import dsac_b200.engine as E
    from dsac_b200 import autograd as A
    E.load()
    gpu = card()
    n, H = a.frames, a.hyps
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream
    coords, pix, gt_cv, gt_jp = E.synth_frames(n, traj=True)
    dc, dp, dg = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (coords, pix, gt_jp))
    eng = E.Engine(max_frames=n, n_hyps=H)

    def fwd():
        eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 0, s)

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        fn()
        t1.record(stream)
        t1.synchronize()
        return t0.elapsed_time(t1)

    # the tracker's prediction for frame f: the refined pose of frame f - 1 (frame 0: its own) and its covariance
    fwd()
    ref = eng.fetch(n).ref_pose
    unc = A.pose_uncertainty(eng, n)
    cov = unc["cov_xi"].cpu().numpy()
    ok = unc["ok"].cpu().numpy().astype(bool)
    Q = np.diag([a.q_rot ** 2] * 3 + [a.q_t ** 2] * 3)
    prev = np.concatenate([[0], np.arange(n - 1)])
    poses = torch.from_numpy(np.ascontiguousarray(ref[prev][:, None, :])).cuda()
    info = np.stack([np.linalg.inv((cov[p] if ok[p] else 0) + Q) for p in prev])[:, None]
    info = torch.from_numpy(np.ascontiguousarray(info)).cuda()

    settings = [("none", None), ("k1_ungated", (poses, None, 0.0)), ("k1_gated", (poses, info, a.gate))]
    for name, pp in settings:
        if pp is None:
            eng.set_pose_priors_device(n, 0, None)
        else:
            eng.set_pose_priors_device(n, 1, pp[0].data_ptr(), pp[1].data_ptr() if pp[1] is not None else None, pp[2], s)
        for _ in range(a.warmup):
            fwd()
        t = [timed(fwd) for _ in range(a.reps)]
        res = eng.fetch(n)
        eng.sampler_profile(True)
        fwd()
        ms, counts = eng.sampler_profile_read()
        eng.sampler_profile(False)
        print(json.dumps({"setting": name, "frames": n, "hyps": H, "gpu": gpu, "step_ms_median": float(np.median(t)),
                          "step_ms_min": float(np.min(t)), "reps": a.reps,
                          "candidates_per_frame": float(res.n_candidates.mean()),
                          "correct_fraction": float(res.correct.mean()), "exhausted_frames": int((res.status & 1).astype(bool).sum()),
                          "bad_prior_frames": int((res.status & E.ST_BAD_PRIOR).astype(bool).sum()),
                          "sampler_profile_ms": {"gen_select": ms[0], "filter": ms[1], "solve": ms[2], "tail": ms[3]},
                          "sampler_profile_counts": {"generated": counts[0], "flagged": counts[1], "accepted": counts[2],
                                                     "rounds": counts[3]}}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
