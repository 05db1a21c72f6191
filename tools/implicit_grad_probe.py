"""Times one backward per coordinate-derivative mode (dsac_set_coord_derivatives) on the GPU: the soft-argmax backward and
the DSAC variant's backward after one forward, the two modes alternated in one process, median of --reps after warm-up.
Prints one JSON line per setting with the card's name and power limit and the refinement CTAs each mode launches.

    python tools/implicit_grad_probe.py --sizes 1 64 1024 --dsac-sizes 1 64 --reps 20
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1, 64, 1024])
    ap.add_argument("--dsac-sizes", type=int, nargs="+", default=[1, 64])
    ap.add_argument("--sub-samples", type=float, nargs="+", default=[0.01, 1.0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    import dsac_b200.engine as E
    E.load()
    gpu = card()
    stream = torch.cuda.current_stream().cuda_stream

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    for pipeline, sizes in (("softam", a.sizes), ("dsac", a.dsac_sizes)):
        for n in sizes:
            coords, pix, gt_cv, gt_jp = E.synth_frames(n)
            for ss in a.sub_samples:
                eng = E.Engine(max_frames=n, n_hyps=256, sub_sample=ss)
                modes = ["central", "implicit"]
                if pipeline == "softam":
                    eng.forward(coords, pix, gt_jp)
                    if ss > 0.01:
                        modes = ["implicit"]   # central mode refuses more than 16 gradient cells per frame
                    def run():
                        eng.backward_device(n, stream=stream)
                else:
                    eng.forward_dsac(coords, pix, gt_jp, random_draw=False)
                    def run():
                        eng.backward_dsac(n)
                times = {m: [] for m in modes}
                jobs = {}
                for m in modes:
                    eng.set_coord_derivatives(m)
                    for _ in range(a.warmup):
                        run()
                for _ in range(a.reps):
                    for m in modes:
                        eng.set_coord_derivatives(m)
                        times[m].append(timed(run))
                for m in modes:
                    eng.set_coord_derivatives(m)
                    if pipeline == "softam":
                        jobs[m] = n * (12 + 1 + 1) if m == "implicit" else n * (12 + 16 * 6)   # refine + replay + IFT CTAs
                    else:
                        bw = eng.backward_dsac(n)
                        # the replay of every hypothesis slot (n H CTAs, those past the selection exit at once), the
                        # refinement jobs, and in implicit mode one k_refine_ift CTA per selected hypothesis
                        jobs[m] = n * 256 + int(bw.n_refine_jobs.sum()) + (int(bw.n_selected.sum()) if m == "implicit" else 0)
                print(json.dumps({"pipeline": pipeline, "n": n, "sub_sample": ss, "gpu": gpu,
                                  "ms_median": {m: float(np.median(v)) for m, v in times.items()},
                                  "refine_ctas": jobs, "reps": a.reps}), flush=True)


if __name__ == "__main__":
    main()
