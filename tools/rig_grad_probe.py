"""Times the rig backward (dsac_backward_rig_device) against the ordinary soft-argmax backward in implicit mode
(dsac_backward_device) on the same synthetic frames, for C in {1, 2, 4} cameras per rig, n in {64, 256} frames and
H in {64, 256} hypotheses per frame with C H <= 1024.  Each backward follows its own forward pass (rig pass, ordinary
pass); only the backward is timed: a host clock around the call and a device synchronise, median of --reps after
--warmup calls of each, the two alternating.  Prints one JSON line per case with the card's name and power limit.

    python tools/rig_grad_probe.py [--reps 20] [--warmup 3]
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


def ring(C):
    import numpy as np
    from scipy.spatial.transform import Rotation
    ext = np.zeros((C, 6))
    for c in range(C):
        a = 2 * np.pi * c / C
        ext[c, :3] = Rotation.from_euler("y", a).as_rotvec()
        ext[c, 3:] = [80.0 * np.sin(a), 0.0, 80.0 * np.cos(a)]
    return ext


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    import dsac_b200.engine as E
    E.load()
    name = card()
    for n in (64, 256):
        coords, pix, gt_cv, gt_jp = E.synth_frames(n, n_streams=2)
        dc = torch.from_numpy(coords).cuda()
        dp = torch.from_numpy(pix).cuda()
        dg = torch.from_numpy(gt_jp).cuda()
        for H in (64, 256):
            eng = E.Engine(max_frames=n, n_hyps=H, n_streams=2)
            eng.set_coord_derivatives("implicit")
            for C in (1, 2, 4):
                if C * H > 1024:
                    continue
                R = n // C
                de = torch.from_numpy(np.tile(ring(C), (R, 1))).cuda()
                dgr = torch.from_numpy(gt_jp[::C].copy()).cuda()   # a rig's ground truth: any pose serves for timing
                dpred = torch.empty((n, E.N, 3), dtype=torch.float32, device="cuda")

                def rig():
                    eng.forward_rig_device(n, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr(), 0, dgr.data_ptr(), 0)
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    eng.backward_rig_device(n, None, None, dpred.data_ptr(), 0.1)
                    torch.cuda.synchronize()
                    return (time.perf_counter() - t) * 1e3

                def ordinary():
                    eng.forward_device(n, dc.data_ptr(), dp.data_ptr(), 0, dg.data_ptr(), 0)
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    eng.backward_device(n, None, None, dpred.data_ptr(), 0.1)
                    torch.cuda.synchronize()
                    return (time.perf_counter() - t) * 1e3

                for _ in range(a.warmup):
                    rig()
                    ordinary()
                tr, to = [], []
                for _ in range(a.reps):
                    tr.append(rig())
                    to.append(ordinary())
                print(json.dumps({"card": name, "frames": n, "cameras": C, "hyps": H, "pool": C * H,
                                  "rig_backward_ms_median": round(float(np.median(tr)), 3),
                                  "ordinary_implicit_backward_ms_median": round(float(np.median(to)), 3)}), flush=True)
            eng.close()


if __name__ == "__main__":
    main()
