"""Times the rig score hooks (dsac_set_rig_score_hooks) on 16 rigs of 4 cameras at H = 64 (64 frames, pools of P = 256):
the closed-form rig pass against the hooked one, the hooked pass with a trivial float64 on-device scorer and with the
score CNN (dsac_b200.score_cnn.ScoreCNN), and the hooked rig backward (dsac_backward_rig_pose_device) with each; host
clock around each call and a device synchronise, median of --reps after --warmup calls, the cases alternating.  Then, in
a separate profiled run (torch.profiler), the device time of k_score_rig with and without the error images, and the
write rate of the error images (n P 1600 fp32) against the H100 SXM's 3.35 TB/s.  Prints one JSON line with the card's
name and power limit, read in the same call.

    python tools/rig_seam_probe.py [--reps 20] [--warmup 3] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

N = 1600
A1, B1, THR = 0.3, 1.5, 10.0   # the trivial scorer: A1 sum_i sigmoid(B1 (THR - d_ji)) in float64
HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


class _W:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}


class Sigmoid:
    """The trivial float64 scorer and its adjoint as hooks, on the stream the engine passes."""

    def __call__(self, dm, n, P, sc, stream):
        import torch
        with torch.cuda.stream(torch.cuda.ExternalStream(stream) if stream else torch.cuda.current_stream()):
            d = torch.as_tensor(_W(dm, (n, P, N), "<f4"), device="cuda")
            s = torch.as_tensor(_W(sc, (n, P), "<f8"), device="cuda")
            s.copy_(A1 * torch.sigmoid(B1 * (THR - d.double())).sum(2))
        return 0

    def backward(self, dm, sg, n, P, out, stream):
        import torch
        with torch.cuda.stream(torch.cuda.ExternalStream(stream) if stream else torch.cuda.current_stream()):
            d = torch.as_tensor(_W(dm, (n, P, N), "<f4"), device="cuda")
            g = torch.as_tensor(_W(sg, (n, P), "<f8"), device="cuda")
            o = torch.as_tensor(_W(out, (n, P, N), "<f8"), device="cuda")
            s = torch.sigmoid(B1 * (THR - d.double()))
            o.copy_(g[:, :, None] * (-A1 * B1) * s * (1 - s))
        return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import dsac_b200.engine as E
    from dsac_b200.score_cnn import ScoreCNN
    from rig_rgbd_probe import card, scene
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    R, C, H = 16, 4, 64
    n, P = R * C, C * H
    coords, pix, _, ext = scene(R, C)
    dev = lambda x, t: torch.from_numpy(np.ascontiguousarray(x, t)).cuda()
    dc, dp, de = dev(coords, np.int16), dev(pix, np.int32), dev(ext, np.float64)
    f64 = dict(dtype=torch.float64, device="cuda")
    ref, st = torch.zeros((R, 6), **f64), torch.zeros(R, dtype=torch.int32, device="cuda")
    seed = torch.ones((R, 6), **f64)
    dpred = torch.zeros((n, N, 3), dtype=torch.float32, device="cuda")
    # one engine per scorer, so that no case re-registers hooks between calls
    plain = E.Engine(max_frames=n, n_hyps=H)
    sig, cnn = Sigmoid(), ScoreCNN()
    eng_sig, eng_cnn = E.Engine(max_frames=n, n_hyps=H), E.Engine(max_frames=n, n_hyps=H)
    eng_sig.set_rig_score_hooks(sig, sig.backward)
    eng_cnn.set_rig_score_hooks(cnn, cnn.backward)

    def rig_pass(eng):
        eng.forward_rig_device(n, C, dc.data_ptr(), dp.data_ptr(), de.data_ptr(), ref_pose=ref.data_ptr(), status=st.data_ptr())

    def backward(eng):
        eng.backward_rig_pose_device(n, seed.data_ptr(), None, dpred.data_ptr())

    calls = {
        "closed_form_pass": lambda: rig_pass(plain),
        "closed_form_backward": lambda: backward(plain),
        "sigmoid_pass": lambda: rig_pass(eng_sig),
        "sigmoid_backward": lambda: backward(eng_sig),
        "cnn_pass": lambda: rig_pass(eng_cnn),
        "cnn_backward": lambda: backward(eng_cnn),
    }
    times = {k: [] for k in calls}
    for i in range(a.warmup + a.reps):
        for k, fn in calls.items():   # (each backward follows its engine's pass)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if i >= a.warmup:
                times[k].append(time.perf_counter() - t0)
    res = {k + "_ms": round(1e3 * float(np.median(v)), 3) for k, v in times.items()}
    res["rigs_refined"] = int(((st.cpu().numpy() & (2 | 256)) == 0).sum())
    # the score kernel alone, in a profiled run of its own: ten passes of each form
    from torch.profiler import ProfilerActivity, profile
    reps = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            rig_pass(plain)
            rig_pass(eng_sig)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            kern[ev.key] = t / 1e3 / reps
    if a.out:
        prof.export_chrome_trace(os.path.join(a.out, "rig_seam.pt.trace.json"))
    dm_ms = sum(v for k, v in kern.items() if "k_score_rig<true" in k)
    plain_ms = sum(v for k, v in kern.items() if "k_score_rig<false" in k)
    dm_bytes = n * P * N * 4
    res["k_score_rig_ms"] = round(plain_ms, 4)
    res["k_score_rig_write_dm_ms"] = round(dm_ms, 4)
    res["diffmap_bytes"] = dm_bytes
    if dm_ms > 0:
        rate = dm_bytes / (dm_ms * 1e-3)
        res["diffmap_write_TBps"] = round(rate / 1e12, 3)
        res["diffmap_write_share_of_3.35TBps"] = round(rate / HBM_BYTES_PER_S, 3)
    res["kernels_ms_per_pass"] = {k: round(v, 4) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])[:12]}
    for e in (plain, eng_sig, eng_cnn):
        e.close()
    print(json.dumps({"card": card(), "R": R, "C": C, "H": H, "frames": n, **res}))


if __name__ == "__main__":
    main()
