"""Measurement: what do per-frame cameras (dsac_set_cameras) cost?  The BASELINE config-4 step (1024 frames x 256
hypotheses x 1600 cells, inputs in HBM, CUDA events, L2 flushed between steps as bench.py does) in three settings:
no cameras, 1024 identical cameras (the config's), 1024 distinct cameras (focal length uniform in 400..1200; their
frames are synthesised for those cameras).  The settings alternate; median of 20 steps after 5 warm-ups each.  Then the
sampler's per-kernel split (dsac_sampler_profile_read; the profile serialises the sampler on one stream, so these are
the kernels' own durations, not the step's).  Needs a GPU: there is nothing to measure without one."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from dsac_b200 import engine as E

NF, WARM, STEPS = 1024, 5, 20
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip(), flush=True)
cfg = E.default_config()
same = np.tile(np.array([cfg.focal, cfg.cx, cfg.cy]), (NF, 1))
rng = np.random.default_rng(0)
distinct = np.stack([rng.uniform(400.0, 1200.0, NF), np.full(NF, cfg.cx), np.full(NF, cfg.cy)], 1)


def frames(cams):
    if cams is None:
        c, p, _, g = E.synth_frames(NF)
    else:
        parts = [E.synth_frames(1, frame0=i, focal=cams[i, 0], cx=cams[i, 1], cy=cams[i, 2]) for i in range(NF)]
        c, p, _, g = (np.concatenate([q[k] for q in parts]) for k in range(4))
    return [torch.from_numpy(a).cuda() for a in (c, p, g)]


std = frames(None)
settings = [("no cameras", None, std), ("1024 identical cameras", same, std), ("1024 distinct cameras", distinct, frames(distinct))]
eng = E.Engine(max_frames=NF)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
stream = torch.cuda.current_stream().cuda_stream


def step(cams, data):
    eng.set_cameras(cams, stream)
    flush.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    eng.forward_device(NF, data[0].data_ptr(), data[1].data_ptr(), 0, data[2].data_ptr(), 0, stream)
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


times = {name: [] for name, _, _ in settings}
for i in range(WARM + STEPS):
    for name, cams, data in settings:
        t = step(cams, data)
        if i >= WARM:
            times[name].append(t)
for name, _, _ in settings:
    t = np.array(times[name])
    print("%-24s step %.3f ms median (min %.3f, max %.3f)" % (name, np.median(t), t.min(), t.max()), flush=True)

eng.sampler_profile(True)
for name, cams, data in settings:
    rows = []
    for i in range(WARM + STEPS):
        step(cams, data)
        ms, counts = eng.sampler_profile_read()
        if i >= WARM:
            rows.append(ms)
    m = np.median(np.array(rows), 0)
    print("%-24s sampler alone: generate+select %.3f  filter %.3f  solve %.3f  resume %.3f ms; %d candidates, %d flagged, %d accepted"
          % (name, m[0], m[1], m[2], m[3], counts[0], counts[1], counts[2]), flush=True)
eng.close()
