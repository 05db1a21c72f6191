"""Measurement: what does an RGB-D pass (dsac_set_cell_depth_device) cost?  The BASELINE config-4 step (1024 frames x
256 hypotheses, inputs in HBM, CUDA events, L2 flushed between steps as bench.py does) on the seeded synthetic RGB-D
frames of tests/rgbd_oracle.py (rho 0.5, sigma 25 mm) in four settings: RGB; RGB-D with full depth; RGB-D with 15 % of
the cells without depth; the same with guided sampling and -inf logits on the cells without depth (zero elsewhere).
Each setting has an engine of its own; the settings alternate; median of 20 steps after 5 warm-ups.  Then the candidates
per frame and the sampler's split (dsac_sampler_profile_read: generate + select, acceptance -- k1_filter + k1_solve in
RGB, k1_kabsch in RGB-D --, tail), alternated as well.  Needs a GPU."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import rgbd_oracle as R
from dsac_b200 import engine as E

NF, WARM, STEPS = 1024, 5, 20
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip(), flush=True)
coords, pix, depth, _, gt_jp = R.synth(NF, seed=2024, rho=0.5, sigma=25.0)
holes = depth.copy()
holes[np.random.default_rng(1).random(holes.shape) < 0.15] = np.nan
guide = np.where(np.isfinite(holes), 0.0, -np.inf).astype(np.float32)
data = [torch.from_numpy(a).cuda() for a in (coords, pix, gt_jp)]
settings = [("RGB", None, None), ("RGB-D", torch.from_numpy(depth).cuda(), None),
            ("RGB-D 15% holes", torch.from_numpy(holes).cuda(), None),
            ("RGB-D 15% holes guided", torch.from_numpy(holes).cuda(), torch.from_numpy(guide).cuda())]
engines = {name: E.Engine(max_frames=NF) for name, _, _ in settings}
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
stream = torch.cuda.current_stream().cuda_stream
for name, d, g in settings:
    engines[name].set_cell_depth_device(NF, d.data_ptr() if d is not None else None, stream)
    engines[name].set_sampling_logits_device(NF, g.data_ptr() if g is not None else None, stream)


def step(name):
    flush.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    engines[name].forward_device(NF, data[0].data_ptr(), data[1].data_ptr(), 0, data[2].data_ptr(), 0, stream)
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


times = {name: [] for name, _, _ in settings}
cand = {}
for i in range(WARM + STEPS):
    for name, _, _ in settings:
        t = step(name)
        if i >= WARM:
            times[name].append(t)
        if i == WARM:
            res = engines[name].fetch(NF)
            cand[name] = (res.n_candidates.mean(), res.correct.mean())
for name, _, _ in settings:
    t = np.array(times[name])
    print("%-24s step %.3f ms median (min %.3f, max %.3f); %.0f candidates per frame; %.3f correct"
          % (name, np.median(t), t.min(), t.max(), cand[name][0], cand[name][1]), flush=True)

for eng in engines.values():
    eng.sampler_profile(True)
rows = {name: [] for name, _, _ in settings}
for i in range(WARM + STEPS):
    for name, _, _ in settings:
        step(name)
        ms, _ = engines[name].sampler_profile_read()
        if i >= WARM:
            rows[name].append(ms)
for name, _, _ in settings:
    m = np.median(np.array(rows[name]), 0)
    print("%-24s sampler alone: generate+select %.3f  acceptance %.3f (filter %.3f + solve %.3f)  tail %.3f ms"
          % (name, m[0], m[1] + m[2], m[1], m[2], m[3]), flush=True)
for eng in engines.values():
    eng.close()
