"""Measurement: what does guided sampling (dsac_set_sampling_logits_device) cost or save?  The BASELINE config-4 step
(1024 frames x 256 hypotheses, synthetic frames with rho 0.5 and sigma 25, inputs in HBM, CUDA events, L2 flushed
between steps as bench.py does) in three settings: the reference's uniform sampler, guided with all-zero logits (the
uniform distribution through the guided path), and guided with logits that put 90 % of each frame's weight on its
inlier cells (reprojection error below thr2d under the ground-truth pose).  Each setting has an engine of its own, so
that the first round of its passes is sized from its own previous pass, as in a training loop that changes the logits
a little per step; the settings alternate; median of 20 steps after 5 warm-ups each.  Then the candidates per frame,
the sampler's per-kernel split (dsac_sampler_profile_read, alternated as well: the profile serialises the sampler on one
stream, so these are the kernels' own durations, not the step's), and the time of dsac_sampling_log_prob_device and of
its backward over the batch.  Needs a GPU."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from dsac_b200 import engine as E
from oracle import oracle as O

NF, WARM, STEPS = 1024, 5, 20
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip(), flush=True)
O.build()
coords, pix, gt_cv, gt_jp = E.synth_frames(NF, rho=0.5, sigma=25.0)
inl = np.stack([O.diff_map(coords[f], pix[f], gt_cv[f, :3], gt_cv[f, 3:]) < 10 for f in range(NF)])
k = np.maximum(inl.sum(1, keepdims=True), 1)
focused = np.where(inl, np.log(0.9 / k), np.log(0.1 / np.maximum(E.N - k, 1))).astype(np.float32)
data = [torch.from_numpy(a).cuda() for a in (coords, pix, gt_jp)]
settings = [("uniform", None), ("guided, zero logits", torch.zeros((NF, E.N), device="cuda")),
            ("guided, 90% on inliers", torch.from_numpy(focused).cuda())]
print("inlier cells per frame: %.1f (mean)" % inl.sum(1).mean(), flush=True)
engines = {name: E.Engine(max_frames=NF) for name, _ in settings}
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
stream = torch.cuda.current_stream().cuda_stream


def step(name, logits):
    eng = engines[name]
    eng.set_sampling_logits_device(NF, logits.data_ptr() if logits is not None else None, stream)
    flush.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    eng.forward_device(NF, data[0].data_ptr(), data[1].data_ptr(), 0, data[2].data_ptr(), 0, stream)
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def candidates(name):
    res = engines[name].fetch(NF)
    return res.n_candidates.mean()


times = {name: [] for name, _ in settings}
cand = {}
for i in range(WARM + STEPS):
    for name, logits in settings:
        t = step(name, logits)
        if i >= WARM:
            times[name].append(t)
        if i == WARM:
            cand[name] = candidates(name)
for name, _ in settings:
    t = np.array(times[name])
    print("%-24s step %.3f ms median (min %.3f, max %.3f); %.0f candidates per frame"
          % (name, np.median(t), t.min(), t.max(), cand[name]), flush=True)

for eng in engines.values():
    eng.sampler_profile(True)
rows = {name: [] for name, _ in settings}
counts = {}
for i in range(WARM + STEPS):
    for name, logits in settings:
        step(name, logits)
        ms, counts[name] = engines[name].sampler_profile_read()
        if i >= WARM:
            rows[name].append(ms)
for name, _ in settings:
    m = np.median(np.array(rows[name]), 0)
    c = counts[name]
    print("%-24s sampler alone: generate+select %.3f  filter %.3f  solve %.3f  tail %.3f ms (sum %.3f); %d candidates, %d flagged, %d accepted"
          % (name, m[0], m[1], m[2], m[3], m.sum(), c[0], c[1], c[2]), flush=True)
for eng in engines.values():
    eng.sampler_profile(False)

logp = torch.empty(NF, dtype=torch.float64, device="cuda")
gl = torch.ones(NF, dtype=torch.float64, device="cuda")
grad = torch.empty((NF, E.N), dtype=torch.float32, device="cuda")
for name, logits in settings[1:]:
    eng = engines[name]
    step(name, logits)
    tf, tb = [], []
    for i in range(WARM + STEPS):
        a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        a.record()
        eng.sampling_log_prob_device(NF, logp.data_ptr(), stream)
        b.record()
        eng.sampling_log_prob_backward_device(NF, gl.data_ptr(), grad.data_ptr(), stream)
        c.record()
        c.synchronize()
        if i >= WARM:
            tf.append(a.elapsed_time(b)); tb.append(b.elapsed_time(c))
    print("%-24s sampling_log_prob %.3f ms, its backward %.3f ms (median of %d over %d frames)"
          % (name, np.median(tf), np.median(tb), STEPS, NF), flush=True)
for eng in engines.values():
    eng.close()
