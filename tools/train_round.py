"""Training-round times of both pipelines through the host entry points, the device entry points and the autograd losses
(development aid; prints one JSON line, writes nothing).

    python tools/train_round.py [--reps 3]

Workloads: the soft-argmax round (forward + backward) on 64 frames per call and the DSAC / RANSAC variant's round
(forward_dsac + backward_dsac) on 16 frames per call, 256 hypotheses, bench.py's seeded synthetic frames.  The same
rounds through the pose-valued outputs: softam_pose with a random seed per frame, and dsac_hypotheses with the
expected-loss form (every hypothesis seeded, as in the loss round) and with only the drawn hypothesis seeded.  Each record is
the wall time of `reps` calls between device synchronisations, per frame.  The card's name and power limit are read in
the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    import dsac_b200.engine as E
    from dsac_b200.autograd import dsac_expected_loss, dsac_hypotheses, softam_loss, softam_pose
    if not torch.cuda.is_available():
        raise SystemExit("train_round.py needs a CUDA device")
    nb3, nb5 = 64, 16
    coords, pix, gt_cv, gt_jp = E.synth_frames(nb3)
    d_coords, d_pix, d_gt = (torch.from_numpy(a).cuda() for a in (coords, pix, gt_jp))
    stream = torch.cuda.current_stream().cuda_stream

    def per_frame_ms(fn, frames):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / (args.reps * frames)

    out = {}
    eng3 = E.Engine(max_frames=nb3)
    pred3 = (d_coords.float() / 1000).contiguous().requires_grad_(True)
    grad3 = torch.empty_like(pred3)

    def softam_host():
        eng3.forward(coords, pix, gt_jp)
        eng3.backward(coords, pix, gt_jp, full=False)

    def softam_device():
        eng3.forward_device(nb3, d_coords.data_ptr(), d_pix.data_ptr(), 0, d_gt.data_ptr(), 0, stream)
        eng3.backward_device(nb3, d_dloss_dpred=grad3.data_ptr(), clamp=0.1, stream=stream)

    def softam_autograd():
        softam_loss(eng3, pred3, d_pix, d_gt).sum().backward()
    w3 = torch.randn((nb3, 6), dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))

    def softam_pose_autograd():   # a random seed on every frame's refined pose
        (softam_pose(eng3, pred3, d_pix) * w3).sum().backward()
    out["softam_64_frames"] = {"host_entries_ms_per_frame": per_frame_ms(softam_host, nb3),
                               "device_entries_ms_per_frame": per_frame_ms(softam_device, nb3),
                               "autograd_ms_per_frame": per_frame_ms(softam_autograd, nb3),
                               "softam_pose_random_seed_ms_per_frame": per_frame_ms(softam_pose_autograd, nb3)}
    eng3.close()

    eng5 = E.Engine(max_frames=nb5)
    c5, p5, g5 = d_coords[:nb5].contiguous(), d_pix[:nb5].contiguous(), d_gt[:nb5].contiguous()
    pred5 = (c5.float() / 1000).contiguous().requires_grad_(True)
    grad5 = torch.empty_like(pred5)
    exp5 = torch.empty(nb5, dtype=torch.float64, device="cuda")

    def dsac_host():
        eng5.forward_dsac(coords[:nb5], pix[:nb5], gt_jp[:nb5], random_draw=True)
        eng5.backward_dsac(nb5)

    def dsac_device():
        eng5.forward_dsac_device(nb5, c5.data_ptr(), p5.data_ptr(), 0, g5.data_ptr(), True, 0, stream, expected_loss=exp5.data_ptr())
        eng5.backward_dsac_device(nb5, d_dloss_dpred=grad5.data_ptr(), clamp=0.1, stream=stream)

    def dsac_autograd():
        dsac_expected_loss(eng5, pred5, p5, g5).sum().backward()
    w5 = torch.randn((nb5, eng5.cfg.n_hyps, 6), dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))

    def hyps_expected():   # expected-loss form: seeds sf_h w_h on every hypothesis, dL/dsf = ref_h . w_h
        sf, ref = dsac_hypotheses(eng5, pred5, p5)
        (sf * (ref * w5).sum(-1)).sum().backward()

    def hyps_drawn():      # the drawn (arg-max) hypothesis only: one seeded hypothesis per frame, no path II
        sf, ref = dsac_hypotheses(eng5, pred5, p5, random_draw=False)
        pick = sf.detach().argmax(1)
        (ref[torch.arange(nb5, device="cuda"), pick] * w5[:, 0]).sum().backward()
    out["dsac_16_frames"] = {"host_entries_ms_per_frame": per_frame_ms(dsac_host, nb5),
                             "device_entries_ms_per_frame": per_frame_ms(dsac_device, nb5),
                             "autograd_ms_per_frame": per_frame_ms(dsac_autograd, nb5),
                             "hypotheses_expected_loss_form_ms_per_frame": per_frame_ms(hyps_expected, nb5),
                             "hypotheses_drawn_only_ms_per_frame": per_frame_ms(hyps_drawn, nb5)}
    eng5.close()
    try:
        card = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        card = "unavailable (%s)" % str(ex)[:80]
    out["gpu"] = {"name": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": card, "reps": args.reps}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
