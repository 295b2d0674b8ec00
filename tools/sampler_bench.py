#!/usr/bin/env python
"""Time DDIM against DPM-Solver++(2M) on one GPU: ``pipe(...)`` end to end at configs[1] shapes (512x512, one 16-frame
window, CFG 3.5, bf16 UNet, synthetic weights and conditioning from bench.build_ours).

  python tools/sampler_bench.py [--arms ddim:25,dpm:10,dpm:15,dpm:25] [--runs 3] [--warmup 1]

The arms alternate within each run, so every arm sees the same drift.  A timed run is one ``pipe(...)`` call from host
inputs to the video in pinned host memory (host clock around a call that ends in a device synchronise).  Prints the card
(name, power limit and max SM clock, read in the same process), one JSON line per run and one summary line per arm:
min / mean / max frames/s, ms per step (call time / steps), and the marginal ms per step between the two DPM arms
with the fewest and most steps (the UNet forward + update of one step, with the fixed decode and prologue removed).
"""
import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from eta_bench import card  # noqa: E402

L, OVERLAP = 16, 8


def call(pipe, steps):
    return pipe(reference_image=None, kps_images=None, audio_waveform=None, width=512, height=512, video_length=L,
                num_inference_steps=steps, guidance_scale=3.5, context_frames=16, context_overlap=OVERLAP,
                reference_attention_weight=0.95, audio_attention_weight=3.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arms", default="ddim:25,dpm:10,dpm:15,dpm:25")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampler_bench.py: no CUDA device (the product has no CPU path)")
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
    arms = [(name, int(steps)) for name, steps in (a.split(":") for a in args.arms.split(","))]
    schedulers = {"ddim": DDIMScheduler(), "dpm": DPMSolverMultistepScheduler()}
    print(json.dumps(dict(card=card())), flush=True)
    pipe, _, _ = bench.build_ours(L, 64, torch.device("cuda", 0))
    for name, steps in arms:
        pipe.scheduler = schedulers[name]
        for _ in range(args.warmup):
            call(pipe, steps)
    times = {arm: [] for arm in arms}
    videos = {}
    for r in range(args.runs):
        for arm in arms:
            pipe.scheduler = schedulers[arm[0]]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            video = call(pipe, arm[1])
            sec = time.perf_counter() - t0
            times[arm].append(sec)
            if arm in videos:
                assert torch.equal(videos[arm], video), f"{arm}: run {r} differs from run 0"
            videos[arm] = video
            print(json.dumps(dict(sampler=arm[0], steps=arm[1], run=r, sec=round(sec, 4),
                                  frames_per_sec=round(L / sec, 4))), flush=True)
    for arm in arms:
        fps = [L / s for s in times[arm]]
        mean = sum(times[arm]) / len(times[arm])
        print(json.dumps(dict(sampler=arm[0], steps=arm[1], frames=L, runs=args.runs,
                              frames_per_sec_min=round(min(fps), 4), frames_per_sec_mean=round(sum(fps) / len(fps), 4),
                              frames_per_sec_max=round(max(fps), 4), ms_per_step=round(1e3 * mean / arm[1], 2),
                              video_sha256=hashlib.sha256(videos[arm].numpy().tobytes()).hexdigest())), flush=True)
    dpm = sorted(a for a in arms if a[0] == "dpm")
    if len(dpm) > 1 and dpm[0][1] != dpm[-1][1]:
        lo, hi = dpm[0], dpm[-1]
        marginal = (sum(times[hi]) / len(times[hi]) - sum(times[lo]) / len(times[lo])) / (hi[1] - lo[1])
        print(json.dumps(dict(marginal_ms_per_step=round(1e3 * marginal, 2), between=[lo[1], hi[1]])), flush=True)
    ddim = [a for a in arms if a[0] == "ddim"]
    for a in ddim:
        for b in dpm:
            if a[1] == b[1]:
                d = (videos[a] - videos[b]).abs().mean().item()
                print(json.dumps(dict(same_steps=a[1], ddim_vs_dpm_mean_abs_difference=d)), flush=True)


if __name__ == "__main__":
    main()
