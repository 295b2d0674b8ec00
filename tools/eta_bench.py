#!/usr/bin/env python
"""Cost of stochastic DDIM (eta > 0) on one GPU: ``pipe(...)`` end to end with eta = 0 and eta = 1, alternating.

  python tools/eta_bench.py [--configs 1,2] [--etas 0,1] [--runs 3] [--warmup 1] [--dump DIR] [--compare DIR]

configs[1] is 512x512, one 16-frame window; configs[2] is 512x512, 96 frames in windows of 16 with overlap 8 (11 windows);
both 25 DDIM steps, CFG 3.5, bf16 UNet, synthetic weights and conditioning (bench.build_ours).  Every call passes a fresh
CPU generator seeded 1234 -- the reference CLI's case, where each step's variance noise is drawn on the host -- so every
run of one (config, eta) computes the same video.  A timed run is one ``pipe(...)`` call from host inputs to the video in
pinned host memory (host clock around a call that ends in a device synchronise).  Prints the card, one JSON line per run
and one summary line per (config, eta) with the min / mean / max frames/s and the SHA-256 of the video's bytes.

``--dump DIR`` writes each (config, eta)'s video to DIR/c<k>_eta<e>.pt (about 300 MB at configs[2], so DIR is best a
scratch directory); ``--compare DIR`` checks that every video this
run computes equals the one of the same name in DIR bit for bit (DIR written by this tool on another build, e.g. the
eta = 0 outputs of a build without eta support).
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

CONFIGS = {1: dict(L=16, overlap=8), 2: dict(L=96, overlap=8)}


def card():
    import subprocess
    p = torch.cuda.get_device_properties(0)
    line = dict(name=p.name, sms=p.multi_processor_count)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        line["power_limit_and_max_sm_clock"] = q[0] if q else None
    except Exception as e:  # the numbers stay valid without the query
        line["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return line


def call(pipe, L, overlap, eta):
    kw = dict(eta=eta, generator=torch.Generator().manual_seed(1234)) if eta else {}
    return pipe(reference_image=None, kps_images=None, audio_waveform=None, width=512, height=512, video_length=L,
                num_inference_steps=25, guidance_scale=3.5, context_frames=16, context_overlap=overlap,
                reference_attention_weight=0.95, audio_attention_weight=3.0, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="1,2")
    ap.add_argument("--etas", default="0,1")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dump", default="")
    ap.add_argument("--compare", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eta_bench.py: no CUDA device (the product has no CPU path)")
    etas = [float(e) for e in args.etas.split(",")]
    print(json.dumps(dict(card=card())), flush=True)
    dev = torch.device("cuda", 0)
    mismatches = 0
    for k in [int(c) for c in args.configs.split(",")]:
        L, overlap = CONFIGS[k]["L"], CONFIGS[k]["overlap"]
        pipe, _, _ = bench.build_ours(L, 64, dev)
        for eta in etas:
            for _ in range(args.warmup):
                call(pipe, L, overlap, eta)
        times = {eta: [] for eta in etas}
        videos = {}
        for r in range(args.runs):
            for eta in etas:                                   # alternating: both arms see the same drift
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                video = call(pipe, L, overlap, eta)
                sec = time.perf_counter() - t0                 # the call ends in a device synchronise
                times[eta].append(sec)
                if eta in videos:
                    assert torch.equal(videos[eta], video), f"configs[{k}] eta={eta}: run {r} differs from run 0"
                videos[eta] = video
                print(json.dumps(dict(config=k, frames=L, eta=eta, run=r, sec=round(sec, 4),
                                      frames_per_sec=round(L / sec, 4))), flush=True)
        for eta in etas:
            fps = [L / s for s in times[eta]]
            name = f"c{k}_eta{eta:g}.pt"
            line = dict(config=k, frames=L, windows=(L - 16) // (16 - overlap) + 1, eta=eta, runs=args.runs,
                        frames_per_sec_min=round(min(fps), 4), frames_per_sec_mean=round(sum(fps) / len(fps), 4),
                        frames_per_sec_max=round(max(fps), 4),
                        video_sha256=hashlib.sha256(videos[eta].numpy().tobytes()).hexdigest())
            if args.dump:
                os.makedirs(args.dump, exist_ok=True)
                torch.save(videos[eta], os.path.join(args.dump, name))
            if args.compare:
                path = os.path.join(args.compare, name)
                if os.path.exists(path):
                    same = torch.equal(torch.load(path), videos[eta])
                    line["equal_to_compare_dir"] = same
                    mismatches += not same
            print(json.dumps(line), flush=True)
        if len(etas) > 1:
            a, b = videos[etas[0]], videos[etas[-1]]
            print(json.dumps(dict(config=k, eta_outputs_differ=not torch.equal(a, b),
                                  mean_abs_difference=(a - b).abs().mean().item())), flush=True)
        del pipe
        torch.cuda.empty_cache()
    if mismatches:
        raise SystemExit(f"eta_bench.py: {mismatches} video(s) differ from {args.compare}")


if __name__ == "__main__":
    main()
