#!/usr/bin/env python
"""Throughput and memory of several samples per call (``num_images_per_prompt``) on one GPU.

  python tools/samples_bench.py --steps K --warmup W [--samples 1,2,4] [--sizes 512,768]

For every n one timed pass is what bench.py times at configs[1] (one 16-frame window, 25 DDIM steps, CFG 3.5, bf16,
synthetic weights): the denoise loop over n samples of the same conditioning -- one UNet forward of 2 n 16 frames per
DDIM step -- followed by the VAE decode of all n x 16 frames, results left on the device.  Prints one JSON line per
(size, n) with per-sample frames/s (n x 16 frames per pass), the UNet time per DDIM step and the peak memory of the pass,
then one line per size with the largest n that a linear fit of the reserved memory over the measured n puts under the
card's memory (an extrapolation: that n is not run).  The first size is timed; the others are only measured for memory
(one DDIM step after a warm-up pass).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

L = 16


def card():
    p = torch.cuda.get_device_properties(0)
    line = dict(name=p.name, sms=p.multi_processor_count, memory_gb=round(p.total_memory / 2 ** 30, 1))
    try:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        line["power_limit_and_max_sm_clock"] = q[0] if q else None
    except Exception as e:  # the numbers stay valid without the query
        line["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return line


def setup(h):
    from vexpress_b200.modules import ReferenceAttentionControl
    dev = torch.device("cuda", 0)
    pipe, host, _ = bench.build_ours(L, h, dev)
    reader = ReferenceAttentionControl(pipe.denoising_unet, do_classifier_free_guidance=True, mode="read",
                                       fusion_blocks="full", reference_attention_weight=0.95, audio_attention_weight=3.0)
    reader.update(pipe.reference_net.writer_view, True, dtype=torch.bfloat16)
    return pipe, host["kps"].to(dev), host["audio"].to(dev), reader


def latents(pipe, n, h):
    """(n,4,L,h,h) drawn by the pipeline's own prepare_latents (bench.py's pipeline overrides it with one fixed sample)."""
    from vexpress_b200.pipelines.v_express_pipeline import VExpressPipeline
    gens = [torch.Generator().manual_seed(100 + i) for i in range(n)]
    lat = VExpressPipeline.prepare_latents(pipe, n, 4, 8 * h, 8 * h, L, torch.bfloat16, None, gens).cuda()
    assert lat.shape == (n, 4, L, h, h)
    return lat


def one_pass(pipe, lat, kps, audio, timesteps):
    out = pipe.denoise(lat.clone(), kps, audio, timesteps, 3.5, 16, 8)
    return pipe.decode_to_device(out, False)


def measure(pipe, kps, audio, n, h, ddim_steps, steps, warmup):
    from vexpress_b200.pipelines.v_express_pipeline import retrieve_timesteps
    timesteps, _ = retrieve_timesteps(pipe.scheduler, ddim_steps, kps.device)
    lat = latents(pipe, n, h)
    pipe._graphs.clear()                   # the captured graphs of the previous n would stay in the reserved pool
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(warmup):
        one_pass(pipe, lat, kps, audio, timesteps)
    row = dict(size=8 * h, n=n, ddim_steps=ddim_steps)
    if steps:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            one_pass(pipe, lat, kps, audio, timesteps)
        e1.record()
        torch.cuda.synchronize()
        sec = e0.elapsed_time(e1) / 1e3 / steps
        e0.record()
        pipe.denoise(lat.clone(), kps, audio, timesteps, 3.5, 16, 8)
        e1.record()
        torch.cuda.synchronize()
        row.update(steps=steps, warmup=warmup, sec_per_pass=sec, frames_per_sec=n * L / sec,
                   frames_per_sec_per_sample=L / sec, unet_ms_per_ddim_step=e0.elapsed_time(e1) / ddim_steps)
    row["peak_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    row["reserved_gb"] = torch.cuda.max_memory_reserved() / 2 ** 30
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--samples", default="1,2,4")
    ap.add_argument("--sizes", default="512,768")
    ap.add_argument("--memory-samples", default="1,2", help="n measured (memory only) at the sizes after the first")
    ap.add_argument("--ddim-steps", type=int, default=25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("samples_bench.py: no CUDA device (the product has no CPU path)")
    ns = [int(x) for x in args.samples.split(",")]
    sizes = [int(x) for x in args.sizes.split(",")]
    print(json.dumps(dict(card=card())), flush=True)
    total_gb = torch.cuda.get_device_properties(0).total_memory / 2 ** 30
    for k, size in enumerate(sizes):
        h = size // 8
        t0 = time.time()
        pipe, kps, audio, reader = setup(h)
        timed = k == 0
        rows = []
        for n in (ns if timed else [int(x) for x in args.memory_samples.split(",")]):
            # memory-only sizes: one DDIM step (after one warm-up pass that captures the graph) is the same peak
            row = measure(pipe, kps, audio, n, h, args.ddim_steps if timed else 1, args.steps if timed else 0,
                          max(args.warmup, 1))
            rows.append(row)
            print(json.dumps(row), flush=True)
        # peak(n) = a + b n over the measured points; the reserved pool, not the live peak, is what runs out
        xs, ys = [r["n"] for r in rows], [r["reserved_gb"] for r in rows]
        mx, my = sum(xs) / len(xs), sum(ys) / len(ys)
        b = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / max(sum((x - mx) ** 2 for x in xs), 1e-9)
        a = my - b * mx
        n_max = int((total_gb - a) / b) if b > 0 else None
        fit = dict(size=size, fit_reserved_gb=dict(a=a, per_sample=b), card_gb=total_gb, predicted_max_n=n_max,
                   seconds=time.time() - t0)
        print(json.dumps(fit), flush=True)
        reader.clear()
        del pipe, kps, audio, reader
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
