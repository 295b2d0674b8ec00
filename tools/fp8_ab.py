#!/usr/bin/env python
"""FP8 mode (UNet3DConditionModel.enable_fp8_linear) against the bf16 default on one GPU.

  python tools/fp8_ab.py [--rounds 3] [--passes 2] [--skip-e2e]

1. The LayerNorm + GEMM pair of every covered shape at configs[1] (512x512, one 16-frame window with CFG: T = 32 h w rows
   per level): ops.layernorm + ops.gemm against ops.layernorm_fp8 + ops.gemm_fp8, CUDA events over windows of >= 300 ms,
   the two modes alternating for --rounds rounds.  Per shape: the median time of each mode and the speed-up; then the sum
   over one forward (the number of such pairs per level of the UNet).
2. configs[1] end to end (25 DDIM steps + VAE decode, what bench.py times), the two modes alternating in this process
   for --passes passes each: frames/s and UNet ms per DDIM step.
3. The decoded videos of the two modes from the same latents: max |difference| and PSNR (8-bit range).
The card's name, power limit and SM clocks are read in the same call.  Prints JSON lines.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

# (level side, C, spatial transformer blocks, motion modules) of one UNet forward at 64x64 latents
LEVELS = ((64, 320, 5, 5), (32, 640, 5, 5), (16, 1280, 5, 5), (8, 1280, 1, 6))
FRAMES = 32                     # one 16-frame window, CFG: uncond | cond


def clocks():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[0] if q else None
    except Exception as e:  # the numbers stay valid without the query
        return f"unavailable: {e}"


def window(fn, min_ms=300.0):
    """ms per call of fn over a window of at least min_ms."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(5):
        fn()
    e1.record()
    torch.cuda.synchronize()
    n = max(5, math.ceil(min_ms / max(e0.elapsed_time(e1) / 5, 1e-3)))
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def pairs(rounds):
    from vexpress_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    total = {"bf16": 0.0, "fp8": 0.0}
    for side, C, n_sp, n_mm in LEVELS:
        HW = side * side
        T = FRAMES * HW
        x = rn(T, C).bfloat16()
        gamma, beta = 1 + 0.1 * rn(C), 0.1 * rn(C)
        pe = rn(16, C)
        # (pair, N, GEGLU, positional encoding, pairs per forward): spatial blocks have the fused qkv, two q (attn1_5,
        # attn2) and a GEGLU; motion modules two fused qkv with the positional encoding and a GEGLU
        shapes = (("qkv", 3 * C, False, False, n_sp), ("qkv+pe", 3 * C, False, True, 2 * n_mm), ("q", C, False, False, 2 * n_sp),
                  ("geglu", 8 * C, True, False, n_sp + n_mm))
        for name, N, geglu, use_pe, count in shapes:
            if count == 0:
                continue
            w = (rn(N, C) / math.sqrt(C)).bfloat16()
            b = rn(N) if geglu else None
            if geglu:
                w, b, _ = ops.pack_geglu(w, b)
            w8, s8 = ops.quantize_fp8_weight(w)
            pe_kw = dict(pe=pe, rows_per_frame=HW) if use_pe else {}

            def bf16():
                n = ops.layernorm(x, gamma, beta, **pe_kw)
                ops.gemm(n, w, b, geglu=geglu)

            def fp8():
                a8, sa = ops.layernorm_fp8(x, gamma, beta, **pe_kw)
                ops.gemm_fp8(a8, sa, w8, s8, b, geglu=geglu)

            t = {"bf16": [], "fp8": []}
            for _ in range(rounds):
                t["bf16"].append(window(bf16))
                t["fp8"].append(window(fp8))
            med = {k: statistics.median(v) for k, v in t.items()}
            flop = 2.0 * T * N * C
            for k in total:
                total[k] += count * med[k]
            print(json.dumps(dict(level=side, C=C, pair=name, M=T, N=N, K=C, per_forward=count,
                                  bf16_ms=t["bf16"], fp8_ms=t["fp8"], speedup=med["bf16"] / med["fp8"],
                                  gemm_tflop=flop / 1e12, pair_tflops_bf16=flop / med["bf16"] / 1e9,
                                  pair_tflops_fp8=flop / med["fp8"] / 1e9)), flush=True)
    print(json.dumps(dict(per_forward_ms=total, speedup=total["bf16"] / total["fp8"], clocks=clocks())), flush=True)


def end_to_end(passes):
    import samples_bench as SB
    from vexpress_b200.pipelines.v_express_pipeline import retrieve_timesteps
    h = 64
    pipe, kps, audio, reader = SB.setup(h)
    unet = pipe.denoising_unet
    timesteps, _ = retrieve_timesteps(pipe.scheduler, 25, kps.device)
    lat = SB.latents(pipe, 1, h)
    videos, rows = {}, {"bf16": [], "fp8": []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for mode in ("bf16", "fp8"):      # warm-up and graph capture of both modes
        unet.enable_fp8_linear() if mode == "fp8" else unet.disable_fp8_linear()
        videos[mode] = SB.one_pass(pipe, lat, kps, audio, timesteps)
    for _ in range(passes):
        for mode in ("bf16", "fp8"):
            unet.enable_fp8_linear() if mode == "fp8" else unet.disable_fp8_linear()
            torch.cuda.synchronize()
            e0.record()
            SB.one_pass(pipe, lat, kps, audio, timesteps)
            e1.record()
            torch.cuda.synchronize()
            sec = e0.elapsed_time(e1) / 1e3
            e0.record()
            pipe.denoise(lat.clone(), kps, audio, timesteps, 3.5, 16, 8)
            e1.record()
            torch.cuda.synchronize()
            rows[mode].append(dict(frames_per_sec=SB.L / sec, unet_ms_per_ddim_step=e0.elapsed_time(e1) / 25))
    print(json.dumps(dict(end_to_end=rows, clocks=clocks())), flush=True)
    a, b = (videos[m].float() for m in ("bf16", "fp8"))
    if a.max() <= 1.0:
        a, b = a * 255, b * 255
    mse = float(((a - b) ** 2).mean())
    print(json.dumps(dict(video_max_abs_diff_8bit=float((a - b).abs().max()),
                          video_psnr_db=10 * math.log10(255 ** 2 / mse) if mse > 0 else math.inf,
                          shape=list(a.shape))), flush=True)
    reader.clear()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--passes", type=int, default=2)
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_ab.py: no CUDA device (the product has no CPU path)")
    p = torch.cuda.get_device_properties(0)
    print(json.dumps(dict(card=p.name, sms=p.multi_processor_count, clocks=clocks())), flush=True)
    pairs(args.rounds)
    if not args.skip_e2e:
        end_to_end(args.passes)


if __name__ == "__main__":
    main()
