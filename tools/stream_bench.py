#!/usr/bin/env python
"""Latency, throughput and device memory of ``VExpressPipeline.stream`` against ``__call__`` on one GPU.

  python tools/stream_bench.py [--compare 240] [--lengths 960,3840] [--ddim-steps 25] [--chunks 4]

Shapes: 512x512, the reference CLI's defaults (24-frame windows, overlap 4, 25 DDIM steps, CFG 3.5), bf16, synthetic
weights (bench.py's full-size UNet and VAE).  The kps features come from a hook that tiles 16 synthetic frames over the
video and the audio tokens repeat a 32-frame bank, so no conditioning of the whole video is ever materialised on the
host.  Prints JSON lines:
  * the card (name, memory, power limit and maximum SM clock);
  * at ``--compare`` L: one untimed 2-step run of each (allocator, lazy state), then ``__call__`` and ``stream`` timed end
    to end (host clock around the whole call, the last chunk on the host): seconds, frames/s, the time from the ``stream``
    call to its first chunk on the host, and ``torch.cuda.max_memory_allocated`` of the whole run.  The two paths share
    the captured UNet graph but not the shape of its kps buffer, so each timed run includes one graph capture;
  * at every ``--lengths`` L: the peak allocated memory of ``stream`` over the run up to its ``--chunks``-th chunk, by
    when every buffer of the steady state -- resident per-frame state, kps ring, captured graph, decoded chunks in
    flight -- has been allocated; later items repeat the same allocations.
``__call__`` runs only at ``--compare`` L: at the longer lengths it would hold the kps features and the video of every
frame on the device.
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
from samples_bench import card  # noqa: E402

H = 64                                       # 512x512 latents


def make_pipeline(dev):
    """bench.py's full-size pipeline (16-frame conditioning it does not use here), with synthetic hooks that produce any
    frame of any length on demand."""
    pipe, host, _ = bench.build_ours(16, H, dev)
    g = torch.Generator().manual_seed(7)
    kps_bank = (0.1 * torch.randn(1, 320, 16, H, H, generator=g)).to(device=dev, dtype=torch.bfloat16)
    audio_bank = bench.ln_rows(torch.randn(1, 32, 5, 768, generator=g)).to(torch.bfloat16)
    state = {}

    def kps_frames(kps_images, start, stop, height, width):
        return kps_bank[:, :, [f % 16 for f in range(start, stop)]]

    def kps_whole(kps_images, height, width, do_cfg):
        L = state["L"]
        feats = kps_frames(None, 0, L, height, width)
        return torch.cat([torch.zeros_like(feats), feats])

    def audio(audio_waveform, video_length, num_pad_audio_frames, do_cfg):
        a = audio_bank[:, [f % 32 for f in range(video_length)]]
        return torch.cat([torch.zeros_like(a), a]).to(dev)

    def latents(batch_size, c, width, height, video_length, dtype, device, generator, latents=None):
        from vexpress_b200.pipelines.v_express_pipeline import VExpressPipeline
        return VExpressPipeline.prepare_latents(pipe, batch_size, c, width, height, video_length, dtype, device,
                                                torch.Generator().manual_seed(100))

    pipe.prepare_kps_feature_frames = kps_frames
    pipe.prepare_kps_feature = kps_whole
    pipe.prepare_audio_embeddings = audio
    pipe.prepare_latents = latents
    return pipe, state


def args_for(L, steps):
    return dict(reference_image=None, kps_images=None, audio_waveform=None, width=8 * H, height=8 * H, video_length=L,
                num_inference_steps=steps, guidance_scale=3.5, context_frames=24, context_overlap=4,
                reference_attention_weight=0.95, audio_attention_weight=3.0)


def run_call(pipe, state, L, steps):
    state["L"] = L
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    video = pipe(**args_for(L, steps))
    sec = time.perf_counter() - t0
    assert video.shape == (1, 3, L, 8 * H, 8 * H)
    return dict(sec=sec, frames_per_sec=L / sec)


def run_stream(pipe, L, steps, max_chunks=None):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, got, frames = None, 0, 0
    gen = pipe.stream(**args_for(L, steps))
    for chunk in gen:
        if first is None:
            first = time.perf_counter() - t0
        assert chunk.start == frames
        frames += chunk.frames.shape[2]
        got += 1
        if max_chunks is not None and got == max_chunks:
            gen.close()
            break
    sec = time.perf_counter() - t0
    return dict(sec=sec, frames=frames, first_chunk_sec=first, frames_per_sec=frames / sec)


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    row = fn()
    torch.cuda.synchronize()
    row["peak_allocated_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compare", type=int, default=240, help="length of the __call__ / stream comparison (0: skip)")
    ap.add_argument("--lengths", default="960,3840", help="lengths of the stream memory measurement")
    ap.add_argument("--ddim-steps", type=int, default=25)
    ap.add_argument("--chunks", type=int, default=4, help="chunks streamed at --lengths")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_bench.py: no CUDA device (the product has no CPU path)")
    lengths = [int(x) for x in args.lengths.split(",") if x]
    T = args.ddim_steps
    print(json.dumps(dict(card=card())), flush=True)
    dev = torch.device("cuda", 0)
    pipe, state = make_pipeline(dev)
    L = args.compare
    if L:
        run_call(pipe, state, L, 2)                              # warm-up of each path
        run_stream(pipe, L, 2)
        call = peak(lambda: run_call(pipe, state, L, T))
        stream = peak(lambda: run_stream(pipe, L, T))
        print(json.dumps(dict(path="__call__", L=L, ddim_steps=T, **call)), flush=True)
        print(json.dumps(dict(path="stream", L=L, ddim_steps=T, **stream,
                              frames_per_sec_vs_call=stream["frames_per_sec"] / call["frames_per_sec"])), flush=True)
    for L in lengths:
        row = peak(lambda: run_stream(pipe, L, T, args.chunks))
        print(json.dumps(dict(path="stream", L=L, ddim_steps=T, chunks=args.chunks, **row)), flush=True)


if __name__ == "__main__":
    main()
