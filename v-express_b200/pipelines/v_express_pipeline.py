"""H100-native ``VExpressPipeline``: drop-in for the reference's ``pipelines/v_express_pipeline.py`` denoising
hot path (``__call__`` -> ``mean_overlap`` :409-589 and ``decode_latents`` :152-166), same call signature and
return value ((n,3,L,H,W) fp32 on the host, values in [0,1], n = ``num_images_per_prompt``).

What differs by design (SURVEY.md 0.5, 8e):
  * latents, kps features and audio tokens stay resident in HBM for the whole video (the reference shuttles every
    window host<->device each step and syncs once per frame);
  * per step, all windows run through one CUDA-graph-captured UNet forward; CFG + /count + overlap accumulation
    is one kernel per window and the DDIM update one kernel per step.  The result equals the reference's
    streaming update (a frame is stepped only after all its windows were visited, :552-572) with identical
    rounding points in the model dtype;
  * context windows shard over the GPUs of one box (``do_multi_devices_inference``, a dead flag in the reference):
    every rank owns a contiguous block of windows and one NCCL all-reduce per step sums the (zero-padded)
    per-frame noise-prediction buffers; the VAE decode is sharded by frame and gathered on rank 0;
  * the VAE decodes all frames of a chunk in one batch;
  * ``num_images_per_prompt`` = n samples of the same conditioning run through ONE UNet forward per window, batched as
    [uncond s0..s(n-1) | cond s0..s(n-1)].  Sample i of an n-sample call is bit-identical to a one-sample call with
    ``generator[i]`` (the reference accepts the argument but its UNet cannot run it);
  * ``stream`` runs the same forwards in a wavefront over the windows (``context.wavefront_schedule``) and yields the
    video chunk by chunk as frames become final, holding kps features only for the windows in flight, so clip length is
    bounded by ~100 KB of resident state per frame rather than by the features and the video (DESIGN.md 5).

Out of the hot path (SURVEY.md 8f), kept as overridable hooks exactly like the reference methods:
``prepare_reference_latent``, ``prepare_kps_feature``, ``prepare_audio_embeddings`` and the ReferenceNet write
pass; they run whatever torch modules the caller registered.
"""
from __future__ import annotations

import math
import os
from typing import Callable, Iterator, List, NamedTuple, Optional, Union

import torch

from .. import _ffi, ops
from ..modules.mutual_self_attention import ReferenceAttentionControl
from ..modules.unet_3d import UNet3DConditionModel
from .context import overlap_plan, wavefront_schedule, window_table
from .scheduler import ddim_coefficients

BF16 = torch.bfloat16
_ALLREDUCE_FP32 = os.environ.get("VX_ALLREDUCE_FP32") == "1"     # A/B switch: reduce the fp32 accumulator instead of its bf16 copy


class VideoChunk(NamedTuple):
    """One piece of a streamed video: frames [start, start + k) of every sample, in a fresh pinned host tensor --
    (n,3,k,H,W) fp32 in [0,1] for ``output="float"``, (n,k,H,W,3) uint8 median-filtered for ``output="uint8"``."""
    start: int
    frames: torch.Tensor


class _HostCopies:
    """Device -> pinned host copies on a side stream, each with an event, so the denoising stream never waits for the
    caller.  The device source is held until its copy has completed.  On a CPU device (the host-side test harness) the
    copy is a plain clone."""

    def __init__(self, dev):
        self.cuda = dev.type == "cuda"
        self.stream = torch.cuda.Stream(dev) if self.cuda else None
        self.pending = []                  # (key, start, host tensor, device source, event), in frame order

    def push(self, key, start, src):
        if not self.cuda:
            self.pending.append((key, start, src.clone(), None, None))
            return
        host = torch.empty(tuple(src.shape), dtype=src.dtype, pin_memory=True)
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            host.copy_(src, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.pending.append((key, start, host, src, ev))

    def ready(self, before_key=None):
        """Pop (in order) the chunks pushed before ``before_key`` (all when None), waiting for their copies."""
        while self.pending and (before_key is None or self.pending[0][0] < before_key):
            _, start, host, _, ev = self.pending.pop(0)
            if ev is not None:
                ev.synchronize()
            yield VideoChunk(start, host)


def retrieve_timesteps(scheduler, num_inference_steps=None, device=None, timesteps=None, **kwargs):
    """Reference pipelines/v_express_pipeline.py:27-68 (custom timestep lists are not used on this path)."""
    if timesteps is not None:
        raise ValueError("custom timestep schedules are not supported by the DDIM hot path")
    scheduler.set_timesteps(num_inference_steps, device=device, **kwargs)
    return scheduler.timesteps, num_inference_steps


def _runs(frames):
    """Sorted frame indices -> lists of consecutive indices."""
    out = []
    for fr in frames:
        if out and out[-1][-1] + 1 == fr:
            out[-1].append(fr)
        else:
            out.append([fr])
    return out


def partition_windows(num_windows: int, world_size: int, rank: int):
    """Contiguous, balanced block of window indices owned by ``rank`` (SURVEY.md 8e: 47 windows over 8 ranks ->
    6,6,6,6,6,6,6,5)."""
    base, rem = divmod(num_windows, world_size)
    start = rank * base + min(rank, rem)
    return list(range(start, start + base + (1 if rank < rem else 0)))


class _GraphedUNet:
    """One CUDA graph of ``UNetEngine.forward_frames`` per (b, n, f, h, w) signature with static I/O buffers of b n f
    frames."""

    def __init__(self, engine, b, f, h, w, enc_tokens, cross_dim, use_graph=True, n=1):
        dev = engine.dev
        self.engine, self.b, self.f, self.n = engine, b, f, n
        self.frames = torch.zeros((b * n * f, 4, h, w), device=dev, dtype=BF16)
        self.enc = torch.zeros((b * n * f, enc_tokens, cross_dim), device=dev, dtype=BF16)
        self.kps_idx = torch.zeros((b * n * f,), device=dev, dtype=torch.int32)
        self.temb = None
        self.kps = None          # static copy of the channels-last kps features (address baked into the graph)
        self.graph = None
        self.out = None
        self.use_graph = use_graph
        self.kps_token = None

    def _run(self):
        extra = {"n": self.n} if self.n > 1 else {}          # a one-sample window is the engine's default call
        return self.engine.forward_frames(self.frames, None, self.enc, self.kps, self.kps_idx, self.b, self.f,
                                          temb=self.temb, **extra)

    def set_kps(self, kps):
        """Per video: (re)load the resident channels-last kps features; same shape keeps the captured graph."""
        if self.kps is None or self.kps.shape != kps.shape:
            self.kps = torch.empty_like(kps)
            self.graph = None
        self.kps.copy_(kps)

    def kps_ring(self, rows, channels):
        """The static kps buffer as a ring of ``rows`` channels-last rows that the caller fills in place between
        replays (``stream``); an existing buffer of that shape is reused, so its captured graph stays valid."""
        if self.kps is None or self.kps.shape != (rows, channels):
            self.set_kps(torch.zeros((rows, channels), device=self.frames.device, dtype=BF16))
        self.kps_token = self.kps
        return self.kps

    def __call__(self, temb):
        if self.temb is None:
            self.temb = torch.empty_like(temb)
        self.temb.copy_(temb)
        if not self.use_graph:
            return self._run()
        if self.graph is None:
            # warm-up on a side stream (allocator + lazy module state), then capture
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._run()
            torch.cuda.current_stream().wait_stream(s)
            self.graph = torch.cuda.CUDAGraph()
            before = _ffi.LAUNCHES
            with torch.cuda.graph(self.graph):
                self.out = self._run()
            self.captured_launches = _ffi.LAUNCHES - before
            _ffi.LAUNCHES = before            # capture enqueues nothing; replays are counted below
        self.graph.replay()
        _ffi.LAUNCHES += self.captured_launches
        return self.out


class VExpressPipeline:
    _optional_components: List[str] = []

    def __init__(self, vae, reference_net, denoising_unet, v_kps_guider, audio_processor, audio_encoder,
                 audio_projection, scheduler, image_proj_model=None, tokenizer=None, text_encoder=None):
        self.vae = vae
        self.reference_net = reference_net
        self.denoising_unet = denoising_unet
        self.v_kps_guider = v_kps_guider
        self.audio_processor = audio_processor
        self.audio_encoder = audio_encoder
        self.audio_projection = audio_projection
        self.scheduler = scheduler
        self.image_proj_model, self.tokenizer, self.text_encoder = image_proj_model, tokenizer, text_encoder
        boc = getattr(getattr(vae, "config", {}), "get", lambda *_: None)("block_out_channels")
        self.vae_scale_factor = 2 ** (len(boc) - 1) if boc else 8
        self.use_cuda_graph = True
        self.vae_chunk = 16
        self._graphs = {}

    # ------------------------------------------------------------------ diffusers-style conveniences
    @property
    def device(self):
        return self.denoising_unet.device

    @property
    def dtype(self):
        return self.denoising_unet.dtype

    def to(self, *args, **kwargs):
        for m in (self.vae, self.reference_net, self.denoising_unet, self.v_kps_guider, self.audio_encoder,
                  self.audio_projection):
            if isinstance(m, torch.nn.Module):
                m.to(*args, **kwargs)
        return self

    def progress_bar(self, iterable=None, total=None):
        from tqdm import tqdm
        return tqdm(iterable, total=total, disable=True)

    # ------------------------------------------------------------------ prologue hooks (outside the hot path)
    @staticmethod
    def _reference_image_to_tensor(image, height, width):
        """The reference's ``reference_image_processor.preprocess`` (VaeImageProcessor(do_convert_rgb=True), default
        do_normalize: [0,1] -> [-1,1], resample "lanczos"; pipelines/v_express_pipeline.py:112-114,344): a PIL image, an HWC
        uint8 array, or a (1,3,H,W) tensor already in [-1,1] -> (1,3,height,width) fp32 in [-1,1]."""
        import numpy as np
        if torch.is_tensor(image):
            if image.dim() == 3:
                image = image.unsqueeze(0)
            if image.shape[-2:] != (height, width):
                raise ValueError(f"reference image tensor must be (1,3,{height},{width}), got {tuple(image.shape)}")
            return image.float()
        if hasattr(image, "convert"):
            image = image.convert("RGB")
            if image.size != (width, height):
                from PIL import Image
                image = image.resize((width, height), resample=Image.LANCZOS)
        arr = np.asarray(image)
        if arr.shape[:2] != (height, width):
            raise ValueError(f"reference image of size {arr.shape[:2]} needs resampling to {(height, width)}: pass a PIL image")
        t = torch.from_numpy(arr.astype(np.float32) / 255.0).permute(2, 0, 1).unsqueeze(0)
        return 2.0 * t - 1.0

    def prepare_reference_latent(self, reference_image, height, width):
        """Reference pipelines/v_express_pipeline.py:343-348: VAE posterior mean of the reference image x 0.18215."""
        x = self._reference_image_to_tensor(reference_image, height, width).to(device=self.device, dtype=self.dtype)
        return self.vae.encode(x).latent_dist.mean * 0.18215

    @staticmethod
    def _condition_images_to_tensor(images, height, width):
        """The reference's ``condition_image_processor.preprocess`` (VaeImageProcessor(do_convert_rgb=True,
        do_normalize=False), pipelines/v_express_pipeline.py:112-115,352-356) for the cases that need no resampling:
        a (b,3,t,H,W) tensor in [0,1], or a list of RGB PIL images / HWC uint8 arrays.  -> (1,3,t,H,W) fp32 in [0,1]."""
        import numpy as np
        if torch.is_tensor(images):
            if images.dim() != 5 or images.shape[-2:] != (height, width):
                raise ValueError(f"kps images tensor must be (b,3,t,{height},{width}), got {tuple(images.shape)}")
            return images.float()
        frames = []
        for img in images:
            if hasattr(img, "convert"):                      # PIL
                img = img.convert("RGB")
                if img.size != (width, height):
                    from PIL import Image
                    img = img.resize((width, height), resample=Image.LANCZOS)   # VaeImageProcessor default "lanczos"
            arr = np.asarray(img)
            if arr.shape[:2] != (height, width):
                raise ValueError(f"kps image of size {arr.shape[:2]} needs resampling to {(height, width)}: pass PIL images")
            frames.append(torch.from_numpy(arr.astype(np.float32) / 255.0).permute(2, 0, 1))
        return torch.stack(frames, 1).unsqueeze(0)

    def prepare_kps_feature(self, kps_images, height, width, do_classifier_free_guidance):
        """Reference pipelines/v_express_pipeline.py:350-372: keypoint images -> VKpsGuider in chunks of 16 frames ->
        (b, 320, L, h, w) with the CFG zero half in front.  The features stay on the device (the reference parks
        them on the CPU and copies a window per step)."""
        if self.v_kps_guider is None:
            raise NotImplementedError("prologue hook: pass a VKpsGuider (vexpress_b200.modules.VKpsGuider or the "
                                      "reference's) or override prepare_kps_feature with precomputed features")
        x = self._condition_images_to_tensor(kps_images, height, width)
        feats = []
        for i in range(0, x.shape[2], 16):
            feats.append(self.v_kps_guider(x[:, :, i:i + 16].to(device=self.device, dtype=self.dtype)))
        kps_feature = torch.cat(feats, dim=2)
        if do_classifier_free_guidance:
            kps_feature = torch.cat([torch.zeros_like(kps_feature), kps_feature], dim=0)
        return kps_feature

    def prepare_kps_feature_frames(self, kps_images, start, stop, height, width):
        """Frames [start, stop) of ``prepare_kps_feature``'s conditional half, (1, 320, stop - start, h, w) on the device,
        for ``stream``, which holds only the frames its windows in flight read.  Converts only the images of the 16-frame
        chunks (aligned at multiples of 16, as ``prepare_kps_feature`` runs them) that hold those frames and runs the
        guider on those chunks, so the result is bit-identical to the slice of the whole-video features."""
        if self.v_kps_guider is None:
            raise NotImplementedError("prologue hook: pass a VKpsGuider (vexpress_b200.modules.VKpsGuider or the "
                                      "reference's) or override prepare_kps_feature_frames with precomputed features")
        c0, c1 = start // 16 * 16, -(-stop // 16) * 16
        images = kps_images[:, :, c0:c1] if torch.is_tensor(kps_images) else kps_images[c0:c1]
        x = self._condition_images_to_tensor(images, height, width)
        feats = [self.v_kps_guider(x[:, :, i:i + 16].to(device=self.device, dtype=self.dtype))
                 for i in range(0, x.shape[2], 16)]
        return torch.cat(feats, dim=2)[:, :, start - c0:stop - c0]

    @staticmethod
    def audio_frame_windows(audio_embeddings, video_length, num_pad_audio_frames):
        """Reference pipelines/v_express_pipeline.py:380-401: encoder states (1,T,d) -> linear interpolation (fp32) to
        2*L steps, 2*num_pad zero rows on both sides, sliding windows (L, 2*(2*num_pad+1), d)."""
        in_dtype = audio_embeddings.dtype
        x = torch.nn.functional.interpolate(audio_embeddings.to(torch.float32).permute(0, 2, 1), size=2 * video_length,
                                            mode="linear")[0].permute(1, 0).to(in_dtype)
        pad = torch.zeros_like(x)[:2 * num_pad_audio_frames]
        x = torch.cat([pad, x, pad], dim=0)
        return torch.stack([x[2 * i:2 * (i + 2 * num_pad_audio_frames + 1)] for i in range(video_length)], dim=0)

    def prepare_audio_embeddings(self, audio_waveform, video_length, num_pad_audio_frames, do_classifier_free_guidance):
        """Reference pipelines/v_express_pipeline.py:374-407.  ``audio_processor`` / ``audio_encoder`` are the caller's
        (wav2vec2, a third-party torch module outside this repo's kernels, SURVEY 8f-f4); the projection is
        ``self.audio_projection`` (vexpress_b200.modules.AudioProjection or the reference's)."""
        if self.audio_encoder is None or self.audio_projection is None:
            raise NotImplementedError("prologue hook: pass audio_processor / audio_encoder / audio_projection or "
                                      "override prepare_audio_embeddings with precomputed tokens")
        wave = audio_waveform
        if self.audio_processor is not None:
            wave = self.audio_processor(audio_waveform, return_tensors="pt", sampling_rate=16000)["input_values"]
        wave = wave.to(self.device, self.dtype)
        states = self.audio_encoder(wave).last_hidden_state                       # (1, T, d)
        windows = self.audio_frame_windows(states, video_length, num_pad_audio_frames)
        audio_embeddings = self.audio_projection(windows).unsqueeze(0)
        if do_classifier_free_guidance:
            audio_embeddings = torch.cat([torch.zeros_like(audio_embeddings), audio_embeddings], dim=0)
        return audio_embeddings

    def run_reference_net(self, reference_image_latents, writer):
        """Reference pipelines/v_express_pipeline.py:502-508: one ReferenceNet pass at t=0 fills the writer banks."""
        enc = torch.zeros((1, 1, 768), dtype=self.dtype, device=self.device)
        self.reference_net(reference_image_latents, timestep=0, encoder_hidden_states=enc, return_dict=False)

    def prepare_latents(self, batch_size, num_channels_latents, width, height, video_length, dtype, device, generator,
                        latents=None):
        """Reference :189-224: noise is drawn on the HOST in the model dtype so seeds reproduce (:514-523).  As diffusers'
        ``randn_tensor``: a list of generators draws sample i as its own (1, ...) tensor from ``generator[i]``, so sample i
        of a batch equals a one-sample draw from the same generator; a single generator (or None) draws the whole batch."""
        shape = (batch_size, num_channels_latents, video_length, height // self.vae_scale_factor,
                 width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an "
                             f"effective batch size of {batch_size}. Make sure the batch size matches the length of "
                             f"the generators.")
        if latents is None:
            if isinstance(generator, list):
                latents = torch.cat([torch.randn((1,) + shape[1:], generator=g, device="cpu", dtype=dtype)
                                     for g in generator])
            else:
                latents = torch.randn(shape, generator=generator, device="cpu", dtype=dtype)
        return latents * self.scheduler.init_noise_sigma

    def get_timesteps(self, num_inference_steps, strength, device):
        init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
        t_start = max(num_inference_steps - init_timestep, 0)
        return self.scheduler.timesteps[t_start * self.scheduler.order:], num_inference_steps - t_start

    # ------------------------------------------------------------------ decode
    @torch.no_grad()
    def decode_latents(self, latents, frame_ids=None, out=None, sample=0):
        """latents (n,4,L,h,w) on the device -> frames of sample ``sample`` in [0,1], fp32, ON THE DEVICE, already in the
        reference's output layout (reference :152-166): ``out`` (3, k, H, W) (allocated when None), frame j of
        ``frame_ids`` (default: all) written to out[:, j].  The conv_out kernel writes through the strides, so no permute
        pass exists.  Frames go through the VAE in chunks of ``vae_chunk`` counted from the first id, whatever the sample,
        so every sample decodes to the bits a one-sample call gives."""
        L = latents.shape[2]
        ids = list(range(L)) if frame_ids is None else list(frame_ids)
        H, W = latents.shape[3] * self.vae_scale_factor, latents.shape[4] * self.vae_scale_factor
        if out is None:
            out = torch.empty((3, len(ids), H, W), device=latents.device, dtype=torch.float32)
        z = latents[sample].permute(1, 0, 2, 3)[ids].contiguous()               # (k,4,h,w)
        for i in range(0, z.shape[0], self.vae_chunk):
            n = min(self.vae_chunk, z.shape[0] - i)
            self.vae.decode_latents(z[i:i + n], out=out[:, i:i + n].permute(1, 0, 2, 3))
        return out

    # ------------------------------------------------------------------ the hot loop
    @torch.no_grad()
    def denoise(self, latents, kps_feature, audio_embeddings, timesteps, guidance_scale, context_frames,
                context_overlap, context_schedule="uniform", distributed=False, callback=None, callback_steps=1):
        """latents (n,4,L,h,w) bf16 device (updated in place and returned); kps_feature (b,C0,L,h,w) device;
        audio_embeddings (b,L,T,768) device.  Steps x windows with overlap averaging, CFG and DDIM
        (reference :486-500,514-589).  The n samples share the conditioning and step together: one UNet forward per window
        on the batch [uncond s0..s(n-1) | cond s0..s(n-1)] whose frames all gather their kps rows from the one resident
        copy, one CFG / overlap launch per window, one DDIM launch per step."""
        unet: UNet3DConditionModel = self.denoising_unet
        eng = unet.engine()
        dev = latents.device
        n, _, L, h, w = latents.shape
        hw = h * w
        do_cfg = guidance_scale > 1.0
        b = 2 if do_cfg else 1
        windows, count = window_table(L, context_frames, context_overlap, context_schedule)
        # reflected tail windows may repeat frames: which slots reach a frame's final sum follows the reference's
        # streaming bookkeeping exactly (context.overlap_plan); tiling lengths give one round with every slot kept
        plan = overlap_plan(windows, count)
        rank, world = 0, 1
        if distributed and torch.distributed.is_available() and torch.distributed.is_initialized():
            rank, world = torch.distributed.get_rank(), torch.distributed.get_world_size()
        mine = partition_windows(len(windows), world, rank)
        count_dev = torch.from_numpy(count).to(device=dev, dtype=torch.int32)
        # channels-last kps of the frames this rank's windows touch, row block (bi*Lloc + frame - lo); stays resident for
        # the whole video.  Only that slice crosses PCIe when the features live on the host.
        own = sorted(set(fr for wi in mine for fr in windows[wi]))
        lo, hi = (own[0], own[-1] + 1) if own else (0, 1)
        Lloc = hi - lo
        C0 = kps_feature.shape[1]
        kps_nhwc = kps_feature[:, :, lo:hi].to(device=dev, dtype=BF16, non_blocking=True) \
            .permute(0, 2, 3, 4, 1).reshape(b * Lloc * hw, C0).contiguous()
        audio = audio_embeddings[:, lo:hi].to(device=dev, dtype=BF16, non_blocking=True)
        T = audio.shape[2]
        acc = torch.zeros((n, 4, L, hw), device=dev, dtype=torch.float32)
        acc_x = torch.empty((n, 4, L, hw), device=dev, dtype=BF16) if world > 1 else None
        win_dev = [torch.tensor(wn, device=dev, dtype=torch.int32) for wn in windows]
        win_long = [t.long() for t in win_dev]
        plan_dev = {wi: [torch.from_numpy(r).to(dev) for r in plan[wi]] for wi in mine}
        # kps row of UNet frame (bi, s, i): the CFG half's copy of window frame i, the same for every sample s
        half_off = torch.arange(b, device=dev, dtype=torch.int32) * Lloc - lo
        kps_idx = {wi: (win_dev[wi][None, None] + half_off[:, None, None]).expand(b, n, len(windows[wi])).reshape(-1)
                   for wi in mine}
        # refresh the projected reference banks (outside any capture) and reuse graphs across calls while valid
        for name in eng.order:
            eng._bank_kv(name, unet.get_submodule(name))
        graphs = self._graphs
        for i, t in enumerate(timesteps):
            temb = eng.time_embedding(int(t))
            acc.zero_()
            for wi in mine:
                window = windows[wi]
                f = len(window)
                key = (b, n, f, h, w, T, bool(self.use_cuda_graph), eng.graph_signature())
                g = graphs.get(key)
                if g is None:
                    for k_old in [k for k in graphs if k[:5] == key[:5] and k != key]:
                        del graphs[k_old]                                       # stale capture of the same shape
                    g = graphs[key] = _GraphedUNet(eng, b, f, h, w, T, audio.shape[-1], self.use_cuda_graph, n)
                x = latents[:, :, win_long[wi]].transpose(1, 2)                 # (n,f,4,h,w)
                g.frames.view(b, n, f, 4, h, w).copy_(x)                        # both CFG halves
                g.enc.view(b, n, f, T, -1).copy_(audio[:, win_long[wi] - lo].unsqueeze(1))
                g.kps_idx.copy_(kps_idx[wi])
                if g.kps_token is not kps_nhwc:
                    g.set_kps(kps_nhwc)
                    g.kps_token = kps_nhwc
                noise = g(temb)                                                 # ((b n f),4,h,w) bf16
                for slots in plan_dev[wi]:
                    if n == 1:
                        ops.cfg_overlap_accumulate(noise, f, hw, L, do_cfg, slots, count_dev, float(guidance_scale),
                                                   acc[0])
                    else:
                        ops.cfg_overlap_accumulate_n(noise, n, f, hw, L, do_cfg, slots, count_dev, float(guidance_scale),
                                                     acc)
            if world > 1:
                # every frame has at most two non-zero bf16 contributions across the ranks (its windows live on one rank
                # or on two neighbours), so the bf16 sum is the reference's own bf16 add -- half the bytes of fp32
                if _ALLREDUCE_FP32:
                    torch.distributed.all_reduce(acc, op=torch.distributed.ReduceOp.SUM)
                else:
                    acc_x.copy_(acc)
                    torch.distributed.all_reduce(acc_x, op=torch.distributed.ReduceOp.SUM)
                    acc.copy_(acc_x)
            sa, sb, sap, sbp = ddim_coefficients(self.scheduler, int(t))
            ops.ddim_step(latents, acc, sa, sb, sap, sbp)                   # elementwise over all n samples
            if callback is not None and i % callback_steps == 0:
                callback(i, t, latents)
        return latents

    @torch.no_grad()
    def denoise_stream(self, latents, kps_images, audio_embeddings, timesteps, guidance_scale, context_frames,
                       context_overlap, context_schedule="uniform", output="float") -> Iterator[VideoChunk]:
        """``denoise`` + decode as a generator of ``VideoChunk``s in frame order, in device memory that does not grow with
        the video beyond latents, acc, audio tokens and the count table.  The same forwards on the same inputs as
        ``denoise``, in the wavefront order of ``context.wavefront_schedule``: a frame gets its DDIM update as soon as its
        last window of the step has contributed (``ops.ddim_step_frames``), and a VAE chunk is decoded as soon as its
        frames are final, so the frames and final latents are bit-identical to ``denoise`` + ``decode_to_device``.

        kps features exist only for the frames of the windows in flight: a ring of frame slots that is the captured
        graph's static kps buffer, filled through ``prepare_kps_feature_frames(kps_images, ...)`` before a frame's first
        read and recycled after its last.  Uncond rows all read slot 0, a zero frame.  latents (n,4,L,h,w) bf16 device
        (updated in place); audio_embeddings (b,L,T,768).  ``output="uint8"`` yields ``ops.median3d_range_u8`` of each
        chunk, which waits for the first frame of the next one."""
        if output not in ("float", "uint8"):
            raise ValueError(f"output must be 'float' or 'uint8', got {output!r}")
        unet: UNet3DConditionModel = self.denoising_unet
        eng = unet.engine()
        dev = latents.device
        n, _, L, h, w = latents.shape
        hw = h * w
        H, W = h * self.vae_scale_factor, w * self.vae_scale_factor
        do_cfg = guidance_scale > 1.0
        b = 2 if do_cfg else 1
        windows, count = window_table(L, context_frames, context_overlap, context_schedule)
        f = len(windows[0])
        if any(len(wn) != f for wn in windows):
            raise ValueError(f"stream needs windows of one size, the {context_schedule!r} schedule gave "
                             f"{sorted(set(len(wn) for wn in windows))}")
        plan = overlap_plan(windows, count)
        sched = wavefront_schedule(windows, len(timesteps), L, self.vae_chunk)
        # kps ring slots, planned on the host: a frame holds its slot from its first read to its last; slot 0 = zeros
        slot_of, free, nslots, fills = {}, [], 0, []
        kps_idx, fin = {}, {}
        for i, (wi, t) in enumerate(sched.order):
            fills.append([])
            for fr in sched.loads[i]:
                if not free:
                    nslots += 1
                    free.append(nslots)
                slot_of[fr] = free.pop()
                fills[i].append(fr)
            if t == 0:
                rows = [0] * (n * f) if do_cfg else []
                kps_idx[wi] = torch.tensor(rows + [slot_of[fr] for fr in windows[wi]] * n, dtype=torch.int32,
                                           device=dev)
                fin[wi] = torch.tensor(sched.finalised[i], dtype=torch.int32, device=dev) if sched.finalised[i] else None
            for fr in sched.releases[i]:
                free.append(slot_of[fr])
        count_dev = torch.from_numpy(count).to(device=dev, dtype=torch.int32)
        audio = audio_embeddings.to(device=dev, dtype=BF16, non_blocking=True)
        T = audio.shape[2]
        acc = torch.zeros((n, 4, L, hw), device=dev, dtype=torch.float32)
        win_long = [torch.tensor(wn, device=dev, dtype=torch.long) for wn in windows]
        plan_dev = [[torch.from_numpy(r).to(dev) for r in rounds] for rounds in plan]
        for name in eng.order:
            eng._bank_kv(name, unet.get_submodule(name))
        key = (b, n, f, h, w, T, bool(self.use_cuda_graph), eng.graph_signature())
        g = self._graphs.get(key)
        if g is None:
            for k_old in [k for k in self._graphs if k[:5] == key[:5] and k != key]:
                del self._graphs[k_old]
            g = self._graphs[key] = _GraphedUNet(eng, b, f, h, w, T, audio.shape[-1], self.use_cuda_graph, n)
        tembs = [eng.time_embedding(int(t)) for t in timesteps]
        coeffs = [ddim_coefficients(self.scheduler, int(t)) for t in timesteps]
        ring = None
        copies = _HostCopies(dev)
        tail = None                     # uint8: decoded frames [tail_start, ...) = halo frame + the chunk not yet filtered
        tail_start = own_start = 0

        def filtered(buf, buf_start, start, stop):
            u8 = torch.empty((n, stop - start, H, W, 3), device=dev, dtype=torch.uint8)
            for s in range(n):
                ops.median3d_range_u8(buf[s], buf_start, start, stop - start, L, out=u8[s])
            return u8

        cur_key = None
        for i, (wi, t) in enumerate(sched.order):
            item_key = t * sched.reach + wi
            if item_key != cur_key:
                if cur_key is not None:
                    yield from copies.ready(before_key=cur_key)    # every item of the key after theirs is enqueued
                cur_key = item_key
            for run in _runs(fills[i]):
                feat = self.prepare_kps_feature_frames(kps_images, run[0], run[-1] + 1, H, W)
                rows = feat[0].to(device=dev, dtype=BF16).permute(1, 2, 3, 0).reshape(len(run), hw, -1)
                if ring is None:
                    ring = g.kps_ring((nslots + 1) * hw, rows.shape[-1]).view(nslots + 1, hw, -1)
                    ring[0].zero_()
                for j, fr in enumerate(run):
                    ring[slot_of[fr]].copy_(rows[j])
            x = latents[:, :, win_long[wi]].transpose(1, 2)                     # (n,f,4,h,w)
            g.frames.view(b, n, f, 4, h, w).copy_(x)
            g.enc.view(b, n, f, T, -1).copy_(audio[:, win_long[wi]].unsqueeze(1))
            g.kps_idx.copy_(kps_idx[wi])
            noise = g(tembs[t])
            for slots in plan_dev[wi]:
                if n == 1:
                    ops.cfg_overlap_accumulate(noise, f, hw, L, do_cfg, slots, count_dev, float(guidance_scale), acc[0])
                else:
                    ops.cfg_overlap_accumulate_n(noise, n, f, hw, L, do_cfg, slots, count_dev, float(guidance_scale), acc)
            if fin[wi] is not None:
                ops.ddim_step_frames(latents, acc, fin[wi], *coeffs[t])
            for c0, c1 in sched.chunks[i]:
                vid = torch.empty((n, 3, c1 - c0, H, W), device=dev, dtype=torch.float32)
                for s in range(n):
                    self.decode_latents(latents, range(c0, c1), out=vid[s], sample=s)
                if output == "float":
                    copies.push(item_key, c0, vid)
                    continue
                if tail is not None:
                    copies.push(item_key, own_start, filtered(torch.cat([tail, vid[:, :, :1]], 2), tail_start, own_start, c0))
                    tail, tail_start = torch.cat([tail[:, :, -1:], vid], 2), c0 - 1
                else:
                    tail = vid
                own_start = c0
        if tail is not None:
            copies.push(cur_key, own_start, filtered(tail, tail_start, own_start, L))
        yield from copies.ready()

    @staticmethod
    def _check_sampling_args(eta, num_images_per_prompt):
        if eta != 0.0:
            raise ValueError("the DDIM hot path is deterministic (eta = 0), like the reference CLI")
        if not isinstance(num_images_per_prompt, int) or num_images_per_prompt < 1:
            raise ValueError(f"num_images_per_prompt must be a positive integer, got {num_images_per_prompt!r}")

    @torch.no_grad()
    def mean_overlap(self, reference_image, kps_images, audio_waveform, width, height, video_length,
                     num_inference_steps, guidance_scale, strength=1., num_images_per_prompt=1, eta: float = 0.0,
                     generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
                     output_type: Optional[str] = "tensor", return_dict: bool = True,
                     callback: Optional[Callable] = None, callback_steps: Optional[int] = 1,
                     context_schedule="uniform", context_frames=24, context_overlap=4, reference_attention_weight=1.,
                     audio_attention_weight=1., num_pad_audio_frames=2, do_multi_devices_inference=False,
                     save_gpu_memory=False, **kwargs):
        self._check_sampling_args(eta, num_images_per_prompt)
        device = self.device
        do_cfg = guidance_scale > 1.0
        batch_size = 1
        timesteps, num_inference_steps = retrieve_timesteps(self.scheduler, num_inference_steps, device, None)
        timesteps, num_inference_steps = self.get_timesteps(num_inference_steps, strength, device)

        writer = ReferenceAttentionControl(self.reference_net, do_classifier_free_guidance=do_cfg, mode="write",
                                           batch_size=batch_size, fusion_blocks="full")
        reader = ReferenceAttentionControl(self.denoising_unet, do_classifier_free_guidance=do_cfg, mode="read",
                                           batch_size=batch_size, fusion_blocks="full",
                                           reference_attention_weight=reference_attention_weight,
                                           audio_attention_weight=audio_attention_weight)
        num_channels_latents = self.denoising_unet.in_channels
        reference_image_latents = self.prepare_reference_latent(reference_image, height, width)
        kps_feature = self.prepare_kps_feature(kps_images, height, width, do_cfg)
        audio_embeddings = self.prepare_audio_embeddings(audio_waveform, video_length, num_pad_audio_frames, do_cfg)
        self.run_reference_net(reference_image_latents, writer)
        reader.update(getattr(self.reference_net, "writer_view", writer), do_cfg, dtype=self.dtype)

        latents = self.prepare_latents(batch_size * num_images_per_prompt, num_channels_latents, width, height,
                                       video_length, self.dtype, torch.device("cpu"), generator)
        latents = latents.to(device=device, dtype=BF16, non_blocking=True)      # one H2D for the whole video
        distributed = bool(do_multi_devices_inference) and torch.distributed.is_available() \
            and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1
        if distributed:
            # every rank drew its own host noise (generator=None, or differently seeded generators): rank 0's is THE video
            torch.distributed.broadcast(latents, src=0)
        try:
            latents = self.denoise(latents, kps_feature, audio_embeddings, timesteps, guidance_scale, context_frames,
                                   context_overlap, context_schedule, distributed, callback, callback_steps)
        finally:
            reader.clear()
            if isinstance(getattr(writer, "unet", None), torch.nn.Module) and hasattr(writer, "clear"):
                writer.clear()
        return self._decode_to_host(latents, distributed)

    def decode_to_device(self, latents, distributed):
        """VAE decode of latents (n,4,L,h,w), sharded by (sample, frame) over the ranks: (n,3,L,H,W) fp32 on rank 0's
        device -- (3,L,H,W) when n = 1 -- and None on the other ranks; the shards meet over NVLink."""
        n, _, L = latents.shape[:3]
        H, W = latents.shape[3] * self.vae_scale_factor, latents.shape[4] * self.vae_scale_factor
        rank, world = 0, 1
        if distributed and torch.distributed.is_available() and torch.distributed.is_initialized():
            rank, world = torch.distributed.get_rank(), torch.distributed.get_world_size()
        if world == 1:
            if n == 1:
                return self.decode_latents(latents)
            out = torch.empty((n, 3, L, H, W), device=latents.device, dtype=torch.float32)
            for s in range(n):
                self.decode_latents(latents, out=out[s], sample=s)
            return out
        # rank r owns items [r per, (r + 1) per) of the sample-major (sample, frame) list: at most one run of frames per
        # sample it touches
        per = math.ceil(n * L / world)
        lo, hi = rank * per, min(n * L, (rank + 1) * per)
        buf = torch.zeros((3, per, H, W), device=latents.device, dtype=torch.float32)
        for s in range(n):
            a, e = max(lo, s * L), min(hi, (s + 1) * L)
            if a < e:
                self.decode_latents(latents, range(a - s * L, e - s * L), out=buf[:, a - lo:e - lo], sample=s)
        gathered = [torch.empty_like(buf) for _ in range(world)] if rank == 0 else None
        torch.distributed.gather(buf, gathered, dst=0)
        if rank != 0:
            return None
        video = torch.cat(gathered, dim=1)[:, :n * L]
        return video if n == 1 else video.view(3, n, L, H, W).transpose(0, 1)

    def _decode_to_host(self, latents, distributed):
        """-> (n,3,L,H,W) fp32 on the host (rank 0): one device->host copy into pinned memory from torch's caching host
        allocator (a fresh tensor per call; the block is recycled when the caller drops it)."""
        video = self.decode_to_device(latents, distributed)
        if video is None:
            return None
        if video.dim() == 4:
            video = video.unsqueeze(0)
        host = torch.empty(tuple(video.shape), dtype=torch.float32, pin_memory=True)
        host.copy_(video, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return host

    def __call__(self, reference_image, kps_images, audio_waveform, width, height, video_length, num_inference_steps,
                 guidance_scale, strength=1., num_images_per_prompt=1, eta: float = 0.0, generator=None,
                 output_type: Optional[str] = "tensor", return_dict: bool = True, callback=None, callback_steps=1,
                 context_schedule="uniform", context_frames=24, context_overlap=4, reference_attention_weight=1.,
                 audio_attention_weight=1., num_pad_audio_frames=2, do_multi_devices_inference=False,
                 save_gpu_memory=False, **kwargs):
        return self.mean_overlap(
            reference_image=reference_image, kps_images=kps_images, audio_waveform=audio_waveform, width=width,
            height=height, video_length=video_length, num_inference_steps=num_inference_steps,
            guidance_scale=guidance_scale, strength=strength, num_images_per_prompt=num_images_per_prompt, eta=eta,
            generator=generator, output_type=output_type, return_dict=return_dict, callback=callback,
            callback_steps=callback_steps, context_schedule=context_schedule, context_frames=context_frames,
            context_overlap=context_overlap, reference_attention_weight=reference_attention_weight,
            audio_attention_weight=audio_attention_weight, num_pad_audio_frames=num_pad_audio_frames,
            do_multi_devices_inference=do_multi_devices_inference, save_gpu_memory=save_gpu_memory, **kwargs)

    def stream(self, reference_image, kps_images, audio_waveform, width, height, video_length, num_inference_steps,
               guidance_scale, strength=1., num_images_per_prompt=1, eta: float = 0.0, generator=None,
               output_type: Optional[str] = "tensor", return_dict: bool = True, context_schedule="uniform",
               context_frames=24, context_overlap=4, reference_attention_weight=1., audio_attention_weight=1.,
               num_pad_audio_frames=2, do_multi_devices_inference=False, save_gpu_memory=False, output="float",
               **kwargs) -> Iterator[VideoChunk]:
        """``__call__`` as a generator of ``VideoChunk(start, frames)`` for videos of any length: chunks of
        ``vae_chunk`` frames in frame order covering [0, video_length) once, each handed out as soon as its frames are
        final, with the device holding the per-frame state of the whole video (latents, accumulator, audio tokens:
        about 100 KB per frame and sample at 512x512) but kps features only for the windows in flight
        (``denoise_stream``).  ``output="float"``: (n,3,k,H,W) fp32 frames equal to the matching frames of ``__call__``;
        ``output="uint8"``: (n,k,H,W,3) median-filtered uint8 frames, the frames ``save_video`` writes.  Runs on one
        GPU.  Arguments are checked when called; the work starts with the first ``next``."""
        self._check_sampling_args(eta, num_images_per_prompt)
        if output not in ("float", "uint8"):
            raise ValueError(f"output must be 'float' or 'uint8', got {output!r}")
        if torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1:
            raise ValueError("stream() runs on one GPU: multi-GPU streaming is not supported "
                             f"(world size {torch.distributed.get_world_size()})")
        return self._stream(reference_image, kps_images, audio_waveform, width, height, video_length,
                            num_inference_steps, guidance_scale, strength, num_images_per_prompt, generator,
                            context_schedule, context_frames, context_overlap, reference_attention_weight,
                            audio_attention_weight, num_pad_audio_frames, output)

    @torch.no_grad()
    def _stream(self, reference_image, kps_images, audio_waveform, width, height, video_length, num_inference_steps,
                guidance_scale, strength, num_images_per_prompt, generator, context_schedule, context_frames,
                context_overlap, reference_attention_weight, audio_attention_weight, num_pad_audio_frames, output):
        device = self.device
        do_cfg = guidance_scale > 1.0
        timesteps, num_inference_steps = retrieve_timesteps(self.scheduler, num_inference_steps, device, None)
        timesteps, num_inference_steps = self.get_timesteps(num_inference_steps, strength, device)
        writer = ReferenceAttentionControl(self.reference_net, do_classifier_free_guidance=do_cfg, mode="write",
                                           batch_size=1, fusion_blocks="full")
        reader = ReferenceAttentionControl(self.denoising_unet, do_classifier_free_guidance=do_cfg, mode="read",
                                           batch_size=1, fusion_blocks="full",
                                           reference_attention_weight=reference_attention_weight,
                                           audio_attention_weight=audio_attention_weight)
        reference_image_latents = self.prepare_reference_latent(reference_image, height, width)
        audio_embeddings = self.prepare_audio_embeddings(audio_waveform, video_length, num_pad_audio_frames, do_cfg)
        self.run_reference_net(reference_image_latents, writer)
        reader.update(getattr(self.reference_net, "writer_view", writer), do_cfg, dtype=self.dtype)
        latents = self.prepare_latents(num_images_per_prompt, self.denoising_unet.in_channels, width, height,
                                       video_length, self.dtype, torch.device("cpu"), generator)
        latents = latents.to(device=device, dtype=BF16, non_blocking=True)
        try:
            yield from self.denoise_stream(latents, kps_images, audio_embeddings, timesteps, guidance_scale,
                                           context_frames, context_overlap, context_schedule, output)
        finally:
            reader.clear()
            if isinstance(getattr(writer, "unet", None), torch.nn.Module) and hasattr(writer, "clear"):
                writer.clear()
