#!/usr/bin/env python
"""Generate tests/golden/pipeline_eta_small.pt and pipeline_eta_nontiling_small.pt: the REFERENCE pipeline's own
``__call__`` at eta > 0 with a seeded CPU generator (stochastic DDIM), on the reduced-width model in fp32.

TEST INFRASTRUCTURE ONLY; needs the reference checkout (VX_REFERENCE, as oracle/gen_golden.py).  It runs
``oracle/gen_golden.py``'s ``gen_pipeline`` unchanged -- the reference's ``pipelines/v_express_pipeline.py`` and UNet
modules imported verbatim over oracle/diffusers_shim -- with two things bound around it:

  * ``VExpressPipeline.__call__`` receives ``eta`` and ``generator`` (torch.Generator().manual_seed(seed)) like any
    caller's keyword arguments; the reference hands both to ``scheduler.step`` (prepare_extra_step_kwargs, :168-187);
  * the scheduler is the shim's ``DDIMScheduler`` with a ``step`` that draws the variance noise as diffusers 0.29.2's
    does -- ``randn_tensor(model_output.shape, generator, device=model_output.device, dtype=model_output.dtype)``, which
    for a CPU generator and host tensors is ``torch.randn(shape, generator=generator, dtype=dtype)`` on the host -- and
    records it before handing it to the shim's step as ``variance_noise``.

Stored: the final latents (fp32), the decoded video of the frames ``video_frames`` (fp16) and, for every
``variance_noise`` in call order, its shape, the SHA-256 of its fp32 bytes and its first 8 values.  One thread, for the
duplicate-index write of the reflected tail window (see oracle/gen_golden.py).

Usage:  python tools/gen_eta_golden.py
"""
import hashlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import gen_golden as G  # noqa: E402  (puts oracle/diffusers_shim on sys.path)

CASES = [
    # tiling: windows of 8 / overlap 4, 3 steps, eta 1
    dict(name="pipeline_eta_small.pt", L=12, S=8, Ov=4, steps=3, eta=1.0, seed=2024, video_frames=[11]),
    # reflected tail window repeating frames 12..18: windows of 16 / overlap 4, 2 steps, eta 0.5
    dict(name="pipeline_eta_nontiling_small.pt", L=20, S=16, Ov=4, steps=2, eta=0.5, seed=2025,
         video_frames=[19]),
]


def digest(x):
    return hashlib.sha256(x.detach().float().contiguous().numpy().tobytes()).hexdigest()


def gen_case(msa, unet3d, pipe, case):
    import diffusers
    draws = []
    shim_scheduler = diffusers.DDIMScheduler

    class RecordingDDIM(shim_scheduler):
        def step(self, model_output, timestep, sample, eta=0.0, use_clipped_model_output=False, generator=None,
                 variance_noise=None, return_dict=True):
            if eta > 0 and variance_noise is None:
                assert isinstance(generator, torch.Generator) and generator.device.type == "cpu"
                assert model_output.device.type == "cpu"
                variance_noise = torch.randn(model_output.shape, generator=generator, dtype=model_output.dtype)
                draws.append(variance_noise.clone())
                generator = None
            return super().step(model_output, timestep, sample, eta=eta,
                                use_clipped_model_output=use_clipped_model_output, generator=generator,
                                variance_noise=variance_noise, return_dict=return_dict)

    real_call = pipe.VExpressPipeline.__call__
    gen = torch.Generator().manual_seed(case["seed"])

    def call(self, *a, **k):
        return real_call(self, *a, eta=case["eta"], generator=gen, **k)
    diffusers.DDIMScheduler = RecordingDDIM
    pipe.VExpressPipeline.__call__ = call
    try:
        G.gen_pipeline(msa, unet3d, pipe, L=case["L"], S=case["S"], Ov=case["Ov"], steps=case["steps"],
                       name=case["name"], with_video=True)
    finally:
        diffusers.DDIMScheduler = shim_scheduler
        pipe.VExpressPipeline.__call__ = real_call
    path = os.path.join(G.GOLD, case["name"])
    out = torch.load(path, weights_only=False)
    ids = case["video_frames"]
    out["video"] = out["video"][:, :, ids].clone()
    out.update(video_frames=ids, eta=case["eta"], seed=case["seed"],
               variance_noise_shapes=[tuple(x.shape) for x in draws],
               variance_noise_sha256=[digest(x) for x in draws],
               variance_noise_head=[x.reshape(-1)[:8].clone() for x in draws])
    torch.save(out, path)
    print(case["name"], ":", len(draws), "draws", out["variance_noise_shapes"], os.path.getsize(path), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(1)
    msa, unet3d, _, pipe = G.import_reference()
    for c in CASES:
        gen_case(msa, unet3d, pipe, c)
