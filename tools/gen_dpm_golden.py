#!/usr/bin/env python
"""Generate tests/golden/pipeline_dpm_small.pt: the REFERENCE pipeline's own ``__call__`` with a DPM-Solver++(2M)
scheduler, on the reduced-width model in fp32.

TEST INFRASTRUCTURE ONLY; needs the reference checkout (VX_REFERENCE, as oracle/gen_golden.py).  It runs
``oracle/gen_golden.py``'s ``gen_pipeline`` unchanged -- the reference's ``pipelines/v_express_pipeline.py`` and UNet
modules imported verbatim over oracle/diffusers_shim -- with the scheduler it constructs from the reference's
noise_scheduler_kwargs replaced by ``tests/dpm_reference.DPMSolverMultistepScheduler`` built from the same keywords (as
diffusers' ``from_config`` would, dropping the DDIM-only ``clip_sample``).

The case is one context window (video_length 8, context_frames 8): the reference calls ``scheduler.step`` once per
window, and the library's scheduler keeps its step index and history across calls, so the reference is well defined with
DPM-Solver++ at one window only.  5 steps: first order at steps 0 and 4, second order at 1-3.  Stored: the final latents
(fp32) and the decoded frame ``video_frames`` (fp16).  One thread, as tools/gen_eta_golden.py.

Usage:  python tools/gen_dpm_golden.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from oracle import gen_golden as G  # noqa: E402  (puts oracle/diffusers_shim on sys.path)
import dpm_reference as R  # noqa: E402

CASE = dict(name="pipeline_dpm_small.pt", L=8, S=8, Ov=4, steps=5, video_frames=[7])


def gen_case(msa, unet3d, ctx, pipe, case):
    import diffusers
    windows = list(ctx.uniform(step=0, num_frames=case["L"], context_size=case["S"], context_stride=1,
                               context_overlap=case["Ov"], closed_loop=False))
    assert len(windows) == 1, windows
    calls = []

    class RecordingDPM(R.DPMSolverMultistepScheduler):
        def step(self, model_output, timestep, sample, **kw):
            out = super().step(model_output, timestep, sample, **kw)
            calls.append((int(timestep), self.step_index - 1, self.lower_order_nums))
            return out

    def build(**kw):
        kw.pop("clip_sample", None)
        return RecordingDPM(**kw)
    ddim = diffusers.DDIMScheduler
    diffusers.DDIMScheduler = build
    try:
        G.gen_pipeline(msa, unet3d, pipe, L=case["L"], S=case["S"], Ov=case["Ov"], steps=case["steps"],
                       name=case["name"], with_video=True)
    finally:
        diffusers.DDIMScheduler = ddim
    assert [c[1] for c in calls] == list(range(case["steps"])), calls
    path = os.path.join(G.GOLD, case["name"])
    out = torch.load(path, weights_only=False)
    ids = case["video_frames"]
    out["video"] = out["video"][:, :, ids].clone()
    out.update(video_frames=ids, sampler="dpmsolver++", solver_order=2, timesteps=[c[0] for c in calls])
    torch.save(out, path)
    print(case["name"], ":", calls, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(1)
    msa, unet3d, ctx, pipe = G.import_reference()
    gen_case(msa, unet3d, ctx, pipe, CASE)
