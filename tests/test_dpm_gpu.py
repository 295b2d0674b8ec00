"""DPM-Solver++ on the H100: the ``vx_dpmpp_step`` / ``vx_dpmpp_step_frames`` kernels against the library-structured
scheduler's eager step on bf16 CUDA tensors (tests/dpm_reference.py), and the public pipeline against the reference
pipeline's own output with that scheduler (tests/golden/pipeline_dpm_small.pt) and against itself streamed."""
import os

import pytest
import torch

import dpm_reference as R
from test_eta_gpu import _fp32_model_pipeline
from test_samples_gpu import _public_pipeline
from test_stream_gpu import _args, _gens, _streaming_pipeline
from test_unet_gpu import _rel

pytestmark = pytest.mark.gpu


def _library_steps(steps, ks, shape, g):
    """Run the library-structured scheduler's ``step`` on bf16 CUDA tensors for steps 0..max(ks); yield, for each k in
    ks, (k, model_output, sample, previous x0 prediction, the library's prev_sample)."""
    lib = R.reference_scheduler()
    lib.set_timesteps(steps)
    for k, t in enumerate(lib.timesteps.tolist()[:max(ks) + 1]):
        x = torch.randn(shape, generator=g).bfloat16().cuda()
        acc = torch.randn(shape, generator=g).bfloat16().float().cuda()
        prev_m = lib.model_outputs[-1]
        out = lib.step(acc.bfloat16(), t, x).prev_sample
        if k in ks:
            yield k, acc, x, prev_m, out, lib.model_outputs[-1]


@pytest.mark.parametrize("shape", [(1, 4, 7, 37), (3, 4, 5, 19 * 19), (2, 4, 16, 4096 + 3)])
@pytest.mark.parametrize("steps,ks", [(5, (0, 1, 3, 4)), (25, (0, 1, 12, 24)), (2, (0, 1))])
def test_dpmpp_step_equals_library_step(shape, steps, ks):
    """Orders 1 (the first step at sigma ~ 4096, the last at sigma_t = 0) and 2, sizes with tails: the kernel's latents
    and history equal the library's prev_sample and x0 prediction, torch.equal."""
    from vexpress_b200 import ops
    from vexpress_b200.pipelines.scheduler import DPMSolverMultistepScheduler, dpm_coefficients
    prod = DPMSolverMultistepScheduler()
    prod.set_timesteps(steps)
    g = torch.Generator().manual_seed(sum(shape) + steps)
    for k, acc, x, prev_m, ref, ref_m in _library_steps(steps, ks, shape, g):
        c = dpm_coefficients(prod, k)
        assert c[-1] == (1 if k in (0, steps - 1) else 2)
        lat = x.clone()
        hist = prev_m.clone() if prev_m is not None else torch.full_like(x, float("nan"))
        ops.dpmpp_step(lat, acc, hist, *c)
        torch.cuda.synchronize()
        assert ref.dtype == torch.bfloat16 and torch.isfinite(lat.float()).all()
        assert torch.equal(lat, ref), (steps, k, (lat.float() - ref.float()).abs().max().item())
        assert torch.equal(hist, ref_m), (steps, k)


@pytest.mark.parametrize("order_step", [0, 2, 4])
def test_dpmpp_step_frames_equals_whole_form(order_step):
    """The frames form updates exactly the listed frames as the whole form does, zeroes their acc entries and leaves
    every other latent, history and acc entry unchanged."""
    from vexpress_b200 import ops
    from vexpress_b200.pipelines.scheduler import DPMSolverMultistepScheduler, dpm_coefficients
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(5)
    c = dpm_coefficients(s, order_step)
    g = torch.Generator(device="cuda").manual_seed(3 + order_step)
    n, L, h = 2, 23, 12
    lat = torch.randn(n, 4, L, h, h, device="cuda", generator=g).bfloat16()
    acc = torch.randn(n, 4, L, h * h, device="cuda", generator=g).bfloat16().float()
    hist = torch.randn(n, 4, L, h * h, device="cuda", generator=g).bfloat16()
    full_lat, full_hist = lat.clone(), hist.clone()
    ops.dpmpp_step(full_lat, acc, full_hist, *c)
    chosen = [0, 3, 4, 11, L - 1]
    got_lat, got_acc, got_hist = lat.clone(), acc.clone(), hist.clone()
    ops.dpmpp_step_frames(got_lat, got_acc, got_hist, torch.tensor(chosen, device="cuda", dtype=torch.int32), *c)
    torch.cuda.synchronize()
    others = [i for i in range(L) if i not in chosen]
    assert torch.equal(got_lat[:, :, chosen], full_lat[:, :, chosen])
    assert torch.equal(got_hist[:, :, chosen], full_hist[:, :, chosen])
    assert torch.equal(got_lat[:, :, others], lat[:, :, others]) and torch.equal(got_hist[:, :, others], hist[:, :, others])
    assert torch.count_nonzero(got_acc[:, :, chosen]) == 0
    assert torch.equal(got_acc[:, :, others], acc[:, :, others])


def test_pipeline_dpm_vs_reference_golden(golden_dir):
    """The reference's own pipeline over the library-structured DPM-Solver++(2M) scheduler (one window, 5 steps): final
    latents within 6e-2 relative L2 and the kept frame within 1.5e-2 mean absolute error -- the tolerances of the DDIM
    golden tests -- eager and graphed runs bit-identical; DDIM at the same steps lands far from the golden."""
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
    g = torch.load(os.path.join(golden_dir, "pipeline_dpm_small.pt"), weights_only=False)
    pipe = _fp32_model_pipeline(g["L"])
    pipe.scheduler = DPMSolverMultistepScheduler()
    captured = {}
    orig = pipe._decode_to_host

    def grab(latents, distributed):
        captured["latents"] = latents.float().cpu()
        return orig(latents, distributed)
    pipe._decode_to_host = grab

    def call():
        return pipe(None, None, None, g["h"] * 8, g["h"] * 8, g["L"], g["steps"], g["guidance_scale"],
                    context_frames=g["S"], context_overlap=g["O"], reference_attention_weight=0.95,
                    audio_attention_weight=3.0)
    videos, e_lat = [], 0.0
    for use_graph in (False, True):
        pipe.use_cuda_graph = use_graph
        video = call()
        assert video.shape == (1, 3, g["L"], g["h"] * 8, g["h"] * 8)
        e_lat = _rel(captured["latents"], g["final_latents"])
        d = (video[:, :, g["video_frames"]] - g["video"].float()).abs().mean().item()
        print(f"DPM-Solver++ graph={use_graph}: final latents rel {e_lat:.3e}; video mean abs {d:.3e}")
        assert e_lat < 6e-2 and d < 1.5e-2
        videos.append(video)
    assert torch.equal(videos[0], videos[1])
    pipe.scheduler = DDIMScheduler()
    call()
    e_ddim = _rel(captured["latents"], g["final_latents"])
    print(f"DDIM at {g['steps']} steps: final latents rel {e_ddim:.3e} from the DPM golden")
    assert e_ddim > max(6e-2, 3 * e_lat), "DDIM should not meet the DPM-Solver++ golden"


@pytest.mark.parametrize("L", [52, 50])
def test_stream_equals_call_under_dpm(L):
    """``stream`` under DPM-Solver++ equals ``__call__`` frame for frame, one and two samples (4 windows of 16 /
    overlap 4: tiling and reflected tail)."""
    from vexpress_b200.pipelines.scheduler import DPMSolverMultistepScheduler
    pipe = _streaming_pipeline(L)
    pipe.scheduler = DPMSolverMultistepScheduler()
    for seeds in ([5], [5, 6]):
        args = dict(_args(L, len(seeds), _gens(seeds)), num_inference_steps=4)
        ref = pipe(**args)
        video = torch.cat([c.frames for c in pipe.stream(**dict(args, generator=_gens(seeds)))], 2)
        print(f"L={L} n={len(seeds)}: max |stream - call| = {(video - ref).abs().max().item()}")
        assert video.shape == ref.shape and torch.equal(video, ref)


def test_three_samples_equal_one_sample_calls_under_dpm():
    from vexpress_b200.pipelines.scheduler import DPMSolverMultistepScheduler
    L, seeds = 20, [5, 6, 7]
    pipe = _public_pipeline(L)
    pipe.scheduler = DPMSolverMultistepScheduler()

    def call(n, gen):
        return pipe(None, None, None, 128, 128, L, 4, 3.5, num_images_per_prompt=n, generator=gen, context_frames=16,
                    context_overlap=4, reference_attention_weight=0.95, audio_attention_weight=3.0)
    video = call(3, _gens(seeds))
    for i, s in enumerate(seeds):
        assert torch.equal(video[i], call(1, _gens([s]))[0]), i
    assert not torch.equal(video[0], video[1])
