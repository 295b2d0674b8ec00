"""Stochastic DDIM (eta > 0) on the H100: the ``vx_ddim_step_eta`` kernel against diffusers' step run eagerly in bf16 on
CUDA, and the public pipeline at eta > 0 against the reference pipeline's own output (tests/golden/pipeline_eta*.pt),
the n-sample contract and torch's default CUDA generator."""
import os

import pytest
import torch

from test_pipeline_gpu import build_pipeline
from test_samples_gpu import _public_pipeline
from test_unet_gpu import _rel

pytestmark = pytest.mark.gpu


def _lib_scheduler(steps):
    import sys
    from oracle import vx_oracle as O
    p = os.path.join(os.path.dirname(os.path.abspath(O.__file__)), "diffusers_shim")
    if p not in sys.path:
        sys.path.insert(0, p)
    import diffusers
    s = diffusers.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                                steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                                timestep_spacing="trailing")
    s.set_timesteps(steps)
    return s


@pytest.mark.parametrize("shape", [(1, 4, 7, 37), (3, 4, 5, 19 * 19), (2, 4, 16, 4096 + 3)])
@pytest.mark.parametrize("noise_dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_ddim_step_eta_kernel_equals_library_step(shape, noise_dtype):
    """bf16 draws: the kernel equals diffusers' ``step(model_output, t, sample, eta, variance_noise=noise)`` on bf16
    CUDA tensors bit for bit.  fp16 / fp32 draws (a model held in that dtype): the latents stay bf16, so the kernel is
    the same bf16 step with the noise product bf16(sigma * noise) taken from the exact fp32 image of the draw -- the
    library's deterministic part of the step plus that term, as eager bf16 CUDA ops."""
    from vexpress_b200 import ops
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, ddim_coefficients_eta
    g = torch.Generator().manual_seed(sum(shape))
    for steps, eta, ts in ((25, 0.3, (959, 499, 39)), (25, 1.0, (959, 39)), (3, 1.0, (999, 665, 332)), (3, 0.5, (999,))):
        lib, prod = _lib_scheduler(steps), DDIMScheduler()
        prod.set_timesteps(steps)
        for t in ts:
            x = torch.randn(shape, generator=g).bfloat16().cuda()
            acc = torch.randn(shape, generator=g).bfloat16().float().cuda()
            noise = torch.randn(shape, generator=g, dtype=noise_dtype).cuda()
            lat = x.clone()
            ops.ddim_step_eta(lat, acc, noise.float(), *ddim_coefficients_eta(prod, t, eta))
            v = acc.bfloat16()
            if noise_dtype == torch.bfloat16:
                ref = lib.step(v, t, x, eta=eta, variance_noise=noise).prev_sample
            else:
                det = lib.step(v, t, x, eta=eta, variance_noise=torch.zeros_like(x)).prev_sample
                std = eta * lib._get_variance(t, t - 1000 // steps) ** 0.5
                ref = det + (float(std) * noise.float()).bfloat16()
            torch.cuda.synchronize()
            assert ref.dtype == torch.bfloat16
            d = (lat.float() - ref.float()).abs().max().item()
            assert torch.equal(lat, ref), (steps, eta, t, d)


def _fp32_model_pipeline(L):
    """The reduced-width pipeline with the UNet held in fp32, as the golden's reference run was, so ``pipe.dtype`` -- the
    dtype the step noise is drawn in -- is fp32 (the engine rounds the weights to bf16 itself)."""
    from oracle import vx_oracle as O
    cfg, vcfg = O.small_cfg(), O.small_vae_cfg()
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), 1234)
    vsd = O.synth_state_dict(O.vae_param_shapes(vcfg), 1235)
    lat, kps, audio, banks = O.synth_inputs(cfg, L, 16, 16, True, 42)
    pipe = build_pipeline(cfg, vcfg, sd, vsd, kps, audio, [b[1:] for b in banks], lat)
    pipe.denoising_unet.float()
    assert pipe.dtype == torch.float32
    return pipe


@pytest.mark.parametrize("name", ["pipeline_eta_small.pt", "pipeline_eta_nontiling_small.pt"])
def test_pipeline_eta_vs_reference_golden(golden_dir, name):
    """The reference's own pipeline at eta > 0 with a seeded CPU generator (tiling L=12, eta 1; reflected tail L=20,
    eta 0.5): final latents within 6e-2 relative L2 and video mean abs error < 1.5e-2 on the decoded frame the golden
    keeps (the last) -- the tolerances of the eta = 0 golden tests -- and the eager and CUDA-graph runs bit-identical."""
    g = torch.load(os.path.join(golden_dir, name), weights_only=False)
    pipe = _fp32_model_pipeline(g["L"])
    captured = {}
    orig = pipe._decode_to_host

    def grab(latents, distributed):
        captured["latents"] = latents.float().cpu()
        return orig(latents, distributed)
    pipe._decode_to_host = grab
    videos = []
    for use_graph in (False, True):
        pipe.use_cuda_graph = use_graph
        video = pipe(None, None, None, g["h"] * 8, g["h"] * 8, g["L"], g["steps"], g["guidance_scale"],
                     eta=g["eta"], generator=torch.Generator().manual_seed(g["seed"]), context_frames=g["S"],
                     context_overlap=g["O"], reference_attention_weight=0.95, audio_attention_weight=3.0)
        assert video.shape == (1, 3, g["L"], g["h"] * 8, g["h"] * 8) and video.dtype == torch.float32
        e_lat = _rel(captured["latents"], g["final_latents"])
        d = (video[:, :, g["video_frames"]] - g["video"].float()).abs()
        print(f"{name} graph={use_graph}: final latents rel {e_lat:.3e}; video mean abs {d.mean().item():.3e}")
        assert e_lat < 6e-2 and d.mean().item() < 1.5e-2
        videos.append(video)
    assert torch.equal(videos[0], videos[1])
    # the noise is what moves the result: the same call at eta = 0 lands far from the eta golden
    det = pipe(None, None, None, g["h"] * 8, g["h"] * 8, g["L"], g["steps"], g["guidance_scale"], context_frames=g["S"],
               context_overlap=g["O"], reference_attention_weight=0.95, audio_attention_weight=3.0)
    assert _rel(captured["latents"], g["final_latents"]) > 0.1, "eta = 0 should not meet the eta golden"
    assert not torch.equal(det, videos[0])


def test_pipeline_eta_three_samples_equal_one_sample_calls():
    """num_images_per_prompt = 3 at eta = 0.8 with a list of generators (initial latents and step noise both come from
    generator[i], as in the reference): sample i equals the one-sample call with generator[i], torch.equal."""
    L, seeds = 20, [5, 6, 7]
    pipe = _public_pipeline(L)

    def call(n, gen):
        return pipe(None, None, None, 128, 128, L, 2, 3.5, num_images_per_prompt=n, generator=gen, eta=0.8,
                    context_frames=16, context_overlap=4, reference_attention_weight=0.95, audio_attention_weight=3.0)
    video = call(3, [torch.Generator().manual_seed(s) for s in seeds])
    assert video.shape == (3, 3, L, 128, 128)
    for i, s in enumerate(seeds):
        one = call(1, [torch.Generator().manual_seed(s)])
        print(f"sample {i}: max |batched - single| = {(video[i] - one[0]).abs().max().item()}")
        assert torch.equal(video[i], one[0]), i
    assert not torch.equal(video[0], video[1])


def test_pipeline_eta_default_cuda_generator_reproduces(monkeypatch):
    """generator=None draws the step noise on the device from torch's default CUDA generator: two calls after the same
    torch.cuda.manual_seed are bit-identical, another seed differs."""
    from vexpress_b200.pipelines import v_express_pipeline as vp
    L = 12
    pipe = _fp32_model_pipeline(L)
    devices = set()
    real = vp._randn

    def rec(shape, generator, device, dtype):
        x = real(shape, generator, device, dtype)
        devices.add(x.device.type)
        return x
    monkeypatch.setattr(vp, "_randn", rec)

    def call(seed):
        torch.cuda.manual_seed(seed)
        return pipe(None, None, None, 128, 128, L, 3, 3.5, eta=1.0, context_frames=8, context_overlap=4,
                    reference_attention_weight=0.95, audio_attention_weight=3.0)
    a, b, c = call(31), call(31), call(32)
    assert devices == {"cuda"}
    assert torch.equal(a, b) and not torch.equal(a, c)
