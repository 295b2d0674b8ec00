"""Several samples per call on the H100 kernels: sample i of an n-sample call is bit-identical to a one-sample call with
``generator[i]`` -- the batched CFG / overlap kernel, the batched UNet forward at full width and the public pipeline."""
import pytest
import torch

from test_pipeline_gpu import build_pipeline
from test_samples_cpu import _ElementwiseEmu
from test_unet_gpu import build_product

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,f,hw,L,S,Ov,do_cfg", [(2, 16, 256, 24, 16, 8, True), (3, 16, 64, 20, 16, 4, True),
                                                   (3, 24, 37, 33, 24, 4, True), (4, 5, 19, 9, 5, 1, False)])
def test_cfg_overlap_n_kernel_equals_emulation(n, f, hw, L, S, Ov, do_cfg):
    """Every window's slots of the overlap plan (non-tiling plans carry -1 slots), accumulated into a running acc
    (n, 4, L, hw): the kernel equals the torch emulation with its rounding points bit for bit, and sample s equals the
    one-sample kernel on its [u | c] blocks."""
    from vexpress_b200 import ops
    from vexpress_b200.pipelines.context import overlap_plan, window_table
    windows, count = window_table(L, S, Ov, "uniform")
    plan = overlap_plan(windows, count)
    g = torch.Generator().manual_seed(n * 100 + f)
    b = 2 if do_cfg else 1
    count_t = torch.from_numpy(count).to(torch.int32)
    count_dev = count_t.cuda()
    acc = torch.randn(n, 4, L, hw, generator=g).bfloat16().float()
    acc_d, acc_1 = acc.cuda(), acc.cuda()
    slots_seen, launches = 0, 0
    for wi, wn in enumerate(windows):
        fw = len(wn)
        if fw != f:
            continue
        noise = torch.randn(b * n * fw, 4, hw, generator=g).bfloat16()
        noise_d = noise.cuda()
        for slots in plan[wi]:
            slots_t = torch.from_numpy(slots)
            slots_d = slots_t.cuda()
            slots_seen += int((slots_t < 0).sum())
            launches += 1
            ops.cfg_overlap_accumulate_n(noise_d, n, fw, hw, L, do_cfg, slots_d, count_dev, 3.5, acc_d)
            _ElementwiseEmu.cfg_overlap_accumulate_n(noise, n, fw, hw, L, do_cfg, slots_t, count_t, 3.5, acc)
            blocks = noise_d.view(b, n, fw, 4, hw)
            for s in range(n):
                ops.cfg_overlap_accumulate(blocks[:, s].contiguous(), fw, hw, L, do_cfg, slots_d, count_dev, 3.5, acc_1[s])
    torch.cuda.synchronize()
    assert torch.equal(acc_d.cpu(), acc)
    assert torch.equal(acc_d, acc_1)
    assert launches >= 2
    if (L, S, Ov) in ((20, 16, 4), (33, 24, 4)):
        assert slots_seen > 0                                # the reflected-window plans exercise the -1 slots


def test_forward_frames_two_samples_equal_one_sample_forwards():
    """Full-width UNet at the configs[0] shape (f = 4, 64x64 latents): one forward of [u s0 | u s1 | c s0 | c s1] equals
    the two one-sample forwards [u s | c s] with torch.equal."""
    from oracle import vx_oracle as O
    cfg = O.DEFAULT_CFG
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), 1234)
    f, h = 4, 64
    lat, kps, audio, banks = O.synth_inputs(cfg, f, h, h, True, 42)
    model, reader = build_product(cfg, sd, [b[1:] for b in banks], 0.95, 3.0)
    eng = model.engine()
    lat2 = torch.randn(lat.shape, generator=torch.Generator().manual_seed(7))
    samples = [lat[0].transpose(0, 1).bfloat16().cuda(), lat2[0].transpose(0, 1).bfloat16().cuda()]   # (f, 4, h, w)
    kps_nhwc = kps.bfloat16().cuda().permute(0, 2, 3, 4, 1).reshape(2 * f * h * h, -1).contiguous()
    enc = audio.reshape(2, f, 5, cfg["cross_attention_dim"]).bfloat16().cuda()
    idx1 = torch.arange(2 * f, device="cuda", dtype=torch.int32)
    with torch.no_grad():
        one = [eng.forward_frames(torch.cat([x, x]), 499, enc.reshape(-1, 5, enc.shape[-1]), kps_nhwc, idx1, 2, f)
               for x in samples]
        frames = torch.cat(samples + samples)                                   # [u s0 | u s1 | c s0 | c s1]
        enc2 = enc.unsqueeze(1).expand(2, 2, f, 5, enc.shape[-1]).reshape(-1, 5, enc.shape[-1]).contiguous()
        idx2 = idx1.view(2, 1, f).expand(2, 2, f).reshape(-1).contiguous()
        two = eng.forward_frames(frames, 499, enc2, kps_nhwc, idx2, 2, f, n=2).view(2, 2, f, 4, h, h)
    torch.cuda.synchronize()
    reader.clear()
    for s in range(2):
        ref = one[s].view(2, f, 4, h, h)
        d = (two[:, s].float() - ref.float()).abs().max().item()
        print(f"sample {s}: max |batched - single| = {d}")
        assert torch.equal(two[:, s], ref), s
    assert not torch.equal(one[0], one[1])


def _public_pipeline(L):
    from oracle import vx_oracle as O
    from vexpress_b200.pipelines.v_express_pipeline import VExpressPipeline
    cfg, vcfg = O.small_cfg(), O.small_vae_cfg()
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), 1234)
    vsd = O.synth_state_dict(O.vae_param_shapes(vcfg), 1235)
    lat, kps, audio, banks = O.synth_inputs(cfg, L, 16, 16, True, 42)
    pipe = build_pipeline(cfg, vcfg, sd, vsd, kps, audio, [b[1:] for b in banks], lat)
    pipe.prepare_latents = VExpressPipeline.prepare_latents.__get__(pipe)        # draw from the caller's generators
    return pipe


def _call(pipe, L, n, generator):
    return pipe(None, None, None, 128, 128, L, 2, 3.5, num_images_per_prompt=n, generator=generator,
                context_frames=16, context_overlap=4, reference_attention_weight=0.95, audio_attention_weight=3.0)


SEEDS = [5, 6, 7]


@pytest.mark.parametrize("use_graph", [False, True])
def test_pipeline_three_samples_equal_one_sample_calls(use_graph):
    """Reduced-width public pipeline, video_length 20 (windows 16 / overlap 4: a reflected tail window): the 3-sample
    call returns (3, 3, L, H, W) and sample i equals the one-sample call with generator[i] bit for bit."""
    L = 20
    pipe = _public_pipeline(L)
    pipe.use_cuda_graph = use_graph
    video = _call(pipe, L, 3, [torch.Generator().manual_seed(s) for s in SEEDS])
    assert video.shape == (3, 3, L, 128, 128) and video.dtype == torch.float32 and video.device.type == "cpu"
    for i, s in enumerate(SEEDS):
        one = _call(pipe, L, 1, [torch.Generator().manual_seed(s)])
        assert one.shape == (1, 3, L, 128, 128)
        d = (video[i] - one[0]).abs().max().item()
        print(f"graph={use_graph} sample {i}: max |batched - single| = {d}")
        assert torch.equal(video[i], one[0]), i
    assert not torch.equal(video[0], video[1])


def test_one_sample_call_equals_fixed_latent_path():
    """n = 1 through the generator route (a list of one generator, or the generator itself) gives the video of the
    existing one-sample path fed the same latents, with the same number of kernel launches."""
    from vexpress_b200 import _ffi
    from vexpress_b200.pipelines.v_express_pipeline import VExpressPipeline
    L = 20
    pipe = _public_pipeline(L)
    fixed = VExpressPipeline.prepare_latents(pipe, 1, 4, 128, 128, L, torch.bfloat16, None,
                                             torch.Generator().manual_seed(SEEDS[0]))
    pipe.prepare_latents = lambda *a, **k: fixed.clone()
    _call(pipe, L, 1, None)                                  # the first call captures the graphs
    l0 = _ffi.LAUNCHES
    ref = _call(pipe, L, 1, None)
    launches = _ffi.LAUNCHES - l0
    pipe.prepare_latents = VExpressPipeline.prepare_latents.__get__(pipe)
    for gen in ([torch.Generator().manual_seed(SEEDS[0])], torch.Generator().manual_seed(SEEDS[0])):
        l0 = _ffi.LAUNCHES
        got = _call(pipe, L, 1, gen)
        assert _ffi.LAUNCHES - l0 == launches
        assert got.shape == ref.shape == (1, 3, L, 128, 128) and torch.equal(got, ref)
