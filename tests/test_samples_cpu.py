"""Several samples per call (``num_images_per_prompt``) on the host side, without a GPU: the batched denoise loop with the
UNet replaced by a cheap deterministic function and the elementwise kernels by torch emulations with the kernels' rounding
points (the harness of tests/test_host_cpu.py, extended with the n-sample CFG / overlap kernel).

The contract: sample i of an n-sample call is bit-identical to a one-sample call with ``generator[i]``."""
import os

import pytest
import torch


def _fake_unet_core(x, kmean, emean, t):
    """x (B,f,4,h,w) fp32; kmean (B,f,1,h,w); emean (B,f,1,1,1) -> (B,f,4,h,w) bf16; mixes the frames of a clip like the
    motion modules do, never across clips."""
    return torch.tanh(0.9 * x + kmean + 0.1 * emean + 0.05 * x.mean(1, keepdim=True) + 1e-3 * t).bfloat16()


class _FakeEngine:
    """Stands in for UNetEngine: every block of f frames of the [uncond s0..s(n-1) | cond s0..s(n-1)] batch is one clip."""
    dev = torch.device("cpu")
    order = []

    def __init__(self):
        self.calls = []

    def time_embedding(self, t):
        return torch.tensor([[float(t)]])

    def graph_signature(self):
        return 0

    def forward_frames(self, frames, timestep, enc, kps, kps_idx, b, f, temb=None, taps=None, n=1):
        NB, _, h, w = frames.shape
        assert NB == b * n * f
        self.calls.append((b, n, f))
        B = b * n
        k = kps.view(-1, h * w, kps.shape[1])[kps_idx.long()].float().mean(-1).view(B, f, 1, h, w)
        e = enc.float().mean((1, 2)).view(B, f, 1, 1, 1)
        out = _fake_unet_core(frames.float().view(B, f, 4, h, w), k, e, float(temb.reshape(-1)[0]))
        return out.view(NB, 4, h, w)


def _rb(t):
    return t.bfloat16().float()


class _ElementwiseEmu:
    """torch emulation of vx_cfg_overlap_accumulate(_n) / vx_ddim_step with the kernels' rounding points
    (csrc/vx_misc.cu)."""

    @staticmethod
    def cfg_overlap_accumulate(noise, f, hw, L, do_cfg, win, count, guidance, acc):
        _ElementwiseEmu.cfg_overlap_accumulate_n(noise, 1, f, hw, L, do_cfg, win, count, guidance, acc.view(1, 4, L, hw))

    @staticmethod
    def cfg_overlap_accumulate_n(noise, n, f, hw, L, do_cfg, win, count, guidance, acc):
        x = noise.reshape(-1, n, f, 4, hw).float()                   # (b, n, f, 4, hw): [u s0..s(n-1) | c s0..s(n-1)]
        win, count = win.cpu(), count.cpu()
        for s in range(n):
            v = _rb(x[0, s] + _rb(guidance * _rb(x[1, s] - x[0, s]))) if do_cfg else x[0, s]
            for i in range(f):
                fr = int(win[i])
                if fr < 0:
                    continue
                acc[s, :, fr] = _rb(acc[s, :, fr] + _rb(v[i].to(acc.device) / float(count[fr])))

    @staticmethod
    def ddim_step(lat, acc, sa, sb, sap, sbp):
        x, v = lat.float().view(acc.shape), _rb(acc)
        x0 = _rb(_rb(sa * x) - _rb(sb * v))
        eps = _rb(_rb(sa * v) + _rb(sb * x))
        lat.copy_((_rb(sap * x0) + _rb(sbp * eps)).bfloat16().view(lat.shape))


class _FakeVae:
    """decode_latents(z (k,4,h,w), out (k,3,8h,8w)): a per-frame map plus (chunk_term = 1) a term that depends on the
    chunk it was decoded in, so a sample decoded in other chunks than a one-sample call would come out different."""

    def __init__(self, chunk_term):
        self.chunks = []
        self.chunk_term = chunk_term

    def decode_latents(self, z, out):
        self.chunks.append(z.shape[0])
        y = z[:, :3].float().repeat_interleave(8, -2).repeat_interleave(8, -1)
        out.copy_(torch.sigmoid(y + self.chunk_term * (1e-3 * z.shape[0] + 1e-4 * z.float().mean())))


def _fake_pipeline(chunk_term=1.0):
    from vexpress_b200.pipelines import v_express_pipeline as vp
    from vexpress_b200.pipelines.scheduler import DDIMScheduler
    eng = _FakeEngine()
    unet = type("U", (), {"engine": lambda self: eng, "get_submodule": lambda self, n: None, "in_channels": 4,
                          "dtype": torch.bfloat16})()
    pipe = vp.VExpressPipeline(vae=_FakeVae(chunk_term), reference_net=None, denoising_unet=unet, v_kps_guider=None,
                               audio_processor=None, audio_encoder=None, audio_projection=None, scheduler=DDIMScheduler())
    pipe.use_cuda_graph = False
    pipe.vae_chunk = 4
    vp.ops = _ElementwiseEmu()
    return pipe, vp, eng


def _fake_conditioning(L, h=4, C0=8):
    g = torch.Generator().manual_seed(1000 + L)
    kps = torch.cat([torch.zeros(1, C0, L, h, h), 0.1 * torch.randn(1, C0, L, h, h, generator=g)]).bfloat16()
    audio = torch.cat([torch.zeros(1, L, 5, 16), torch.randn(1, L, 5, 16, generator=g)]).bfloat16()
    return kps, audio


def _draw(pipe, seeds, L, h=4):
    return pipe.prepare_latents(len(seeds), 4, 8 * h, 8 * h, L, torch.bfloat16, torch.device("cpu"),
                                [torch.Generator().manual_seed(s) for s in seeds])


def _run(L, S, Ov, seeds, steps=3, distributed=False, callback=None, chunk_term=1.0):
    """-> (final latents (n,4,L,h,w), decoded video, fake engine, fake vae) of one denoise + decode on the host."""
    from vexpress_b200 import ops as real_ops
    from vexpress_b200.pipelines.v_express_pipeline import retrieve_timesteps
    pipe, vp, eng = _fake_pipeline(chunk_term)
    try:
        kps, audio = _fake_conditioning(L)
        ts, _ = retrieve_timesteps(pipe.scheduler, steps, None)
        lat = pipe.denoise(_draw(pipe, seeds, L), kps, audio, ts, 3.5, S, Ov, distributed=distributed, callback=callback)
        video = pipe.decode_to_device(lat, distributed)
        return lat, video, eng, pipe.vae
    finally:
        vp.ops = real_ops


SEEDS = [11, 22, 33]


@pytest.mark.parametrize("L,S,Ov", [(24, 16, 8), (20, 16, 4), (33, 24, 4)])
def test_n_samples_equal_one_sample_calls(L, S, Ov):
    """Tiling and non-tiling lengths (reflected tail windows): each sample of a 3-sample denoise + decode equals the
    one-sample run with its generator, bit for bit; every window is one forward of all 3 samples."""
    seen = []
    lat, video, eng, vae = _run(L, S, Ov, SEEDS, callback=lambda i, t, x: seen.append(tuple(x.shape)))
    assert lat.shape == (3, 4, L, 4, 4) and video.shape == (3, 3, L, 32, 32)
    assert seen == [(3, 4, L, 4, 4)] * 3
    assert eng.calls and all(c[:2] == (2, 3) for c in eng.calls)
    for i, s in enumerate(SEEDS):
        lat1, video1, eng1, vae1 = _run(L, S, Ov, [s])
        assert video1.shape == (3, L, 32, 32)
        assert torch.equal(lat[i], lat1[0]), i
        assert torch.equal(video[i], video1), i
        assert len(eng1.calls) == len(eng.calls) and all(c[:2] == (2, 1) for c in eng1.calls)
        assert vae.chunks == vae1.chunks * 3                       # every sample decodes in the one-sample chunks
    assert not torch.equal(lat[0], lat[1])


def _gloo_worker(rank, world, port, L, S, Ov, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lat, video, _, _ = _run(L, S, Ov, SEEDS, distributed=True, chunk_term=0.0)
    if rank == 0:
        ret.put((lat.float().numpy(), video.numpy()))
    else:
        assert video is None
    dist.destroy_process_group()


@pytest.mark.parametrize("L,S,Ov", [(40, 16, 8), (20, 16, 4)])
def test_n_samples_sharded_over_two_ranks_equal_one_rank(L, S, Ov):
    """denoise(distributed=True) with 3 samples under gloo: the all-reduce covers acc (n, 4, L, hw), the decode is sharded
    by (sample, frame) and gathered on rank 0 -- bit-identical to one rank.  (A rank decodes its frames in other chunks
    than one rank would -- the real VAE's GroupNorm then differs in the last bits, tests/test_multigpu_gpu.py -- so the
    fake decode here does not depend on the chunk: what is checked is that every (sample, frame) lands in its place.)"""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + ((os.getpid() * 11 + L) % 2000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, L, S, Ov, ret)) for r in range(2)]
    for p in procs:
        p.start()
    got_lat, got_vid = (torch.from_numpy(t) for t in ret.get(timeout=120))
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    lat, video, _, _ = _run(L, S, Ov, SEEDS, chunk_term=0.0)
    assert got_vid.shape == video.shape == (3, 3, L, 32, 32)
    assert torch.equal(got_lat, lat.float()) and torch.equal(got_vid, video)


def _randn_tensor(shape, generator, dtype):
    """diffusers.utils.torch_utils.randn_tensor on the host, restated: a list draws sample i as (1, ...) from generator[i]."""
    if isinstance(generator, list):
        shape = (1,) + tuple(shape[1:])
        return torch.cat([torch.randn(shape, generator=g, device="cpu", dtype=dtype) for g in generator], dim=0)
    return torch.randn(shape, generator=generator, device="cpu", dtype=dtype)


def test_prepare_latents_matches_randn_tensor():
    from vexpress_b200.pipelines.scheduler import DDIMScheduler
    from vexpress_b200.pipelines.v_express_pipeline import VExpressPipeline
    pipe = VExpressPipeline(vae=None, reference_net=None, denoising_unet=None, v_kps_guider=None, audio_processor=None,
                            audio_encoder=None, audio_projection=None, scheduler=DDIMScheduler())
    shape = (3, 4, 6, 8, 8)
    gens = lambda: [torch.Generator().manual_seed(s) for s in SEEDS]
    got = pipe.prepare_latents(3, 4, 64, 64, 6, torch.bfloat16, torch.device("cpu"), gens())
    assert got.dtype == torch.bfloat16 and torch.equal(got, _randn_tensor(shape, gens(), torch.bfloat16))
    for i, s in enumerate(SEEDS):                             # sample i == a one-sample draw from generator i
        one = pipe.prepare_latents(1, 4, 64, 64, 6, torch.bfloat16, None, [torch.Generator().manual_seed(s)])
        assert torch.equal(got[i:i + 1], one)
        assert torch.equal(one, pipe.prepare_latents(1, 4, 64, 64, 6, torch.bfloat16, None, torch.Generator().manual_seed(s)))
    single = pipe.prepare_latents(3, 4, 64, 64, 6, torch.float32, None, torch.Generator().manual_seed(5))
    assert torch.equal(single, _randn_tensor(shape, torch.Generator().manual_seed(5), torch.float32))
    torch.manual_seed(3)
    unseeded = pipe.prepare_latents(3, 4, 64, 64, 6, torch.float32, None, None)
    torch.manual_seed(3)
    assert torch.equal(unseeded, _randn_tensor(shape, None, torch.float32))


def test_bad_sample_counts_raise():
    from vexpress_b200.pipelines.scheduler import DDIMScheduler
    from vexpress_b200.pipelines.v_express_pipeline import VExpressPipeline
    pipe = VExpressPipeline(vae=None, reference_net=None, denoising_unet=None, v_kps_guider=None, audio_processor=None,
                            audio_encoder=None, audio_projection=None, scheduler=DDIMScheduler())
    with pytest.raises(ValueError, match="list of generators of length 2"):
        pipe.prepare_latents(3, 4, 64, 64, 6, torch.bfloat16, None, [torch.Generator(), torch.Generator()])
    with pytest.raises(ValueError, match="list of generators of length 1"):
        pipe.prepare_latents(2, 4, 64, 64, 6, torch.bfloat16, None, [torch.Generator()])
    for bad in (0, -1, 1.5):
        with pytest.raises(ValueError, match="num_images_per_prompt"):
            pipe(None, None, None, 64, 64, 6, 2, 3.5, num_images_per_prompt=bad)
