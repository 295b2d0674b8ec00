"""Streaming on the H100 kernels: ``VExpressPipeline.stream`` equals ``__call__`` bit for bit on the reduced-width
pipeline (eager and graphed, one and two samples, tiling and non-tiling lengths of four windows), its uint8 output equals
the median filter of the whole video, the two kernels it adds equal their whole-video forms, and its peak device memory
does not grow with the video beyond the resident per-frame state."""
import numpy as np
import pytest
import torch

from test_samples_gpu import _public_pipeline

pytestmark = pytest.mark.gpu

STEPS, S, OV = 2, 16, 4


def _args(L, n=1, generator=None):
    return dict(reference_image=None, kps_images=None, audio_waveform=None, width=128, height=128, video_length=L,
                num_inference_steps=STEPS, guidance_scale=3.5, num_images_per_prompt=n, generator=generator,
                context_frames=S, context_overlap=OV, reference_attention_weight=0.95, audio_attention_weight=3.0)


def _streaming_pipeline(L):
    """The reduced-width public pipeline; its kps hook for ``stream`` slices the features ``prepare_kps_feature``
    returns for ``__call__``."""
    pipe = _public_pipeline(L)
    kps = pipe.prepare_kps_feature(None, 128, 128, True)
    assert torch.count_nonzero(kps[0]) == 0                  # the CFG zero half every uncond row of the ring reads
    pipe.prepare_kps_feature_frames = lambda images, a, e, height, width: kps[1:, :, a:e]
    return pipe


def _gens(seeds):
    return [torch.Generator().manual_seed(s) for s in seeds]


@pytest.mark.parametrize("L", [52, 50])                       # 4 windows of 16 / overlap 4: tiling, reflected tail
@pytest.mark.parametrize("use_graph", [False, True])
def test_stream_float_equals_call(L, use_graph):
    pipe = _streaming_pipeline(L)
    pipe.use_cuda_graph = use_graph
    ref = pipe(**_args(L, 1, _gens([5])))
    chunks = list(pipe.stream(**_args(L, 1, _gens([5]))))
    assert [c.start for c in chunks] == list(range(0, L, pipe.vae_chunk))
    assert all(c.frames.is_pinned() and c.frames.dtype == torch.float32 for c in chunks)
    video = torch.cat([c.frames for c in chunks], 2)
    assert video.shape == ref.shape == (1, 3, L, 128, 128)
    print(f"L={L} graph={use_graph}: max |stream - call| = {(video - ref).abs().max().item()}")
    assert torch.equal(video, ref)
    # a second stream on the same pipeline (ring and graph reused) gives the same frames
    assert torch.equal(torch.cat([c.frames for c in pipe.stream(**_args(L, 1, _gens([5])))], 2), ref)


@pytest.mark.parametrize("L", [52, 50])
def test_stream_two_samples_and_uint8(L):
    """n = 2 with a list of generators (graphed): float frames equal ``__call__``; uint8 frames equal ``median3d_u8`` of
    each sample of the ``__call__`` video."""
    from vexpress_b200 import ops
    pipe = _streaming_pipeline(L)
    ref = pipe(**_args(L, 2, _gens([5, 6])))
    video = torch.cat([c.frames for c in pipe.stream(**_args(L, 2, _gens([5, 6])))], 2)
    assert video.shape == ref.shape == (2, 3, L, 128, 128) and torch.equal(video, ref)
    chunks = list(pipe.stream(**_args(L, 2, _gens([5, 6])), output="uint8"))
    assert [c.start for c in chunks] == list(range(0, L, pipe.vae_chunk))
    frames = torch.cat([c.frames for c in chunks], 1)
    assert frames.dtype == torch.uint8 and frames.shape == (2, L, 128, 128, 3)
    for s in range(2):
        assert torch.equal(frames[s], ops.median3d_u8(ref[s].cuda().contiguous()).cpu()), s


def test_ddim_step_frames_equals_ddim_step():
    from vexpress_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    n, L, h = 2, 23, 12
    lat = torch.randn(n, 4, L, h, h, device="cuda", generator=g).bfloat16()
    acc = torch.randn(n, 4, L, h * h, device="cuda", generator=g).bfloat16().float()
    coeffs = (0.8, 0.6, 0.9, 0.43588989)
    full_lat = lat.clone()
    ops.ddim_step(full_lat, acc, *coeffs)
    chosen = [0, 3, 4, 11, L - 1]
    got_lat, got_acc = lat.clone(), acc.clone()
    ops.ddim_step_frames(got_lat, got_acc, torch.tensor(chosen, device="cuda", dtype=torch.int32), *coeffs)
    torch.cuda.synchronize()
    others = [i for i in range(L) if i not in chosen]
    assert torch.equal(got_lat[:, :, chosen], full_lat[:, :, chosen])
    assert torch.equal(got_lat[:, :, others], lat[:, :, others])
    assert torch.count_nonzero(got_acc[:, :, chosen]) == 0
    assert torch.equal(got_acc[:, :, others], acc[:, :, others])


@pytest.mark.parametrize("T,runs", [(37, [(0, 16), (16, 32), (32, 37), (5, 6), (36, 37)]), (2, [(0, 1), (1, 2), (0, 2)])])
def test_median_range_equals_whole_video(T, runs):
    """Chunks at the start, in the middle and at the end, each from a buffer of its frames plus one halo frame on each
    side that exists: the uint8 frames of ``median3d_u8`` on the whole video, bit for bit."""
    from vexpress_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(T)
    video = torch.rand(3, T, 24, 20, device="cuda", generator=g)
    video[:, :, :3] = 0.5                                   # ties
    full = ops.median3d_u8(video)
    for a, e in runs:
        lo, hi = max(a - 1, 0), min(e + 1, T)
        got = ops.median3d_range_u8(video[:, lo:hi].contiguous(), lo, a, e - a, T)
        assert torch.equal(got, full[a:e]), (a, e)
    with pytest.raises(Exception, match="must cover"):
        ops.median3d_range_u8(video[:, 1:3].contiguous(), 1, 1, 1, T) if T > 2 else \
            ops.median3d_range_u8(video[:, 1:2].contiguous(), 1, 1, 1, T)


def test_prepare_kps_feature_frames_equals_slices():
    """The default hook on the reduced VKpsGuider, for a (1,3,L,H,W) tensor and for a list of uint8 images: slices of
    ``prepare_kps_feature``'s conditional half, bit for bit, across 16-frame chunk boundaries."""
    from oracle import vx_oracle as O
    from vexpress_b200.modules.prologue import VKpsGuider
    from vexpress_b200.pipelines.scheduler import DDIMScheduler
    from vexpress_b200.pipelines.v_express_pipeline import VExpressPipeline
    m = VKpsGuider(320, block_out_channels=(16, 32, 96, 256))
    m.load_state_dict(O.synth_state_dict(O.kps_guider_param_shapes(O.KPS_CFG), 77))
    m = m.to(device="cuda", dtype=torch.bfloat16)
    unet = type("U", (), {"device": torch.device("cuda"), "dtype": torch.bfloat16})()
    pipe = VExpressPipeline(vae=None, reference_net=None, denoising_unet=unet, v_kps_guider=m, audio_processor=None,
                            audio_encoder=None, audio_projection=None, scheduler=DDIMScheduler())
    L = 40
    imgs = torch.rand(1, 3, L, 64, 64, generator=torch.Generator().manual_seed(4))
    as_list = [np.ascontiguousarray((imgs[0, :, i].permute(1, 2, 0) * 255).to(torch.uint8).numpy()) for i in range(L)]
    for images in (imgs, as_list):
        whole = pipe.prepare_kps_feature(images, 64, 64, True)
        assert whole.shape == (2, 320, L, 8, 8)
        for a, e in [(0, 5), (13, 35), (16, 32), (30, 40), (39, 40)]:
            got = pipe.prepare_kps_feature_frames(images, a, e, 64, 64)
            assert got.shape == (1, 320, e - a, 8, 8) and torch.equal(got, whole[1:, :, a:e]), (a, e)


def _peak_growth(run):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    run()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_stream_peak_memory_flat_in_length():
    """Peak device memory of ``stream`` from L to 3L grows by no more than the resident per-frame state (latents bf16,
    acc fp32, audio tokens of both CFG halves, count) x 2L plus a fixed slack, while ``__call__`` grows by the whole
    video's kps features and decoded frames.  One pipeline serves every length (conditioning sliced from a 3L clip)."""
    from oracle import vx_oracle as O
    L1, L3 = 48, 144
    pipe = _public_pipeline(L3)
    pipe.use_cuda_graph = False
    kps, audio = pipe.prepare_kps_feature(None, 128, 128, True), pipe.prepare_audio_embeddings(None, L3, 2, True)
    cur = {}
    pipe.prepare_kps_feature = lambda *a, **k: kps[:, :, :cur["L"]]
    pipe.prepare_audio_embeddings = lambda *a, **k: audio[:, :cur["L"]]
    pipe.prepare_kps_feature_frames = lambda images, a, e, height, width: kps[1:, :, a:e]
    runs = {"stream": lambda L: [None for _ in pipe.stream(**_args(L, 1, _gens([5])))],
            "call": lambda L: pipe(**_args(L, 1, _gens([5])))}
    growth = {}
    for name, run in runs.items():
        peaks = []
        for L in (L1, L1, L3):                              # the first run allocates what later runs reuse
            cur["L"] = L
            peaks.append(_peak_growth(lambda: run(L)))
        growth[name] = peaks[2] - peaks[1]
    hw, T, cad = 16 * 16, 5, O.small_cfg()["cross_attention_dim"]
    per_frame = 4 * hw * (2 + 4) + 2 * T * cad * 2 + 4
    slack = 4 << 20
    bound = per_frame * 2 * L1 + slack
    print(f"peak growth L={L1}->{L3}: stream {growth['stream']} B, __call__ {growth['call']} B; bound {bound} B")
    assert 0 <= growth["stream"] <= bound
    assert 2 * bound < growth["call"]
