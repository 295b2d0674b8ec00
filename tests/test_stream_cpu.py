"""Streaming (``VExpressPipeline.stream`` / ``denoise_stream``) on the host side, without a GPU: the wavefront schedule's
integer properties, and the streamed frames and final latents against ``denoise`` + ``decode_to_device`` bit for bit,
with the UNet replaced by the cheap deterministic function and the elementwise kernels by the torch emulations of
tests/test_samples_cpu.py (plus ``ddim_step_frames`` and the range median)."""
import os

import pytest
import torch
import torch.nn.functional as F

from test_samples_cpu import _ElementwiseEmu, _FakeEngine, _fake_pipeline, _rb

# (L, context, overlap): tiling, non-tiling (reflected tail window), overlap >= stride (R = 2), L <= context
CASES = [(24, 8, 4), (20, 16, 4), (33, 24, 4), (26, 8, 5), (6, 8, 4)]


class _StreamEmu(_ElementwiseEmu):
    @staticmethod
    def ddim_step_frames(lat, acc, frames, sa, sb, sap, sbp):
        """vx_ddim_step_frames: vx_ddim_step on the listed frames, their acc entries zeroed."""
        idx = frames.long()
        a = acc.view(lat.shape[0], 4, lat.shape[2], -1)
        x, v = lat[:, :, idx].float().reshape(a[:, :, idx].shape), _rb(a[:, :, idx])
        x0 = _rb(_rb(sa * x) - _rb(sb * v))
        eps = _rb(_rb(sa * v) + _rb(sb * x))
        lat[:, :, idx] = (_rb(sap * x0) + _rb(sbp * eps)).bfloat16().view(lat[:, :, idx].shape)
        a[:, :, idx] = 0

    @staticmethod
    def median3d_range_u8(buf, buf_start, own_start, own_count, video_length, out=None):
        res = _median_u8(buf, buf_start, own_start, own_count, video_length)
        if out is not None:
            out.copy_(res)
        return res


def _median_u8(buf, buf_start, own_start, own_count, T):
    """The reference's 3x3x3 reflect-padded median + (v * 255).astype(uint8) on frames [own_start, +own_count) of a
    T-frame video held from buf_start in buf (C,k,H,W)."""
    refl = lambda i: -i if i < 0 else (2 * (T - 1) - i if i >= T else i)
    out = []
    for t in range(own_start, own_start + own_count):
        x = buf[:, [refl(t + d) - buf_start for d in (-1, 0, 1)]]             # (C,3,H,W)
        xp = F.pad(x, (1, 1, 1, 1), mode="reflect")
        nb = xp.unfold(2, 3, 1).unfold(3, 3, 1)                               # (C,3,H,W,3,3)
        m = nb.permute(0, 2, 3, 1, 4, 5).reshape(*nb.shape[:1], *nb.shape[2:4], 27).median(-1).values
        out.append((m * 255).to(torch.uint8).permute(1, 2, 0))
    return torch.stack(out)


class _LoggingEngine(_FakeEngine):
    """Records (window frames, timestep) of every forward: the cond block of sample 0 carries the frame index in its
    first audio token."""

    def forward_frames(self, frames, timestep, enc, kps, kps_idx, b, f, temb=None, taps=None, n=1):
        row0 = (b - 1) * n * f
        self.log.append((tuple(int(enc[row0 + i, 0, 0]) for i in range(f)), float(temb.reshape(-1)[0])))
        return super().forward_frames(frames, timestep, enc, kps, kps_idx, b, f, temb, taps, n)


def _conditioning(L, h=4, C0=8):
    g = torch.Generator().manual_seed(1000 + L)
    kps = torch.cat([torch.zeros(1, C0, L, h, h), 0.1 * torch.randn(1, C0, L, h, h, generator=g)]).bfloat16()
    audio = torch.cat([torch.zeros(1, L, 5, 16), torch.randn(1, L, 5, 16, generator=g)])
    audio[1, :, 0, 0] = torch.arange(L, dtype=torch.float32)
    return kps, audio.bfloat16()


def _pipe(kps):
    from vexpress_b200.pipelines import v_express_pipeline as vp
    pipe, vp, _ = _fake_pipeline()
    eng = _LoggingEngine()
    eng.log = []
    pipe.denoising_unet.engine = lambda: eng
    vp.ops = _StreamEmu()
    live = {"requests": []}

    def frames(kps_images, start, stop, height, width):
        assert (height, width) == (kps.shape[-2] * 8, kps.shape[-1] * 8)
        live["requests"].append((start, stop))
        return kps[1:, :, start:stop]
    pipe.prepare_kps_feature_frames = frames
    return pipe, vp, eng, live


def _run_both(L, S, Ov, seeds, steps, output="float"):
    from vexpress_b200 import ops as real_ops
    from vexpress_b200.pipelines.v_express_pipeline import retrieve_timesteps
    kps, audio = _conditioning(L)
    pipe, vp, eng, live = _pipe(kps)
    try:
        ts, _ = retrieve_timesteps(pipe.scheduler, steps, None)
        draw = lambda: pipe.prepare_latents(len(seeds), 4, 32, 32, L, torch.bfloat16, torch.device("cpu"),
                                            [torch.Generator().manual_seed(s) for s in seeds])
        lat_ref = pipe.denoise(draw(), kps, audio, ts, 3.5, S, Ov)
        video_ref = pipe.decode_to_device(lat_ref, False)
        if video_ref.dim() == 4:
            video_ref = video_ref.unsqueeze(0)
        eng.log.clear()
        lat = draw()
        chunks = list(pipe.denoise_stream(lat, None, audio, ts, 3.5, S, Ov, output=output))
        ring = [g.kps for g in pipe._graphs.values()]
        return dict(lat_ref=lat_ref, video_ref=video_ref, lat=lat, chunks=chunks, log=list(eng.log),
                    ts=[float(t) for t in ts], ring=ring, pipe=pipe, live=live)
    finally:
        vp.ops = real_ops


def _windows(L, S, Ov):
    from vexpress_b200.pipelines.context import window_table
    return window_table(L, S, Ov)[0]


@pytest.mark.parametrize("L,S,Ov", CASES)
@pytest.mark.parametrize("n,steps", [(1, 1), (1, 3), (2, 5), (2, 3)])
def test_stream_equals_denoise_and_decode(L, S, Ov, n, steps):
    r = _run_both(L, S, Ov, [11, 22][:n], steps)
    chunks, vc = r["chunks"], r["pipe"].vae_chunk
    assert [c.start for c in chunks] == list(range(0, L, vc))                 # frame order, multiples of vae_chunk
    assert all(c.frames.shape == (n, 3, min(vc, L - c.start), 32, 32) for c in chunks)
    video = torch.cat([c.frames for c in chunks], 2)
    assert video.shape == r["video_ref"].shape
    assert torch.equal(video, r["video_ref"])
    assert torch.equal(r["lat"], r["lat_ref"])
    # every (window, step) forward exactly once, each after the forwards it depends on
    windows = _windows(L, S, Ov)
    items = [(windows.index(list(fr)), r["ts"].index(t)) for fr, t in r["log"]]
    assert len(items) == len(set(items)) == steps * len(windows)
    assert sorted(items) == sorted((w, t) for w in range(len(windows)) for t in range(steps))
    done = set()
    for w, t in items:
        if t > 0:
            assert all((u, t - 1) in done for u in range(len(windows)) if set(windows[u]) & set(windows[w])), (w, t)
        done.add((w, t))


@pytest.mark.parametrize("L,S,Ov", [(20, 16, 4), (33, 24, 4), (26, 8, 5), (6, 8, 4)])
def test_stream_uint8_equals_median_of_whole_video(L, S, Ov):
    r = _run_both(L, S, Ov, [11, 22], 3, output="uint8")
    chunks, vc = r["chunks"], r["pipe"].vae_chunk
    assert [c.start for c in chunks] == list(range(0, L, vc))
    frames = torch.cat([c.frames for c in chunks], 1)
    assert frames.dtype == torch.uint8 and frames.shape == (2, L, 32, 32, 3)
    for s in range(2):
        assert torch.equal(frames[s], _median_u8(r["video_ref"][s], 0, 0, L, L)), s


def _max_live(sched):
    live = peak = 0
    for ld, rel in zip(sched.loads, sched.releases):
        live += len(ld)
        peak = max(peak, live)
        live -= len(rel)
    return peak


@pytest.mark.parametrize("L,S,Ov", [(130, 24, 4), (40, 8, 5), (40, 8, 4)])
@pytest.mark.parametrize("steps", [1, 3, 5])
def test_kps_ring_is_bounded_and_flat_in_length(L, S, Ov, steps):
    """The kps ring holds at most the frames of the R (T - 1) + 1 windows in flight (plus the zero frame), the same
    number for a video 4x longer; every frame's features are requested once.  L has more windows than are ever in
    flight."""
    from vexpress_b200.pipelines.context import wavefront_schedule
    rings = []
    for length in (L, 4 * L):
        r = _run_both(length, S, Ov, [11], steps)
        windows = _windows(length, S, Ov)
        sched = wavefront_schedule(windows, steps, length, 4)
        assert len(r["ring"]) == 1
        frames = r["ring"][0].shape[0] // 16 - 1
        assert frames == _max_live(sched) <= (sched.reach * (steps - 1) + 1) * S
        asked = sorted(f for a, e in r["live"]["requests"] for f in range(a, e))
        assert asked == list(range(length))
        rings.append(frames)
    assert rings[0] == rings[1]


@pytest.mark.parametrize("L,S,Ov,R", [(24, 8, 4, 1), (20, 16, 4, 1), (33, 24, 4, 1), (26, 8, 5, 2), (6, 8, 4, 0),
                                      (40, 8, 6, 3)])
@pytest.mark.parametrize("T", [1, 3, 5])
def test_wavefront_schedule(L, S, Ov, R, T):
    from vexpress_b200.pipelines.context import wavefront_schedule
    windows = _windows(L, S, Ov)
    W = len(windows)
    sched = wavefront_schedule(windows, T, L, 4)
    assert sched.reach == R
    assert sorted(sched.order) == sorted((w, t) for w in range(W) for t in range(T))
    pos = {it: i for i, it in enumerate(sched.order)}
    last = [max(w for w in range(W) if fr in windows[w]) for fr in range(L)]
    for (w, t), i in pos.items():
        for u in range(W):
            if set(windows[u]) & set(windows[w]):
                if t > 0:
                    assert pos[(u, t - 1)] < i                         # neighbours' previous step first
                assert (pos[(u, t)] < i) == (u < w)                      # within a step: window order
        # frames are stepped after their last window of the step, and before any window reads them at the next step
        assert sched.finalised[i] == sorted(fr for fr in set(windows[w]) if last[fr] == w)
    step_at = {}
    for i, fins in enumerate(sched.finalised):
        for fr in fins:
            step_at[(fr, sched.order[i][1])] = i
    assert len(step_at) == L * T
    for (w, t), i in pos.items():
        for fr in set(windows[w]):
            if t > 0:
                assert step_at[(fr, t - 1)] < i
            assert step_at[(fr, t)] >= i
    # chunks: in frame order, each once, only after all its frames got their last step
    emitted = [(i, c) for i, cs in enumerate(sched.chunks) for c in cs]
    assert [c for _, c in emitted] == [(a, min(a + 4, L)) for a in range(0, L, 4)]
    for i, (a, e) in emitted:
        assert all(step_at[(fr, T - 1)] <= i for fr in range(a, e))
    # kps lifetimes: loaded at the first read, released after the last
    for fr in range(L):
        reads = [pos[(w, t)] for w in range(W) if fr in windows[w] for t in range(T)]
        assert fr in sched.loads[min(reads)] and fr in sched.releases[max(reads)]
    assert sorted(f for fs in sched.loads for f in fs) == list(range(L)) == sorted(f for fs in sched.releases for f in fs)


def test_stream_rejects_eta_and_bad_output():
    pipe, _, _, _ = _pipe(_conditioning(8)[0])
    with pytest.raises(ValueError, match="eta"):
        next(pipe.stream(None, None, None, 32, 32, 8, 2, 3.5, eta=0.5))
    with pytest.raises(ValueError, match="num_images_per_prompt"):
        pipe.stream(None, None, None, 32, 32, 8, 2, 3.5, num_images_per_prompt=0)
    with pytest.raises(ValueError, match="output"):
        pipe.stream(None, None, None, 32, 32, 8, 2, 3.5, output="png")


def _gloo_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        pipe, _, _, _ = _pipe(_conditioning(8)[0])
        try:
            pipe.stream(None, None, None, 32, 32, 8, 2, 3.5)
            ret.put((rank, "no error"))
        except ValueError as e:
            ret.put((rank, str(e)))
    finally:
        dist.destroy_process_group()


def test_stream_rejects_world_size_above_one():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + ((os.getpid() * 13 + 7) % 2000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(ret.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert all("one GPU" in got[r] for r in range(2)), got
