"""Stochastic DDIM (eta > 0) on the host side, without a GPU: the eta scalar tables, the variance-noise draws in the
reference's order (context.step_frame_ids, diffusers' randn_tensor semantics, last write wins on repeated frames) and the
denoise loop with the UNet replaced by a cheap deterministic function and the elementwise kernels by torch emulations with
the kernels' rounding points (the harness of tests/test_samples_cpu.py), against the oracle's restatement of the
reference loop and the noise the reference pipeline itself drew (tests/golden/pipeline_eta*_small.pt)."""
import math
import os

import numpy as np
import pytest
import torch

from test_host_cpu import _fake_unet_fn
from test_samples_cpu import _ElementwiseEmu, _draw, _fake_conditioning, _fake_pipeline


def _rb(t):
    return t.bfloat16().float()


class _EtaEmu(_ElementwiseEmu):
    """+ vx_ddim_step_eta (csrc/vx_misc.cu) with its rounding points."""

    @staticmethod
    def ddim_step_eta(lat, acc, noise, sa, sb, sap, c_dir, sigma):
        assert noise.dtype == torch.float32 and noise.shape == acc.shape
        x, v = lat.float().view(acc.shape), _rb(acc)
        x0 = _rb(_rb(sa * x) - _rb(sb * v))
        eps = _rb(_rb(sa * v) + _rb(sb * x))
        prev = _rb(_rb(sap * x0) + _rb(c_dir * eps))
        lat.copy_((prev + _rb(sigma * noise)).bfloat16().view(lat.shape))


def _shim():
    import sys
    from oracle import vx_oracle as O
    p = os.path.join(os.path.dirname(os.path.abspath(O.__file__)), "diffusers_shim")
    if p not in sys.path:
        sys.path.insert(0, p)
    import diffusers
    return diffusers


def _lib_scheduler():
    return _shim().DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                                 steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                                 timestep_spacing="trailing")


# ---------------------------------------------------------------------------------------------------------- tables
@pytest.mark.parametrize("steps", [3, 25])
@pytest.mark.parametrize("eta", [0.3, 1.0])
def test_eta_tables_against_closed_form_and_library_scalars(steps, eta):
    """sigma and c_dir at every step: within fp32 rounding of the float64 closed form on the same a_t / a_prev, and bit
    for bit the scalars of the library-structured scheduler's ``step`` (the 0-d fp32 tensor arithmetic of diffusers).
    The one exception is eta = 1 at t = 999 of 25 steps, where a_t = 0 and the library's radicand 1 - a_prev - sigma^2
    rounds to -1 ulp: its ``** 0.5`` is NaN (and so is every latent after that step), the product's c_dir the exact 0."""
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, ddim_coefficients_eta
    prod, lib = DDIMScheduler(), _lib_scheduler()
    prod.set_timesteps(steps)
    lib.set_timesteps(steps)
    nan_steps = 0
    for t in prod.timesteps.tolist():
        sa, sb, sap, c_dir, sigma = ddim_coefficients_eta(prod, t, eta)
        prev = t - 1000 // steps
        a_t = lib.alphas_cumprod[t]
        a_p = lib.alphas_cumprod[prev] if prev >= 0 else lib.final_alpha_cumprod
        # float64 closed forms on the fp32 table entries
        a, ap = float(a_t), float(a_p)
        var64 = (1 - ap) / (1 - a) * (1 - a / ap)
        sig64 = eta * math.sqrt(var64)
        u = 2.0 ** -23
        assert abs(sigma - sig64) <= 4 * u * max(sig64, 1e-30), (t, sigma, sig64)
        # c_dir is the root of a difference that cancels to 0 at a_t = 0, eta = 1: compare its square
        assert abs(c_dir ** 2 - (1 - ap - sig64 ** 2)) <= 8 * u, (t, c_dir, 1 - ap - sig64 ** 2)
        assert (sa, sb, sap) == (float(a_t ** 0.5), float((1 - a_t) ** 0.5), float(a_p ** 0.5))
        # the library's own scalars (schedulers/scheduling_ddim.py step, 0.29.2)
        std = eta * lib._get_variance(t, prev) ** 0.5
        lib_c_dir = (1 - a_p - std ** 2) ** 0.5
        assert np.float32(sigma).tobytes() == np.float32(float(std)).tobytes(), t
        if torch.isnan(lib_c_dir):
            nan_steps += 1
            assert (steps, eta, t) == (25, 1.0, 999) and c_dir == 0.0
        else:
            assert np.float32(c_dir).tobytes() == np.float32(float(lib_c_dir)).tobytes(), t
    assert nan_steps == (1 if (steps, eta) == (25, 1.0) else 0)


@pytest.mark.parametrize("steps", [2, 3, 25, 50])
def test_eta_zero_tables_equal_deterministic_tables(steps):
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, ddim_coefficients, ddim_coefficients_eta
    s = DDIMScheduler()
    s.set_timesteps(steps)
    for t in s.timesteps.tolist():
        sa, sb, sap, sbp = ddim_coefficients(s, t)
        assert ddim_coefficients_eta(s, t, 0.0) == (sa, sb, sap, sbp, 0.0)


@pytest.mark.parametrize("bad", [-0.1, 1.0001, 2.0, float("nan"), float("inf"), "0.5x", None])
def test_out_of_range_eta_raises(bad):
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, ddim_coefficients_eta
    pipe, _, _ = _fake_pipeline()
    from vexpress_b200 import ops as real_ops
    from vexpress_b200.pipelines import v_express_pipeline as vp
    vp.ops = real_ops
    with pytest.raises(ValueError, match="eta"):
        pipe(None, None, None, 32, 32, 8, 2, 3.5, eta=bad)
    if isinstance(bad, float):
        s = DDIMScheduler()
        s.set_timesteps(3)
        with pytest.raises(ValueError, match="eta"):
            ddim_coefficients_eta(s, 999, bad)


# ----------------------------------------------------------------------------------------------- step_frame_ids
@pytest.mark.parametrize("L,S,Ov", [(12, 8, 4), (20, 16, 4), (33, 24, 4), (40, 16, 8), (96, 16, 8), (7, 16, 4)])
def test_step_frame_ids_follow_the_overlap_replay(L, S, Ov):
    """Every frame is stepped in exactly one window (its last), once per occurrence there (so reflected windows repeat
    frames), and the slots of its last occurrence's sum are the ones the overlap plan keeps."""
    from vexpress_b200.pipelines.context import overlap_plan, step_frame_ids, window_table
    windows, count = window_table(L, S, Ov)
    steps, plan = step_frame_ids(windows, count), overlap_plan(windows, count)
    assert sorted(set(f for ids in steps for f in ids)) == list(range(L))
    for wi, ids in enumerate(steps):
        for f in set(ids):
            assert max(w for w, win in enumerate(windows) if f in win) == wi
            assert ids.count(f) == windows[wi].count(f)
            last = max(li for li, fr in enumerate(windows[wi]) if fr == f)
            assert any(r[last] == f for r in plan[wi])
    if (L, S, Ov) == (20, 16, 4):
        assert any(len(ids) != len(set(ids)) for ids in steps)


# ------------------------------------------------------------------------------------------- harness + oracle
def _run(L, S, Ov, seeds, noise_gen, eta, steps=3, distributed=False, dtype=torch.bfloat16, chunk_term=1.0):
    """-> (final latents (n,4,L,h,w), decoded video) of one host-side denoise + decode at eta."""
    from vexpress_b200 import ops as real_ops
    from vexpress_b200.pipelines.v_express_pipeline import retrieve_timesteps
    pipe, vp, eng = _fake_pipeline(chunk_term)
    pipe.denoising_unet.dtype = dtype
    vp.ops = _EtaEmu()
    try:
        kps, audio = _fake_conditioning(L)
        ts, _ = retrieve_timesteps(pipe.scheduler, steps, None)
        lat = pipe.denoise(_draw(pipe, seeds, L), kps, audio, ts, 3.5, S, Ov, distributed=distributed, eta=eta,
                           generator=noise_gen)
        return lat, pipe.decode_to_device(lat, distributed)
    finally:
        vp.ops = real_ops


def _randn_tensor(shape, generator, device, dtype):
    """diffusers 0.29.2 ``randn_tensor``, restated: a CPU generator draws on the host, a list draws sample i as (1, ...)
    from generator[i] (a list of one is the generator), None draws on ``device``; the result moves to ``device``."""
    device = torch.device(device)
    rand_device = device
    if generator is not None:
        gtype = (generator[0] if isinstance(generator, list) else generator).device.type
        if gtype != device.type:
            assert gtype == "cpu", gtype
            rand_device = torch.device("cpu")
    if isinstance(generator, list) and len(generator) == 1:
        generator = generator[0]
    if isinstance(generator, list):
        one = (1,) + tuple(shape[1:])
        return torch.cat([torch.randn(one, generator=g, device=rand_device, dtype=dtype) for g in generator]).to(device)
    return torch.randn(tuple(shape), generator=generator, device=rand_device, dtype=dtype).to(device)


def _oracle(L, S, Ov, seeds, noise_gen, eta, steps, monkeypatch):
    """The oracle's restatement of the reference loop (``O.denoise``) with the step of diffusers 0.29.2 at ``eta`` with
    ``generator`` -- what the reference's ``extra_step_kwargs`` hand to every step call -- and the step's rounding on
    the device the reference runs on (CUDA: fp32 scalars times bf16 tensors rounded once to bf16; CPU eager would round
    the scalar first)."""
    from oracle import vx_oracle as O
    pipe, _, _ = _fake_pipeline()
    lat = _draw(pipe, seeds, L)
    kps, audio = _fake_conditioning(L)

    def step_cuda_semantics(self, model_output, timestep, sample, **_):
        a_t, a_prev = self.coeffs(int(timestep))
        x, v = sample.float(), model_output.float()
        std = eta * ((1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev)) ** 0.5          # _get_variance, fp32 0-d
        sa, sb, sap = float(a_t ** 0.5), float((1 - a_t) ** 0.5), float(a_prev ** 0.5)
        cd, sg = float((1 - a_prev - std ** 2) ** 0.5), float(std)
        x0 = _rb(_rb(sa * x) - _rb(sb * v))
        eps = _rb(_rb(sa * v) + _rb(sb * x))
        prev = _rb(_rb(sap * x0) + _rb(cd * eps))
        noise = _randn_tensor(model_output.shape, noise_gen, model_output.device, model_output.dtype)
        return O._StepOut((prev + _rb(sg * noise.float())).bfloat16())

    def unet_fn(x, t, aud, kps):
        """n samples share the conditioning: the batch [u s0..s(n-1) | c s0..s(n-1)] repeats each CFG half's rows."""
        b = kps.shape[0]
        n = x.shape[0] // b
        aud = aud.view(b, -1, *aud.shape[1:]).repeat_interleave(n, 0).flatten(0, 1)
        return _fake_unet_fn(x, t, aud, kps.repeat_interleave(n, 0))
    monkeypatch.setattr(O.DDIM, "step", step_cuda_semantics)
    return O.denoise(None, None, lat, kps, audio, None, steps, 3.5, S, Ov, unet_fn=unet_fn)


@pytest.mark.parametrize("L,S,Ov,eta,n", [(12, 8, 4, 1.0, 1), (24, 16, 8, 0.5, 1), (20, 16, 4, 0.5, 1),
                                          (33, 24, 4, 0.3, 1), (20, 16, 4, 1.0, 2)])
def test_denoise_at_eta_equals_reference_loop(L, S, Ov, eta, n, monkeypatch):
    """Tiling and non-tiling lengths (reflected tail windows repeat frames): bit-identical to the oracle's reference loop
    drawing through diffusers' randn_tensor from the same seeded generator; n = 2 with one generator draws (2, ...)."""
    seeds = [11, 22][:n]
    out, _ = _run(L, S, Ov, seeds, torch.Generator().manual_seed(77), eta)
    ref = _oracle(L, S, Ov, seeds, torch.Generator().manual_seed(77), eta, 3, monkeypatch)
    assert out.dtype == torch.bfloat16 and ref.dtype == torch.bfloat16
    assert torch.equal(out, ref)
    det, _ = _run(L, S, Ov, seeds, torch.Generator().manual_seed(77), 0.0)
    assert not torch.equal(out, det)


def test_single_generator_draws_whole_batch_per_window(monkeypatch):
    """n = 2 with one generator: every step call draws one (2, 4, k, h, w) tensor in the model dtype, k counting the
    frames the window steps (repeats included), in window order -- diffusers' randn_tensor on a single generator."""
    from vexpress_b200.pipelines import v_express_pipeline as vp
    from vexpress_b200.pipelines.context import step_frame_ids, window_table
    shapes = []
    real = vp._randn

    def rec(shape, generator, device, dtype):
        shapes.append((tuple(shape), dtype, torch.device(device).type))
        return real(shape, generator, device, dtype)
    monkeypatch.setattr(vp, "_randn", rec)
    L, S, Ov = 20, 16, 4
    _run(L, S, Ov, [11, 22], torch.Generator().manual_seed(5), 0.5, steps=2)
    ks = [len(ids) for ids in step_frame_ids(*window_table(L, S, Ov))]
    assert shapes[0] == ((2, 4, L, 4, 4), torch.bfloat16, "cpu")        # prepare_latents: the initial latents
    assert shapes[1:] == [((2, 4, k, 4, 4), torch.bfloat16, "cpu") for k in ks] * 2
    assert sum(ks) > L                                                   # the reflected tail repeats frames


def test_generator_list_sample_equals_one_sample_call():
    """num_images_per_prompt = 3 with a list of generators: sample i (latents and decoded video) equals the one-sample
    call with generator[i], given as a list of one or as the generator itself, with torch.equal."""
    L, S, Ov, eta = 20, 16, 4, 0.7
    seeds, nseeds = [11, 22, 33], [501, 502, 503]
    lat, video = _run(L, S, Ov, seeds, [torch.Generator().manual_seed(s) for s in nseeds], eta)
    assert lat.shape == (3, 4, L, 4, 4) and video.shape == (3, 3, L, 32, 32)
    for i in range(3):
        for gen in ([torch.Generator().manual_seed(nseeds[i])], torch.Generator().manual_seed(nseeds[i])):
            lat1, video1 = _run(L, S, Ov, [seeds[i]], gen, eta)
            assert torch.equal(lat[i], lat1[0]), i
            assert torch.equal(video[i], video1), i
    assert not torch.equal(lat[0], lat[1])


def test_eta_zero_leaves_generator_untouched():
    g = torch.Generator().manual_seed(9)
    state = g.get_state()
    lat0, _ = _run(20, 16, 4, [11], g, 0.0)
    assert torch.equal(g.get_state(), state)
    _run(20, 16, 4, [11], g, 0.5)
    assert not torch.equal(g.get_state(), state)
    # and eta = 0 with a generator is the deterministic loop
    lat1, _ = _run(20, 16, 4, [11], None, 0.0)
    assert torch.equal(lat0, lat1)


def test_mismatched_generator_list_raises():
    with pytest.raises(ValueError, match="list of generators of length 2"):
        _run(12, 8, 4, [11, 22, 33], [torch.Generator(), torch.Generator()], 0.5)


# ---------------------------------------------------------------------------------- golden: the reference's draws
@pytest.mark.parametrize("name", ["pipeline_eta_small.pt", "pipeline_eta_nontiling_small.pt"])
def test_draws_equal_reference_variance_noise(golden_dir, name, monkeypatch):
    """The reference pipeline (fp32, seeded CPU generator, tools/gen_eta_golden.py) recorded the shape, SHA-256 and first
    values of every variance_noise its scheduler drew.  The product, held in fp32 as the golden was, draws the same
    tensors bit for bit in the same order and shapes, and each step's noise buffer holds, per frame, the element of the
    frame's last occurrence (the reference's sequential write-back: the last write wins)."""
    import hashlib
    from vexpress_b200.pipelines import v_express_pipeline as vp
    from vexpress_b200.pipelines.context import step_frame_ids, window_table
    g = torch.load(os.path.join(golden_dir, name), weights_only=False)
    L, S, Ov, steps, h = g["L"], g["S"], g["O"], g["steps"], g["h"]
    windows, count = window_table(L, S, Ov)
    ids = [x for x in step_frame_ids(windows, count) if x]
    assert [tuple(s) for s in g["variance_noise_shapes"]] == [(1, 4, len(x), h, h) for x in ids] * steps
    draws = []
    real = vp._randn

    def rec(shape, generator, device, dtype):
        x = real(shape, generator, device, dtype)
        draws.append(x.clone())
        return x
    monkeypatch.setattr(vp, "_randn", rec)
    noise = vp._StepNoise(windows, count, (1, 4, L, h, h), torch.float32, torch.Generator().manual_seed(g["seed"]),
                          torch.device("cpu"))
    for step in range(steps):
        noise.draw()
        expect = torch.full((1, 4, L, h * h), float("nan"))
        for k, fr_ids in enumerate(ids):
            x = draws[step * len(ids) + k].view(1, 4, len(fr_ids), h * h)
            for j, fr in enumerate(fr_ids):
                expect[:, :, fr] = x[:, :, j]
        assert torch.equal(noise.buf, expect), step
    assert [tuple(x.shape) for x in draws] == [tuple(s) for s in g["variance_noise_shapes"]]
    assert all(x.dtype == torch.float32 for x in draws)
    assert all(torch.equal(x.reshape(-1)[:8], head) for x, head in zip(draws, g["variance_noise_head"]))
    assert [hashlib.sha256(x.contiguous().numpy().tobytes()).hexdigest() for x in draws] == g["variance_noise_sha256"]


# ------------------------------------------------------------------------------------------------- several ranks
def _gloo_worker(rank, world, port, L, S, Ov, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lat, _ = _run(L, S, Ov, [11, 22], torch.Generator().manual_seed(900 + rank), 0.8, distributed=True, chunk_term=0.0)
    if rank == 0:
        ret.put(lat.float().numpy())
    dist.destroy_process_group()


@pytest.mark.parametrize("L,S,Ov,world", [(40, 16, 8, 2), (20, 16, 4, 2), (56, 16, 8, 3)])
def test_sharded_eta_equals_one_rank_seeded_like_rank0(L, S, Ov, world):
    """denoise(distributed=True) at eta > 0 under gloo with a differently seeded generator per rank: rank 0 draws and
    broadcasts each step's noise, so the result is bit-identical to one rank seeded like rank 0."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + ((os.getpid() * 13 + L + world) % 2000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, L, S, Ov, ret)) for r in range(world)]
    for p in procs:
        p.start()
    got = torch.from_numpy(ret.get(timeout=180))
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    lat, _ = _run(L, S, Ov, [11, 22], torch.Generator().manual_seed(900), 0.8, chunk_term=0.0)
    assert torch.equal(got, lat.float())
    other, _ = _run(L, S, Ov, [11, 22], torch.Generator().manual_seed(901), 0.8, chunk_term=0.0)
    assert not torch.equal(other, lat)
