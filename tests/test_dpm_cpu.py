"""DPM-Solver++ sampling on the host side, without a GPU: the scheduler tables against the library-structured restatement
(tests/dpm_reference.py) and float64 closed forms, the solver's accuracy on a Gaussian toy problem in float64, and the
denoise / stream loops with the UNet replaced by a cheap deterministic function and the elementwise kernels by torch
emulations with the kernels' rounding points (the harness of tests/test_samples_cpu.py), against the reference loop over
the restatement (one window) and the per-frame oracle (several windows)."""
import math
import os

import numpy as np
import pytest
import torch

import dpm_reference as R
from test_host_cpu import _fake_unet_fn
from test_samples_cpu import _ElementwiseEmu, _draw, _fake_conditioning, _fake_pipeline


def _rb(t):
    return t.bfloat16().float()


def _bits(x):
    return np.float32(x).tobytes()


class _DpmEmu(_ElementwiseEmu):
    """+ vx_dpmpp_step / vx_dpmpp_step_frames (csrc/vx_misc.cu) with their rounding points."""

    @staticmethod
    def _update(x, acc, hist, alpha_s, sigma_s, ratio, c0, inv_r0, c0h, order):
        x, v = x.float(), _rb(acc)
        m0 = _rb(_rb(alpha_s * x) - _rb(sigma_s * v))
        out = ratio * x - _rb(c0 * m0)
        if order == 2:
            out = out - _rb(c0h * _rb(inv_r0 * _rb(m0 - hist.float())))
        return out.bfloat16(), m0.bfloat16()

    @staticmethod
    def dpmpp_step(lat, acc, hist, *c):
        assert lat.dtype == torch.bfloat16 and acc.dtype == torch.float32 and hist.dtype == torch.bfloat16
        out, m0 = _DpmEmu._update(lat.view(acc.shape), acc, hist.view(acc.shape), *c)
        lat.copy_(out.view(lat.shape))
        hist.copy_(m0.view(hist.shape))

    @staticmethod
    def dpmpp_step_frames(lat, acc, hist, frames, *c):
        n, ch, L = lat.shape[:3]
        ids = frames.long().cpu()
        lat3, acc3, hist3 = lat.view(n, ch, L, -1), acc.view(n, ch, L, -1), hist.view(n, ch, L, -1)
        out, m0 = _DpmEmu._update(lat3[:, :, ids], acc3[:, :, ids], hist3[:, :, ids], *c)
        lat3[:, :, ids] = out
        hist3[:, :, ids] = m0
        acc3[:, :, ids] = 0


# ---------------------------------------------------------------------------------------------------------- tables
@pytest.mark.parametrize("steps", [5, 10, 25])
def test_tables_equal_library_and_closed_forms(steps):
    """Timesteps are DDIM's trailing ones; alphas_cumprod and sigmas equal the library-structured restatement bit for
    bit, and each step's scalars equal the ones its update computes; all within a few fp32 ulps of float64 closed forms
    on the same table entries."""
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, DPMSolverMultistepScheduler, dpm_coefficients
    prod, lib, ddim = DPMSolverMultistepScheduler(), R.reference_scheduler(), DDIMScheduler()
    for s in (prod, lib, ddim):
        s.set_timesteps(steps)
    assert prod.timesteps.tolist() == lib.timesteps.tolist() == ddim.timesteps.tolist()
    assert torch.equal(prod.alphas_cumprod, lib.alphas_cumprod) and float(prod.alphas_cumprod[-1]) == 2 ** -24
    assert torch.equal(prod.alphas_cumprod[:-1], ddim.alphas_cumprod[:-1])
    assert prod.sigmas.dtype == torch.float32 and torch.equal(prod.sigmas, lib.sigmas) and float(prod.sigmas[-1]) == 0
    u = 2.0 ** -23
    for k, t in enumerate(prod.timesteps.tolist()):
        a = float(prod.alphas_cumprod[t])
        assert abs(float(prod.sigmas[k]) - math.sqrt((1 - a) / a)) <= 2 * u * math.sqrt((1 - a) / a)
        a_s, s_s, ratio, c0, inv_r0, c0h, order = dpm_coefficients(prod, k)
        assert order == (1 if k in (0, steps - 1) else 2)
        # the library's scalars
        lib._step_index = k
        st, ss = lib.sigmas[k + 1], lib.sigmas[k]
        al_t, sg_t = lib._sigma_to_alpha_sigma_t(st)
        al_s, sg_s = lib._sigma_to_alpha_sigma_t(ss)
        h = (torch.log(al_t) - torch.log(sg_t)) - (torch.log(al_s) - torch.log(sg_s))
        assert _bits(a_s) == _bits(al_s) and _bits(s_s) == _bits(sg_s)
        assert _bits(ratio) == _bits(sg_t / sg_s) and _bits(c0) == _bits(al_t * (torch.exp(-h) - 1.0))
        # float64 closed forms: alpha_s = sqrt(abar), sigma_s = sqrt(1 - abar), c0 = alpha_t (e^-h - 1)
        assert abs(a_s - math.sqrt(a)) <= 4 * u * math.sqrt(a) and abs(s_s - math.sqrt(1 - a)) <= 4 * u
        if k == steps - 1:
            assert (ratio, c0) == (0.0, -1.0)
            continue
        ap = float(prod.alphas_cumprod[prod.timesteps[k + 1]])
        lam = lambda x: 0.5 * math.log(x / (1 - x))
        h64 = lam(ap) - lam(a)
        assert abs(ratio - math.sqrt((1 - ap) / (1 - a))) <= 8 * u * math.sqrt((1 - ap) / (1 - a))
        assert abs(c0 - math.sqrt(ap) * math.expm1(-h64)) <= 16 * u * math.sqrt(ap)
        if order == 2:
            a1 = float(prod.alphas_cumprod[prod.timesteps[k - 1]])
            h0 = lam(a) - lam(a1)
            r0_64 = h0 / h64
            assert _bits(c0h) == _bits(0.5 * (al_t * (torch.exp(-h) - 1.0)))
            st1 = lib.sigmas[k - 1]
            al_1, sg_1 = lib._sigma_to_alpha_sigma_t(st1)
            r0 = ((torch.log(al_s) - torch.log(sg_s)) - (torch.log(al_1) - torch.log(sg_1))) / h
            assert _bits(inv_r0) == _bits(1.0 / r0)
            assert abs(inv_r0 - 1 / r0_64) <= 64 * u * abs(1 / r0_64), (k, inv_r0, 1 / r0_64)


def test_order_follows_history_solver_order_and_last_step():
    from vexpress_b200.pipelines.scheduler import DPMSolverMultistepScheduler, dpm_coefficients
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(5)
    assert [dpm_coefficients(s, k)[-1] for k in range(5)] == [1, 2, 2, 2, 1]
    assert [dpm_coefficients(s, k, first=k == 2)[-1] for k in range(2, 5)] == [1, 2, 1]     # a strength slice
    s1 = DPMSolverMultistepScheduler(solver_order=1)
    s1.set_timesteps(5)
    assert [dpm_coefficients(s1, k)[-1] for k in range(5)] == [1] * 5


# ------------------------------------------------------------------------------------------ float64 solver checks
def _abar():
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
    return DDIMScheduler().alphas_cumprod.double().numpy(), DPMSolverMultistepScheduler().alphas_cumprod.double().numpy()


def _dpm64(ts, abar, x, x0_fn, solver_order=2, upto=None):
    """DPM-Solver++ in float64 on the sigma table of ``abar`` at ``ts`` (final sigma 0): x after ``upto`` steps."""
    sig = [math.sqrt((1 - abar[t]) / abar[t]) for t in ts] + [0.0]
    al = lambda s: 1 / math.sqrt(s * s + 1)
    lam = lambda s: math.log(1 / s) if s > 0 else math.inf
    m_prev = None
    for k in range(len(ts) if upto is None else upto):
        a_s, s_s, a_t, s_t = al(sig[k]), sig[k] * al(sig[k]), al(sig[k + 1]), sig[k + 1] * al(sig[k + 1])
        h = lam(sig[k + 1]) - lam(sig[k])
        m0 = x0_fn(x, a_s, s_s)
        c0 = a_t * (math.exp(-h) - 1.0)
        x_new = (s_t / s_s) * x - c0 * m0
        if solver_order == 2 and m_prev is not None and k < len(ts) - 1:
            r0 = (lam(sig[k]) - lam(sig[k - 1])) / h
            x_new = x_new - 0.5 * c0 * (m0 - m_prev) / r0
        x, m_prev = x_new, m0
    return x


def _ddim64(ts, abar, x, x0_fn, upto):
    for k in range(upto):
        a, ap = abar[ts[k]], abar[ts[k + 1]] if k + 1 < len(ts) else 1.0
        x0 = x0_fn(x, math.sqrt(a), math.sqrt(1 - a))
        eps = (x - math.sqrt(a) * x0) / math.sqrt(1 - a)
        x = math.sqrt(ap) * x0 + math.sqrt(1 - ap) * eps
    return x


@pytest.mark.parametrize("solver_order", [1, 2])
def test_constant_x0_predictor_is_integrated_exactly(solver_order):
    """With an x0 predictor constant along the path, the exponential integrator is exact: every state is
    alpha_t c + sigma_t z and the last step returns c -- in float64, at orders 1 and 2."""
    _, abar = _abar()
    rng = np.random.default_rng(1)
    c, z = rng.standard_normal(64), rng.standard_normal(64)
    for steps in (5, 10, 25):
        ts = [int(t) for t in np.round(np.arange(1000, 0, -1000 / steps)).astype(np.int64) - 1]
        a0 = math.sqrt(abar[ts[0]])
        x_T = a0 * c + math.sqrt(1 - a0 * a0) * z
        for upto in range(1, steps):
            x = _dpm64(ts, abar, x_T, lambda x, a, s: c, solver_order, upto)
            a = math.sqrt(abar[ts[upto]])
            assert np.abs(x - (a * c + math.sqrt(1 - a * a) * z)).max() <= 1e-12, (steps, upto)
        assert np.array_equal(_dpm64(ts, abar, x_T, lambda x, a, s: c, solver_order), c)


def _toy_errors(steps):
    """Relative L2 error of DDIM and DPM-Solver++(2M) at the last nonzero noise level on the Gaussian toy."""
    abar_ddim, abar_dpm = _abar()
    mu, s, x_T = R.toy_problem()
    x0 = lambda x, a, sg: R.toy_x0(mu, s, x, a, sg)
    ts = [int(t) for t in np.round(np.arange(1000, 0, -1000 / steps)).astype(np.int64) - 1]
    a = math.sqrt(abar_ddim[ts[-1]])
    want = R.toy_ode_state(mu, s, x_T, a, math.sqrt(1 - a * a))
    rel = lambda x: float(np.linalg.norm(x - want) / np.linalg.norm(want))
    return rel(_ddim64(ts, abar_ddim, x_T, x0, steps - 1)), rel(_dpm64(ts, abar_dpm, x_T, x0, 2, steps - 1))


def test_gaussian_toy_accuracy():
    """DPM-Solver++(2M) below 0.35x DDIM's error at 10 steps; its error falls >= 3x from 5 to 10 steps and >= 2.5x from
    10 to 20 (second-order convergence; DDIM is first order)."""
    err = {n: _toy_errors(n) for n in (5, 8, 10, 20, 25)}
    for n, (d, p) in err.items():
        print(f"{n:3d} steps: DDIM {d:.3e}  DPM-Solver++(2M) {p:.3e}")
    assert err[10][1] < 0.35 * err[10][0]
    assert err[5][1] >= 3 * err[10][1] and err[10][1] >= 2.5 * err[20][1]
    assert err[8][1] < err[25][0]


# ------------------------------------------------------------------------------------------- harness + oracles
def _fake_dpm_pipeline(chunk_term=1.0, scheduler=None):
    from vexpress_b200.pipelines.scheduler import DPMSolverMultistepScheduler
    pipe, vp, eng = _fake_pipeline(chunk_term)
    pipe.scheduler = scheduler if scheduler is not None else DPMSolverMultistepScheduler()
    vp.ops = _DpmEmu()
    return pipe, vp, eng


def _run(L, S, Ov, seeds, steps=5, distributed=False, eta=0.0, generator=None, chunk_term=1.0, scheduler=None):
    """-> (final latents (n,4,L,h,w), decoded video) of one host-side DPM denoise + decode."""
    from vexpress_b200 import ops as real_ops
    from vexpress_b200.pipelines.v_express_pipeline import retrieve_timesteps
    pipe, vp, eng = _fake_dpm_pipeline(chunk_term, scheduler)
    try:
        kps, audio = _fake_conditioning(L)
        ts, _ = retrieve_timesteps(pipe.scheduler, steps, None)
        lat = pipe.denoise(_draw(pipe, seeds, L), kps, audio, ts, 3.5, S, Ov, distributed=distributed, eta=eta,
                           generator=generator)
        return lat, pipe.decode_to_device(lat, distributed)
    finally:
        vp.ops = real_ops


def _unet_fn(x, t, aud, kps):
    """n samples share the conditioning: the batch [u s0..s(n-1) | c s0..s(n-1)] repeats each CFG half's rows."""
    b = kps.shape[0]
    n = x.shape[0] // b
    aud = aud.view(b, -1, *aud.shape[1:]).repeat_interleave(n, 0).flatten(0, 1)
    return _fake_unet_fn(x, t, aud, kps.repeat_interleave(n, 0))


def _inputs(L, seeds):
    pipe, _, _ = _fake_pipeline()
    return (_draw(pipe, seeds, L),) + _fake_conditioning(L)


@pytest.mark.parametrize("steps,n", [(5, 1), (8, 2), (3, 1)])
def test_one_window_equals_reference_loop_over_library_class(steps, n, monkeypatch):
    """One context window: the reference's loop (the oracle's restatement of :527-572) stepping the library-structured
    scheduler -- its step index and history kept across calls, its rounding points on CUDA -- is bit-identical to the
    product's denoise, and so is the per-frame oracle."""
    from oracle import vx_oracle as O
    L, seeds = 8, [11, 22][:n]
    out, _ = _run(L, 8, 4, seeds, steps)
    lat, kps, audio = _inputs(L, seeds)
    monkeypatch.setattr(O, "DDIM", lambda: R.reference_scheduler())
    with R.cuda_rounding():
        ref = O.denoise(None, None, lat, kps, audio, None, steps, 3.5, 8, 4, unet_fn=_unet_fn)
    assert out.dtype == ref.dtype == torch.bfloat16
    assert torch.equal(out, ref)
    assert torch.equal(out, R.denoise_per_frame(lat, kps, audio, steps, 3.5, 8, 4, _unet_fn))
    monkeypatch.undo()                                                   # the DDIM loop lands elsewhere
    assert not torch.equal(out, O.denoise(None, None, lat, kps, audio, None, steps, 3.5, 8, 4, unet_fn=_unet_fn))


@pytest.mark.parametrize("L,S,Ov,n,order", [(12, 8, 4, 1, 2), (20, 16, 4, 1, 2), (33, 24, 4, 2, 2), (24, 16, 8, 1, 1),
                                            (20, 16, 4, 2, 1)])
def test_several_windows_equal_per_frame_oracle(L, S, Ov, n, order):
    """Tiling and reflected-tail lengths: bit-identical to the per-frame oracle (one update per frame and step, each
    frame with its own history), at solver orders 2 and 1."""
    from vexpress_b200.pipelines.scheduler import DPMSolverMultistepScheduler
    seeds = [11, 22][:n]
    out, _ = _run(L, S, Ov, seeds, 5, scheduler=DPMSolverMultistepScheduler(solver_order=order))
    lat, kps, audio = _inputs(L, seeds)
    assert torch.equal(out, R.denoise_per_frame(lat, kps, audio, 5, 3.5, S, Ov, _unet_fn, order))


@pytest.mark.parametrize("L", [52, 50])
def test_stream_equals_denoise_and_decode(L):
    """``denoise_stream`` (the wavefront, ``vx_dpmpp_step_frames``) gives the latents and frames of ``denoise`` +
    decode, for one and two samples."""
    from vexpress_b200 import ops as real_ops
    from vexpress_b200.pipelines.v_express_pipeline import retrieve_timesteps
    for seeds in ([11], [11, 22]):
        ref_lat, ref_video = _run(L, 16, 4, seeds, 4)
        pipe, vp, _ = _fake_dpm_pipeline()
        try:
            kps, audio = _fake_conditioning(L)
            pipe.prepare_kps_feature_frames = lambda images, a, e, height, width: kps[1:, :, a:e]
            ts, _ = retrieve_timesteps(pipe.scheduler, 4, None)
            lat = _draw(pipe, seeds, L)
            chunks = list(pipe.denoise_stream(lat, None, audio, ts, 3.5, 16, 4))
        finally:
            vp.ops = real_ops
        video = torch.cat([c.frames for c in chunks], 2)
        assert torch.equal(lat, ref_lat)
        assert torch.equal(video, ref_video if len(seeds) > 1 else ref_video.unsqueeze(0))


def test_three_samples_equal_one_sample_calls():
    L, S, Ov, seeds = 20, 16, 4, [11, 22, 33]
    lat, video = _run(L, S, Ov, seeds)
    for i, s in enumerate(seeds):
        lat1, video1 = _run(L, S, Ov, [s])
        assert torch.equal(lat[i], lat1[0]) and torch.equal(video[i], video1), i
    assert not torch.equal(lat[0], lat[1])


def test_eta_draws_nothing_under_dpm():
    """eta > 0 is ignored by DPM-Solver++ (the library's step takes no eta): the result equals eta = 0 and the generator
    is not advanced."""
    g = torch.Generator().manual_seed(9)
    state = g.get_state()
    lat1, _ = _run(20, 16, 4, [11], eta=1.0, generator=g)
    assert torch.equal(g.get_state(), state)
    lat0, _ = _run(20, 16, 4, [11])
    assert torch.equal(lat0, lat1)


def _gloo_worker(rank, world, port, L, S, Ov, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lat, _ = _run(L, S, Ov, [11, 22], distributed=True, chunk_term=0.0)
    if rank == 0:
        ret.put(lat.float().numpy())
    dist.destroy_process_group()


@pytest.mark.parametrize("L,S,Ov", [(40, 16, 8), (20, 16, 4)])
def test_two_ranks_equal_one_rank(L, S, Ov):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + ((os.getpid() * 17 + L) % 2000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, L, S, Ov, ret)) for r in range(2)]
    for p in procs:
        p.start()
    got = torch.from_numpy(ret.get(timeout=180))
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    lat, _ = _run(L, S, Ov, [11, 22], chunk_term=0.0)
    assert torch.equal(got, lat.float())


# ------------------------------------------------------------------------------------------ configuration surface
@pytest.mark.parametrize("option,value", [("beta_schedule", "linear"), ("prediction_type", "epsilon"),
                                          ("timestep_spacing", "leading"), ("algorithm_type", "sde-dpmsolver++"),
                                          ("solver_type", "heun"), ("solver_order", 3),
                                          ("final_sigmas_type", "sigma_min"), ("use_karras_sigmas", True),
                                          ("use_lu_lambdas", True), ("thresholding", True),
                                          ("lambda_min_clipped", -5.1), ("variance_type", "learned_range"),
                                          ("trained_betas", [0.1] * 1000)])
def test_unsupported_configurations_raise(option, value):
    from vexpress_b200.pipelines.scheduler import DPMSolverMultistepScheduler
    with pytest.raises(ValueError, match=option):
        DPMSolverMultistepScheduler(**{option: value})


def test_reference_kwargs_and_from_config():
    """``DPMSolverMultistepScheduler(**noise_scheduler_kwargs)`` with the reference's DDIM keywords, and ``from_config``
    of a DDIM config (DDIM-only keys dropped); lower_order_final / euler_at_final are accepted either way."""
    from vexpress_b200.pipelines.scheduler import DDIMScheduler, DPMSolverMultistepScheduler
    kw = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, steps_offset=1,
              prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")
    a = DPMSolverMultistepScheduler(**kw)
    b = DPMSolverMultistepScheduler.from_config(vars(DDIMScheduler().config))
    c = DPMSolverMultistepScheduler.from_config(dict(kw, _class_name="DDIMScheduler", set_alpha_to_one=True,
                                                     lower_order_final=False, euler_at_final=True))
    for s in (a, b, c):
        s.set_timesteps(10)
        assert torch.equal(s.sigmas, a.sigmas) and s.config.solver_order == 2
    with pytest.raises(TypeError, match="bogus"):
        DPMSolverMultistepScheduler(bogus=1)


class DPMSolverMultistepScheduler:
    """A diffusers-like DPM scheduler: only the class name, ``config`` and the methods the pipeline calls."""
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, **config):
        self.config = type("FrozenDict", (dict,), {})(config)
        self.timesteps = torch.arange(999, -1, -1)
        self.num_inference_steps = None

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        self.timesteps = torch.from_numpy(np.round(np.arange(1000, 0, -1000 / num_inference_steps)).astype(np.int64) - 1)

    def step(self, *a, **k):
        raise AssertionError("the pipeline never calls a foreign scheduler's step")

    def scale_model_input(self, sample, timestep=None):
        return sample


def test_duck_typed_diffusers_scheduler_is_accepted():
    """An object named DPMSolverMultistepScheduler with a diffusers-style config dict runs the product's DPM update,
    bit-identical to the product's own class; any other class keeps the DDIM update."""
    from vexpress_b200.pipelines.scheduler import dpm_scheduler
    c = R.reference_scheduler().config
    cfg = {k: getattr(c, k) for k in dir(c) if not k.startswith("_")}
    foreign = DPMSolverMultistepScheduler(_class_name="DPMSolverMultistepScheduler", _diffusers_version="0.29.2", **cfg)
    got, _ = _run(20, 16, 4, [11], scheduler=foreign)
    want, _ = _run(20, 16, 4, [11])
    assert torch.equal(got, want)
    assert dpm_scheduler(R.reference_scheduler()) is not None           # the restatement carries the library's name
    assert dpm_scheduler(type("EulerDiscreteScheduler", (DPMSolverMultistepScheduler,), {})()) is None
