"""DPM-Solver++ references for the tests and tools/gen_dpm_golden.py (test infrastructure only; imports nothing of the
product).

* ``DPMSolverMultistepScheduler``: diffusers 0.29.2's class (schedulers/scheduling_dpmsolver_multistep.py) restated in
  the library's structure for its deterministic algorithm ``dpmsolver++`` -- ``step_index``, ``model_outputs``,
  ``lower_order_nums``, the zero-SNR clamp ``alphas_cumprod[-1] = 2**-24``, the fp32 upcast of the sample in ``step``
  and the cast back to the model dtype.  Like the library it keeps its history across ``step`` calls, so the reference
  pipeline, which calls ``step`` once per context window, is only well defined with it at one window.
* ``cuda_rounding``: CPU eager rounds a 0-d fp32 tensor to bf16 before multiplying a bf16 tensor by it, where CUDA keeps
  the fp32 scalar and rounds the product once.  Under this mode the CPU products follow CUDA, so the library-structured
  step on host tensors gives the bits it gives on the GPU.
* ``PerFrameDPM`` / ``denoise_per_frame``: a specialised restatement of the per-frame semantics the product implements
  for videos of several windows -- each frame gets one update per step, from its averaged model output, and keeps its
  own history of x0 predictions -- written with explicit rounding points.
* The library's class name is kept, so the pipeline recognises the restatement as a diffusers DPM scheduler.

The rounding points are diffusers' eager arithmetic on bf16 CUDA tensors as restated here; the library itself is not
a dependency of this project, so they are held to its structure, not to its installed code."""
import os
import sys

import numpy as np
import torch
from torch.overrides import TorchFunctionMode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _shim_schedulers():
    p = os.path.join(ROOT, "oracle", "diffusers_shim")
    if p not in sys.path:
        sys.path.insert(0, p)
    import diffusers.schedulers as s
    return s


class SchedulerOutput:
    def __init__(self, prev_sample):
        self.prev_sample = prev_sample


class DPMSolverMultistepScheduler:
    order = 1

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                 dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                 solver_type="midpoint", lower_order_final=True, euler_at_final=False, use_karras_sigmas=False,
                 use_lu_lambdas=False, final_sigmas_type="zero", lambda_min_clipped=-float("inf"), variance_type=None,
                 timestep_spacing="linspace", steps_offset=0, rescale_betas_zero_snr=False):
        self.config = type("Config", (), dict(
            num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
            beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
            prediction_type=prediction_type, thresholding=thresholding,
            dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
            algorithm_type=algorithm_type, solver_type=solver_type, lower_order_final=lower_order_final,
            euler_at_final=euler_at_final, use_karras_sigmas=use_karras_sigmas, use_lu_lambdas=use_lu_lambdas,
            final_sigmas_type=final_sigmas_type, lambda_min_clipped=lambda_min_clipped, variance_type=variance_type,
            timestep_spacing=timestep_spacing, steps_offset=steps_offset,
            rescale_betas_zero_snr=rescale_betas_zero_snr))()
        shim = _shim_schedulers()
        if trained_betas is not None:
            self.betas = torch.tensor(trained_betas, dtype=torch.float32)
        elif beta_schedule == "linear":
            self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        elif beta_schedule == "scaled_linear":
            self.betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        elif beta_schedule == "squaredcos_cap_v2":
            self.betas = shim.betas_for_alpha_bar(num_train_timesteps)
        else:
            raise NotImplementedError(f"{beta_schedule} is not implemented for {self.__class__}")
        if rescale_betas_zero_snr:
            self.betas = shim.rescale_zero_terminal_snr(self.betas)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        if rescale_betas_zero_snr:
            # Close to 0 without being 0 so first sigma is not inf
            self.alphas_cumprod[-1] = 2 ** -24
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.sigmas = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5
        self.init_noise_sigma = 1.0
        if algorithm_type != "dpmsolver++":
            raise NotImplementedError(f"{algorithm_type} is not restated here")
        if solver_type not in ("midpoint", "heun"):
            raise NotImplementedError(f"{solver_type} is not implemented for {self.__class__}")
        if use_karras_sigmas or use_lu_lambdas or thresholding or variance_type is not None:
            raise NotImplementedError("Karras / Lu sigmas, thresholding and learned variances are not restated here")
        self.num_inference_steps = None
        timesteps = np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=np.float32)[::-1].copy()
        self.timesteps = torch.from_numpy(timesteps)
        self.model_outputs = [None] * solver_order
        self.lower_order_nums = 0
        self._step_index = None
        self._begin_index = None

    @property
    def step_index(self):
        return self._step_index

    def set_timesteps(self, num_inference_steps=None, device=None):
        clipped_idx = torch.searchsorted(torch.flip(self.lambda_t, [0]), self.config.lambda_min_clipped)
        last_timestep = ((self.config.num_train_timesteps - clipped_idx).numpy()).item()
        if self.config.timestep_spacing == "linspace":
            timesteps = np.linspace(0, last_timestep - 1, num_inference_steps + 1).round()[::-1][:-1].copy() \
                .astype(np.int64)
        elif self.config.timestep_spacing == "leading":
            step_ratio = last_timestep // (num_inference_steps + 1)
            timesteps = (np.arange(0, num_inference_steps + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            timesteps += self.config.steps_offset
        elif self.config.timestep_spacing == "trailing":
            step_ratio = self.config.num_train_timesteps / num_inference_steps
            timesteps = np.arange(last_timestep, 0, -step_ratio).round().copy().astype(np.int64)
            timesteps -= 1
        else:
            raise ValueError(f"{self.config.timestep_spacing} is not supported")
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
        if self.config.final_sigmas_type == "sigma_min":
            sigma_last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5
        elif self.config.final_sigmas_type == "zero":
            sigma_last = 0
        else:
            raise ValueError(f"final_sigmas_type must be 'zero' or 'sigma_min', got {self.config.final_sigmas_type}")
        sigmas = np.concatenate([sigmas, [sigma_last]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        self.timesteps = torch.from_numpy(timesteps).to(device=device, dtype=torch.int64)
        self.num_inference_steps = len(timesteps)
        self.model_outputs = [None] * self.config.solver_order
        self.lower_order_nums = 0
        self._step_index = None
        self._begin_index = None
        self.sigmas = self.sigmas.to("cpu")

    def _sigma_to_alpha_sigma_t(self, sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        sigma_t = sigma * alpha_t
        return alpha_t, sigma_t

    def convert_model_output(self, model_output, sample=None):
        if self.config.prediction_type == "epsilon":
            sigma = self.sigmas[self.step_index]
            alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma)
            x0_pred = (sample - sigma_t * model_output) / alpha_t
        elif self.config.prediction_type == "sample":
            x0_pred = model_output
        elif self.config.prediction_type == "v_prediction":
            sigma = self.sigmas[self.step_index]
            alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma)
            x0_pred = alpha_t * sample - sigma_t * model_output
        else:
            raise ValueError(f"prediction_type given as {self.config.prediction_type} is not supported")
        return x0_pred

    def dpm_solver_first_order_update(self, model_output, sample=None, noise=None):
        sigma_t, sigma_s = self.sigmas[self.step_index + 1], self.sigmas[self.step_index]
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma_t)
        alpha_s, sigma_s = self._sigma_to_alpha_sigma_t(sigma_s)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s = torch.log(alpha_s) - torch.log(sigma_s)
        h = lambda_t - lambda_s
        x_t = (sigma_t / sigma_s) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * model_output
        return x_t

    def multistep_dpm_solver_second_order_update(self, model_output_list, sample=None, noise=None):
        sigma_t, sigma_s0, sigma_s1 = (self.sigmas[self.step_index + 1], self.sigmas[self.step_index],
                                       self.sigmas[self.step_index - 1])
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma_t)
        alpha_s0, sigma_s0 = self._sigma_to_alpha_sigma_t(sigma_s0)
        alpha_s1, sigma_s1 = self._sigma_to_alpha_sigma_t(sigma_s1)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
        m0, m1 = model_output_list[-1], model_output_list[-2]
        h, h_0 = lambda_t - lambda_s0, lambda_s0 - lambda_s1
        r0 = h_0 / h
        D0, D1 = m0, (1.0 / r0) * (m0 - m1)
        if self.config.solver_type == "midpoint":
            x_t = ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                   - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1)
        else:
            x_t = ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                   + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1)
        return x_t

    def index_for_timestep(self, timestep, schedule_timesteps=None):
        if schedule_timesteps is None:
            schedule_timesteps = self.timesteps
        index_candidates = (schedule_timesteps == timestep).nonzero()
        if len(index_candidates) == 0:
            return len(self.timesteps) - 1
        if len(index_candidates) > 1:
            return index_candidates[1].item()
        return index_candidates[0].item()

    def _init_step_index(self, timestep):
        if self._begin_index is None:
            if isinstance(timestep, torch.Tensor):
                timestep = timestep.to(self.timesteps.device)
            self._step_index = self.index_for_timestep(timestep)
        else:
            self._step_index = self._begin_index

    def step(self, model_output, timestep, sample, generator=None, variance_noise=None, return_dict=True):
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the "
                             "scheduler")
        if self.step_index is None:
            self._init_step_index(timestep)
        lower_order_final = (self.step_index == len(self.timesteps) - 1) and (
            self.config.euler_at_final or (self.config.lower_order_final and len(self.timesteps) < 15)
            or self.config.final_sigmas_type == "zero")
        lower_order_second = ((self.step_index == len(self.timesteps) - 2) and self.config.lower_order_final
                              and len(self.timesteps) < 15)
        model_output = self.convert_model_output(model_output, sample=sample)
        for i in range(self.config.solver_order - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
        self.model_outputs[-1] = model_output
        # Upcast to avoid precision issues when computing prev_sample
        sample = sample.to(torch.float32)
        noise = None
        if self.config.solver_order == 1 or self.lower_order_nums < 1 or lower_order_final:
            prev_sample = self.dpm_solver_first_order_update(model_output, sample=sample, noise=noise)
        elif self.config.solver_order == 2 or self.lower_order_nums < 2 or lower_order_second:
            prev_sample = self.multistep_dpm_solver_second_order_update(self.model_outputs, sample=sample, noise=noise)
        else:
            raise NotImplementedError("third-order DPM-Solver++ is not restated here")
        if self.lower_order_nums < self.config.solver_order:
            self.lower_order_nums += 1
        # Cast sample back to expected dtype
        prev_sample = prev_sample.to(model_output.dtype)
        self._step_index += 1
        if not return_dict:
            return (prev_sample,)
        return SchedulerOutput(prev_sample=prev_sample)

    def scale_model_input(self, sample, *args, **kwargs):
        return sample


def reference_scheduler(**overrides):
    """The class above with the reference's noise_scheduler_kwargs (inference_v2.yaml:24-33)."""
    kw = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", steps_offset=1,
              prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")
    kw.update(overrides)
    return DPMSolverMultistepScheduler(**kw)


class cuda_rounding(TorchFunctionMode):
    """CPU products of a 0-d fp32 tensor and a bf16 tensor computed as CUDA computes them: the fp32 product, rounded
    once to bf16."""

    _MULS = (torch.Tensor.mul, torch.Tensor.__mul__, torch.Tensor.__rmul__, torch.mul)

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func in self._MULS and len(args) == 2 and not kwargs:
            for s, t in (args, args[::-1]):
                if isinstance(s, torch.Tensor) and isinstance(t, torch.Tensor) and s.dim() == 0 \
                        and s.dtype == torch.float32 and t.dim() > 0 and t.dtype == torch.bfloat16 \
                        and t.device.type == "cpu":
                    return (s * t.float()).bfloat16()
        return func(*args, **kwargs)


def _rb(t):
    return t.bfloat16().float()


class PerFrameDPM:
    """DPM-Solver++(2M) at the reference's configuration with one history per frame: ``step(k, frames, v, x)`` updates
    the listed frames at step k of the call from their model outputs v and latents x (both bf16, (n,4,len(frames),...)),
    with the kernel's rounding points.  Scalars are the fp32 0-d arithmetic of the library's update, written out for
    v-prediction on the clamped zero-SNR table."""

    def __init__(self, steps, solver_order=2):
        from oracle import vx_oracle as O
        ddim = O.DDIM()
        abar = ddim.alphas_cumprod.clone()
        abar[-1] = 2 ** -24
        ddim.set_timesteps(steps)
        self.timesteps = [int(t) for t in ddim.timesteps]
        table = ((1 - abar) / abar) ** 0.5
        self.sig = torch.cat([table[torch.tensor(self.timesteps)], torch.zeros(1)])
        self.solver_order = solver_order
        self.hist = {}                        # frame -> (step index of its last update, its x0 prediction)

    def _lam(self, k):
        s = self.sig[k]
        a = 1 / ((s ** 2 + 1) ** 0.5)
        return a, s * a, torch.log(a) - torch.log(s * a)

    def step(self, k, frames, v, x):
        a_s, s_s, l_s = self._lam(k)
        a_t, s_t, l_t = self._lam(k + 1)
        h = l_t - l_s
        c0 = float(a_t * (torch.exp(-h) - 1.0))
        ratio = float(s_t / s_s)
        x, v = x.float(), v.float()
        m0 = _rb(_rb(float(a_s) * x) - _rb(float(s_s) * v))
        out = ratio * x - _rb(c0 * m0)
        last = k == len(self.timesteps) - 1
        for j, fr in enumerate(frames):
            prev = self.hist.get(fr)
            if self.solver_order == 2 and not last and prev is not None:
                assert prev[0] == k - 1, (fr, prev[0], k)
                _, _, l_s1 = self._lam(k - 1)
                inv_r0 = float(1.0 / ((l_s - l_s1) / h))
                d1 = _rb(inv_r0 * _rb(m0[:, :, j] - prev[1]))
                out[:, :, j] = out[:, :, j] - _rb(float(0.5 * (a_t * (torch.exp(-h) - 1.0))) * d1)
            self.hist[fr] = (k, m0[:, :, j].clone())
        return out.bfloat16()


def denoise_per_frame(latents, kps_feature, audio_embeddings, steps, guidance_scale, context_frames, context_overlap,
                      unet_fn, solver_order=2):
    """The reference's window loop (pipelines/v_express_pipeline.py:527-572) with the per-frame DPM-Solver++ step: a
    window's finalised frames are stepped once each, from the model output of their last occurrence (the one the
    reference's sequential write-back keeps when a reflected window repeats a frame)."""
    from oracle import vx_oracle as O
    sched = PerFrameDPM(steps, solver_order)
    L = latents.shape[2]
    do_cfg = guidance_scale > 1.0
    windows = O.context_windows(L, context_frames, context_overlap)
    nfc = torch.from_numpy(O.num_frame_context(windows, L))
    latents = latents.clone()
    for k, t in enumerate(sched.timesteps):
        counter = torch.zeros(L, dtype=torch.long)
        noise_preds = [None] * L
        for window in windows:
            aud = audio_embeddings[:, window]
            x = latents[:, :, window].repeat(2 if do_cfg else 1, 1, 1, 1, 1)
            noise_pred = unet_fn(x, t, aud.reshape(-1, aud.shape[-2], aud.shape[-1]), kps_feature[:, :, window])
            if do_cfg:
                u, c = noise_pred.chunk(2)
                noise_pred = u + guidance_scale * (c - u)
            counter[window] += 1
            noise_pred = noise_pred / nfc[window][None, None, :, None, None]
            kept = {}
            for li, fi in enumerate(window):
                if noise_preds[fi] is None:
                    noise_preds[fi] = noise_pred[:, :, li].clone()
                else:
                    noise_preds[fi] += noise_pred[:, :, li]
                if counter[fi] == nfc[fi]:
                    kept[fi] = noise_preds[fi]           # a repeated frame: the last occurrence wins
                    noise_preds[fi] = None
            if kept:
                ids = sorted(kept)
                stepped = sched.step(k, ids, torch.stack([kept[i] for i in ids], 2), latents[:, :, ids])
                latents[:, :, ids] = stepped
    assert all(v[0] == len(sched.timesteps) - 1 for v in sched.hist.values()) and len(sched.hist) == L
    return latents


def toy_problem(dims=20000, seed=0):
    """The Gaussian toy: x0 ~ N(mu, s^2) per dimension, mu ~ N(0,1), s = exp(0.5 N(0,1)); x_T ~ N(0,1); float64."""
    rng = np.random.default_rng(seed)
    mu = rng.standard_normal(dims)
    s = np.exp(0.5 * rng.standard_normal(dims))
    return mu, s, rng.standard_normal(dims)


def toy_x0(mu, s, x, alpha, sigma):
    """The exact posterior mean E[x0 | x_t = x] of the toy at (alpha, sigma)."""
    return mu + alpha * s ** 2 * (x - alpha * mu) / (alpha ** 2 * s ** 2 + sigma ** 2)


def toy_ode_state(mu, s, x_T, alpha, sigma):
    """The probability-flow ODE state from x_T at (alpha, sigma), in closed form."""
    return alpha * mu + np.sqrt(alpha ** 2 * s ** 2 + sigma ** 2) * x_T
