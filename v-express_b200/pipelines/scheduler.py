"""DDIM and DPM-Solver++ schedulers restated for the hot path (diffusers 0.29.2 ``DDIMScheduler`` and
``DPMSolverMultistepScheduler`` with the reference's configuration inference_v2.yaml:23-33: scaled-linear betas,
zero-terminal-SNR rescale, v-prediction, trailing timestep spacing; SURVEY.md Appendix B.5).  Host-side scalar tables
only: the tensor update itself is the fused ``vx_ddim_step`` kernel (``vx_ddim_step_eta`` for stochastic DDIM, eta > 0)
or ``vx_dpmpp_step``."""
import inspect
import math
from types import SimpleNamespace

import numpy as np
import torch


def _scaled_linear_betas(num_train_timesteps, beta_start, beta_end, rescale_betas_zero_snr):
    """diffusers' "scaled_linear" betas in fp32, rescaled to zero terminal SNR (arXiv:2305.08891 Algorithm 1) when asked."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    if rescale_betas_zero_snr:
        root = torch.cumprod(1.0 - betas, 0).sqrt()
        first, last = root[0].clone(), root[-1].clone()
        root = (root - last) * (first / (first - last))
        abar = root ** 2
        betas = 1 - torch.cat([abar[:1], abar[1:] / abar[:-1]])
    return betas


class DDIMScheduler:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 clip_sample=False, set_alpha_to_one=True, steps_offset=1, prediction_type="v_prediction",
                 rescale_betas_zero_snr=True, timestep_spacing="trailing", **_):
        if beta_schedule != "scaled_linear" or prediction_type != "v_prediction" or timestep_spacing != "trailing" \
                or clip_sample:
            raise ValueError("vexpress_b200.DDIMScheduler implements the reference's inference_v2.yaml configuration only")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, clip_sample=clip_sample,
                                      set_alpha_to_one=set_alpha_to_one, steps_offset=steps_offset,
                                      prediction_type=prediction_type, rescale_betas_zero_snr=rescale_betas_zero_snr,
                                      timestep_spacing=timestep_spacing)
        self.betas = betas = _scaled_linear_betas(num_train_timesteps, beta_start, beta_end, rescale_betas_zero_snr)
        self.alphas = 1.0 - betas
        self.alphas_cumprod = torch.cumprod(self.alphas, 0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_inference_steps = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1, dtype=torch.int64)

    def set_timesteps(self, num_inference_steps, device=None):
        n = self.config.num_train_timesteps
        self.num_inference_steps = num_inference_steps
        ts = np.round(np.arange(n, 0, -n / num_inference_steps)).astype(np.int64) - 1
        self.timesteps = torch.from_numpy(ts)  # kept on the host: the step loop never syncs on a device tensor

    def scale_model_input(self, sample, timestep=None):
        return sample


def ddim_coefficients(scheduler, timestep: int):
    """(sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev)) as python floats from fp32 scalar math, exactly the
    scalars diffusers' ``step`` multiplies the model-dtype tensors with."""
    cfg = scheduler.config
    if getattr(cfg, "prediction_type", "v_prediction") != "v_prediction":
        raise ValueError("only v_prediction is supported")
    n_train = cfg.num_train_timesteps
    prev = int(timestep) - n_train // scheduler.num_inference_steps
    a_t = scheduler.alphas_cumprod[int(timestep)].float().cpu()
    a_p = (scheduler.alphas_cumprod[prev] if prev >= 0 else scheduler.final_alpha_cumprod).float().cpu()
    b_t = 1 - a_t
    return float(a_t ** 0.5), float(b_t ** 0.5), float(a_p ** 0.5), float((1 - a_p) ** 0.5)


def ddim_coefficients_eta(scheduler, timestep: int, eta: float):
    """(sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), c_dir, sigma) for the stochastic step (``vx_ddim_step_eta``), from the
    fp32 0-d tensor arithmetic of diffusers' ``step`` / ``_get_variance``:

        variance = (1-a_prev)/(1-a_t) * (1 - a_t/a_prev);  sigma = eta * variance ** 0.5
        c_dir    = (1 - a_prev - sigma ** 2) ** 0.5

    so each scalar equals the library's bit for bit -- with one exception: where that radicand rounds below zero
    (eta = 1 at a_t = 0, the first trailing step of a zero-terminal-SNR schedule: sigma ** 2 rounds one ulp above
    1 - a_prev at 25 steps), the library's 0-d ``** 0.5`` is NaN and the whole video with it; c_dir is 0 here, the exact
    value.  At eta = 0, sigma = 0 and c_dir = sqrt(1 - a_prev): the first four entries and c_dir are ``ddim_coefficients``."""
    if not 0.0 <= eta <= 1.0:
        raise ValueError(f"eta must lie in [0, 1], got {eta!r}")
    cfg = scheduler.config
    if getattr(cfg, "prediction_type", "v_prediction") != "v_prediction":
        raise ValueError("only v_prediction is supported")
    prev = int(timestep) - cfg.num_train_timesteps // scheduler.num_inference_steps
    a_t = scheduler.alphas_cumprod[int(timestep)].float().cpu()
    a_p = (scheduler.alphas_cumprod[prev] if prev >= 0 else scheduler.final_alpha_cumprod).float().cpu()
    b_t, b_p = 1 - a_t, 1 - a_p
    variance = (b_p / b_t) * (1 - a_t / a_p)
    sigma = eta * variance ** 0.5
    c_dir = (1 - a_p - sigma ** 2).clamp_min(0) ** 0.5
    return float(a_t ** 0.5), float(b_t ** 0.5), float(a_p ** 0.5), float(c_dir), float(sigma)


class DPMSolverMultistepScheduler:
    """diffusers 0.29.2 ``DPMSolverMultistepScheduler`` (DPM-Solver++(2M), arXiv:2211.01095) for the reference's
    configuration: the constructor keywords of the library class with the inference_v2.yaml:24-33 values as defaults, so
    ``DPMSolverMultistepScheduler(**noise_scheduler_kwargs)`` works (DDIM-only keys such as ``clip_sample`` are
    ignored).  Only the tables live here; the multistep history is per call and per frame in the pipeline, so one
    object serves any number of calls."""
    order = 1
    init_noise_sigma = 1.0
    _DDIM_ONLY = ("clip_sample", "clip_sample_range", "set_alpha_to_one")

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 trained_betas=None, solver_order=2, prediction_type="v_prediction", thresholding=False,
                 dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                 solver_type="midpoint", lower_order_final=True, euler_at_final=False, use_karras_sigmas=False,
                 use_lu_lambdas=False, final_sigmas_type="zero", lambda_min_clipped=-float("inf"), variance_type=None,
                 timestep_spacing="trailing", steps_offset=1, rescale_betas_zero_snr=True, **ddim_only):
        unknown = sorted(set(ddim_only) - set(self._DDIM_ONLY))
        if unknown:
            raise TypeError(f"DPMSolverMultistepScheduler got unexpected keyword arguments {unknown}")
        required = dict(trained_betas=(trained_betas, None), beta_schedule=(beta_schedule, "scaled_linear"),
                        prediction_type=(prediction_type, "v_prediction"), timestep_spacing=(timestep_spacing, "trailing"),
                        algorithm_type=(algorithm_type, "dpmsolver++"), solver_type=(solver_type, "midpoint"),
                        final_sigmas_type=(final_sigmas_type, "zero"), thresholding=(thresholding, False),
                        use_karras_sigmas=(use_karras_sigmas, False), use_lu_lambdas=(use_lu_lambdas, False),
                        variance_type=(variance_type, None))
        for name, (value, want) in required.items():
            if value is not want and value != want:
                raise ValueError(f"vexpress_b200.DPMSolverMultistepScheduler supports {name}={want!r} only, got {value!r}")
        if solver_order not in (1, 2):
            raise ValueError(f"vexpress_b200.DPMSolverMultistepScheduler supports solver_order 1 or 2, got {solver_order!r}")
        if not (isinstance(lambda_min_clipped, (int, float)) and math.isinf(lambda_min_clipped) and lambda_min_clipped < 0):
            raise ValueError(f"vexpress_b200.DPMSolverMultistepScheduler supports lambda_min_clipped=-inf only, got "
                             f"{lambda_min_clipped!r}")
        self.config = SimpleNamespace(
            num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
            beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
            prediction_type=prediction_type, thresholding=thresholding,
            dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
            algorithm_type=algorithm_type, solver_type=solver_type, lower_order_final=lower_order_final,
            euler_at_final=euler_at_final, use_karras_sigmas=use_karras_sigmas, use_lu_lambdas=use_lu_lambdas,
            final_sigmas_type=final_sigmas_type, lambda_min_clipped=lambda_min_clipped, variance_type=variance_type,
            timestep_spacing=timestep_spacing, steps_offset=steps_offset, rescale_betas_zero_snr=rescale_betas_zero_snr)
        self.betas = _scaled_linear_betas(num_train_timesteps, beta_start, beta_end, rescale_betas_zero_snr)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, 0)
        if rescale_betas_zero_snr:
            self.alphas_cumprod[-1] = 2 ** -24      # the library's clamp: the first sigma is finite (about 4096)
        self.num_inference_steps = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1, dtype=torch.int64)
        self.sigmas = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5

    @classmethod
    def from_config(cls, config):
        """From a dict or a config object (a diffusers scheduler's ``config``); keys this class does not take, such as
        DDIM's or diffusers' ``_class_name``, are ignored."""
        items = dict(config) if isinstance(config, dict) else \
            {k: getattr(config, k) for k in dir(config) if not k.startswith("_")}
        keys = set(inspect.signature(cls.__init__).parameters) - {"self", "ddim_only"}
        return cls(**{k: v for k, v in items.items() if k in keys})

    def set_timesteps(self, num_inference_steps, device=None):
        """Trailing spacing (DDIM's timesteps) and their sigmas followed by a final 0; both stay on the host."""
        n = self.config.num_train_timesteps
        self.num_inference_steps = num_inference_steps
        ts = np.round(np.arange(n, 0, -n / num_inference_steps)).astype(np.int64) - 1
        self.timesteps = torch.from_numpy(ts)
        table = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5
        self.sigmas = torch.cat([table[self.timesteps], torch.zeros(1)])

    def scale_model_input(self, sample, timestep=None):
        return sample


def dpm_scheduler(scheduler):
    """The ``DPMSolverMultistepScheduler`` that ``scheduler`` stands for: itself, or one built from the ``config`` of a
    diffusers ``DPMSolverMultistepScheduler`` (recognised by class name and its ``config`` / ``set_timesteps`` /
    ``step``, since diffusers is not a dependency) with the same ``set_timesteps`` applied.  None for every other
    scheduler, which runs the DDIM update."""
    if isinstance(scheduler, DPMSolverMultistepScheduler):
        return scheduler
    if type(scheduler).__name__ != "DPMSolverMultistepScheduler" or not all(
            hasattr(scheduler, a) for a in ("config", "set_timesteps", "step", "timesteps")):
        return None
    dpm = DPMSolverMultistepScheduler.from_config(scheduler.config)
    if getattr(scheduler, "num_inference_steps", None) is not None:
        dpm.set_timesteps(scheduler.num_inference_steps)
    return dpm


def _alpha_sigma(sigma):
    """diffusers' ``_sigma_to_alpha_sigma_t`` on a 0-d fp32 tensor."""
    alpha = 1 / ((sigma ** 2 + 1) ** 0.5)
    return alpha, sigma * alpha


def dpm_coefficients(scheduler, step_index, first=None):
    """(alpha_s, sigma_s, sigma_t / sigma_s, c0, 1 / r0, c0h, order) of step ``step_index`` (a position in the full
    ``scheduler.timesteps``) for ``vx_dpmpp_step``, as python floats from the fp32 0-d tensor arithmetic of diffusers'
    ``convert_model_output`` / ``dpm_solver_first_order_update`` / ``multistep_dpm_solver_second_order_update``:

        alpha = 1 / sqrt(sigma^2 + 1), sigma_vp = sigma * alpha, lambda = log(alpha) - log(sigma_vp)
        h = lambda_t - lambda_s,  c0 = alpha_t (e^-h - 1),  r0 = (lambda_s - lambda_s1) / h,  c0h = 0.5 c0

    The step is first order on the first step of a call (``first``, default ``step_index == 0``: no history yet), at
    ``solver_order == 1`` and on the last step; otherwise second order (1 / r0 and c0h are 0 at first order).  On the
    last step sigma_t = 0: lambda_t = +inf, e^-h = 0, c0 = -1 and the ratio 0, so the update returns the x0 prediction."""
    sig = scheduler.sigmas
    n = len(scheduler.timesteps)
    if not 0 <= step_index < n:
        raise ValueError(f"step_index {step_index} outside the {n}-step schedule")
    first = step_index == 0 if first is None else first
    order = 1 if first or scheduler.config.solver_order == 1 or step_index == n - 1 else 2
    alpha_t, sigma_t = _alpha_sigma(sig[step_index + 1])
    alpha_s, sigma_s = _alpha_sigma(sig[step_index])
    lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
    lambda_s = torch.log(alpha_s) - torch.log(sigma_s)
    h = lambda_t - lambda_s
    c0 = alpha_t * (torch.exp(-h) - 1.0)
    inv_r0 = c0h = 0.0
    if order == 2:
        alpha_s1, sigma_s1 = _alpha_sigma(sig[step_index - 1])
        r0 = (lambda_s - (torch.log(alpha_s1) - torch.log(sigma_s1))) / h
        inv_r0, c0h = float(1.0 / r0), float(0.5 * c0)
    return float(alpha_s), float(sigma_s), float(sigma_t / sigma_s), float(c0), inv_r0, c0h, order
