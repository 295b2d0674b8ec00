"""DDIM scheduler restated for the hot path (diffusers 0.29.2 ``DDIMScheduler`` with the reference's
configuration inference_v2.yaml:23-33: scaled-linear betas, zero-terminal-SNR rescale, v-prediction, trailing
timestep spacing; SURVEY.md Appendix B.5).  Host-side scalar tables only: the tensor update itself is the fused
``vx_ddim_step`` kernel, or ``vx_ddim_step_eta`` for stochastic DDIM (eta > 0)."""
from types import SimpleNamespace

import numpy as np
import torch


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
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        if rescale_betas_zero_snr:
            root = torch.cumprod(1.0 - betas, 0).sqrt()
            first, last = root[0].clone(), root[-1].clone()
            root = (root - last) * (first / (first - last))
            abar = root ** 2
            betas = 1 - torch.cat([abar[:1], abar[1:] / abar[:-1]])
        self.betas = betas
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
