"""diffusers 0.25.0 EulerDiscreteScheduler, EulerAncestralDiscreteScheduler and DPMSolverMultistepScheduler restated
literally in torch [third-party recollection; omg_b200/scheduler.py lists what it rests on].  TEST INFRASTRUCTURE: the
step() arithmetic as diffusers writes it, float32 tables, the sample's dtype for the arithmetic, indexed by the step
index i instead of the timestep.  The tests check omg_b200/scheduler.py's coefficient form against these classes, and
run oracle.pipeline.denoise with one of them in place of its default Euler (`oracle_schedule`).  `configs()` lists the
host schedules every supported rule gives, for the CPU and kernel tests alike."""
import contextlib

import numpy as np
import torch


def _betas(cfg):
    N = cfg["num_train_timesteps"]
    if cfg["beta_schedule"] == "scaled_linear":
        return torch.linspace(cfg["beta_start"] ** 0.5, cfg["beta_end"] ** 0.5, N, dtype=torch.float32) ** 2
    return torch.linspace(cfg["beta_start"], cfg["beta_end"], N, dtype=torch.float32)


def _sigma_to_t(sigma, log_sigmas):
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low = log_sigmas[low_idx]
    high = log_sigmas[high_idx]
    w = (low - log_sigma) / (low - high)
    w = np.clip(w, 0, 1)
    t = (1 - w) * low_idx + w * high_idx
    return t.reshape(sigma.shape)


def _convert_to_karras(in_sigmas, num_inference_steps):
    sigma_min = in_sigmas[-1].item()
    sigma_max = in_sigmas[0].item()
    rho = 7.0
    ramp = np.linspace(0, 1, num_inference_steps)
    min_inv_rho = sigma_min ** (1 / rho)
    max_inv_rho = sigma_max ** (1 / rho)
    return (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho


class _Discrete:
    def __init__(self, noise_source=None, **cfg):
        self.config = cfg
        self.noise_source = noise_source   # i -> the noise step i draws (the generator's draws, replayed)
        self.alphas_cumprod = torch.cumprod(1.0 - _betas(cfg), dim=0)
        self.timesteps = self.sigmas = None

    def _euler_timesteps(self, n):
        cfg, N = self.config, self.config["num_train_timesteps"]
        if cfg["timestep_spacing"] == "linspace":
            return np.linspace(0, N - 1, n, dtype=np.float32)[::-1].copy()
        if cfg["timestep_spacing"] == "leading":
            step_ratio = N // n
            timesteps = (np.arange(0, n) * step_ratio).round()[::-1].copy().astype(np.float32)
            return timesteps + cfg["steps_offset"]
        step_ratio = N / n
        timesteps = (np.arange(N, 0, -step_ratio)).round().copy().astype(np.float32)
        return timesteps - 1

    @property
    def init_noise_sigma(self):
        max_sigma = self.sigmas.max()
        if self.config["timestep_spacing"] in ["linspace", "trailing"]:
            return float(max_sigma)
        return float((max_sigma ** 2 + 1) ** 0.5)

    def scale_model_input(self, sample, i):
        return sample / ((self.sigmas[i] ** 2 + 1) ** 0.5)

    def _pred_original(self, model_output, sample, sigma):
        if self.config["prediction_type"] == "epsilon":
            return sample - sigma * model_output
        return model_output * (-sigma / (sigma ** 2 + 1) ** 0.5) + (sample / (sigma ** 2 + 1))


class EulerDiscreteScheduler(_Discrete):
    def set_timesteps(self, n):
        timesteps = self._euler_timesteps(n)
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        log_sigmas = np.log(sigmas)
        sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
        if self.config.get("use_karras_sigmas", False):
            sigmas = _convert_to_karras(in_sigmas=sigmas, num_inference_steps=n)
            timesteps = np.array([_sigma_to_t(sigma, log_sigmas) for sigma in sigmas])
        sigmas = torch.from_numpy(sigmas).to(dtype=torch.float32)
        self.timesteps = torch.from_numpy(timesteps.astype(np.float32))
        self.sigmas = torch.cat([sigmas, torch.zeros(1)])
        return self.timesteps

    def step(self, model_output, i, sample, noise=None):
        sigma = self.sigmas[i]
        pred_original_sample = self._pred_original(model_output, sample, sigma)
        derivative = (sample - pred_original_sample) / sigma
        dt = self.sigmas[i + 1] - sigma
        return sample + derivative * dt


class EulerAncestralDiscreteScheduler(_Discrete):
    def set_timesteps(self, n):
        timesteps = self._euler_timesteps(n)
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
        sigmas = np.concatenate([sigmas, [0.0]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        self.timesteps = torch.from_numpy(timesteps)
        return self.timesteps

    def step(self, model_output, i, sample, noise=None):
        sigma = self.sigmas[i]
        pred_original_sample = self._pred_original(model_output, sample, sigma)
        sigma_from = self.sigmas[i]
        sigma_to = self.sigmas[i + 1]
        sigma_up = (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5
        sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
        derivative = (sample - pred_original_sample) / sigma
        dt = sigma_down - sigma
        prev_sample = sample + derivative * dt
        noise = self.noise_source(i) if noise is None else noise
        return prev_sample + noise.to(sample.dtype) * sigma_up


class DPMSolverMultistepScheduler(_Discrete):
    init_noise_sigma = 1.0

    def set_timesteps(self, n):
        cfg, N = self.config, self.config["num_train_timesteps"]
        last_timestep = N
        if cfg["timestep_spacing"] == "linspace":
            timesteps = np.linspace(0, last_timestep - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif cfg["timestep_spacing"] == "leading":
            step_ratio = last_timestep // (n + 1)
            timesteps = (np.arange(0, n + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            timesteps += cfg["steps_offset"]
        else:
            step_ratio = N / n
            timesteps = np.arange(last_timestep, 0, -step_ratio).round().copy().astype(np.int64)
            timesteps -= 1
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        log_sigmas = np.log(sigmas)
        if cfg.get("use_karras_sigmas", False):
            sigmas = np.flip(sigmas).copy()
            sigmas = _convert_to_karras(in_sigmas=sigmas, num_inference_steps=n)
            timesteps = np.array([_sigma_to_t(sigma, log_sigmas) for sigma in sigmas]).round()
            sigmas = np.concatenate([sigmas, sigmas[-1:]]).astype(np.float32)
        else:
            sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
            sigma_last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5
            sigmas = np.concatenate([sigmas, [sigma_last]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        _, unique_indices = np.unique(timesteps, return_index=True)
        timesteps = timesteps[np.sort(unique_indices)]
        self.timesteps = torch.from_numpy(timesteps).to(dtype=torch.int64)
        self.model_outputs = [None] * cfg.get("solver_order", 2)
        self.lower_order_nums = 0
        return self.timesteps

    def scale_model_input(self, sample, i):
        return sample

    @staticmethod
    def _sigma_to_alpha_sigma_t(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        sigma_t = sigma * alpha_t
        return alpha_t, sigma_t

    def convert_model_output(self, model_output, i, sample):
        sigma = self.sigmas[i]
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma)
        if self.config["prediction_type"] == "epsilon":
            return (sample - sigma_t * model_output) / alpha_t
        return alpha_t * sample - sigma_t * model_output

    def first_order_update(self, model_output, i, sample, noise):
        sigma_t, sigma_s = self.sigmas[i + 1], self.sigmas[i]
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma_t)
        alpha_s, sigma_s = self._sigma_to_alpha_sigma_t(sigma_s)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s = torch.log(alpha_s) - torch.log(sigma_s)
        h = lambda_t - lambda_s
        if self.config["algorithm_type"] == "dpmsolver++":
            return (sigma_t / sigma_s) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * model_output
        return ((sigma_t / sigma_s * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * model_output
                + sigma_t * torch.sqrt(1.0 - torch.exp(-2 * h)) * noise)

    def second_order_update(self, model_output_list, i, sample, noise):
        sigma_t, sigma_s0, sigma_s1 = self.sigmas[i + 1], self.sigmas[i], self.sigmas[i - 1]
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
        midpoint = self.config["solver_type"] == "midpoint"
        if self.config["algorithm_type"] == "dpmsolver++":
            if midpoint:
                return ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                        - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1)
            return ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                    + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1)
        if midpoint:
            return ((sigma_t / sigma_s0 * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * D0
                    + 0.5 * (alpha_t * (1 - torch.exp(-2.0 * h))) * D1
                    + sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h)) * noise)
        return ((sigma_t / sigma_s0 * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * D0
                + (alpha_t * ((1.0 - torch.exp(-2.0 * h)) / (-2.0 * h) + 1.0)) * D1
                + sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h)) * noise)

    def step(self, model_output, i, sample, noise=None):
        cfg = self.config
        n = len(self.timesteps)
        lower_order_final = (i == n - 1) and (cfg.get("euler_at_final", False)
                                              or (cfg.get("lower_order_final", True) and n < 15))
        model_output = self.convert_model_output(model_output, i, sample)
        order = cfg.get("solver_order", 2)
        for k in range(order - 1):
            self.model_outputs[k] = self.model_outputs[k + 1]
        self.model_outputs[-1] = model_output
        if cfg["algorithm_type"] == "dpmsolver++":
            noise = None
        else:
            noise = (self.noise_source(i) if noise is None else noise).to(sample.dtype)
        if order == 1 or self.lower_order_nums < 1 or lower_order_final:
            prev_sample = self.first_order_update(model_output, i, sample, noise)
        else:
            prev_sample = self.second_order_update(self.model_outputs, i, sample, noise)
        if self.lower_order_nums < order:
            self.lower_order_nums += 1
        return prev_sample


def make(cls_name: str, config: dict, noise_source=None):
    """The oracle class of that name from a full config dict (omg_b200.scheduler classes' `config`)."""
    return {"EulerDiscreteScheduler": EulerDiscreteScheduler,
            "EulerAncestralDiscreteScheduler": EulerAncestralDiscreteScheduler,
            "DPMSolverMultistepScheduler": DPMSolverMultistepScheduler}[cls_name](noise_source, **config)


def configs():
    """Every supported rule (name, host schedule) over the three spacings, built from SDXL-base's config as users do.
    The one function here that uses omg_b200.scheduler: the restatements above stay independent of it."""
    from omg_b200 import scheduler as S
    BASE = S.SDXL_BASE_CONFIG
    out = []
    for sp in ("leading", "trailing", "linspace"):
        for k in (False, True):
            for pt in ("epsilon", "v_prediction"):
                out.append((f"euler-{sp}-karras{int(k)}-{pt}",
                            S.EulerDiscreteScheduler.from_config(BASE, timestep_spacing=sp, use_karras_sigmas=k,
                                                                 prediction_type=pt)))
        for pt in ("epsilon", "v_prediction"):
            out.append((f"euler_a-{sp}-{pt}",
                        S.EulerAncestralDiscreteScheduler.from_config(BASE, timestep_spacing=sp, prediction_type=pt)))
        for k in (False, True):
            for alg in ("dpmsolver++", "sde-dpmsolver++"):
                for st in ("midpoint", "heun"):
                    for pt in ("epsilon", "v_prediction"):
                        out.append((f"dpm-{sp}-karras{int(k)}-{alg}-{st}-{pt}",
                                    S.DPMSolverMultistepScheduler.from_config(
                                        BASE, timestep_spacing=sp, use_karras_sigmas=k, algorithm_type=alg,
                                        solver_type=st, prediction_type=pt)))
    out.append(("dpm-order1", S.DPMSolverMultistepScheduler.from_config(BASE, solver_order=1)))
    out.append(("dpm-no-lower-order-final", S.DPMSolverMultistepScheduler.from_config(BASE, lower_order_final=False)))
    out.append(("dpm-euler-at-final", S.DPMSolverMultistepScheduler.from_config(BASE, euler_at_final=True)))
    out.append(("euler-linear-betas", S.EulerDiscreteScheduler.from_config(BASE, beta_schedule="linear",
                                                                           beta_start=0.0001, beta_end=0.02)))
    return out


@contextlib.contextmanager
def oracle_schedule(schedule):
    """oracle.pipeline.denoise with `schedule` in place of its default EulerDiscrete() (the loop builds its scheduler
    by calling that name): the same oracle loop, another scheduler."""
    from oracle import pipeline as op
    default = op.EulerDiscrete
    op.EulerDiscrete = lambda: schedule
    try:
        yield
    finally:
        op.EulerDiscrete = default
