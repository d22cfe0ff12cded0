"""Sampling schedules (host side; the per-step arithmetic itself runs inside omg_fuse_step / omg_solver_step).

Restates the diffusers 0.25.0 schedulers the reference can be given (`KarrasDiffusionSchedulers`,
src/pipelines/lora_pipeline.py:176, instantid_pipeline.py:179; requirements.txt pins diffusers 0.25.0) [3P]:

  EulerDiscreteScheduler           timestep_spacing leading | trailing | linspace, steps_offset, use_karras_sigmas,
                                   interpolation_type linear, prediction_type epsilon | v_prediction,
                                   beta_schedule scaled_linear | linear
  EulerAncestralDiscreteScheduler  the same spacings, betas and prediction types (no Karras sigmas in 0.25)
  DPMSolverMultistepScheduler      algorithm_type dpmsolver++ | sde-dpmsolver++, solver_order 1 | 2,
                                   solver_type midpoint | heun, lower_order_final, euler_at_final,
                                   use_karras_sigmas, the three spacings, epsilon | v_prediction

Any other class or value raises ValueError naming the key and the value; nothing falls back silently.  The surface is
diffusers': `config` (a dict), `from_config(config, **overrides)` (keys the class does not take are ignored, as
diffusers does, so `DPMSolverMultistepScheduler.from_config(euler.config)` carries timestep_spacing and steps_offset
over), `set_timesteps(n)`, `timesteps`, `sigmas`, `init_noise_sigma`, `order`.  Tables are numpy arrays (they live on
the host; the kernels take per-step scalars).

What the code rests on, restated from memory of the diffusers 0.25.0 sources [3P] (tests/util_schedulers.py restates the
same recollection literally, in torch, with the classes' step() arithmetic):
  * betas: linear = linspace(beta_start, beta_end, N); scaled_linear = linspace(sqrt(start), sqrt(end), N)^2, float32;
    alphas_cumprod = cumprod(1 - betas); training sigmas = sqrt((1 - acp) / acp) in float32.
  * Euler / Euler-a set_timesteps: linspace = linspace(0, N-1, n)[::-1]; leading = arange(n) * (N // n), reversed,
    + steps_offset; trailing = round(arange(N, 0, -N/n)) - 1.  Sigmas: np.interp(timesteps, arange(N), sigmas);
    Euler + use_karras_sigmas: Karras rho = 7 ramp between the interpolated schedule's first and last sigma, and
    timesteps = _sigma_to_t(sigma) (float, log-sigma interpolation).  A final sigma of 0 is appended.
    init_noise_sigma = sigma_max for linspace / trailing, sqrt(sigma_max^2 + 1) for leading.
    scale_model_input divides by sqrt(sigma^2 + 1).
  * Euler step (s_churn 0): x0 = x - sigma * eps (epsilon) or eps * (-sigma / sqrt(sigma^2+1)) + x / (sigma^2+1)
    (v_prediction); x' = x + (x - x0) / sigma * (sigma' - sigma).
  * Euler-a step: sigma_up = sqrt(sigma'^2 (sigma^2 - sigma'^2) / sigma^2), sigma_down = sqrt(sigma'^2 - sigma_up^2);
    x' = x + (x - x0) / sigma * (sigma_down - sigma) + z * sigma_up, with z = randn(model_output.shape, fp16,
    generator) drawn on every step, the last (sigma_up = 0) included.
  * DPM-Solver++ set_timesteps: linspace = round(linspace(0, N-1, n+1))[::-1][:-1]; leading = arange(n+1) * (N // (n+1)),
    reversed, last dropped, + steps_offset; trailing = round(arange(N, 0, -N/n)) - 1; int64.  Non-Karras: interpolated
    sigmas + sigma_last = sqrt((1 - acp[0]) / acp[0]).  Karras: the ramp spans the full training sigmas, timesteps =
    round(_sigma_to_t(sigma)), and sigmas[-1] is repeated (the last step has h = 0).  Duplicate timesteps are dropped
    (np.unique, order kept) without touching the sigmas.  init_noise_sigma = 1, scale_model_input is the identity.
  * DPM-Solver++ step, with alpha = 1/sqrt(sigma^2+1), sigma_vp = sigma * alpha, lambda = log alpha - log sigma_vp:
    x0 = (x - sigma_vp * eps) / alpha (epsilon) or alpha * x - sigma_vp * v (v_prediction); first order when
    solver_order == 1, on the first step, or on the last step when euler_at_final or (lower_order_final and fewer than
    15 steps); else the multistep second-order update on D0 = x0, D1 = (x0 - x0_prev) / r0, r0 = h_prev / h.  The SDE
    variant draws z = randn(model_output.shape, fp16, generator) on every step.

Each schedule states, per step i, what the step kernel computes (float64 here, rounded to fp32 for the kernel):
    x0 = c_x * x + c_eps * eps;   x' = a * x + b * x0 + c * x0_prev + d * z;   next inputs = x' * s.
"""
import json
import math
import os
from typing import NamedTuple

import numpy as np

SDXL_BASE_CONFIG = {  # stable-diffusion-xl-base-1.0/scheduler/scheduler_config.json [3P]
    "_class_name": "EulerDiscreteScheduler", "beta_end": 0.012, "beta_schedule": "scaled_linear",
    "beta_start": 0.00085, "clip_sample": False, "interpolation_type": "linear", "num_train_timesteps": 1000,
    "prediction_type": "epsilon", "sample_max_value": 1.0, "set_alpha_to_one": False, "skip_prk_steps": True,
    "steps_offset": 1, "timestep_spacing": "leading", "trained_betas": None, "use_karras_sigmas": False,
}


class StepCoeffs(NamedTuple):
    """One step of x0 = c_x x + c_eps eps;  x' = a x + b x0 + c x0_prev + d z;  next inputs = x' * s."""
    c_x: float
    c_eps: float
    a: float
    b: float
    c: float
    d: float
    s: float


def _require(cls_name, key, value, allowed):
    if value not in allowed:
        raise ValueError(f"{cls_name}: {key}={value!r} is not supported (supported: {', '.join(map(repr, allowed))})")


def _sigma_to_t(sigma, log_sigmas):
    """diffusers _sigma_to_t: piecewise-linear interpolation of the timestep in log sigma [3P]."""
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    t = (1 - w) * low_idx + w * high_idx
    return t.reshape(np.shape(sigma))


def _karras(sigma_min: float, sigma_max: float, n: int, rho: float = 7.0):
    ramp = np.linspace(0, 1, n)
    min_inv, max_inv = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    return (max_inv + ramp * (min_inv - max_inv)) ** rho


class _Schedule:
    """Config handling and the tables every class shares."""
    order = 1
    stochastic = False      # draws z every step
    _defaults: dict = {}
    _class_name = ""

    def __init__(self, **kwargs):
        cfg = dict(self._defaults)
        for k, v in kwargs.items():
            if k not in cfg:
                raise ValueError(f"{self._class_name}: unknown argument {k!r}")
            cfg[k] = v
        self.config = dict(cfg, _class_name=self._class_name)
        n = self._class_name
        _require(n, "beta_schedule", cfg["beta_schedule"], ("scaled_linear", "linear"))
        _require(n, "trained_betas", cfg["trained_betas"], (None,))
        _require(n, "prediction_type", cfg["prediction_type"], ("epsilon", "v_prediction"))
        _require(n, "timestep_spacing", cfg["timestep_spacing"], ("leading", "trailing", "linspace"))
        if "rescale_betas_zero_snr" in cfg:
            _require(n, "rescale_betas_zero_snr", cfg["rescale_betas_zero_snr"], (False,))
        N = int(cfg["num_train_timesteps"])
        if cfg["beta_schedule"] == "scaled_linear":
            betas = np.linspace(cfg["beta_start"] ** 0.5, cfg["beta_end"] ** 0.5, N, dtype=np.float32) ** 2
        else:
            betas = np.linspace(cfg["beta_start"], cfg["beta_end"], N, dtype=np.float32)
        self.alphas_cumprod = np.cumprod((1.0 - betas).astype(np.float32), dtype=np.float32)
        self.num_train_timesteps = N
        self.steps_offset = int(cfg["steps_offset"])
        self.prediction_type = cfg["prediction_type"]
        self.timesteps = None
        self.sigmas = None

    @classmethod
    def from_config(cls, config, **overrides):
        """diffusers' `from_config`: the keys of `config` this class takes, then `overrides` (which must be its keys)."""
        kw = {k: v for k, v in dict(config).items() if k in cls._defaults}
        kw.update(overrides)
        return cls(**kw)

    def _train_sigmas(self):
        return ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5   # float32

    def _spaced_timesteps(self, n: int):
        """Euler / Euler-a spacing (float32)."""
        N, sp = self.num_train_timesteps, self.config["timestep_spacing"]
        if sp == "linspace":
            return np.linspace(0, N - 1, n, dtype=np.float32)[::-1].copy()
        if sp == "leading":
            ts = (np.arange(0, n) * (N // n)).round()[::-1].copy().astype(np.float32)
            return ts + self.steps_offset
        ts = np.arange(N, 0, -N / n).round().copy().astype(np.float32)
        return ts - 1

    @property
    def num_steps(self) -> int:
        return len(self.timesteps)

    def scheduler_key(self) -> str:
        """Canonical text of the config (cache keys)."""
        return json.dumps(self.config, sort_keys=True, default=str)

    # per-step values of the step kernel ------------------------------------------------------------------------
    @property
    def uses_fuse_step(self) -> bool:
        """True when the step is plain Euler on epsilon, the update omg_fuse_step computes."""
        return False

    @property
    def uses_history(self) -> bool:
        """True when a step reads the previous step's x0 (the caller keeps an fp32 history buffer)."""
        return False

    def input_scale(self, i: int) -> float:
        """Scale of the model inputs of step i (scale_model_input); i == num_steps gives the scale after the last step."""
        return 1.0

    def step_coeffs(self, i: int) -> StepCoeffs:
        raise NotImplementedError


class _EulerFamily(_Schedule):
    def _x0_coeffs(self, sigma: float):
        if self.prediction_type == "epsilon":
            return 1.0, -sigma
        return 1.0 / (sigma * sigma + 1.0), -sigma / math.sqrt(sigma * sigma + 1.0)

    @property
    def init_noise_sigma(self) -> float:
        smax = self.sigmas.max()
        if self.config["timestep_spacing"] in ("linspace", "trailing"):
            return float(smax)
        return float((smax ** 2 + 1) ** 0.5)

    def input_scale(self, i: int) -> float:
        return float(1.0 / (self.sigmas[i] ** 2 + 1) ** 0.5)


class EulerDiscreteScheduler(_EulerFamily):
    _class_name = "EulerDiscreteScheduler"
    _defaults = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                     trained_betas=None, prediction_type="epsilon", interpolation_type="linear",
                     use_karras_sigmas=False, sigma_min=None, sigma_max=None, timestep_spacing="linspace",
                     timestep_type="discrete", steps_offset=0, rescale_betas_zero_snr=False)

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        n = self._class_name
        _require(n, "interpolation_type", self.config["interpolation_type"], ("linear",))
        _require(n, "use_karras_sigmas", self.config["use_karras_sigmas"], (False, True))
        _require(n, "timestep_type", self.config["timestep_type"], ("discrete",))
        _require(n, "sigma_min", self.config["sigma_min"], (None,))
        _require(n, "sigma_max", self.config["sigma_max"], (None,))

    def set_timesteps(self, num_inference_steps: int):
        ts = self._spaced_timesteps(num_inference_steps)
        train = self._train_sigmas()
        sig = np.interp(ts, np.arange(0, len(train)), train)
        if self.config["use_karras_sigmas"]:
            sig = _karras(float(sig[-1]), float(sig[0]), num_inference_steps)
            log_sigmas = np.log(train)
            ts = np.array([_sigma_to_t(s, log_sigmas) for s in sig])
        self.sigmas = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.timesteps = ts.astype(np.float32)
        return self.timesteps

    @property
    def uses_fuse_step(self) -> bool:
        return self.prediction_type == "epsilon"

    def step_coeffs(self, i: int) -> StepCoeffs:
        s, s1 = float(self.sigmas[i]), float(self.sigmas[i + 1])
        c_x, c_eps = self._x0_coeffs(s)
        return StepCoeffs(c_x, c_eps, s1 / s, 1.0 - s1 / s, 0.0, 0.0, self.input_scale(i + 1))


class EulerDiscreteSchedule(EulerDiscreteScheduler):
    """EulerDiscreteScheduler configured by SDXL-base's scheduler_config.json (the default of both pipelines)."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 steps_offset: int = 1):
        super().__init__(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule="scaled_linear", timestep_spacing="leading", steps_offset=steps_offset)
        self.config["_class_name"] = "EulerDiscreteScheduler"

    @classmethod
    def from_config(cls, config, **overrides):
        return EulerDiscreteScheduler.from_config(config, **overrides)


class EulerAncestralDiscreteScheduler(_EulerFamily):
    _class_name = "EulerAncestralDiscreteScheduler"
    stochastic = True
    _defaults = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                     trained_betas=None, prediction_type="epsilon", timestep_spacing="linspace", steps_offset=0,
                     rescale_betas_zero_snr=False)

    def set_timesteps(self, num_inference_steps: int):
        ts = self._spaced_timesteps(num_inference_steps)
        train = self._train_sigmas()
        sig = np.interp(ts, np.arange(0, len(train)), train)
        self.sigmas = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.timesteps = ts.astype(np.float32)
        return self.timesteps

    def step_coeffs(self, i: int) -> StepCoeffs:
        s, s1 = float(self.sigmas[i]), float(self.sigmas[i + 1])
        c_x, c_eps = self._x0_coeffs(s)
        up = math.sqrt(s1 * s1 * (s * s - s1 * s1) / (s * s))
        down = math.sqrt(max(s1 * s1 - up * up, 0.0))
        return StepCoeffs(c_x, c_eps, down / s, 1.0 - down / s, 0.0, up, self.input_scale(i + 1))


class DPMSolverMultistepScheduler(_Schedule):
    _class_name = "DPMSolverMultistepScheduler"
    _defaults = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                     trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                     dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                     solver_type="midpoint", lower_order_final=True, euler_at_final=False, use_karras_sigmas=False,
                     use_lu_lambdas=False, lambda_min_clipped=-float("inf"), variance_type=None,
                     timestep_spacing="linspace", steps_offset=0)
    init_noise_sigma = 1.0

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        n, cfg = self._class_name, self.config
        _require(n, "solver_order", cfg["solver_order"], (1, 2))
        _require(n, "algorithm_type", cfg["algorithm_type"], ("dpmsolver++", "sde-dpmsolver++"))
        _require(n, "solver_type", cfg["solver_type"], ("midpoint", "heun"))
        _require(n, "thresholding", cfg["thresholding"], (False,))
        _require(n, "use_lu_lambdas", cfg["use_lu_lambdas"], (False,))
        _require(n, "variance_type", cfg["variance_type"], (None,))
        _require(n, "lambda_min_clipped", cfg["lambda_min_clipped"], (-float("inf"),))
        _require(n, "use_karras_sigmas", cfg["use_karras_sigmas"], (False, True))
        self.order = int(cfg["solver_order"])
        self.stochastic = cfg["algorithm_type"] == "sde-dpmsolver++"

    def set_timesteps(self, num_inference_steps: int):
        N, n, sp = self.num_train_timesteps, num_inference_steps, self.config["timestep_spacing"]
        last = N  # lambda_min_clipped = -inf clips nothing
        if sp == "linspace":
            ts = np.linspace(0, last - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif sp == "leading":
            ts = (np.arange(0, n + 1) * (last // (n + 1))).round()[::-1][:-1].copy().astype(np.int64)
            ts += self.steps_offset
        else:
            ts = np.arange(last, 0, -N / n).round().copy().astype(np.int64)
            ts -= 1
        train = self._train_sigmas()
        if self.config["use_karras_sigmas"]:
            log_sigmas = np.log(train)
            flipped = np.flip(train).copy()
            sig = _karras(float(flipped[-1]), float(flipped[0]), n)
            ts = np.array([_sigma_to_t(s, log_sigmas) for s in sig]).round()
            sig = np.concatenate([sig, sig[-1:]]).astype(np.float32)
        else:
            sig = np.interp(ts, np.arange(0, len(train)), train)
            sig_last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5
            sig = np.concatenate([sig, [sig_last]]).astype(np.float32)
        self.sigmas = sig
        _, first = np.unique(ts, return_index=True)
        self.timesteps = ts[np.sort(first)].astype(np.int64)
        return self.timesteps

    @property
    def uses_history(self) -> bool:
        return self.order == 2

    def _first_order(self, i: int) -> bool:
        n, cfg = self.num_steps, self.config
        final = i == n - 1 and (cfg["euler_at_final"] or (cfg["lower_order_final"] and n < 15))
        return self.order == 1 or i == 0 or final

    def step_coeffs(self, i: int) -> StepCoeffs:
        s0, st = float(self.sigmas[i]), float(self.sigmas[i + 1])
        a0 = 1.0 / math.sqrt(s0 * s0 + 1.0)
        if self.prediction_type == "epsilon":   # x0 = (x - sigma_vp eps) / alpha, sigma_vp / alpha = sigma
            c_x, c_eps = 1.0 / a0, -s0
        else:                                   # x0 = alpha x - sigma_vp v
            c_x, c_eps = a0, -s0 * a0
        if st == s0:
            # h = 0 (the repeated final Karras sigma): every update term vanishes and x' = x.  diffusers' midpoint
            # arithmetic gives exactly that; its heun coefficient (e^-h - 1)/h + 1 is 0/0 there, here its limit 0.
            return StepCoeffs(c_x, c_eps, 1.0, 0.0, 0.0, 0.0, 1.0)
        at = 1.0 / math.sqrt(st * st + 1.0)
        h = math.log(s0) - math.log(st)              # lambda_t - lambda_s0 with lambda = -log sigma
        sde = self.stochastic
        if sde:
            a = (st * at) / (s0 * a0) * math.exp(-h)
            B = at * -math.expm1(-2.0 * h)           # coefficient of D0
            d = st * at * math.sqrt(-math.expm1(-2.0 * h))
        else:
            a = (st * at) / (s0 * a0)
            B = -at * math.expm1(-h)
            d = 0.0
        if self._first_order(i):
            return StepCoeffs(c_x, c_eps, a, B, 0.0, d, 1.0)
        s1 = float(self.sigmas[i - 1])
        inv_r0 = h / (math.log(s1) - math.log(s0))   # 1 / r0 = h / h_0
        if self.config["solver_type"] == "midpoint":
            C = 0.5 * B                               # coefficient of D1
        elif sde:
            C = at * (-math.expm1(-2.0 * h) / (-2.0 * h) + 1.0)
        else:
            C = at * (math.expm1(-h) / h + 1.0)
        # D1 = (x0 - x0_prev) / r0
        return StepCoeffs(c_x, c_eps, a, B + C * inv_r0, -C * inv_r0, d, 1.0)


CLASSES = {c._class_name: c for c in (EulerDiscreteScheduler, EulerAncestralDiscreteScheduler,
                                       DPMSolverMultistepScheduler)}

# --scheduler of the CLIs: name -> (class, from_config overrides)
CLI_CHOICES = {
    "euler": (EulerDiscreteScheduler, {}),
    "euler_a": (EulerAncestralDiscreteScheduler, {}),
    "dpmpp_2m": (DPMSolverMultistepScheduler, {}),
    "dpmpp_2m_karras": (DPMSolverMultistepScheduler, {"use_karras_sigmas": True}),
    "dpmpp_2m_sde": (DPMSolverMultistepScheduler, {"algorithm_type": "sde-dpmsolver++"}),
    "dpmpp_2m_sde_karras": (DPMSolverMultistepScheduler, {"algorithm_type": "sde-dpmsolver++",
                                                          "use_karras_sigmas": True}),
}


def from_config(config: dict) -> _Schedule:
    """The class `config["_class_name"]` names, built from `config` (what diffusers' pipeline loading does)."""
    name = config.get("_class_name")
    if name not in CLASSES:
        raise ValueError(f"scheduler _class_name={name!r} is not supported (supported: {', '.join(CLASSES)})")
    return CLASSES[name].from_config(config)


def load_scheduler(model_dir) -> _Schedule:
    """`<model_dir>/scheduler/scheduler_config.json` when present, else SDXL-base's Euler (EulerDiscreteSchedule)."""
    path = os.path.join(os.fspath(model_dir), "scheduler", "scheduler_config.json")
    if not os.path.isfile(path):
        return EulerDiscreteSchedule()
    with open(path) as f:
        return from_config(json.load(f))


def cli_scheduler(name: str, config: dict) -> _Schedule:
    """`--scheduler name`: the class it names, `from_config(config, ...)` of the checkpoint's config."""
    if name not in CLI_CHOICES:
        raise ValueError(f"--scheduler {name!r} is not supported (supported: {', '.join(CLI_CHOICES)})")
    cls, over = CLI_CHOICES[name]
    return cls.from_config(config, **over)
