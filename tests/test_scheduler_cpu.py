"""CPU tests of the sampling schedules (omg_b200/scheduler.py): tables and per-step coefficients against the literal
diffusers 0.25.0 restatements of tests/util_schedulers.py, config handling, omg_solver_step's argument checks and the CLI
flag."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from omg_b200 import scheduler as S
import util_schedulers as O  # noqa: E402
from util_schedulers import configs  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = S.SDXL_BASE_CONFIG
STEPS = (2, 3, 14, 15, 16, 20, 25, 30, 50)


CONFIGS = configs()


def oracle_of(s):
    return O.make(s.config["_class_name"], {k: v for k, v in s.config.items() if k != "_class_name"})


@pytest.mark.parametrize("name,s", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_tables_match_the_oracle(name, s):
    """Timesteps, sigmas, init_noise_sigma and input scales.  The host builds its float32 betas with numpy (as the
    SDXL-base schedule always has), the oracle with torch as diffusers does: the two differ in the last bits of
    alphas_cumprod, hence rtol 1e-5 on sigmas and a 1e-3 tolerance on the log-sigma-interpolated Karras timesteps of
    Euler (integer timesteps are exact)."""
    for n in STEPS:
        ts = s.set_timesteps(n)
        o = oracle_of(s)
        ots = o.set_timesteps(n).numpy()
        assert ts.dtype == ots.dtype and ts.shape == ots.shape, (n, ts.dtype, ots.dtype)
        if ts.dtype == np.int64 or not s.config.get("use_karras_sigmas"):
            assert np.array_equal(ts, ots), n
        else:
            np.testing.assert_allclose(ts, ots, atol=1e-3, rtol=0)
        np.testing.assert_allclose(s.sigmas, o.sigmas.numpy(), rtol=1e-5, atol=0)
        assert math.isclose(s.init_noise_sigma, o.init_noise_sigma, rel_tol=1e-6)
        x = torch.ones(1, dtype=torch.float64)
        for i in range(len(ts)):
            assert math.isclose(s.input_scale(i), float(o.scale_model_input(x, i)), rel_tol=1e-6)
        assert np.all(np.isfinite(s.sigmas))


def test_sdxl_sigma_range_and_base_config_reproduces_the_default_schedule():
    s = S.DPMSolverMultistepScheduler.from_config(BASE, use_karras_sigmas=True)
    s.set_timesteps(25)
    assert abs(s.sigmas[0] - 14.6146) < 1e-3 and abs(s.sigmas[-1] - 0.0292) < 1e-4
    text = json.dumps(BASE)   # the checkpoint's file as it is read
    for n in STEPS:
        a, b = S.from_config(json.loads(text)), S.EulerDiscreteSchedule()
        assert type(a) is S.EulerDiscreteScheduler and a.uses_fuse_step
        assert np.array_equal(a.set_timesteps(n), b.set_timesteps(n))
        assert np.array_equal(a.sigmas, b.sigmas) and a.init_noise_sigma == b.init_noise_sigma
        assert all(a.input_scale(i) == b.input_scale(i) for i in range(n + 1))


def test_from_config_carries_spacing_and_offset():
    euler = S.EulerDiscreteScheduler.from_config(BASE)
    dpm = S.DPMSolverMultistepScheduler.from_config(euler.config, use_karras_sigmas=False)
    assert dpm.config["timestep_spacing"] == "leading" and dpm.config["steps_offset"] == 1
    assert "interpolation_type" not in dpm.config      # not a DPM argument: ignored
    ts = dpm.set_timesteps(20)
    assert ts[0] == 20 * (1000 // 21) + 1 and ts[-1] == 1000 // 21 + 1
    assert dpm.init_noise_sigma == 1.0 and dpm.input_scale(3) == 1.0 and dpm.order == 2


def test_load_scheduler_reads_the_checkpoint_config(tmp_path):
    assert type(S.load_scheduler(tmp_path)) is S.EulerDiscreteSchedule
    os.makedirs(tmp_path / "scheduler")
    cfg = dict(BASE, _class_name="DPMSolverMultistepScheduler", use_karras_sigmas=True)
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(cfg))
    s = S.load_scheduler(tmp_path)
    assert type(s) is S.DPMSolverMultistepScheduler and s.config["use_karras_sigmas"]


@pytest.mark.parametrize("make,msg", [
    (lambda: S.from_config(dict(BASE, _class_name="UniPCMultistepScheduler")), "UniPCMultistepScheduler"),
    (lambda: S.from_config(dict(BASE, _class_name="HeunDiscreteScheduler")), "HeunDiscreteScheduler"),
    (lambda: S.DPMSolverMultistepScheduler.from_config(BASE, solver_order=3), "solver_order=3"),
    (lambda: S.DPMSolverMultistepScheduler.from_config(BASE, algorithm_type="dpmsolver"), "algorithm_type='dpmsolver'"),
    (lambda: S.DPMSolverMultistepScheduler.from_config(BASE, solver_type="bh2"), "solver_type='bh2'"),
    (lambda: S.DPMSolverMultistepScheduler.from_config(BASE, thresholding=True), "thresholding=True"),
    (lambda: S.EulerDiscreteScheduler.from_config(BASE, trained_betas=[0.1] * 1000), "trained_betas="),
    (lambda: S.EulerDiscreteScheduler.from_config(BASE, rescale_betas_zero_snr=True), "rescale_betas_zero_snr=True"),
    (lambda: S.EulerDiscreteScheduler.from_config(BASE, prediction_type="sample"), "prediction_type='sample'"),
    (lambda: S.EulerDiscreteScheduler.from_config(BASE, interpolation_type="log_linear"), "interpolation_type="),
    (lambda: S.EulerDiscreteScheduler.from_config(BASE, timestep_spacing="even"), "timestep_spacing='even'"),
    (lambda: S.EulerDiscreteScheduler.from_config(BASE, beta_schedule="squaredcos_cap_v2"), "beta_schedule="),
    (lambda: S.EulerAncestralDiscreteScheduler.from_config(BASE, use_karras_sigmas=True), "use_karras_sigmas"),
    (lambda: S.cli_scheduler("lms", BASE), "'lms'"),
])
def test_unsupported_values_raise_naming_them(make, msg):
    with pytest.raises(ValueError, match=None) as e:
        make()
    assert msg in str(e.value), str(e.value)


def run_trajectory(s, n, coeff_form: bool):
    """A whole float64 trajectory with a fake model (a fixed nonlinear map of x and t) and fixed noise: the host's
    coefficient form, or the oracle's literal step() sequence."""
    g = torch.Generator().manual_seed(n)
    x = torch.randn(2, 4, 6, 5, generator=g, dtype=torch.float64)
    noises = [torch.randn(2, 4, 6, 5, generator=g, dtype=torch.float64) for _ in range(60)]
    ts = s.set_timesteps(n)
    o = None if coeff_form else oracle_of(s)
    if o is not None:
        o.set_timesteps(n)
        o.sigmas = torch.from_numpy(s.sigmas)   # same float32 table on both sides: the algebra is under test
    x = x * s.init_noise_sigma
    hist = torch.zeros_like(x)
    for i in range(len(ts)):
        xin = x * s.input_scale(i)
        eps = torch.tanh(xin) * (1 + float(ts[i]) / 1000) + 0.1 * xin
        if coeff_form:
            k = s.step_coeffs(i)
            x0 = k.c_x * x + k.c_eps * eps
            x = k.a * x + k.b * x0 + k.c * hist + k.d * noises[i]
            hist = x0
        else:
            x = o.step(eps, i, x, noise=noises[i])
    return x


@pytest.mark.parametrize("name,s", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_coefficient_form_matches_the_literal_steps(name, s):
    heun_h0 = "karras1" in name and "heun" in name
    for n in STEPS:
        mine = run_trajectory(s, n, True)
        ref = run_trajectory(s, n, False)
        assert torch.isfinite(mine).all(), (name, n)
        if torch.isnan(ref).any():
            # diffusers' heun coefficient (e^-h - 1)/h + 1 is 0/0 on the repeated final Karras sigma (h = 0) of a
            # second-order last step, a NaN times D1 = 0; the host takes its limit, 0, which leaves x as it is
            m = len(s.timesteps)
            assert heun_h0 and n >= 15 and s.sigmas[m] == s.sigmas[m - 1], (name, n)
            continue
        # the oracle forms its scalar factors (dt, sigma_up, h, ...) from float32 0-d tensors as diffusers does, the
        # host in float64: 1e-5 bounds that rounding; an algebra slip shows up at O(1)
        err = ((mine - ref).abs().max() / ref.abs().max()).item()
        assert err < 1e-5, (name, n, err)


def test_karras_final_step_is_the_identity_and_lower_order_final():
    s = S.DPMSolverMultistepScheduler.from_config(BASE, use_karras_sigmas=True)
    s.set_timesteps(20)
    assert s.sigmas[-1] == s.sigmas[-2]
    k = s.step_coeffs(19)
    assert (k.a, k.b, k.c, k.d, k.s) == (1.0, 0.0, 0.0, 0.0, 1.0)
    s.set_timesteps(10)   # fewer than 15 steps: the last step is first order (no history term)
    assert s.step_coeffs(9).c == 0.0 and s.step_coeffs(8).c != 0.0 and s.step_coeffs(0).c == 0.0
    s.set_timesteps(20)
    assert s.step_coeffs(18).c != 0.0


def test_euler_ancestral_last_step_has_no_noise_term():
    s = S.EulerAncestralDiscreteScheduler.from_config(BASE)
    s.set_timesteps(20)
    k = s.step_coeffs(19)
    assert k.d == 0.0 and k.a == 0.0 and k.b == 1.0 and s.stochastic
    assert all(s.step_coeffs(i).d > 0 for i in range(19))


def test_cli_choices_map_to_from_config():
    for name, (cls, over) in S.CLI_CHOICES.items():
        s = S.cli_scheduler(name, BASE)
        assert type(s) is cls
        assert s.config["timestep_spacing"] == "leading" and s.config["steps_offset"] == 1
        for k, v in over.items():
            assert s.config[k] == v
    assert S.cli_scheduler("dpmpp_2m_sde_karras", BASE).stochastic


@pytest.mark.parametrize("cli", ["inference_lora.py", "inference_instantid.py"])
def test_cli_flag_parsing(cli):
    r = subprocess.run([sys.executable, os.path.join(ROOT, cli), "--help"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and "--scheduler" in r.stdout
    for name in S.CLI_CHOICES:
        assert name in r.stdout
    r = subprocess.run([sys.executable, os.path.join(ROOT, cli), "--scheduler", "ddim", "--synthetic"],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 2 and "invalid choice: 'ddim'" in r.stderr


def test_solver_step_rejects_bad_descriptors_before_touching_the_gpu():
    from omg_b200 import _lib as L
    lib = L.load()
    ok, off8, off4 = 0x1000, 0x1008, 0x1004

    def solver(**kw):
        d = L.SolverDesc()
        f = d.fuse
        f.n_concepts, f.HW, f.guidance = 1, 64, 7.5
        f.noise_main = f.latents = f.next_main_in = f.next_concept_in = f.latents_f16 = ok
        f.noise_concept[0] = f.mask[0] = ok
        d.c_x, d.c_eps, d.a, d.b, d.c, d.d, d.input_scale = 1.0, -1.0, 0.5, 0.5, 0.25, 0.1, 1.0
        d.history, d.noise, d.store_x0 = ok, ok, 1
        for k, v in kw.items():
            if k == "noise_concept":
                f.noise_concept[0] = v
            elif hasattr(f, k):
                setattr(f, k, v)
            else:
                setattr(d, k, v)
        return lib.omg_solver_step(C.byref(d), None)

    cases = [
        (lambda: lib.omg_solver_step(None, None), "omg_solver_step: null pointer"),
        (lambda: solver(noise_main=None), "omg_solver_step: null pointer"),
        (lambda: solver(latents=None), "omg_solver_step: null pointer"),
        (lambda: solver(n_concepts=9), "omg_solver_step: n_concepts=9 out of range"),
        (lambda: solver(n_concepts=-1), "omg_solver_step: n_concepts=-1 out of range"),
        (lambda: solver(HW=0), "omg_solver_step: empty latent"),
        (lambda: solver(noise_concept=None), "omg_solver_step: concept 0 has a mask but no noise prediction"),
        (lambda: solver(noise=None), "omg_solver_step: d=0.1 needs noise"),
        (lambda: solver(history=None), "omg_solver_step: c=0.25 / store_x0=1 needs history"),
        (lambda: solver(history=None, c=0.0), "omg_solver_step: c=0 / store_x0=1 needs history"),
        (lambda: solver(latents=off8), "omg_solver_step: latents must be 16 B"),
        (lambda: solver(next_main_in=off8), "omg_solver_step: next_main_in must be 16 B"),
        (lambda: solver(next_concept_in=off8), "omg_solver_step: next_concept_in must be 16 B"),
        (lambda: solver(noise_main=off4), "omg_solver_step: noise_main must be 8 B"),
        (lambda: solver(noise_concept=off4), "omg_solver_step: noise_concept must be 8 B"),
        (lambda: solver(latents_f16=off8 + 2), "omg_solver_step: latents_f16 must be 4 B"),
        (lambda: solver(history=off8), "omg_solver_step: history must be 16 B"),
        (lambda: solver(noise=ok + 1), "omg_solver_step: noise must be 2 B"),
    ]
    for call, msg in cases:
        n0 = lib.omg_launch_count()
        rc = call()
        e = lib.omg_last_error().decode()
        assert rc == 1 and e.startswith(msg), (msg, rc, e)
        assert lib.omg_launch_count() == n0, msg
    # no noise needed when d == 0, no history when c == 0 and x0 is not stored: those pass validation (no call here
    # launches: the device pointers are fake, so only the checks are exercised above)
