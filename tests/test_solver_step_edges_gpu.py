"""Edge tests of the sampling step kernels (omg_solver_step, omg_fuse_step) through the C ABI, in the conventions of
test_kernel_edges_gpu.py:

* `check` bounds every element:  |out - ref| <= 4 u |ref| + k u rms(ref)  with u = 2^-24 (fp32) or 2^-11 (fp16), plus
  "no NaN / inf".  `pytest -s` prints the k each case needs.
* Every output lies inside a flat NaN-filled `Guard` buffer whose outside must stay bit-identical; every fp16 noise row
  carries NaN in channels 4..7, and every input buffer is followed by NaN, so a read outside an operand shows up as NaN.
* An operand a step must not read (the history when c == 0, the noise z when d == 0) is NaN.

Whole schedules: every supported configuration runs end to end through the kernel, with a fake model that reads the
kernel's own fp16 next inputs as the UNet does.  The float64 reference applies fusion, guidance and the coefficient form
to the predictions and noise the kernel was given (recorded), so the two runs differ only by rounding; the kernel's
error after every step is bounded relative to what diffusers' own float32 arithmetic (the literal restatement of
util_schedulers.py) makes of the same inputs.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from util_schedulers import configs, make  # noqa: E402

PAD = 8
U32, U16 = 2.0 ** -24, 2.0 ** -11
GUIDANCE = 7.5
H, W = 24, 40                # 960 latent pixels: rectangular, not a multiple of the kernel's 128-pixel blocks
HW = H * W
# DPM's final step is first order below 15 steps and second order from 15 on; with Karras sigmas it is the identity
STEP_COUNTS = (3, 10, 15, 20)

# Bounds, with what the cases need on an NVIDIA H100 80GB HBM3 at a 700 W power limit.  Whole schedules: the kernel's
# per-element k of the fp32 latents / history, worst over the steps of a case, is at most K_FACTOR times the k the
# float32 literal restatement needs on the same inputs, or K_FLOOR.  Measured: at most 1.78 x the literal's k for the
# latents and 1.52 x for the history; the largest k where the factor does not cover it is 36.8 (literal 20.7,
# DPM-Solver++ 2M heun, Karras, 3 steps); the largest k overall is 1346 (literal 1423, Euler on linear betas, whose
# sigma_max of 157 dominates the absolute error; the error of the sigma ~ 14 SDXL schedules stays below 850).
K_FACTOR = 2.5
K_FLOOR = 64.0
K_NEXT = 1.0      # fp16 next inputs (u = 2^-11): measured 0.08
K_STEP = 4.0      # one step, fp32 outputs, coefficients exact in fp32: measured 1.86 (latents), 1.19 (history)


def need(out, ref, u):
    o, r = out.double(), ref.double()
    assert torch.isfinite(o).all(), "non-finite output"
    rms = r.pow(2).mean().sqrt().clamp_min(1e-30)
    return (((o - r).abs() - 4 * u * r.abs()) / (u * rms)).max().item()


def check(out, ref, k, u, what):
    n = need(out, ref, u)
    print(f"[check] {what}: k needed {n:.2f} (bound {k})")
    assert n <= k, f"{what}: per-element error needs k = {n:.2f} > {k}"


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


class Guard:
    """Contiguous output view of `shape` inside a NaN-filled buffer, PAD elements before and after."""

    def __init__(self, shape, dtype=torch.float16):
        n = math.prod(shape)
        self.buf = torch.full((n + 2 * PAD,), float("nan"), dtype=dtype, device="cuda")
        self.out = self.buf[PAD:PAD + n].view(shape)
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        self.inside[PAD:PAD + n] = True
        self.before = self.buf.clone()

    def intact(self):
        return bool(((_bits(self.buf) == _bits(self.before)) | self.inside).all())

    def untouched(self):
        return same_bits(self.buf, self.before)


def tailed(t):
    """t (contiguous) at the start of a NaN-filled buffer with PAD rows of NaN after it."""
    row = t.shape[-1] if t.dim() > 1 else 1
    buf = torch.full((t.numel() + PAD * row,), float("nan"), dtype=t.dtype, device="cuda")
    v = buf[:t.numel()].view(t.shape)
    v.copy_(t)
    return v


def noise_rows(vals):
    """fp16 [rows, HW, 8] prediction buffer: `vals` [rows, HW, 4] in channels 0..3, NaN in 4..7 and after the end."""
    t = torch.full(vals.shape[:-1] + (8,), float("nan"), dtype=torch.float16, device="cuda")
    t[..., :4] = vals.half()
    return tailed(t)


def twice(run):
    """run() -> list of output tensors; a second run from the same state must reproduce them bit for bit."""
    a, b = run(), run()
    for x, y in zip(a, b):
        assert same_bits(x, y), "second run differs"
    return a


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


def guided(nm, ncs, masks, dtype):
    """Region fusion and guidance of fp16 predictions (channels 0..3) in `dtype`: the guided eps of images 0 and 1,
    [2, hw, 4].  Concepts accumulate in index order inside their mask (`mask == 1`), as the kernel does."""
    n = nm[..., :4].to(dtype)
    hw = n.shape[1]
    u1, c1 = n[1].clone(), n[3].clone()
    union = torch.zeros(hw, dtype=torch.bool, device=n.device)
    au = torch.zeros(hw, 4, dtype=dtype, device=n.device)
    ac = torch.zeros(hw, 4, dtype=dtype, device=n.device)
    for nc, m in zip(ncs, masks):
        if m is None:
            continue
        sel = m.to(n.device) == 1
        union |= sel
        au[sel] += nc[0, sel, :4].to(dtype)
        ac[sel] += nc[1, sel, :4].to(dtype)
    u1[union], c1[union] = au[union], ac[union]
    return torch.stack([n[0] + GUIDANCE * (n[2] - n[0]), u1 + GUIDANCE * (c1 - u1)])


# ------------------------------------------------------------------------------------------------------ whole schedules
def _region_masks():
    m = torch.zeros(2, H, W, device="cuda")
    m[0, 2:20, 3:26] = 1
    m[1, 6:23, 14:38] = 1        # overlaps concept 0 on rows 6..19, columns 14..25
    return [tailed(m[0].reshape(HW).contiguous()), tailed(m[1].reshape(HW).contiguous())]


def fake_model(xin, t, gains):
    """A fixed nonlinear map of the fp16 model inputs (channels 0..3) and the timestep, one gain per batch row (so the
    cond rows differ from the uncond rows and guidance matters), rounded to fp16 as the UNet's output is.  It vanishes
    at a fixed O(1) pattern rather than at 0, so the latents a schedule ends on stay O(1): a map that vanishes at 0
    drives them to ~1e-6, where the absolute rounding error of the sigma ~ 14 steps swamps any relative bound."""
    x = xin[..., :4].double()
    idx = torch.arange(x.shape[1] * 4, dtype=torch.float64, device=x.device).view(x.shape[1], 4)
    y = x - torch.sin(0.37 * idx) * 1.5
    g = torch.tensor(gains, dtype=torch.float64, device=x.device).view(-1, 1, 1)
    return (torch.tanh(y) * (1 + t / 1000) * g + 0.1 * y).half()


MAIN_GAINS = (1.0, 0.95, 1.3, 1.4)          # uncond0, uncond1, cond0, cond1
CONCEPT_GAINS = ((0.9, 1.25), (1.1, 1.5))   # (uncond, cond) of each concept


def _cases():
    out = []
    for name, s in configs():
        kernels = ("solver", "fuse") if s.uses_fuse_step else ("solver",)
        for n in STEP_COUNTS:
            for kern in kernels:
                out.append(pytest.param(name, s, n, kern, id=f"{name}-n{n}-{kern}"))
    return out


@pytest.mark.parametrize("name,s,n,kernel", _cases())
def test_whole_schedule(ops, name, s, n, kernel):
    ts = s.set_timesteps(n)
    m = len(ts)
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + len(name))
    x_init = torch.randn(2, H, W, 4, generator=g, device="cuda") * s.init_noise_sigma
    masks = _region_masks()
    lat = Guard((2, H, W, 4), torch.float32)
    hist = Guard((2, H, W, 4), torch.float32)      # NaN: step 0 has c = 0 and must not read it
    nxt, nxc, l16 = Guard((4, HW, 8)), Guard((2, HW, 8)), Guard((2, H, W, 4))
    lat.out.copy_(x_init)
    s0 = s.input_scale(0)
    xin = (x_init * s0).reshape(2, HW, 4)
    nxt.out.zero_()
    nxt.out[..., :4] = torch.cat([xin, xin]).half()
    nxc.out.zero_()
    nxc.out[..., :4] = torch.stack([xin[1], xin[1]]).half()
    nan_z = tailed(torch.full((2, 4, H, W), float("nan"), dtype=torch.float16, device="cuda"))

    # float64 reference and float32 literal restatement, both on the recorded inputs
    xr, hr = x_init.double(), None
    o = make(s.config["_class_name"], {a: v for a, v in s.config.items() if a != "_class_name"})
    o.set_timesteps(n)
    o.sigmas = torch.from_numpy(s.sigmas)
    xl = x_init.cpu()
    dpm = s.config["_class_name"] == "DPMSolverMultistepScheduler"
    worst = {"latents": [0.0, 0.0], "history": [0.0, 0.0], "next_main_in": 0.0, "next_concept_in": 0.0}
    literal_ok = True

    for i in range(m):
        k = s.step_coeffs(i)
        t = float(ts[i])
        nm = noise_rows(fake_model(nxt.out, t, MAIN_GAINS))
        ncs = [noise_rows(fake_model(nxc.out, t, gk)) for gk in CONCEPT_GAINS]
        z = None
        if s.stochastic:
            z = tailed(torch.randn((2, 4, H, W), generator=g, device="cuda", dtype=torch.float16))
        before = lat.out.clone()
        if kernel == "fuse":
            ops.fuse_step(nm, ncs, masks, GUIDANCE, float(s.sigmas[i]), float(s.sigmas[i + 1]), lat.out, nxt.out,
                          nxc.out, latents_f16=l16.out)
        else:
            ops.solver_step(nm, ncs, masks, GUIDANCE, k, lat.out, nxt.out, nxc.out, l16.out, history=hist.out,
                            store_x0=True, noise=None if z is None else (z if k.d != 0 else nan_z))
        torch.cuda.synchronize()
        what = f"{name} n={n} {kernel} step {i}"
        assert lat.intact() and hist.intact() and nxt.intact() and nxc.intact() and l16.intact(), what

        eps = guided(nm, ncs, masks, torch.float64).view(2, H, W, 4)
        x0r = k.c_x * xr + k.c_eps * eps
        xn = k.a * xr + k.b * x0r
        if k.c != 0:
            xn = xn + k.c * hr
        if k.d != 0:
            xn = xn + k.d * z.double().permute(0, 2, 3, 1)
        xr, hr = xn, x0r

        if literal_ok:
            e32 = guided(nm.cpu(), [c.cpu() for c in ncs], [mk.cpu() for mk in masks], torch.float32).view(2, H, W, 4)
            zl = None if z is None else z.float().permute(0, 2, 3, 1).cpu()
            x0l = None if dpm else o._pred_original(e32, xl, o.sigmas[i])
            xl = o.step(e32, i, xl, noise=zl)
            if dpm:
                x0l = o.model_outputs[-1]   # the converted model output of this step: its x0
            if torch.isfinite(xl).all():
                worst["latents"][1] = max(worst["latents"][1], need(xl, xr.cpu(), U32))
                worst["history"][1] = max(worst["history"][1], need(x0l, x0r.cpu(), U32))
            else:
                # diffusers' heun coefficient is 0/0 on the repeated final Karras sigma (see test_scheduler_cpu.py)
                assert i == m - 1 and s.sigmas[i] == s.sigmas[i + 1], what
                literal_ok = False

        worst["latents"][0] = max(worst["latents"][0], need(lat.out, xr, U32))
        if kernel == "solver":
            worst["history"][0] = max(worst["history"][0], need(hist.out, x0r, U32))
        sc = (xr * k.s).reshape(2, HW, 4)
        worst["next_main_in"] = max(worst["next_main_in"], need(nxt.out[..., :4], torch.cat([sc, sc]), U16))
        worst["next_concept_in"] = max(worst["next_concept_in"],
                                       need(nxc.out[..., :4], torch.stack([sc[1], sc[1]]), U16))
        assert (_bits(nxt.out[..., 4:]) == 0).all() and (_bits(nxc.out[..., 4:]) == 0).all(), what
        assert same_bits(l16.out, lat.out.half()), what
        if (k.a, k.b, k.c, k.d) == (1.0, 0.0, 0.0, 0.0):
            assert same_bits(lat.out, before), f"{what}: the identity step changed the latents"

    print(f"[schedule] {name} n={n} {kernel}: latents k {worst['latents'][0]:.1f} (literal fp32 "
          f"{worst['latents'][1]:.1f}), history k {worst['history'][0]:.1f} (literal fp32 {worst['history'][1]:.1f}), "
          f"next_main_in k {worst['next_main_in']:.2f}, next_concept_in k {worst['next_concept_in']:.2f}")
    for q in ("latents", "history") if kernel == "solver" else ("latents",):
        mine, lit = worst[q]
        bound = max(K_FACTOR * lit, K_FLOOR)
        assert mine <= bound, f"{name} n={n} {kernel} {q}: k = {mine:.1f} > {bound:.1f} (literal fp32 {lit:.1f})"
    assert worst["next_main_in"] <= K_NEXT and worst["next_concept_in"] <= K_NEXT, worst


# ---------------------------------------------------------------------------------------- single-step coefficient patterns
def _f32(*v):
    return tuple(float(np.float32(x)) for x in v)


# (c_x, c_eps, a, b, c, d, s), store_x0: every pattern the schedules produce, and c != 0 without a store (the ABI allows it)
PATTERNS = {
    "c0": (_f32(1.0, -3.1, 0.62, 0.38, 0.0, 0.0, 0.41), False),                 # Euler without a history buffer
    "c0_store": (_f32(1.07, -0.52, 0.71, 0.29, 0.0, 0.0, 1.0), True),           # DPM first / first-order step
    "c_store": (_f32(1.07, -0.52, 0.71, 0.41, -0.12, 0.0, 1.0), True),          # DPM second-order step
    "c_readonly": (_f32(1.07, -0.52, 0.71, 0.41, -0.12, 0.0, 1.0), False),      # history read, not written
    "d": (_f32(0.93, -0.37, 0.55, 0.47, -0.09, 0.31, 1.0), True),               # SDE second-order step
    "identity": (_f32(1.02, -0.2, 1.0, 0.0, 0.0, 0.0, 1.0), True),             # repeated final Karras sigma
}


@pytest.mark.parametrize("null", ["none", "next_main_in", "next_concept_in", "latents_f16"])
@pytest.mark.parametrize("pattern", list(PATTERNS))
@pytest.mark.parametrize("hw", [1, 127, 128, 129, 16385])
def test_single_step_patterns(ops, hw, pattern, null):
    """One step of each coefficient pattern around the 128-pixel block edge and at the SDXL 1024^2 latent (+1); each
    optional output is also passed as NULL, and its buffer must stay untouched."""
    from omg_b200.scheduler import StepCoeffs
    coeffs, store = PATTERNS[pattern]
    k = StepCoeffs(*coeffs)
    g = torch.Generator(device="cuda").manual_seed(hw * 7 + len(pattern))
    nm = noise_rows(torch.randn(4, hw, 4, generator=g, device="cuda"))
    ncs = [noise_rows(torch.randn(2, hw, 4, generator=g, device="cuda")) for _ in range(3)]
    masks = [tailed((torch.rand(hw, generator=g, device="cuda") < 0.5).float()) for _ in range(2)] + [None]
    lat0 = torch.randn(2, hw, 4, generator=g, device="cuda") * 3
    hist0 = torch.randn(2, hw, 4, generator=g, device="cuda")
    if k.c == 0:
        hist0.fill_(float("nan"))            # not read
    z = tailed(torch.randn(2, 4, hw, generator=g, device="cuda").half())
    if k.d == 0:
        z.fill_(float("nan"))                # not read

    def run():
        lat, hist = Guard((2, hw, 4), torch.float32), Guard((2, hw, 4), torch.float32)
        lat.out.copy_(lat0)
        hist.out.copy_(hist0)
        lat.before, hist.before = lat.buf.clone(), hist.buf.clone()
        nxt, nxc, l16 = Guard((4, hw, 8)), Guard((2, hw, 8)), Guard((2, hw, 4))
        ops.solver_step(nm, ncs, masks, GUIDANCE, k, lat.out, None if null == "next_main_in" else nxt.out,
                        None if null == "next_concept_in" else nxc.out, None if null == "latents_f16" else l16.out,
                        history=hist.out, store_x0=store, noise=z)
        torch.cuda.synchronize()
        assert lat.intact() and hist.intact() and nxt.intact() and nxc.intact() and l16.intact()
        for gd, nm_ in ((nxt, "next_main_in"), (nxc, "next_concept_in"), (l16, "latents_f16")):
            if null == nm_:
                assert gd.untouched(), f"{nm_} written through a NULL pointer"
        if not store:
            assert hist.untouched(), "history written without store_x0"
        return [lat.out.clone(), hist.out.clone(), nxt.out.clone(), nxc.out.clone(), l16.out.clone()]

    lat, hist, nxt, nxc, l16 = twice(run)
    eps = guided(nm, ncs, masks, torch.float64)
    x = lat0.double()
    x0 = k.c_x * x + k.c_eps * eps
    ref = k.a * x + k.b * x0
    if k.c != 0:
        ref = ref + k.c * hist0.double()
    if k.d != 0:
        ref = ref + k.d * z.double().reshape(2, 4, hw).transpose(1, 2)
    what = f"solver step {pattern} HW={hw} null={null}"
    if pattern == "identity":
        assert same_bits(lat, lat0), what
    check(lat, ref, K_STEP, U32, f"{what} latents")
    if store:
        check(hist, x0, K_STEP, U32, f"{what} history")
    sc = ref * k.s
    if null != "next_main_in":
        check(nxt[..., :4], torch.cat([sc, sc]), K_NEXT, U16, f"{what} next_main_in")
        assert (_bits(nxt[..., 4:]) == 0).all()
    if null != "next_concept_in":
        check(nxc[..., :4], torch.stack([sc[1], sc[1]]), K_NEXT, U16, f"{what} next_concept_in")
        assert (_bits(nxc[..., 4:]) == 0).all()
    if null != "latents_f16":
        assert same_bits(l16, lat.half()), what


# ------------------------------------------------------------------------------------------------------ launch-plan replay
def test_plan_replays_solver_and_fuse_steps(ops):
    """One omg_solver_step (history read and stored, noise) and one omg_fuse_step recorded in an omg_plan and replayed
    from C on the restored state: bit-identical to the recorded launches, history included."""
    from omg_b200.scheduler import StepCoeffs
    hw = 1000
    g = torch.Generator(device="cuda").manual_seed(3)
    nm = noise_rows(torch.randn(4, hw, 4, generator=g, device="cuda"))
    ncs = [noise_rows(torch.randn(2, hw, 4, generator=g, device="cuda")) for _ in range(2)]
    masks = [tailed((torch.rand(hw, generator=g, device="cuda") < 0.5).float()) for _ in range(2)]
    z = tailed(torch.randn(2, 4, hw, generator=g, device="cuda").half())
    lat0 = [torch.randn(2, hw, 4, generator=g, device="cuda") * 3 for _ in range(2)]
    hist0 = torch.randn(2, hw, 4, generator=g, device="cuda")
    k = StepCoeffs(*PATTERNS["d"][0])
    lat = [t.clone() for t in lat0]
    hist = hist0.clone()
    outs = [torch.empty(4, hw, 8, dtype=torch.float16, device="cuda"), torch.empty(2, hw, 8, dtype=torch.float16,
                                                                                    device="cuda"),
            torch.empty(2, hw, 4, dtype=torch.float16, device="cuda"),
            torch.empty(4, hw, 8, dtype=torch.float16, device="cuda"), torch.empty(2, hw, 8, dtype=torch.float16,
                                                                                    device="cuda"),
            torch.empty(2, hw, 4, dtype=torch.float16, device="cuda")]

    plan = ops.LaunchPlan()
    with plan:
        ops.solver_step(nm, ncs, masks, GUIDANCE, k, lat[0], outs[0], outs[1], outs[2], history=hist, store_x0=True,
                        noise=z)
        ops.fuse_step(nm, ncs, masks, GUIDANCE, 3.2, 2.7, lat[1], outs[3], outs[4], latents_f16=outs[5])
    assert len(plan) == 2
    torch.cuda.synchronize()
    recorded = [t.clone() for t in lat + [hist] + outs]
    for t, t0 in zip(lat, lat0):
        t.copy_(t0)
    hist.copy_(hist0)
    for o in outs:
        o.fill_(float("nan"))
    plan.run()
    torch.cuda.synchronize()
    for a, b in zip(recorded, lat + [hist] + outs):
        assert torch.isfinite(a.float()).all() and same_bits(a, b)
    assert not same_bits(recorded[0], lat0[0]) and not same_bits(recorded[2], hist0)
