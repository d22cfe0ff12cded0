"""The bf16 decode path on the H100: the bf16 variants of omg_gemm, omg_groupnorm and omg_softmax_rows against float64
references on the same bf16 operands, the bf16 VAE decoder against the fp32 oracle (oracle/vae.py), the fp16 overflow
the reference up-casts for, the pipelines, launch plans, the loader and the InstantID CLI.

* Per-element bound `check`:  |out - ref| <= u |ref| + k u rms(ref)  with u = 2^-8, the unit roundoff of bf16 (8
  significant bits): rounding the fp32 result to bf16 alone may cost u |ref|.  k is set per kernel family below.
* Outputs sit in NaN-filled buffers (`Guard`) whose other bytes must be unchanged; operands sit in NaN-filled buffers
  with wider rows (`poisoned`), so a read outside an operand shows up as NaN.
* Every kernel case runs twice and must be bit-identical.  `pytest -s` prints the measured values behind each bound.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF = torch.bfloat16
U = 2.0 ** -8   # bf16 unit roundoff
PAD = 8

# Per-element k with the worst value the cases need, measured on an NVIDIA H100 80GB HBM3 at a 400 W power limit (a
# value <= 0 means every element is within u |ref|: the fp32 accumulation error is far below bf16's rounding)
K_GEMM = 0.25     # measured 0.00 (GEMM tile families, convs with shortcut, upsample conv)
K_NORM = 0.25     # measured 0.005 (GroupNorm at 1e5 and |mean| / sigma = 32)
K_SOFTMAX = 0.25  # measured 0.00
# Decoder vs the fp32 oracle on bf16-rounded weights and latents, same card: rel-L2 of the image and max abs error of
# the postprocessed image, about 1.8x the worst measured value (rel-L2 1.11e-2 tiny 16x16, abs 2.20e-2 SDXL 32x32; the
# overflow cases 9.9e-3 and 1.5e-2)
DEC_REL_L2 = 2e-2
DEC_ATOL = 4e-2


def check(out, ref, k, what=""):
    o, r = out.double(), ref.double()
    assert torch.isfinite(o).all(), f"{what}: non-finite output"
    rms = r.pow(2).mean().sqrt().clamp_min(1e-300)
    need = (((o - r).abs() - U * r.abs()) / (U * rms)).max().item()
    rl = ((o - r).norm() / r.norm().clamp_min(1e-300)).item()
    print(f"[check] {what}: rel_l2 {rl:.3e}, k needed {need:.3f} (bound {k})")
    assert need <= k, f"{what}: per-element error needs k = {need:.3f} > {k}"
    return need


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


class Guard:
    """Output view of `shape` inside a NaN-filled buffer: PAD rows before and 2 PAD after along dim -2, PAD columns on
    both sides."""

    def __init__(self, shape, dtype=BF):
        full = list(shape)
        full[-2] += 3 * PAD
        full[-1] += 2 * PAD
        self.buf = torch.full(full, float("nan"), dtype=dtype, device="cuda")
        idx = (slice(None),) * (len(shape) - 2) + (slice(PAD, PAD + shape[-2]), slice(PAD, PAD + shape[-1]))
        self.out = self.buf[idx]
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        self.inside[idx] = True
        self.before = self.buf.clone()

    def intact(self):
        return bool(((_bits(self.buf) == _bits(self.before)) | self.inside).all())


def poisoned(t, rows=0):
    full = list(t.shape)
    full[-2] += rows
    full[-1] += 2 * PAD
    buf = torch.full(full, float("nan"), dtype=t.dtype, device="cuda")
    v = buf[..., :t.shape[-2], PAD:PAD + t.shape[-1]]
    v.copy_(t)
    return v


def rnd(*shape, scale=1.0, seed=0, dtype=BF):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


def twice(run):
    a, b = run(), run()
    for x, y in zip(a, b):
        assert same_bits(x, y), "second run differs"
    return a


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


# ---------------------------------------------------------------------------------------------------------------- GEMM
# family -> (block_n, cta_pair, N with a partial last n-tile; 320 needs N % 320 == 0)
FAMILIES = {"64": (64, 1, 224), "128": (128, 1, 352), "160": (160, 1, 224), "160-tall": (160, 3, 224),
            "256": (256, 1, 288), "320": (320, 1, 640)}
# output magnitude per K: 1e-3 up to 1e6 (fp16's largest finite value is 65504)
SCALE = {8: 1e-3, 40: 1.0, 200: 1e3, 1000: 1e6}


def _linear_case(ops, M, N, K, bn, cta_pair, scale, seed=0, dtype=BF, ints=False):
    def opnd(*shape, s, sd):
        if ints:  # integer values: exact in fp16 and bf16
            g = torch.Generator(device="cuda").manual_seed(sd)
            return torch.randint(-2, 3, shape, generator=g, device="cuda").to(dtype)
        return rnd(*shape, scale=s, seed=sd, dtype=dtype)

    x = poisoned(opnd(M, K, s=math.sqrt(scale), sd=seed + 1))
    wbuf = torch.full((N + PAD, K), float("nan"), dtype=dtype, device="cuda")
    w = wbuf[:N]
    w.copy_(opnd(N, K, s=math.sqrt(scale / K), sd=seed + 2))
    bbuf = torch.full((N + PAD,), float("nan"), dtype=dtype, device="cuda")
    b = bbuf[:N]
    b.copy_(opnd(N, s=scale, sd=seed + 3))
    r = poisoned(opnd(M, N, s=scale, sd=seed + 4))

    def run():
        g = Guard((M, N), dtype)
        ops.linear(x, w, bias=b, residual=r, out=g.out, block_n=bn, cta_pair=cta_pair)
        torch.cuda.synchronize()
        assert g.intact(), "write outside the output window"
        return [g.out.clone()]

    out, = twice(run)
    return out, x.double() @ w.double().t() + b.double() + r.double()


@pytest.mark.parametrize("K", [8, 40, 200, 1000])
@pytest.mark.parametrize("M", [1, 127, 129, 383])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_bf16_gemm_tile_families_with_tails(ops, family, M, K):
    bn, cta_pair, N = FAMILIES[family]
    out, ref = _linear_case(ops, M, N, K, bn, cta_pair, SCALE[K])
    assert out.dtype == BF
    check(out, ref, K_GEMM, what=f"bf16 gemm {family} M={M} N={N} K={K} |out|~{SCALE[K]:g}")
    if cta_pair == 3:  # tall tiles compute exactly what single 128-row tiles compute
        single, _ = _linear_case(ops, M, N, K, bn, 1, SCALE[K])
        assert same_bits(out, single)


@pytest.mark.parametrize("family", list(FAMILIES))
def test_bf16_gemm_same_arithmetic_as_fp16(ops, family):
    """Integer operands with |result| <= 256 are exact in both types, so the bf16 and fp16 GEMMs must agree exactly."""
    bn, cta_pair, N = FAMILIES[family]
    ob, ref = _linear_case(ops, 383, N, 40, bn, cta_pair, 1.0, seed=20, dtype=BF, ints=True)
    oh, _ = _linear_case(ops, 383, N, 40, bn, cta_pair, 1.0, seed=20, dtype=torch.float16, ints=True)
    assert ref.abs().max().item() <= 256
    assert torch.equal(ob.double(), ref) and torch.equal(oh.double(), ref)


@pytest.mark.parametrize("W,H,scale", [(5, 7, 1.0), (96, 3, 1e5), (130, 3, 1e-3)])
def test_bf16_conv3x3_shortcut_and_residual(ops, W, H, scale):
    """A ResBlock conv2: 9 taps of a 40-channel NaN-poisoned input plus a 24-channel 1x1 shortcut K-segment, bias and a
    residual (the decoder's residual trunk), at magnitudes up to 1e5."""
    B, Cin, Cs, N = 2, 40, 24, 96
    s = math.sqrt(scale)
    x = poisoned(rnd(B, H, W, Cin, scale=s, seed=1))
    sc = poisoned(rnd(B, H, W, Cs, scale=s, seed=2))
    wt = rnd(N, Cin, 3, 3, scale=s * (9 * Cin) ** -0.5, seed=3)
    ws = rnd(N, Cs, scale=s * Cs ** -0.5, seed=4)
    bias, res = rnd(N, scale=scale, seed=5), rnd(B, H, W, N, scale=scale, seed=6)
    w = torch.cat([ops.pack_conv3x3_weight(wt), ws], dim=1).contiguous()

    def run():
        g = Guard((B, H, W, N))
        ops.conv3x3(x, w, bias=bias, residual=res, out=g.out, shortcut=[(sc, 9 * Cin)])
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), bias.double(), padding=1) \
        + F.conv2d(sc.double().permute(0, 3, 1, 2), ws.double()[:, :, None, None]) + res.double().permute(0, 3, 1, 2)
    check(out.permute(0, 3, 1, 2), ref, K_GEMM, what=f"bf16 conv+shortcut W={W} H={H} |out|~{scale:g}")


@pytest.mark.parametrize("H,W", [(5, 7), (16, 16)])
def test_bf16_upsample_conv_phase_views(ops, H, W):
    """Nearest-2x upsample + 3x3 conv: four phase convs through strided output views (odd and even sizes)."""
    B, Cin, N = 2, 40, 64
    x = rnd(B, H, W, Cin, scale=30.0, seed=1)
    wt, bias = rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2), rnd(N, seed=3)

    def run():
        g = Guard((B, 2 * H, 2 * W, N))
        ops.upsample2x_conv3x3(x, ops.pack_conv3x3_weight(wt), bias=bias, out=g.out)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    ref = F.conv2d(F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest"), wt.double(),
                   bias.double(), padding=1)
    check(out.permute(0, 3, 1, 2), ref, K_GEMM, what=f"bf16 upsample conv {H} x {W}")


def test_bf16_ops_reject_mixed_operands_and_unsupported_features(ops):
    x, w = rnd(128, 64), rnd(64, 64)
    with pytest.raises(ValueError, match="mixed"):
        ops.linear(x, w.half())
    with pytest.raises(ValueError, match="mixed"):
        ops.linear(x.half(), w)
    with pytest.raises(ValueError, match="mixed"):
        ops.groupnorm(x.view(1, 128, 64), torch.ones(64, device="cuda").half(), torch.zeros(64, device="cuda", dtype=BF),
                      1e-6, 0)
    with pytest.raises(RuntimeError, match="bf16 supports only OMG_EPI_NONE"):
        ops.linear(x, w, epilogue=2)
    with pytest.raises(ValueError):   # ops without a bf16 variant keep rejecting it
        ops.layernorm(x, w[0], w[1])
    assert ops.linear(x, w).dtype == BF


# ---------------------------------------------------------------------------------------------------- GroupNorm, softmax
@pytest.mark.parametrize("silu", [0, 1])
@pytest.mark.parametrize("B,HW,C1,C2", [(2, 37, 64, 0), (1, 4099, 96, 32), (3, 1, 512, 0)])
def test_groupnorm_bf16_large_offset_inputs(ops, B, HW, C1, C2, silu):
    """Inputs at 1e5 with each (image, group) offset to |mean| / sigma = 32 (well past fp16's range), odd HW, a two-source
    channel concatenation; fp32 statistics of the bf16 values, normalised and activated output in bf16."""
    C = C1 + C2
    g = torch.Generator(device="cuda").manual_seed(B * HW + C)
    sign = torch.randint(0, 2, (B, 1, 32, 1), generator=g, device="cuda") * 2.0 - 1.0
    z = torch.randn(B, HW, 32, C // 32, generator=g, device="cuda") + 32.0 * sign
    x = (z * 1e5).reshape(B, HW, C).to(BF)
    x1, x2 = x[..., :C1].contiguous(), (x[..., C1:].contiguous() if C2 else None)
    gamma, beta = rnd(C, scale=0.5, seed=7) + 1, rnd(C, scale=0.5, seed=8)
    # the output is contiguous: it sits in a flat NaN-filled buffer with PAD elements on either side
    buf = torch.full((B * HW * C + 2 * PAD,), float("nan"), dtype=BF, device="cuda")
    out = buf[PAD:PAD + B * HW * C].view(B, HW, C)
    before = buf.clone()

    def run():
        ops.groupnorm(x1, gamma, beta, 1e-6, silu, x2=x2, out=out)
        torch.cuda.synchronize()
        return [out.clone()]

    got, = twice(run)
    assert same_bits(buf[:PAD], before[:PAD]) and same_bits(buf[-PAD:], before[-PAD:])
    xd = x.double().view(B, HW, 32, C // 32)
    mean = xd.mean(dim=(1, 3), keepdim=True)
    var = xd.var(dim=(1, 3), unbiased=False, keepdim=True)
    ref = ((xd - mean) / torch.sqrt(var + 1e-6)).view(B, HW, C) * gamma.double() + beta.double()
    if silu:
        ref = ref * torch.sigmoid(ref)
    check(got, ref, K_NORM, what=f"groupnorm_bf16 B={B} HW={HW} C={C1}+{C2} silu={silu}")


@pytest.mark.parametrize("rows,cols,scale", [(7, 64, 1.0), (33, 1024, 0.5), (16, 16384, 0.044), (5, 32768, 1.0)])
def test_softmax_rows_bf16(ops, rows, cols, scale):
    g = torch.Generator().manual_seed(rows + cols)
    x = (torch.randn(rows, cols, generator=g) * 4).to(BF).cuda()
    ref = torch.softmax(x.double() * scale, dim=-1)
    big = torch.full((rows, cols + 8), float("nan"), dtype=BF, device="cuda")  # strided rows, NaN tails
    big[:, :cols] = x

    def run():
        big[:, :cols] = x
        ops.softmax_rows(big[:, :cols], scale)
        torch.cuda.synchronize()
        return [big.clone()]

    got, = twice(run)
    check(got[:, :cols], ref, K_SOFTMAX, what=f"softmax_rows_bf16 {rows} x {cols}")
    assert torch.allclose(got[:, :cols].double().sum(-1), torch.ones(rows, dtype=torch.float64, device="cuda"),
                          atol=2 * U)
    assert bool(got[:, cols:].isnan().all())


# -------------------------------------------------------------------------------------------------------------- decoder
def _bf16_round(sd):
    return {k: v.to(BF).float() for k, v in sd.items()}


def _latents(batch, h, w, seed=5):
    return (torch.randn(batch, 4, h, w, generator=torch.Generator().manual_seed(seed)) * 0.13025 * 3).to(BF).float()


@pytest.mark.parametrize("which,h,w,batch", [("tiny", 16, 16, 2), ("tiny", 8, 24, 1), ("sdxl", 32, 32, 1)])
def test_bf16_decode_matches_oracle(which, h, w, batch):
    from omg_b200 import synthetic
    from omg_b200.vae import PackedVaeDecoder, VaeConfig
    from oracle import vae as ov
    cfg = VaeConfig.tiny() if which == "tiny" else VaeConfig.sdxl()
    ocfg = ov.VaeConfig(block_out_channels=cfg.block_out_channels)
    sd = _bf16_round(synthetic.make_vae_state_dict(cfg, seed=3))
    lat = _latents(batch, h, w)
    torch.set_num_threads(32)
    ref = ov.decode(sd, lat, ocfg)
    dec = PackedVaeDecoder(sd, cfg, device="cuda", dtype=BF)
    assert all(t.dtype == BF for t in dec.p.values())
    got = dec.decode(lat.cuda())
    assert got.dtype == BF and got.shape == ref.shape == (batch, 3, 8 * h, 8 * w)
    err = ((got.float().cpu() - ref).norm() / ref.norm()).item()
    img = dec(lat.cuda(), "pt")
    atol = (img.cpu() - ov.postprocess(ref)).abs().max().item()
    print(f"[decoder] bf16 {which} {h}x{w}: image rel-L2 {err:.3e}, postprocessed max abs {atol:.3e}")
    assert err < DEC_REL_L2 and atol < DEC_ATOL
    assert same_bits(dec.decode(lat.cuda()), got)


def _overflow_state_dict(cfg, scale):
    """Random VAE weights with conv_in and the mid / up ResNets' conv2 and conv_shortcut scaled so that the residual
    trunk carries values of order `scale` (what the original SDXL VAE weights do to fp16 activations)."""
    from omg_b200 import synthetic
    sd = synthetic.make_vae_state_dict(cfg, seed=4)
    for k in list(sd):
        if k.startswith("decoder.conv_in.") or (".resnets." in k and (".conv2." in k or ".conv_shortcut." in k)):
            sd[k] = sd[k] * (scale if ".conv_shortcut." not in k else 1.0)
    return _bf16_round(sd)


def _oracle_trunk_max(sd, lat, ocfg):
    """max |x| of the oracle's residual trunk after conv_in and after every mid / up block."""
    from oracle import vae as ov
    g = ocfg.norm_num_groups
    z = F.conv2d(lat.float() / ocfg.scaling_factor, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
    x = F.conv2d(z, sd["decoder.conv_in.weight"], sd["decoder.conv_in.bias"], padding=1)
    peak = x.abs().max().item()
    x = ov._res(x, sd, "decoder.mid_block.resnets.0", g)
    x = ov._attn(x, sd, "decoder.mid_block.attentions.0", g)
    x = ov._res(x, sd, "decoder.mid_block.resnets.1", g)
    peak = max(peak, x.abs().max().item())
    for i in range(len(ocfg.block_out_channels)):
        for j in range(ocfg.layers_per_block + 1):
            x = ov._res(x, sd, f"decoder.up_blocks.{i}.resnets.{j}", g)
            peak = max(peak, x.abs().max().item())
        if i < len(ocfg.block_out_channels) - 1:
            x = F.interpolate(x, scale_factor=2.0, mode="nearest")
            x = F.conv2d(x, sd[f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"],
                         sd[f"decoder.up_blocks.{i}.upsamplers.0.conv.bias"], padding=1)
    return peak


@pytest.mark.parametrize("which,h,w", [("tiny", 16, 16), ("sdxl", 16, 16)])
def test_fp16_overflow_decodes_in_bf16(which, h, w):
    from omg_b200.vae import PackedVaeDecoder, VaeConfig
    from oracle import vae as ov
    cfg = VaeConfig.tiny() if which == "tiny" else VaeConfig.sdxl()
    ocfg = ov.VaeConfig(block_out_channels=cfg.block_out_channels)
    sd = _overflow_state_dict(cfg, 3e4)
    lat = _latents(1, h, w, seed=6)
    torch.set_num_threads(32)
    peak = _oracle_trunk_max(sd, lat, ocfg)
    print(f"[overflow] {which}: oracle residual trunk max |x| = {peak:.3e}")
    assert peak > 65504.0
    with pytest.raises(FloatingPointError, match="fp16"):
        PackedVaeDecoder(sd, cfg, dtype=torch.float16)(lat.cuda(), "pt")
    ref = ov.decode(sd, lat, ocfg)
    dec = PackedVaeDecoder(sd, cfg, dtype=BF)
    got = dec.decode(lat.cuda()).float().cpu()
    err = ((got - ref).norm() / ref.norm()).item()
    atol = (dec(lat.cuda(), "pt").cpu() - ov.postprocess(ref)).abs().max().item()
    print(f"[overflow] {which}: bf16 image rel-L2 {err:.3e}, postprocessed max abs {atol:.3e}")
    assert err < DEC_REL_L2 and atol < DEC_ATOL


# ------------------------------------------------------------------------------------------------------------ pipelines
def _check_images(dec, lat, pt, pil):
    ref = dec(lat, "pt")
    assert pt.shape == ref.shape and torch.equal(pt, ref)
    arr = (ref.permute(0, 2, 3, 1).cpu().numpy() * 255).round().astype("uint8")
    assert len(pil) == lat.shape[0]
    for a, im in zip(arr, pil):
        assert im.size == (lat.shape[3] * 8, lat.shape[2] * 8)
        assert (a == np.array(im)).all()


def test_lora_pipeline_with_bf16_decoder():
    from omg_b200 import factory, synthetic
    from omg_b200.config import UNetConfig
    from omg_b200.vae import PackedVaeDecoder, VaeConfig
    wl = factory.build_lora_workload(UNetConfig.tiny(), 128, 2, 8, 4, 7.5)
    dec = PackedVaeDecoder(synthetic.make_vae_state_dict(VaeConfig.tiny(), 1), VaeConfig.tiny(), dtype=BF)
    wl.pipe.vae_decoder = dec
    lat0 = torch.randn(1, 4, 16, 16, generator=torch.Generator().manual_seed(0)).half()
    out = {}
    for ot in ("latent", "pt", "pil"):
        kw = dict(wl.call_kwargs)
        kw["output_type"] = ot
        out[ot] = wl.pipe(stage=1, latents=lat0, **kw).images
    assert out["pt"].shape == (2, 3, 128, 128)
    _check_images(dec, out["latent"], out["pt"], out["pil"])


def test_instantid_pipeline_with_bf16_decoder():
    import argparse
    import importlib.util
    from omg_b200 import synthetic
    from omg_b200.vae import PackedVaeDecoder, VaeConfig
    spec = importlib.util.spec_from_file_location("cli_instantid", os.path.join(ROOT, "inference_instantid.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    args = argparse.Namespace(tiny=True, image_size=128, prompt="two people")
    pipe, controller, cm = cli.build_synthetic(args, torch.device("cuda"))
    cm.set_ip_adapter_scale(0.8)
    dec = PackedVaeDecoder(synthetic.make_vae_state_dict(VaeConfig.tiny(), 2), VaeConfig.tiny(), dtype=BF)
    pipe.vae_decoder = dec
    g = torch.Generator().manual_seed(1)
    faces = [torch.nn.functional.normalize(torch.randn(512, generator=g), dim=0) for _ in range(2)]
    regions = [("a man", "bad", None), ("a woman", "bad", None)]
    lat0 = torch.randn(1, 4, 16, 16, generator=torch.Generator().manual_seed(3)).half()
    out = {}
    for ot in ("latent", "pt", "pil"):
        controller.reset()
        out[ot] = pipe(prompt=[["two people"] * 2, regions], negative_prompt=["noisy"] * 2, guidance_scale=3.0,
                       num_inference_steps=3, concept_models=cm, controller=controller, stage=1,
                       controlnet_conditioning_scale=0.8, face_embeds=faces, height=128, width=128, output_type=ot,
                       latents=lat0).images
    _check_images(dec, out["latent"], out["pt"], out["pil"])


# --------------------------------------------------------------------------------------------------------- launch plans
def test_bf16_launch_plan_replays_bit_identically(ops):
    x, w, b = rnd(256, 128, seed=1), rnd(192, 128, scale=128 ** -0.5, seed=2), rnd(192, seed=3)
    gamma, beta = rnd(192, scale=0.1, seed=4) + 1, rnd(192, scale=0.1, seed=5)
    s0 = rnd(64, 1024, scale=4.0, seed=6)
    y = torch.empty(256, 192, dtype=BF, device="cuda")
    z = torch.empty(2, 128, 192, dtype=BF, device="cuda")
    s = s0.clone()
    ws = torch.empty(2 * (10240 + 64 * 256), dtype=torch.float32, device="cuda")
    plan = ops.LaunchPlan()
    with plan:
        ops.linear(x, w, bias=b, out=y)
        ops.groupnorm(y.view(2, 128, 192), gamma, beta, 1e-6, 1, out=z, stats_ws=ws)
        ops.softmax_rows(s, 0.5)
    assert len(plan) == 3  # one step per C-ABI call (the GroupNorm call is three kernel launches)
    torch.cuda.synchronize()
    eager = [y.clone(), z.clone(), s.clone()]
    y.fill_(float("nan"))
    z.fill_(float("nan"))
    s.copy_(s0)
    plan.run()
    torch.cuda.synchronize()
    for a, e in zip((y, z, s), eager):
        assert same_bits(a, e)


def test_bf16_decode_issues_as_many_launches_as_fp16():
    from omg_b200 import _lib, synthetic
    from omg_b200.vae import PackedVaeDecoder, VaeConfig
    cfg = VaeConfig.tiny()
    sd = synthetic.make_vae_state_dict(cfg, 0)
    lat = _latents(2, 16, 16).cuda()
    counts = {}
    for dt in (torch.float16, BF):
        dec = PackedVaeDecoder(sd, cfg, dtype=dt)
        dec.decode(lat)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        dec.decode(lat)
        torch.cuda.synchronize()
        counts[dt] = _lib.launch_count() - n0
    print("[launches] decode:", counts)
    assert counts[BF] == counts[torch.float16] > 0


# ---------------------------------------------------------------------------------------------------------- loader, CLI
def test_from_pretrained_resolves_the_fp16_variant(tmp_path):
    from safetensors.torch import save_file
    from omg_b200 import synthetic
    from omg_b200.vae import PackedVaeDecoder, VaeConfig
    cfg = VaeConfig.tiny()
    sd = {k: v.half() for k, v in synthetic.make_vae_state_dict(cfg, 5).items()}
    os.makedirs(tmp_path / "vae")
    save_file(sd, str(tmp_path / "vae" / "diffusion_pytorch_model.fp16.safetensors"))
    loaded = PackedVaeDecoder.from_pretrained(str(tmp_path), cfg=cfg)
    direct = PackedVaeDecoder(sd, cfg, dtype=BF)
    assert loaded.dtype == BF
    assert all(torch.equal(loaded.p[k], direct.p[k]) for k in direct.p)
    lat = _latents(1, 8, 8).cuda()
    assert same_bits(loaded.decode(lat), direct.decode(lat))


def test_instantid_cli_decodes_and_runs_sam_on_the_stage1_image(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "inference_instantid.py"), "--synthetic", "--tiny", "--decode",
                        "--image_size", "128", "--num_inference_steps", "3", "--sam_boxes", "8,16,60,112|68,16,120,112",
                        "--save_dir", str(tmp_path)], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    from PIL import Image
    for name in ("stage-1", "stage-2"):
        p = tmp_path / "seed_53" / (name + ".png")
        assert p.exists(), r.stdout
        assert Image.open(p).size == (128, 128)
    assert "SAM mask 0" in r.stdout and "SAM mask 1" in r.stdout
