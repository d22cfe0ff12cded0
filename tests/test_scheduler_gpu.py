"""GPU tests of the sampling schedules: omg_solver_step against a float64 restatement, and the two-stage pipelines on
every rule against oracle.pipeline.denoise run with the same schedule (tests/util_schedulers.py) (tiny topology, 18 steps so that fusion runs).
Pipeline tolerances are the measured error x 1.25 (H100 SXM); stochastic rules replay the noise of the same seeded
generator in the oracle."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from util_models import lora, ocfg, oracle_lora, r16, rel, weights  # noqa: E402
from util_schedulers import oracle_schedule  # noqa: E402

from omg_b200 import scheduler as S  # noqa: E402

STEPS = 18
BASE = S.SDXL_BASE_CONFIG
RULES = {
    "dpmpp_2m_karras": lambda: S.cli_scheduler("dpmpp_2m_karras", BASE),
    "dpmpp_2m_sde": lambda: S.cli_scheduler("dpmpp_2m_sde", BASE),
    "euler_a": lambda: S.cli_scheduler("euler_a", BASE),
    "euler_trailing_v": lambda: S.EulerDiscreteScheduler.from_config(BASE, timestep_spacing="trailing",
                                                                     prediction_type="v_prediction"),
}
K_F32 = 32.0   # fp32 latents / history, in units of 2^-24 x rms (the bound of test_kernel_edges_gpu.py)
K_F16 = 2.0    # fp16 next inputs, in units of 2^-11 x rms


def check(out, ref, k, u, what):
    o, r = out.double().cpu(), ref.double().cpu()
    assert torch.isfinite(o).all(), what
    rms = r.pow(2).mean().sqrt().clamp_min(1e-30)
    need = (((o - r).abs() - 4 * u * r.abs()) / (u * rms)).max().item()
    print(f"[check] {what}: k needed {need:.2f} (bound {k})")
    assert need <= k, f"{what}: per-element error needs k = {need:.2f} > {k}"


def _kernel_coeffs(rule):
    s = {"euler_v": lambda: S.EulerDiscreteScheduler.from_config(BASE, prediction_type="v_prediction"),
         "euler_a": RULES["euler_a"], "dpmpp_2m": lambda: S.cli_scheduler("dpmpp_2m", BASE),
         "dpmpp_2m_sde_heun": lambda: S.DPMSolverMultistepScheduler.from_config(
             BASE, algorithm_type="sde-dpmsolver++", solver_type="heun")}[rule]()
    s.set_timesteps(20)
    return s.step_coeffs(5), s


@pytest.mark.parametrize("rule", ["euler_v", "euler_a", "dpmpp_2m", "dpmpp_2m_sde_heun"])
@pytest.mark.parametrize("n_concepts", [0, 2, 8])
@pytest.mark.parametrize("hw", [(64, 64), (25, 40)])     # 4096 pixels, and 1000: not a multiple of 128
def test_solver_step_kernel(rule, n_concepts, hw):
    from omg_b200 import ops
    h, w = hw
    HW = h * w
    g = torch.Generator().manual_seed(n_concepts * 7 + h)
    k, sch = _kernel_coeffs(rule)
    nm = torch.randn(4, HW, 8, generator=g).half()
    ncs = [torch.randn(2, HW, 8, generator=g).half() for _ in range(n_concepts)]
    masks = [(torch.rand(HW, generator=g) < 0.3).float() for _ in range(n_concepts)]
    if n_concepts == 8:
        masks[3] = None                                          # a skipped concept
    lat = torch.randn(2, h, w, 4, generator=g) * 3
    hist = torch.randn(2, h, w, 4, generator=g)
    z = torch.randn(2, 4, h, w, generator=g).half()
    gs = 7.5
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    lat_d, hist_d = lat.cuda(), hist.cuda()
    nxt = torch.full((4, h, w, 8), float("nan"), dtype=torch.float16, device="cuda")
    nxc = torch.full((2, h, w, 8), float("nan"), dtype=torch.float16, device="cuda")
    f16 = torch.empty(2, h, w, 4, dtype=torch.float16, device="cuda")
    ops.solver_step(nm.cuda(), [dev(n) for n in ncs], [dev(m) for m in masks], gs, k, lat_d, nxt, nxc, f16,
                    history=hist_d, store_x0=True, noise=z.cuda() if k.d != 0 else None)
    torch.cuda.synchronize()
    # float64 restatement: fusion, guidance, x0, update
    e = nm.double()[..., :4]
    u1, c1 = e[1].clone(), e[3].clone()
    union = torch.zeros(HW, dtype=torch.bool)
    au, ac = torch.zeros(HW, 4, dtype=torch.float64), torch.zeros(HW, 4, dtype=torch.float64)
    for n, m in zip(ncs, masks):
        if m is None:
            continue
        sel = m == 1
        union |= sel
        au[sel] += n.double()[0, sel, :4]
        ac[sel] += n.double()[1, sel, :4]
    u1[union], c1[union] = au[union], ac[union]
    eps = torch.stack([e[0] + gs * (e[2] - e[0]), u1 + gs * (c1 - u1)]).reshape(2, h, w, 4)
    x = lat.double()
    x0 = k.c_x * x + k.c_eps * eps
    zz = z.double().permute(0, 2, 3, 1) if k.d != 0 else 0.0
    ref = k.a * x + k.b * x0 + k.c * hist.double() + k.d * zz
    check(lat_d, ref, K_F32, 2.0 ** -24, f"{rule} latents")
    check(hist_d, x0, K_F32, 2.0 ** -24, f"{rule} history")
    sc = ref * k.s
    check(nxt[..., :4], torch.cat([sc, sc]), K_F16, 2.0 ** -11, f"{rule} next_main_in")
    check(nxc[..., :4], torch.stack([sc[1], sc[1]]), K_F16, 2.0 ** -11, f"{rule} next_concept_in")
    assert (nxt[..., 4:] == 0).all() and (nxc[..., 4:] == 0).all()
    check(f16, ref, K_F16, 2.0 ** -11, f"{rule} latents_f16")


def _masks(size):
    m1 = torch.zeros(size, size)
    m2 = torch.zeros(size, size)
    m1[size // 8: 7 * size // 8, size // 16: 7 * size // 16] = 1
    m2[size // 8: 7 * size // 8, 9 * size // 16: 15 * size // 16] = 1
    return m1, m2


def _oracle_schedule(s, seed, h, w):
    """The literal restatement of schedule s, replaying the noise the pipeline draws from seed."""
    from util_schedulers import make
    return make(s.config["_class_name"], {k: v for k, v in s.config.items() if k != "_class_name"},
                _noise_source(s, seed, h, w))


def _noise_source(s, seed, h, w):
    """The per-step noise the pipeline draws from torch.Generator("cuda").manual_seed(seed) (no latent draw: the
    latents are given)."""
    if not s.stochastic:
        return None
    g = torch.Generator("cuda").manual_seed(seed)
    zs = [torch.randn((2, 4, h, w), generator=g, device="cuda", dtype=torch.float16).float().cpu() for _ in range(STEPS)]
    return lambda i: zs[i]


# measured on an H100 80GB HBM3 (700 W) x 1.25: 2.02e-3, 2.92e-3, 2.97e-3, 2.22e-3 (larger image-1 error of the two)
LORA_TOL = {"dpmpp_2m_karras": 2.6e-3, "dpmpp_2m_sde": 3.7e-3, "euler_a": 3.8e-3, "euler_trailing_v": 2.8e-3}


@pytest.mark.parametrize("rule", list(RULES))
def test_lora_two_stage_pipeline_on_each_schedule(rule):
    from omg_b200.config import UNetConfig
    from omg_b200.pipelines import ConceptModels, LoraMultiConceptPipeline, revise_regionally_controlnet_forward
    from omg_b200.prompt_attention import AttentionReplace
    from omg_b200.unet import PackedUNet
    from oracle import p2p as op2p
    from oracle import unet as ou
    from oracle.pipeline import Concept, denoise
    cfg = UNetConfig.tiny()
    sd = weights(cfg, 0)
    size = 256
    prompts = ["a man and a woman on the beach"] * 2
    regions = [("a man smiling", "blurry"), ("a woman smiling", "blurry")]
    pipe = LoraMultiConceptPipeline(PackedUNet(cfg, sd))
    pipe.scheduler = RULES[rule]()
    controller = AttentionReplace(prompts, 50, {"default_": 1.0}, 0.4, width=8, height=8)
    revise_regionally_controlnet_forward(pipe, controller)
    cm = ConceptModels(pipe.unet)
    loras = [lora(cfg, 101), lora(cfg, 102)]
    cm.load_lora_weights(loras[0], adapter_name="manA")
    cm.load_lora_weights(loras[1], adapter_name="womanB")
    lat0 = torch.randn(1, 4, size // 8, size // 8, generator=torch.Generator().manual_seed(14)).half()
    masks = list(_masks(size))
    seed = 77
    out = pipe(prompt=[prompts, regions], negative_prompt=["noisy"] * 2, guidance_scale=7.5, num_inference_steps=STEPS,
               cross_attention_kwargs={"scale": 0.8}, concept_models=cm, lora_list=["manA", "womanB"], styleL=False,
               height=size, width=size, output_type="latent", latents=lat0, stage=2, region_masks=masks,
               generator=torch.Generator("cuda").manual_seed(seed)).images
    assert torch.isfinite(out.float()).all()
    pe, ne, pp, np_ = pipe.encode_prompt(prompts, ["noisy"] * 2, 0.8)
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32)
    octrl = op2p.AttentionReplaceOracle(prompts, 50, {"default_": 1.0}, 0.4, 8, 8)
    octrl.num_att_layers = len(ou.attention_names(ocfg(cfg)))
    main = ou.Ctx(sd, ocfg(cfg), attn_core=ou.make_p2p_attn_core(octrl))
    concepts = []
    for k, (rp, rn) in enumerate(regions):
        e, n_, p_, np2 = cm.encode_prompt(rp, negative_prompt=rn)
        concepts.append(Concept(r16(torch.cat([n_, e])), r16(torch.cat([np2, p_])), tid.repeat(2, 1), masks[k],
                                unet=ou.Ctx(sd, ocfg(cfg), lora=oracle_lora([(loras[k], 1.0)], 0.8))))
    with oracle_schedule(_oracle_schedule(pipe.scheduler, seed, size // 8, size // 8)):
        ref = denoise(main, lat0.float(), r16(torch.cat([ne, pe])), r16(torch.cat([np_, pp])), tid.repeat(4, 1),
                      concepts, 2, STEPS, 7.5)
    e0, e1 = rel(out[0], ref[0]), rel(out[1], ref[1])
    print(f"{rule}: lora pipeline final-latent rel err: layout {e0:.3e} fused {e1:.3e}")
    assert e0 < LORA_TOL[rule] and e1 < LORA_TOL[rule]


def test_instantid_pipeline_with_a_multistep_schedule():
    from omg_b200 import synthetic
    from omg_b200.config import UNetConfig
    from omg_b200.pipelines import ConceptModels, InstantidMultiConceptPipeline, revise_regionally_controlnet_forward
    from omg_b200.prompt_attention import AttentionReplace
    from omg_b200.unet import PackedUNet
    from oracle import p2p as op2p
    from oracle import unet as ou
    from oracle.pipeline import Concept, denoise
    from oracle.resampler import resampler_forward
    cfg = UNetConfig.tiny()
    sd = weights(cfg, 0)
    idsd = weights(cfg, 41, controlnet=True)
    size = 128
    rs = torch.load(os.path.join(os.path.dirname(__file__), "golden", "resampler.pt"))
    rs["sd"] = {k: v.float() for k, v in rs["sd"].items()}
    ipw = {k: (r16(a), r16(b)) for k, (a, b) in synthetic.make_ip_adapter(cfg, 31).items()}
    pipe = InstantidMultiConceptPipeline(PackedUNet(cfg, sd), controlnet=PackedUNet(cfg, idsd, controlnet=True))
    pipe.scheduler = S.cli_scheduler("dpmpp_2m_sde_karras", BASE)
    prompts = ["two people"] * 2
    controller = AttentionReplace(prompts, 50, {"default_": 1.0}, 0.4, width=4, height=4)
    revise_regionally_controlnet_forward(pipe, controller)
    cm = ConceptModels(pipe.unet)
    cm.load_ip_adapter_instantid(rs["sd"], ipw, heads=rs["heads"], dim_head=rs["dim_head"], num_tokens=16)
    cm.set_ip_adapter_scale(0.8)
    g = torch.Generator().manual_seed(53)
    lat0 = torch.randn(1, 4, size // 8, size // 8, generator=g).half()
    faces = [torch.nn.functional.normalize(torch.randn(512, generator=g), dim=0) for _ in range(2)]
    kps = r16(torch.rand(3, size, size, generator=g))
    masks = list(_masks(size))
    regions = [("a man", "bad", None), ("a woman", "bad", None)]
    out = pipe(prompt=[prompts, regions], negative_prompt=["noisy"] * 2, guidance_scale=3.0,
               num_inference_steps=STEPS, concept_models=cm, stage=2, region_masks=masks, image=kps,
               controlnet_conditioning_scale=0.8, face_embeds=faces, height=size, width=size, output_type="latent",
               latents=lat0, generator=torch.Generator("cuda").manual_seed(5)).images
    pe, ne, pp, np_ = pipe.encode_prompt(prompts, ["noisy"] * 2)
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32)
    octrl = op2p.AttentionReplaceOracle(prompts, 50, {"default_": 1.0}, 0.4, 4, 4)
    octrl.num_att_layers = len(ou.attention_names(ocfg(cfg)))
    main = ou.Ctx(sd, ocfg(cfg), attn_core=ou.make_p2p_attn_core(octrl))
    concepts = []
    for k, reg in enumerate(regions):
        e, n_, p_, np2 = pipe.encode_prompt(reg[0], reg[1])
        emb = faces[k].reshape(1, 1, 512)
        tokens = resampler_forward(rs["sd"], torch.cat([torch.zeros_like(emb), emb]), rs["heads"], rs["dim_head"])
        concepts.append(Concept(r16(torch.cat([n_, e])), r16(torch.cat([np2, p_])), tid.repeat(2, 1), masks[k],
                                unet=ou.Ctx(sd, ocfg(cfg), ip_weights=ipw, ip_tokens=16, ip_scale=0.8),
                                image_tokens=r16(tokens)))
    with oracle_schedule(_oracle_schedule(pipe.scheduler, 5, size // 8, size // 8)):
        ref = denoise(main, lat0.float(), r16(torch.cat([ne, pe])), r16(torch.cat([np_, pp])), tid.repeat(4, 1),
                      concepts, 2, STEPS, 3.0, identitynet=ou.Ctx(idsd, ocfg(cfg)),
                      identity_cond=kps[None].repeat(2, 1, 1, 1), identity_scale=0.8)
    e = rel(out, ref)
    print(f"instantid dpmpp_2m_sde_karras pipeline final-latent rel err {e:.3e}")
    assert e < 1.5e-3   # measured 1.17e-3 x 1.25


@pytest.mark.parametrize("rule", list(RULES))
def test_dedup_agrees_on_each_schedule(rule):
    """Dedup on and off agree (the bound of the default-Euler dedup test).  A stochastic schedule gives the two
    images different noise from step 0, so its twin rows are not deduplicated; the stage-2 prefix still is."""
    from omg_b200 import factory
    from omg_b200.config import UNetConfig
    wl = factory.build_lora_workload(UNetConfig.tiny(), 256, 2, 8, STEPS, 7.5)
    wl.pipe.scheduler = RULES[rule]()
    lat0 = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(14)).half()
    pipe, ctrl = wl.pipe, wl.controller
    kw = dict(wl.call_kwargs)

    def two_stage():
        counts = []
        o1 = pipe(stage=1, latents=lat0, generator=torch.Generator("cuda").manual_seed(9), **kw).images.clone()
        counts.append(pipe.sample_forwards)
        ctrl.reset()
        o2 = pipe(stage=2, latents=lat0, region_masks=wl.masks, generator=torch.Generator("cuda").manual_seed(9),
                  **kw).images.clone()
        counts.append(pipe.sample_forwards)
        ctrl.reset()
        return o1, o2, counts

    a1, a2, ca = two_stage()
    assert ca == [4 * STEPS, 4 * STEPS + 2 * 4]
    pipe.dedup = True
    d1, d2, cd = two_stage()
    stochastic = pipe.scheduler.stochastic
    assert cd == ([4 * STEPS, 4 * 2 + 2 * 4] if stochastic else [2 * STEPS, 2 * 8]), cd
    print(f"{rule}: dedup vs as-executed:", rel(d1, a1), rel(d2, a2))
    assert rel(d1, a1) < 1e-3 and rel(d2, a2) < 1e-3
    assert torch.equal(d1[0], d1[1]) != stochastic
    # without a generator a stochastic schedule draws from the global RNG: no prefix reuse
    if stochastic:
        pipe(stage=2, latents=lat0, region_masks=wl.masks, **kw)
        ctrl.reset()
        assert pipe.sample_forwards == 4 * STEPS + 2 * 4


def test_callback_replacing_latents_with_a_multistep_schedule():
    from omg_b200 import factory
    from omg_b200.config import UNetConfig
    wl = factory.build_lora_workload(UNetConfig.tiny(), 256, 2, 8, 6, 7.5)
    wl.pipe.scheduler = S.cli_scheduler("dpmpp_2m_karras", BASE)
    kw = dict(wl.call_kwargs)
    lat0 = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(3)).half()
    seen = []
    out = wl.pipe(stage=1, latents=lat0, callback_on_step_end=lambda p, i, t, d: seen.append(d["latents"].clone()) or {},
                  **kw).images
    wl.controller.reset()
    out2 = wl.pipe(stage=1, latents=lat0, callback_on_step_end=lambda p, i, t, d: {"latents": seen[i].clone()},
                   **kw).images
    wl.controller.reset()
    assert rel(out2, out) < 1e-3
    out3 = wl.pipe(stage=1, latents=lat0, callback_on_step_end=lambda p, i, t, d: {"latents": d["latents"] * 0.5}
                   if i == 2 else {}, **kw).images
    wl.controller.reset()
    assert rel(out3, out) > 1e-2 and torch.isfinite(out3.float()).all()


def test_sdxl_base_config_pipeline_equals_the_default(tmp_path):
    from omg_b200 import factory
    from omg_b200.config import UNetConfig
    wl = factory.build_lora_workload(UNetConfig.tiny(), 256, 2, 8, STEPS, 7.5)
    kw = dict(wl.call_kwargs)
    lat0 = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(14)).half()
    a = wl.pipe(stage=2, latents=lat0, region_masks=wl.masks, **kw).images.clone()
    wl.controller.reset()
    os.makedirs(tmp_path / "scheduler")
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(BASE))
    wl.pipe.scheduler = S.load_scheduler(tmp_path)
    b = wl.pipe(stage=2, latents=lat0, region_masks=wl.masks, **kw).images
    wl.controller.reset()
    assert type(wl.pipe.scheduler) is S.EulerDiscreteScheduler and torch.equal(a, b)
