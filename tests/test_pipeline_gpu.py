"""GPU parity of the full two-stage loops (LoRA and InstantID variants) against oracle.pipeline.denoise on the tiny
topology: 18 steps so that the fusion window (step index > 15) is exercised, P2P self-replace threshold 8x8 tokens,
two concepts with disjoint masks.  Final-latent tolerances allow for 18 chained UNet calls at fp16 storage vs the fp32
oracle."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from util_models import lora, ocfg, oracle_lora, r16, rel, weights  # noqa: E402

STEPS = 18
G = os.path.join(os.path.dirname(__file__), "golden")


def _masks(size):
    m1 = torch.zeros(size, size)
    m2 = torch.zeros(size, size)
    m1[size // 8: 7 * size // 8, size // 16: 7 * size // 16] = 1
    m2[size // 8: 7 * size // 8, 9 * size // 16: 15 * size // 16] = 1
    return m1, m2


@pytest.mark.parametrize("share,lora_mode", [(False, "merged"), (True, "merged"), (True, "unmerged")])
def test_lora_two_stage_pipeline(share, lora_mode, monkeypatch):
    """share=True: the concept UNet is the main UNet's packed weights -> fusion steps run as ONE grouped forward
    (main rows + both concepts' rows); share=False: separate concept forwards."""
    from omg_b200.config import UNetConfig
    from omg_b200.pipelines import ConceptModels, LoraMultiConceptPipeline, revise_regionally_controlnet_forward
    from omg_b200.prompt_attention import AttentionReplace
    from omg_b200.unet import PackedUNet
    from oracle import p2p as op2p
    from oracle import unet as ou
    from oracle.pipeline import Concept, denoise
    monkeypatch.setenv("OMG_LORA", lora_mode)
    cfg = UNetConfig.tiny()
    sd = weights(cfg, 0)
    size = 256
    prompt = "a man and a woman on the beach"
    prompts = [prompt] * 2
    regions = [("a man smiling", "blurry"), ("a woman smiling", "blurry")]
    pipe = LoraMultiConceptPipeline(PackedUNet(cfg, sd))
    controller = AttentionReplace(prompts, 50, {"default_": 1.0}, 0.4, width=8, height=8)
    revise_regionally_controlnet_forward(pipe, controller)
    cm = ConceptModels(pipe.unet if share else PackedUNet(cfg, sd))
    loras = [lora(cfg, 101), lora(cfg, 102)]
    cm.load_lora_weights(loras[0], adapter_name="manA")
    cm.load_lora_weights(loras[1], adapter_name="womanB")
    g = torch.Generator().manual_seed(14)
    lat0 = torch.randn(1, 4, size // 8, size // 8, generator=g).half()
    masks = list(_masks(size))
    common = dict(prompt=[prompts, regions], negative_prompt=["noisy"] * 2, guidance_scale=7.5,
                  num_inference_steps=STEPS, cross_attention_kwargs={"scale": 0.8}, concept_models=cm,
                  lora_list=["manA", "womanB"], styleL=False, height=size, width=size, output_type="latent",
                  latents=lat0)
    out1 = pipe(stage=1, **common).images
    assert controller.cur_step == STEPS
    controller.reset()
    out2 = pipe(stage=2, region_masks=masks, **common).images
    assert torch.equal(out1[0], out1[1])                      # stage 1: both rows identical trajectories
    if share:   # grouped B=8 launches may tile differently from B=4: equal up to fp16 rounding noise
        assert rel(out2[0], out1[0]) < 2e-3
    else:
        assert torch.equal(out2[0], out1[0])                  # image 0 of stage 2 reproduces the layout image
    assert not torch.equal(out2[1], out2[0])

    # ---- oracle
    pe, ne, pp, np_ = pipe.encode_prompt(prompts, ["noisy"] * 2, 0.8)
    ctx4, pooled4 = r16(torch.cat([ne, pe])), r16(torch.cat([np_, pp]))
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32)
    octrl = op2p.AttentionReplaceOracle(prompts, 50, {"default_": 1.0}, 0.4, 8, 8)
    octrl.num_att_layers = len(ou.attention_names(ocfg(cfg)))
    main = ou.Ctx(sd, ocfg(cfg), attn_core=ou.make_p2p_attn_core(octrl))
    concepts = []
    for k, (rp, rn) in enumerate(regions):
        e, n_, p_, np2 = cm.encode_prompt(rp, negative_prompt=rn)
        concepts.append(Concept(r16(torch.cat([n_, e])), r16(torch.cat([np2, p_])), tid.repeat(2, 1), masks[k],
                                unet=ou.Ctx(sd, ocfg(cfg), lora=oracle_lora([(loras[k], 1.0)], 0.8))))
    ref2 = denoise(main, lat0.float(), ctx4, pooled4, tid.repeat(4, 1), concepts, 2, STEPS, 7.5)
    e0, e1 = rel(out2[0], ref2[0]), rel(out2[1], ref2[1])
    print("lora pipeline final-latent rel err: layout", e0, "fused", e1)
    assert e0 < 2.8e-3 and e1 < 2.8e-3


def test_lora_pipeline_skips_concept_without_mask_and_style_adapter():
    from omg_b200.config import UNetConfig
    from omg_b200.pipelines import ConceptModels, LoraMultiConceptPipeline
    from omg_b200.unet import PackedUNet
    from oracle import unet as ou
    from oracle.pipeline import Concept, denoise
    cfg = UNetConfig.tiny()
    sd = weights(cfg, 0)
    size = 128
    pipe = LoraMultiConceptPipeline(PackedUNet(cfg, sd))           # no controller installed: plain attention
    cm = ConceptModels(PackedUNet(cfg, sd))
    loras = {"a": lora(cfg, 201), "b": lora(cfg, 202), "style": lora(cfg, 203)}
    for k, v in loras.items():
        cm.load_lora_weights(v, adapter_name=k)
    g = torch.Generator().manual_seed(3)
    lat0 = torch.randn(1, 4, size // 8, size // 8, generator=g).half()
    m1, _ = _masks(size)
    regions = [("x", "y"), ("z", "w")]
    out = pipe(prompt=[["p"] * 2, regions], negative_prompt=["n"] * 2, guidance_scale=5.0, num_inference_steps=STEPS,
               cross_attention_kwargs={"scale": 0.8}, concept_models=cm, lora_list=["a", "b"], styleL=True, stage=2,
               region_masks=[m1, None], height=size, width=size, output_type="latent", latents=lat0).images
    pe, ne, pp, np_ = pipe.encode_prompt(["p"] * 2, ["n"] * 2)
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32)
    concepts = []
    for k, (rp, rn) in enumerate(regions):
        e, n_, p_, np2 = cm.encode_prompt(rp, negative_prompt=rn)
        lo = oracle_lora([(loras["ab"[k]], 0.7), (loras["style"], 0.5)], 0.8)
        concepts.append(Concept(r16(torch.cat([n_, e])), r16(torch.cat([np2, p_])), tid.repeat(2, 1),
                                m1 if k == 0 else None, unet=ou.Ctx(sd, ocfg(cfg), lora=lo)))
    ref = denoise(ou.Ctx(sd, ocfg(cfg)), lat0.float(), r16(torch.cat([ne, pe])), r16(torch.cat([np_, pp])),
                  tid.repeat(4, 1), concepts, 2, STEPS, 5.0)
    e = rel(out, ref)
    print("style/None-mask pipeline rel err", e)
    assert e < 2.2e-3


@pytest.mark.parametrize("share", [False, True])
def test_instantid_two_stage_pipeline(share):
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
    rs = torch.load(os.path.join(G, "resampler.pt"))
    rs["sd"] = {k: v.float() for k, v in rs["sd"].items()}  # stored as fp16 (fp16-representable values)
    ipw = {k: (r16(a), r16(b)) for k, (a, b) in synthetic.make_ip_adapter(cfg, 31).items()}
    pipe = InstantidMultiConceptPipeline(PackedUNet(cfg, sd), controlnet=PackedUNet(cfg, idsd, controlnet=True))
    prompts = ["two people"] * 2
    controller = AttentionReplace(prompts, 50, {"default_": 1.0}, 0.4, width=4, height=4)
    revise_regionally_controlnet_forward(pipe, controller)
    cm = ConceptModels(pipe.unet if share else PackedUNet(cfg, sd))
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
               latents=lat0).images
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
    ref = denoise(main, lat0.float(), r16(torch.cat([ne, pe])), r16(torch.cat([np_, pp])), tid.repeat(4, 1), concepts,
                  2, STEPS, 3.0, identitynet=ou.Ctx(idsd, ocfg(cfg)), identity_cond=kps[None].repeat(2, 1, 1, 1),
                  identity_scale=0.8)
    e = rel(out, ref)
    print("instantid pipeline final-latent rel err", e)
    assert e < 1.3e-3


def test_dedup_mode_reproduces_the_as_executed_result():
    """Opt-in exact de-duplication (SURVEY 8d): twin rows run B=2 until the first fusion step, stage 2 resumes from the
    latents stage 1 had after step 15.  Same results, 172/296 of the UNet sample-forwards at 30 steps (here, at 18
    steps: 52 instead of 152)."""
    from omg_b200 import factory
    from omg_b200.config import UNetConfig
    wl = factory.build_lora_workload(UNetConfig.tiny(), 256, 2, 8, STEPS, 7.5)
    lat0 = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(14)).half()
    pipe, ctrl = wl.pipe, wl.controller
    kw = dict(wl.call_kwargs)

    def two_stage():
        counts = []
        o1 = pipe(stage=1, latents=lat0, **kw).images.clone()
        counts.append(pipe.sample_forwards)
        assert ctrl.cur_step == STEPS
        ctrl.reset()
        o2 = pipe(stage=2, latents=lat0, region_masks=wl.masks, **kw).images.clone()
        counts.append(pipe.sample_forwards)
        assert ctrl.cur_step == STEPS
        ctrl.reset()
        return o1, o2, counts

    a1, a2, ca = two_stage()
    assert ca == [4 * STEPS, 4 * STEPS + 2 * 4]  # fusion in steps 16, 17 with two concepts
    pipe.dedup = True
    d1, d2, cd = two_stage()
    assert cd == [2 * STEPS, 2 * 8]
    print("dedup vs as-executed:", rel(d1, a1), rel(d2, a2), "bitwise", torch.equal(d1, a1), torch.equal(d2, a2))
    assert rel(d1, a1) < 1e-3 and rel(d2, a2) < 1e-3
    assert torch.equal(d1[0], d1[1])  # stage 1: image 1 is image 0
    # a different seed in stage 2 must not resume from the cached prefix
    lat1 = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(15)).half()
    pipe(stage=2, latents=lat1, region_masks=wl.masks, **kw)
    assert pipe.sample_forwards == 2 * 16 + 2 * 8
    ctrl.reset()


def test_generator_only_latent_path_matches_the_reference_call():
    """A15: with `generator=` and no `latents=` the pipeline draws randn((1,4,h,w), generator, fp16) on the generator's
    device exactly like prepare_latents / randn_tensor (lora_pipeline.py:397-409; the CLIs pass
    torch.Generator(device).manual_seed(seed), inference_lora.py:262,291), so a seed reproduces the reference's noise."""
    from omg_b200 import factory
    from omg_b200.config import UNetConfig
    wl = factory.build_lora_workload(UNetConfig.tiny(), 256, 2, 8, 4, 7.5)
    kw = dict(wl.call_kwargs)
    for gdev in ("cpu", "cuda"):
        a = wl.pipe(stage=1, generator=torch.Generator(gdev).manual_seed(14), **kw).images.clone()
        wl.controller.reset()
        lat0 = torch.randn((1, 4, 32, 32), generator=torch.Generator(gdev).manual_seed(14), device=gdev, dtype=torch.float16)
        b = wl.pipe(stage=1, latents=lat0, **kw).images.clone()
        wl.controller.reset()
        assert torch.equal(a, b)
    c = wl.pipe(stage=1, generator=torch.Generator("cuda").manual_seed(15), **kw).images
    wl.controller.reset()
    assert not torch.equal(a, c)


def test_callback_on_step_end_sees_and_may_replace_latents():
    """callback_on_step_end(pipe, i, t, {"latents": (2,4,h,w)}) after every scheduler step (lora_pipeline.py:617-625)."""
    from omg_b200 import factory
    from omg_b200.config import UNetConfig
    wl = factory.build_lora_workload(UNetConfig.tiny(), 256, 2, 8, 4, 7.5)
    kw = dict(wl.call_kwargs)
    lat0 = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(3)).half()
    seen = []
    out = wl.pipe(stage=1, latents=lat0, callback_on_step_end=lambda p, i, t, d: seen.append((i, float(t), d["latents"].clone())) or {},
                  **kw).images
    wl.controller.reset()
    assert [s[0] for s in seen] == [0, 1, 2, 3] and seen[0][2].shape == (2, 4, 32, 32)
    assert torch.equal(seen[-1][2].half(), out)
    # replacing the latents after step 1 with the recorded ones is a no-op; replacing them with zeros is not
    out2 = wl.pipe(stage=1, latents=lat0, callback_on_step_end=lambda p, i, t, d: {"latents": seen[i][2].clone()}, **kw).images
    wl.controller.reset()
    assert rel(out2, out) < 1e-3
    out3 = wl.pipe(stage=1, latents=lat0, callback_on_step_end=lambda p, i, t, d: {"latents": torch.zeros_like(d["latents"])} if i == 1 else {},
                   **kw).images
    wl.controller.reset()
    assert rel(out3, out) > 1e-2


def test_main_pass_controlnet_condition_change_with_graphs():
    """The LoRA pipeline with a spatial ControlNet on the main pass (lora_pipeline.py:519-540), called twice with two
    different condition images through CUDA graphs: the captured ControlNet graph reads the condition embedding from a
    persistent buffer, so the second call must see the new image (advisor finding of round 1) - each call is compared with
    a fresh eager pipeline on the same image and with the oracle."""
    from omg_b200.config import UNetConfig
    from omg_b200.pipelines import ConceptModels, LoraMultiConceptPipeline
    from omg_b200.unet import PackedUNet
    from oracle import unet as ou
    from oracle.pipeline import Concept, denoise
    cfg = UNetConfig.tiny()
    sd, csd = weights(cfg, 0), weights(cfg, 21, controlnet=True)
    size, steps = 128, 4
    g = torch.Generator().manual_seed(5)
    lat0 = torch.randn(1, 4, size // 8, size // 8, generator=g).half()
    conds = [r16(torch.rand(3, size, size, generator=g)) for _ in range(2)]
    regions = [("x", "y"), ("z", "w")]
    common = dict(prompt=[["p"] * 2, regions], negative_prompt=["n"] * 2, guidance_scale=5.0, num_inference_steps=steps,
                  cross_attention_kwargs={"scale": 0.8}, lora_list=[], styleL=False, stage=1, height=size, width=size,
                  output_type="latent", latents=lat0, controlnet_conditioning_scale=0.7)

    def build(use_graphs):
        unet = PackedUNet(cfg, sd)
        pipe = LoraMultiConceptPipeline(unet, controlnet=PackedUNet(cfg, csd, controlnet=True), use_graphs=use_graphs)
        return pipe, ConceptModels(unet)

    pipe, cm = build(True)
    outs = [pipe(image=[c, c], concept_models=cm, **common).images.clone() for c in conds]
    outs.append(pipe(image=[conds[0], conds[0]], concept_models=cm, **common).images.clone())   # back to the first image
    assert torch.equal(outs[0], outs[2]) and not torch.equal(outs[0], outs[1])
    # the same loop with every forward replayed from a C-ABI launch plan (omg_plan) instead of a CUDA graph
    planned, cm3 = build(False)
    planned.executor = "plan"
    for k, c in enumerate(conds):
        assert rel(planned(image=[c, c], concept_models=cm3, **common).images, outs[k]) < 1e-5
    assert sum(len(r.plans) for r in planned._runners.values()) >= 2 and not any(r.graphs for r in planned._runners.values())
    pe, ne, pp, np_ = pipe.encode_prompt(["p"] * 2, ["n"] * 2)
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32)
    for k, c in enumerate(conds):
        eager, cm2 = build(False)
        ref_eager = eager(image=[c, c], concept_models=cm2, **common).images
        assert rel(outs[k], ref_eager) < 1e-5
        ref = denoise(ou.Ctx(sd, ocfg(cfg)), lat0.float(), r16(torch.cat([ne, pe])), r16(torch.cat([np_, pp])), tid.repeat(4, 1),
                      [], 1, steps, 5.0, controlnet=ou.Ctx(csd, ocfg(cfg)), controlnet_cond=c[None].repeat(4, 1, 1, 1),
                      controlnet_scale=0.7)
        e = rel(outs[k], ref)
        print("main-pass controlnet pipeline rel err", e)
        assert e < 3.5e-3   # measured on H100: 2.5e-3 / 2.6e-3: 4 large Euler steps at guidance 5 (main UNet + ControlNet per step)


def test_instantid_main_pass_controlnet_together_with_identitynet():
    """InstantID with BOTH a spatial ControlNet on the main pass (controlnet2, instantid_pipeline.py:574-616) and the
    IdentityNet on the concept pass (:639-674) while the concept UNet shares the packed base weights: one grouped forward
    with two residual slots (rows 0-3 <- controlnet2, concept rows <- IdentityNet)."""
    from omg_b200 import synthetic
    from omg_b200.config import UNetConfig
    from omg_b200.pipelines import ConceptModels, InstantidMultiConceptPipeline
    from omg_b200.unet import PackedUNet
    from oracle import unet as ou
    from oracle.pipeline import Concept, denoise
    from oracle.resampler import resampler_forward
    cfg = UNetConfig.tiny()
    sd, idsd, c2sd = weights(cfg, 0), weights(cfg, 41, controlnet=True), weights(cfg, 42, controlnet=True)
    size = 128
    rs = torch.load(os.path.join(G, "resampler.pt"))
    rs["sd"] = {k: v.float() for k, v in rs["sd"].items()}  # stored as fp16 (fp16-representable values)
    ipw = {k: (r16(a), r16(b)) for k, (a, b) in synthetic.make_ip_adapter(cfg, 31).items()}
    pipe = InstantidMultiConceptPipeline(PackedUNet(cfg, sd), controlnet=PackedUNet(cfg, idsd, controlnet=True))
    pipe.controlnet2 = PackedUNet(cfg, c2sd, controlnet=True)
    cm = ConceptModels(pipe.unet)
    cm.load_ip_adapter_instantid(rs["sd"], ipw, heads=rs["heads"], dim_head=rs["dim_head"], num_tokens=16)
    cm.set_ip_adapter_scale(0.8)
    g = torch.Generator().manual_seed(53)
    lat0 = torch.randn(1, 4, size // 8, size // 8, generator=g).half()
    faces = [torch.nn.functional.normalize(torch.randn(512, generator=g), dim=0) for _ in range(2)]
    kps, pose = r16(torch.rand(3, size, size, generator=g)), r16(torch.rand(3, size, size, generator=g))
    masks = list(_masks(size))
    regions = [("a man", "bad", None), ("a woman", "bad", None)]
    prompts = ["two people"] * 2
    out = pipe(prompt=[prompts, regions], negative_prompt=["noisy"] * 2, guidance_scale=3.0, num_inference_steps=STEPS,
               concept_models=cm, stage=2, region_masks=masks, image=kps, controlnet_conditioning_scale=0.8, t2i_image=pose,
               t2i_controlnet_conditioning_scale=0.6, face_embeds=faces, height=size, width=size, output_type="latent",
               latents=lat0).images
    pe, ne, pp, np_ = pipe.encode_prompt(prompts, ["noisy"] * 2)
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32)
    concepts = []
    for k, reg in enumerate(regions):
        e, n_, p_, np2 = pipe.encode_prompt(reg[0], reg[1])
        emb = faces[k].reshape(1, 1, 512)
        tokens = resampler_forward(rs["sd"], torch.cat([torch.zeros_like(emb), emb]), rs["heads"], rs["dim_head"])
        concepts.append(Concept(r16(torch.cat([n_, e])), r16(torch.cat([np2, p_])), tid.repeat(2, 1), masks[k],
                                unet=ou.Ctx(sd, ocfg(cfg), ip_weights=ipw, ip_tokens=16, ip_scale=0.8), image_tokens=r16(tokens)))
    ref = denoise(ou.Ctx(sd, ocfg(cfg)), lat0.float(), r16(torch.cat([ne, pe])), r16(torch.cat([np_, pp])), tid.repeat(4, 1), concepts,
                  2, STEPS, 3.0, controlnet=ou.Ctx(c2sd, ocfg(cfg)), controlnet_cond=pose[None].repeat(4, 1, 1, 1), controlnet_scale=0.6,
                  identitynet=ou.Ctx(idsd, ocfg(cfg)), identity_cond=kps[None].repeat(2, 1, 1, 1), identity_scale=0.8)
    e = rel(out, ref)
    print("instantid + main-pass controlnet pipeline rel err", e)
    assert e < 1.3e-3   # measured on H100: 0.96e-3
