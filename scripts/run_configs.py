"""BASELINE.json configs 3, 4 on one GPU (config 2 is bench.py's workload, config 5 its --gpus sweep).

  (config 1, the full-width parity check against the fp32 oracle, is tests/test_config1_gpu.py)
  config 3  OMG + InstantID, 2 identities (IP-adapter concept UNet + IdentityNet), 1024^2, 30 steps: s / image.
  config 4  4 LoRA concepts + style LoRA + spatial ControlNet on the main pass, 1024^2, 30 steps: s / image.
Prints one JSON object per config; results are copied into BASELINE.md section 5.
"""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from omg_b200 import synthetic  # noqa: E402
from omg_b200.config import UNetConfig  # noqa: E402
from omg_b200.pipelines import (ConceptModels, InstantidMultiConceptPipeline, LoraMultiConceptPipeline,  # noqa: E402
                                revise_regionally_controlnet_forward)
from omg_b200.prompt_attention import AttentionReplace  # noqa: E402
from omg_b200.unet import PackedUNet  # noqa: E402

dev = "cuda"
cfg = UNetConfig.sdxl()
which = sys.argv[1:] or ["3", "4"]


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


def timed_image(fn, warm=1, reps=1):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


sd = synthetic.make_state_dict(cfg, seed=0, device=dev, dtype=torch.float16)

if "3" in which:
    size = 1024
    unet = PackedUNet(cfg, sd, device=dev)
    idnet = PackedUNet(cfg, synthetic.make_state_dict(cfg, seed=1, controlnet=True, device=dev, dtype=torch.float16),
                       device=dev, controlnet=True)
    pipe = InstantidMultiConceptPipeline(unet, controlnet=idnet)
    prompt = "two people on a beach"
    ctrl = AttentionReplace([prompt] * 2, 50, {"default_": 1.0}, 0.4, size // 32, size // 32)
    revise_regionally_controlnet_forward(pipe, ctrl)
    cm = ConceptModels(unet)
    dim, depth, heads = 1280, 4, 20
    g = torch.Generator().manual_seed(7)

    def rn(*s):
        return torch.randn(*s, generator=g) * (s[-1] ** -0.5)

    rs = {"latents": rn(1, 16, dim), "proj_in.weight": rn(dim, 512), "proj_in.bias": torch.zeros(dim),
          "proj_out.weight": rn(2048, dim), "proj_out.bias": torch.zeros(2048), "norm_out.weight": torch.ones(2048),
          "norm_out.bias": torch.zeros(2048)}
    for li in range(depth):
        a, f = f"layers.{li}.0", f"layers.{li}.1"
        for nm in ("norm1", "norm2"):
            rs[f"{a}.{nm}.weight"], rs[f"{a}.{nm}.bias"] = torch.ones(dim), torch.zeros(dim)
        rs[f"{a}.to_q.weight"], rs[f"{a}.to_kv.weight"], rs[f"{a}.to_out.weight"] = rn(dim, dim), rn(2 * dim, dim), rn(dim, dim)
        rs[f"{f}.0.weight"], rs[f"{f}.0.bias"] = torch.ones(dim), torch.zeros(dim)
        rs[f"{f}.1.weight"], rs[f"{f}.3.weight"] = rn(4 * dim, dim), rn(dim, 4 * dim)
    cm.load_ip_adapter_instantid(rs, synthetic.make_ip_adapter(cfg, 31, device=dev), heads=heads, dim_head=64, num_tokens=16)
    cm.set_ip_adapter_scale(0.8)
    faces = [torch.nn.functional.normalize(torch.randn(512, generator=torch.Generator().manual_seed(s)), dim=0) for s in (1, 2)]
    cond = torch.rand(3, size, size, generator=g)
    masks = synthetic.rect_masks(2, (size, size))
    regions = [("a man", "bad", None), ("a woman", "bad", None)]
    common = dict(prompt=[[prompt] * 2, regions], negative_prompt=["noisy"] * 2, guidance_scale=3.0,
                  num_inference_steps=30, concept_models=cm, image=cond, controlnet_conditioning_scale=0.8,
                  face_embeds=faces, height=size, width=size, output_type="latent")

    def image():
        gen = torch.Generator().manual_seed(53)
        lat0 = torch.randn(1, 4, size // 8, size // 8, generator=gen).half()
        pipe(stage=1, latents=lat0, **common)
        ctrl.reset()
        o = pipe(stage=2, latents=lat0, region_masks=masks, **common).images
        ctrl.reset()
        return o

    t = timed_image(image, warm=2, reps=1)
    o = image()
    print(json.dumps({"config": 3, "desc": "OMG+InstantID, 2 identities (IP-adapter concept streams + IdentityNet), 1024^2, "
                                           "30 steps per stage, guidance 3.0", "s_per_image": t, "images_per_s": 1 / t,
                      "finite": bool(torch.isfinite(o).all())}), flush=True)
    del pipe, cm, idnet, unet
    torch.cuda.empty_cache()

if "4" in which:
    size = 1024
    unet = PackedUNet(cfg, sd, device=dev)
    cn = PackedUNet(cfg, synthetic.make_state_dict(cfg, seed=2, controlnet=True, device=dev, dtype=torch.float16),
                    device=dev, controlnet=True)
    pipe = LoraMultiConceptPipeline(unet, controlnet=cn)
    prompt = "four friends in a park"
    ctrl = AttentionReplace([prompt] * 2, 50, {"default_": 1.0}, 0.4, size // 32, size // 32)
    revise_regionally_controlnet_forward(pipe, ctrl)
    style = synthetic.make_lora(cfg, seed=999, rank=32, device=dev)
    pipe.load_lora_weights(style, adapter_name="style")
    cm = ConceptModels(unet)
    cm.load_lora_weights(style, adapter_name="style")
    names = []
    for k in range(4):
        cm.load_lora_weights(synthetic.make_lora(cfg, seed=1000 + k, rank=32, device=dev), adapter_name=f"c{k}")
        names.append(f"c{k}")
    masks = []
    for qy in range(2):
        for qx in range(2):
            m = torch.zeros(size, size)
            m[qy * 512 + 32:(qy + 1) * 512 - 32, qx * 512 + 32:(qx + 1) * 512 - 32] = 1
            masks.append(m)
    cond = torch.rand(3, size, size, generator=torch.Generator().manual_seed(5))
    regions = [(f"person {k}", "bad") for k in range(4)]
    common = dict(prompt=[[prompt] * 2, regions], negative_prompt=["noisy"] * 2, guidance_scale=7.5,
                  num_inference_steps=30, cross_attention_kwargs={"scale": 0.8}, concept_models=cm, lora_list=names,
                  styleL=True, image=[cond, cond], height=size, width=size, output_type="latent")

    def image4():
        gen = torch.Generator().manual_seed(14)
        lat0 = torch.randn(1, 4, size // 8, size // 8, generator=gen).half()
        pipe(stage=1, latents=lat0, **common)
        ctrl.reset()
        o = pipe(stage=2, latents=lat0, region_masks=masks, **common).images
        ctrl.reset()
        return o

    t = timed_image(image4, warm=2, reps=1)
    o = image4()
    print(json.dumps({"config": 4, "desc": "4 LoRA concepts (each + style adapter, weights [0.7, 0.5]) + style LoRA on the "
                                           "main pass + spatial ControlNet (B=4) on the main pass, 1024^2, 30 steps per stage",
                      "s_per_image": t, "images_per_s": 1 / t, "finite": bool(torch.isfinite(o).all())}), flush=True)
