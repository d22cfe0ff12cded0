"""BASELINE config 1 at FULL SDXL widths (2.57 G parameters): one fusion step of stage 2 (step index 16) at 64x64
latents, main UNet rows (B=4, prompt-to-prompt self-replace window active) + one LoRA concept (B=2) as ONE grouped
forward, then omg_fuse_step; compared with the fp32 oracle on the host cores.  Tolerances (1.25 x measured): 2.2e-3 / 2.9e-3 on the noise
prediction, 3e-3 on the latents after the step."""
import os
import time

import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


def test_config1_full_width_fusion_step():
    from omg_b200 import ops, synthetic
    from omg_b200.config import UNetConfig
    from omg_b200.pipelines import LoraMultiConceptPipeline, revise_regionally_controlnet_forward
    from omg_b200.prompt_attention import AttentionReplace
    from omg_b200.unet import PackedUNet, RowGroup, UNetRunner
    from oracle import p2p as op2p
    from oracle import unet as ou
    from oracle.pipeline import fuse_noise
    from oracle.scheduler import EulerDiscrete
    dev = "cuda"
    cfg = UNetConfig.sdxl()
    sd = synthetic.make_state_dict(cfg, seed=0, device=dev, dtype=torch.float16)
    torch.set_num_threads(min(32, len(os.sched_getaffinity(0))))
    H = W = 64
    size = H * 8
    lo = synthetic.make_lora(cfg, seed=1000, rank=32, device=dev)
    unet = PackedUNet(cfg, sd, device=dev)
    unet.add_lora_set("c0", [(lo, 1.0)], 0.8)
    g = torch.Generator().manual_seed(0)
    ctx4 = torch.randn(2, 77, 2048, generator=g).half().float()
    ctx4 = torch.cat([ctx4[:1], ctx4[:1], ctx4[1:], ctx4[1:]])
    pooled4 = torch.randn(2, 1280, generator=g).half().float()
    pooled4 = torch.cat([pooled4[:1], pooled4[:1], pooled4[1:], pooled4[1:]])
    cctx = torch.randn(2, 77, 2048, generator=g).half().float()
    cpooled = torch.randn(2, 1280, generator=g).half().float()
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32)
    sched = EulerDiscrete()
    ts = sched.set_timesteps(30)
    i = 16
    lat = (torch.randn(2, 4, H, W, generator=g) * float(sched.sigmas[i])).half().float()
    mask = torch.zeros(size, size)
    mask[:, : size // 2] = 1
    lmi = sched.scale_model_input(torch.cat([lat] * 2), i).half().float()
    # --- CUDA path: grouped forward (main rows + concept rows) and the fused step kernel
    prompts = ["x y z"] * 2
    ctrl = AttentionReplace(prompts, 50, {"default_": 1.0}, 0.4, size // 32, size // 32)
    pipe = LoraMultiConceptPipeline(unet, use_graphs=False)
    revise_regionally_controlnet_forward(pipe, ctrl)
    ctrl.cur_step = i
    groups = [RowGroup(0, 4, None, False), RowGroup(4, 6, "c0", False)]
    r = UNetRunner(unet, 6, H, W, use_graphs=False, groups=groups)
    pipe._update_p2p_context([], ctrl, ctx4, first=True)
    r.set_conditioning([float(ts[i])], [(ctx4, None, False), (cctx, "c0", False)], torch.cat([pooled4, cpooled]),
                       tid.repeat(6, 1), extra_ctx=pipe._p2p_rows)
    x = torch.zeros(6, H, W, 8, dtype=torch.float16, device=dev)
    x[:4, ..., :4] = lmi.permute(0, 2, 3, 1).half().to(dev)
    x[4:, ..., :4] = torch.cat([lmi[3:4]] * 2).permute(0, 2, 3, 1).half().to(dev)
    r.sample_in.copy_(x)
    variant, _ = pipe._p2p_variant(r, ctrl, False)
    variant["self_items"] = variant["self_items"][:4] + [(4, 4, 4, 4), (5, 5, 5, 5)]
    variant["cross_items"] = [variant["cross_items"][0][:4] + [(4, 4, 6, 6), (5, 5, 7, 7)]]
    variant["ip_items"] = []
    noise = r.forward(0, variant)
    lat_dev = lat.permute(0, 2, 3, 1).contiguous().to(dev)
    m_lat = (torch.nn.functional.interpolate(mask[None, None], size=(H, W), mode="nearest")[0, 0] == 1).float().reshape(-1).to(dev)
    ops.fuse_step(noise[0:4], [noise[4:6]], [m_lat], 7.5, float(sched.sigmas[i]), float(sched.sigmas[i + 1]), lat_dev)
    torch.cuda.synchronize()
    noise_gpu = noise[..., :4].permute(0, 3, 1, 2).float().cpu()
    # --- fp32 oracle on the host cores (weights = the same fp16-rounded values)
    t0 = time.perf_counter()
    sd_cpu = {k: v.float().cpu() for k, v in sd.items()}
    ocfg = ou.UNetConfig()
    octrl = op2p.AttentionReplaceOracle(prompts, 50, {"default_": 1.0}, 0.4, size // 32, size // 32)
    octrl.num_att_layers = 140
    octrl.cur_step = i
    with torch.no_grad():
        n_main = ou.unet_forward(ou.Ctx(sd_cpu, ocfg, attn_core=ou.make_p2p_attn_core(octrl)), lmi, float(ts[i]), ctx4,
                                 pooled4, tid.repeat(4, 1))
        olo = {k: [(a.float().cpu(), b.float().cpu(), s * 0.8)] for k, (a, b, s) in lo.items()}
        n_c = ou.unet_forward(ou.Ctx(sd_cpu, ocfg, lora=olo), torch.cat([lmi[3:4]] * 2), float(ts[i]), cctx, cpooled,
                              tid.repeat(2, 1))
    fused = fuse_noise(n_main, [n_c], [mask])
    nu, nt = fused.chunk(2)
    ref_lat = sched.step(nu + 7.5 * (nt - nu), i, lat)
    out = {"config": 1, "desc": "SDXL widths, 64x64 latents, stage-2 step 16 (main B=4 under P2P + 1 LoRA concept B=2 as one "
                                "grouped forward), fp32 CPU oracle vs CUDA",
           "noise_rel_err_main": rel(noise_gpu[:4], n_main), "noise_rel_err_concept": rel(noise_gpu[4:], n_c),
           "latent_rel_err_after_step": rel(lat_dev.permute(0, 3, 1, 2), ref_lat), "oracle_cpu_s": time.perf_counter() - t0,
           "cpu_threads": torch.get_num_threads()}
    # --- the reference's own arithmetic for context: the same restatement run as fp16 torch eager on the GPU
    # (fp16 weights and activations, materialised fp16 probabilities, un-merged LoRA = the diffusers / peft library
    # path): how far THAT is from fp32, and how far the CUDA path is from it
    sd_h = {k: v.half().to(dev) for k, v in sd.items()}
    hctrl = op2p.AttentionReplaceOracle(prompts, 50, {"default_": 1.0}, 0.4, size // 32, size // 32)
    hctrl.num_att_layers, hctrl.cur_step = 140, i
    hctrl.mapper = hctrl.mapper.to(dev)
    hctrl.cross_replace_alpha = hctrl.cross_replace_alpha.to(dev).half()
    hd = lambda t: t.half().to(dev)  # noqa: E731
    with torch.no_grad():
        h_main = ou.unet_forward(ou.Ctx(sd_h, ocfg, attn_core=ou.make_p2p_attn_core(hctrl)), hd(lmi), float(ts[i]),
                                 hd(ctx4), hd(pooled4), tid.repeat(4, 1).to(dev))
        hlo = {k: [(hd(a), hd(b), s * 0.8)] for k, (a, b, s) in lo.items()}
        h_c = ou.unet_forward(ou.Ctx(sd_h, ocfg, lora=hlo), hd(torch.cat([lmi[3:4]] * 2)), float(ts[i]), hd(cctx),
                              hd(cpooled), tid.repeat(2, 1).to(dev))
    out["fp16_eager_rel_err_main"] = rel(h_main, n_main)
    out["fp16_eager_rel_err_concept"] = rel(h_c, n_c)
    out["cuda_vs_fp16_eager_main"] = rel(noise_gpu[:4], h_main)
    print(out)
    assert out["noise_rel_err_main"] < 2.2e-3 and out["noise_rel_err_concept"] < 2.9e-3
    assert out["latent_rel_err_after_step"] < 1.4e-3
    # never worse than the reference's own library arithmetic (fp16 eager) against fp32, measured in the same run
    assert out["noise_rel_err_main"] < out["fp16_eager_rel_err_main"]
    assert out["noise_rel_err_concept"] < out["fp16_eager_rel_err_concept"]

