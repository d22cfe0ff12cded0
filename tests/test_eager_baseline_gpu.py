"""The number to beat on the same GPU (SURVEY 8d, CPU-baseline row): the reference's actual library path - torch eager
fp16 (cuBLAS / cuDNN), probabilities materialised for the prompt-to-prompt controller - restated by the oracle and run
on the same GPU, timed for one main-UNet call (B=4, 128x128 latents) next to the CUDA path's graph replay.  Test
infrastructure: the only assertion is that the hand-written path is faster."""
import time

import pytest
import torch

pytestmark = pytest.mark.gpu


def test_main_unet_step_vs_torch_eager_fp16():
    from omg_b200 import factory, synthetic
    from omg_b200.config import UNetConfig
    from oracle import p2p as op2p
    from oracle import unet as ou
    dev = "cuda"
    cfg = UNetConfig.sdxl()
    wl = factory.build_lora_workload(cfg, 1024, 2, 32, 30, 7.5)
    pipe = wl.pipe
    kw = dict(wl.call_kwargs)
    lat0 = torch.randn(1, 4, 128, 128, generator=torch.Generator().manual_seed(0)).half()
    pipe(stage=1, latents=lat0, **{**kw, "num_inference_steps": 3})  # builds and captures the main runner
    wl.controller.reset()
    main = pipe._runner("main", pipe.unet, 4, 128, 128)
    key = next(iter(main.graphs))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        main.graphs[key].replay()
    e1.record()
    torch.cuda.synchronize()
    ours_ms = e0.elapsed_time(e1) / 5

    sd_h = synthetic.make_state_dict(cfg, seed=0, device=dev, dtype=torch.float16)
    prompts = kw["prompt"][0]
    ctrl = op2p.AttentionReplaceOracle(prompts, 50, {"default_": 1.0}, 0.4, 32, 32)
    ctrl.num_att_layers = 140
    ctrl.mapper = ctrl.mapper.to(dev)
    ctrl.cross_replace_alpha = ctrl.cross_replace_alpha.to(dev).half()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4, 4, 128, 128, generator=g).half().to(dev)
    ctx = torch.randn(4, 77, 2048, generator=g).half().to(dev)
    pooled = torch.randn(4, 1280, generator=g).half().to(dev)
    tid = torch.tensor([[1024, 1024, 0, 0, 1024, 1024]], dtype=torch.float32, device=dev).repeat(4, 1)
    c = ou.Ctx(sd_h, ou.UNetConfig(), attn_core=ou.make_p2p_attn_core(ctrl))
    ts = []
    with torch.no_grad():
        for it in range(4):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            y = ou.unet_forward(c, x, 500.0, ctx, pooled, tid)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
    eager_ms = sorted(ts[1:])[1]
    print({"main_unet_b4_128x128_ms": {"omg_b200_graph_replay": round(ours_ms, 2), "torch_eager_fp16_materialised_probs": round(eager_ms, 2)},
           "speedup": round(eager_ms / ours_ms, 2), "finite": bool(torch.isfinite(y).all())})
    assert ours_ms < eager_ms
