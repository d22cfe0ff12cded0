"""Cost of LoCon adapters in the grouped forward: main rows (B = 4) + two concepts (B = 2 each) at 128 x 128 latents,
SDXL width, synthetic weights, CUDA-graph replay.  The concepts carry a transformer-only LoRA in one runner and a LoCon
adapter (the same Linears plus every ResBlock / down-sampler / up-sampler module) in the other; timed windows alternate
between the two in one process.  Prints one JSON line: median and min-max ms per forward of both, kernel launches per
forward of both, the HBM bytes of the conv weight planes, card name and power limit.  Needs a GPU (there is no CPU timing).

  python scripts/lora_conv_bench.py [--windows 7] [--iters 10] [--size 128]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--size", type=int, default=128, help="latent height = width")
    ap.add_argument("--rank", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_conv_bench.py needs a CUDA device")
    from omg_b200 import synthetic
    from omg_b200.config import UNetConfig
    from omg_b200.unet import PackedUNet, RowGroup, UNetRunner
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    gpu = q.stdout.strip() or torch.cuda.get_device_name(0)
    dev = "cuda"
    cfg = UNetConfig.sdxl()
    model = PackedUNet(cfg, synthetic.make_state_dict(cfg, seed=0, device=dev, dtype=torch.float16), device=dev)
    H = W = a.size
    g = torch.Generator().manual_seed(0)
    ctx = torch.randn(8, 77, cfg.cross_attention_dim, generator=g)
    pooled = torch.randn(8, cfg.pooled_dim, generator=g)
    tid = torch.tensor([[H * 8, W * 8, 0, 0, H * 8, W * 8]], dtype=torch.float32).repeat(8, 1)
    x = torch.randn(8, H, W, 8, generator=g).half().to(dev)
    x[..., 4:] = 0
    runners, launches, plane_bytes = {}, {}, {}
    for kind in ("linear", "locon"):
        for k in range(2):
            lo = synthetic.make_lora(cfg, seed=1000 + k, rank=a.rank, device=dev, conv=kind == "locon")
            model.add_lora_set(f"{kind}{k}", [(lo, 1.0)], 0.8)
        groups = [RowGroup(0, 4, None), RowGroup(4, 6, f"{kind}0"), RowGroup(6, 8, f"{kind}1")]
        r = UNetRunner(model, 8, H, W, groups=groups, use_graphs=True)
        r.set_conditioning([500.0], [(ctx[gr.start:gr.stop], gr.lora_key, False) for gr in groups], pooled, tid)
        r.sample_in.copy_(x)
        for _ in range(3):   # eager warm-up, capture, replay
            r.forward(0, key=("k",))
        torch.cuda.synchronize()
        runners[kind], launches[kind] = r, r.graph_launches[("k",)]
        plane_bytes[kind] = sum(v[0].numel() * 2 for k, v in r._b2_cache.items() if k.startswith("conv|"))
        if not r.merge_lora:
            print("note: OMG_LORA=unmerged - the convs run once per stream instead of on weight planes", file=sys.stderr)
    ms = {"linear": [], "locon": []}
    for _ in range(a.windows):
        for kind, r in runners.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                r.forward(0, key=("k",))
            e1.record()
            torch.cuda.synchronize()
            ms[kind].append(e0.elapsed_time(e1) / a.iters)
    out = {"workload": f"grouped UNet forward B=4+2+2, {H}x{W} latents, SDXL width, rank {a.rank}, graph replay", "gpu": gpu,
           "windows": a.windows, "iters": a.iters}
    for kind in ms:
        out[kind] = {"median_ms": round(statistics.median(ms[kind]), 3), "min_ms": round(min(ms[kind]), 3),
                     "max_ms": round(max(ms[kind]), 3), "launches": launches[kind],
                     "conv_plane_gb": round(plane_bytes[kind] / 1e9, 3)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
