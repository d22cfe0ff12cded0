"""Graph-replay time of the main (B=4) and the grouped fusion-step (B=8) UNet forward at 128x128 latents, under the
executor's A/B switches (each variant in its own process: the switches are read once).

  python scripts/forward_ms.py                       # prints one JSON line per variant
  python scripts/forward_ms.py --one                 # this process, current environment
"""
import json
import os
import subprocess
import sys

VARIANTS = [("default", {}), ("gn_stats_pass", {"OMG_GN_FUSE": "0"}), ("trunk_fp32_twins", {"OMG_TRUNK_F32": "1"}),
            ("launch_plan_executor", {"OMG_EXECUTOR": "plan"})]
if "--variants" in sys.argv:
    want = sys.argv[sys.argv.index("--variants") + 1].split(",")
    VARIANTS = [v for v in VARIANTS if v[0] in want]


def one():
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from omg_b200 import factory
    from omg_b200.config import UNetConfig
    wl = factory.build_lora_workload(UNetConfig.sdxl(), 1024, 2, 32, 30, 7.5)
    pipe, cm, kw = wl.pipe, wl.concept_models, dict(wl.call_kwargs)
    lat0 = torch.randn(1, 4, 128, 128, generator=torch.Generator().manual_seed(14)).half()
    # two short pipeline calls build, warm and capture every runner / graph the loop uses
    kw["num_inference_steps"] = 20
    pipe(stage=1, latents=lat0, **kw)
    wl.controller.reset()
    pipe(stage=2, latents=lat0, region_masks=wl.masks, **kw)
    wl.controller.reset()
    torch.cuda.synchronize()
    out = {}
    for tag, r in pipe._runners.items():
        for key, g in r.graphs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(3):
                g.replay()
            e0.record()
            for _ in range(10):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            out[f"{tag[0]}_b{tag[2]}:{'/'.join(str(k) for k in key)}"] = {"ms": round(e0.elapsed_time(e1) / 10, 3),
                                                                           "launches": r.graph_launches[key]}
        for key, pl in r.plans.items():   # OMG_EXECUTOR=plan: the forward replayed from C (omg_plan_run), no CUDA graph
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(3):
                pl.run()
            e0.record()
            for _ in range(10):
                pl.run()
            e1.record()
            torch.cuda.synchronize()
            out[f"{tag[0]}_b{tag[2]}:{'/'.join(str(k) for k in key)}"] = {"ms": round(e0.elapsed_time(e1) / 10, 3),
                                                                           "launches": len(pl), "executor": "plan"}
    print(json.dumps(out))


if __name__ == "__main__":
    if "--one" in sys.argv:
        one()
    else:
        for name, env in VARIANTS:
            e = dict(os.environ)
            e.update(env)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one"], env=e, capture_output=True, text=True)
            line = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else r.stderr[-400:]
            print(json.dumps({"variant": name, "env": env, "result": json.loads(line) if line.startswith("{") else line}), flush=True)
