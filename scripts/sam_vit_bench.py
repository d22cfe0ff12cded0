"""SAM ViT-H `set_image` at 1024² (synthetic weights): SamPredictor on the kernels against the same card's fp16 torch
restatement of ImageEncoderViT (oracle/sam_vit.py on fp16 weights, softmax materialised as segment_anything computes
it).  Timed windows alternate between the two; medians are reported with TFLOP/s from shapes, card and power limit.

  python scripts/sam_vit_bench.py [--kind vit_h] [--windows 7] [--iters 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def encoder_flops(C, depth, glob, T=4096, grid=64, window=14, out=256):
    """Multiply-adds x 2 of ImageEncoderViT at 1024²: patch embedding, per block qkv / proj / MLP (24 T C²), attention
    (Q K^T and P V, 4 n² C per group) with the rel-pos products (2 n (Sh + Sw) C), and the neck."""
    f = 2 * T * 768 * C
    nwin = (-(-grid // window)) ** 2
    for i in range(depth):
        f += 24 * T * C * C
        if i in glob:
            f += 4 * T * T * C + 2 * T * 2 * grid * C
        else:
            n = window * window
            f += nwin * (4 * n * n * C + 2 * n * 2 * window * C)
    return f + 2 * T * C * out + 2 * T * 9 * out * out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kind", default="vit_h")
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sam_vit_bench.py measures on the GPU; no CUDA device found")
    from omg_b200 import synthetic
    from omg_b200.sam import SamPredictor, sam_model_registry
    from omg_b200.sam_vit import KINDS
    from oracle.sam_decoder import preprocess
    from oracle.sam_vit import image_encoder
    C, depth, _, glob = KINDS[a.kind]
    sd = synthetic.make_sam_vit_state_dict(a.kind, 0, device="cuda", dtype=torch.float16)
    pred = SamPredictor(sam_model_registry[a.kind](state_dict=sd))
    osd = {k[len("image_encoder."):]: v for k, v in sd.items() if k.startswith("image_encoder.")}
    img = (np.random.default_rng(0).random((1024, 1024, 3)) * 255).astype(np.uint8)

    def kern():
        pred.set_image(img)

    def ref():
        with torch.no_grad():
            return image_encoder(preprocess(img).cuda().half(), osd)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.iters):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / a.iters

    kern()
    r = ref()
    rl = ((pred.get_image_embedding().float() - r.float()).norm() / r.float().norm()).item()
    tk, tt = [], []
    for _ in range(a.windows):
        tk.append(timed(kern))
        tt.append(timed(ref))
    fl = encoder_flops(C, depth, glob)
    mk, mt = statistics.median(tk), statistics.median(tt)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(json.dumps({"card": q[0] if q else torch.cuda.get_device_name(), "kind": a.kind, "tflop_per_image": fl / 1e12,
                      "set_image_ms": round(mk, 2), "torch_fp16_encoder_ms": round(mt, 2),
                      "kernel_tflops": round(fl / mk / 1e9, 1), "torch_tflops": round(fl / mt / 1e9, 1),
                      "embedding_rel_l2_vs_torch_fp16": rl}))


if __name__ == "__main__":
    main()
