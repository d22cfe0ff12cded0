"""omg_attention_relpos at SAM ViT-H's shapes (16 heads of 80, 64 x 64 tokens at the 1024² input): a global block and a
14 x 14-window block, against the same card's fp16 torch restatement of segment_anything's Attention (softmax
materialised, as segment_anything computes it).  Timed windows alternate between the two; the median of the windows is
reported with TFLOP/s from shapes (the two attention GEMMs plus the two bias products), card name and power limit.

  python scripts/relpos_bench.py [--heads 16] [--hd 80] [--windows 9] [--iters 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def flops(heads, hd, window, H=64, W=64):
    """Per image: S = Q K^T and O = P V (2 n^2 hd each per group and head) + the bias products (2 n S hd, both tables)."""
    if window:
        groups, n, S = (-(-H // window)) * (-(-W // window)), window * window, window
    else:
        groups, n, S = 1, H * W, H
    return heads * groups * (4 * n * n * hd + 2 * n * 2 * S * hd)


def torch_relpos(qkv, H, W, heads, hd, th, tw, window, bias):
    from oracle.sam_vit import attention_core, window_unpartition
    B, C = qkv.shape[0], heads * hd
    x = qkv.view(B, H, W, 3 * C)
    if window:
        Hp, Wp = -(-H // window) * window, -(-W // window) * window
        full = bias.view(1, 1, 1, 3 * C).expand(B, Hp, Wp, 3 * C).clone()
        full[:, :H, :W] = x
        wins = full.view(B, Hp // window, window, Wp // window, window, 3 * C).permute(0, 1, 3, 2, 4, 5)
        y = attention_core(wins.reshape(-1, window, window, 3 * C), heads, th, tw)
        return window_unpartition(y, window, (Hp, Wp), (H, W))
    return attention_core(x, heads, th, tw)


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", type=int, default=16)
    ap.add_argument("--hd", type=int, default=80)
    ap.add_argument("--windows", type=int, default=9)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("relpos_bench.py measures on the GPU; no CUDA device found")
    from omg_b200 import ops
    H = W = 64
    C = a.heads * a.hd
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(1, H * W, 3 * C, generator=g, device="cuda").half()
    bias = torch.randn(3 * C, generator=g, device="cuda").half()
    res = {"card": card(), "heads": a.heads, "head_dim": a.hd}
    for window in (0, 14):
        S = window or H
        th = (torch.randn(2 * S - 1, a.hd, generator=g, device="cuda") * 0.1).half()
        tw = (torch.randn(2 * S - 1, a.hd, generator=g, device="cuda") * 0.1).half()
        out = torch.empty(1, H * W, C, dtype=torch.float16, device="cuda")
        kern = lambda: ops.attention_relpos(qkv, H, W, a.heads, a.hd, th, tw, window=window, k_bias=bias[C:2 * C],
                                            v_bias=bias[2 * C:], out=out)
        ref = lambda: torch_relpos(qkv, H, W, a.heads, a.hd, th, tw, window, bias)
        for f in (kern, ref):
            f()
        torch.cuda.synchronize()
        rel = ((out.float() - ref().reshape(1, H * W, C).float()).norm() / ref().float().norm()).item()
        tk, tt = [], []
        for _ in range(a.windows):
            tk.append(timed(kern, a.iters))
            tt.append(timed(ref, a.iters))
        fl = flops(a.heads, a.hd, window)
        mk, mt = statistics.median(tk), statistics.median(tt)
        res["global" if window == 0 else "window14"] = {
            "kernel_ms": round(mk, 4), "torch_fp16_ms": round(mt, 4), "gflop": round(fl / 1e9, 2),
            "kernel_tflops": round(fl / mk / 1e9, 1), "torch_tflops": round(fl / mt / 1e9, 1), "rel_l2_vs_torch": rel}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
