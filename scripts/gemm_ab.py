"""Tall 256x160 tiles vs 128x320 tiles on the narrow-N GEMM / conv shapes of the SDXL UNet (B=4):
median of 20 timed launches each, L2 flushed between launches.  One JSON line per shape."""
import json
import sys

import torch

sys.path.insert(0, ".")
from omg_b200 import ops  # noqa: E402

dev = "cuda"
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def rnd(*s, scale=1.0):
    return (torch.randn(*s, device=dev) * scale).half()


for (M, N, K, tag) in [(4096, 1280, 1280, "out1280"), (4096, 1280, 5120, "ff2_1280"), (16384, 640, 640, "out640"),
                       (16384, 640, 2560, "ff2_640"), (8192, 1280, 1280, "out1280_b8"), (8192, 1280, 5120, "ff2_1280_b8")]:
    x, w, res = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(M, N)
    out = torch.empty(M, N, device=dev, dtype=torch.float16)
    r = {"name": tag, "gflop": 2.0 * M * N * K / 1e9}
    for name, kw in (("tall160", dict(block_n=160, cta_pair=3)), ("pair320", dict(block_n=320))):
        ms = timeit(lambda: ops.linear(x, w, residual=res, out=out, **kw))
        r[name] = {"us": round(ms * 1e3, 1), "tflops": round(r["gflop"] / ms, 1)}
    print(json.dumps(r), flush=True)
for (B, H, Cin, N, tag) in [(4, 128, 320, 320, "conv320@128"), (4, 64, 640, 640, "conv640@64"), (4, 32, 1280, 1280, "conv1280@32"),
                            (4, 32, 2560, 1280, "conv2560->1280@32"), (4, 128, 960, 320, "conv960->320@128")]:
    x = rnd(B, H, H, Cin)
    w = ops.pack_conv3x3_weight(rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
    out = torch.empty(B, H, H, N, device=dev, dtype=torch.float16)
    r = {"name": tag, "gflop": 2.0 * B * H * H * N * 9 * Cin / 1e9}
    for name, kw in (("tall160", dict(block_n=160, cta_pair=3)), ("pair320", dict(block_n=320))):
        ms = timeit(lambda: ops.conv3x3(x, w, out=out, **kw))
        r[name] = {"us": round(ms * 1e3, 1), "tflops": round(r["gflop"] / ms, 1)}
    print(json.dumps(r), flush=True)
