"""Per-kernel timing on the GPU (CUDA events, L2 flushed between iterations) for the SDXL shapes of the hot path,
next to the torch library call (cuBLAS / cuDNN / SDPA) the reference would make.  Prints TFLOP/s and GB/s."""
import json
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from omg_b200 import ops  # noqa: E402

dev = "cuda"
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=8, warm=3):
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


res = []


def report(name, ms, flops=None, bytes_=None, ref_ms=None):
    r = {"name": name, "ms": round(ms, 4)}
    if flops:
        r["tflops"] = round(flops / ms / 1e9, 1)
    if bytes_:
        r["gbs"] = round(bytes_ / ms / 1e6, 1)
    if ref_ms:
        r["torch_ms"] = round(ref_ms, 4)
        if flops:
            r["torch_tflops"] = round(flops / ref_ms / 1e9, 1)
    res.append(r)
    print(json.dumps(r), flush=True)


# ---- linears (B=4 main pass): tokens 4*4096 @ c=640, 4*1024 @ c=1280
for (M, N, K, tag) in [(16384, 1920, 640, "qkv640"), (16384, 640, 640, "out640"), (16384, 5120, 640, "ff1_640"),
                       (16384, 640, 2560, "ff2_640"), (4096, 3840, 1280, "qkv1280"), (4096, 1280, 1280, "out1280"),
                       (4096, 10240, 1280, "ff1_1280"), (4096, 1280, 5120, "ff2_1280"), (8192, 1280, 5120, "ff2_1280_b8"),
                       (8192, 10240, 1280, "ff1_1280_b8")]:
    x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    out = torch.empty(M, N, device=dev, dtype=torch.float16)
    ref = timeit(lambda: F.linear(x, w))
    for bn in ([0] if "ff1" in tag else [0, 128, 160, 256]):
        if bn == 160 and N % 160:
            continue
        ms = timeit(lambda: ops.linear(x, w, out=out, block_n=bn))
        report(f"linear_{tag}_bn{bn}", ms, 2.0 * M * N * K, ref_ms=ref)
    if "ff1" in tag:
        wi, _ = ops.pack_geglu_weight(w)
        o2 = torch.empty(M, N // 2, device=dev, dtype=torch.float16)
        ms = timeit(lambda: ops.linear(x, wi, out=o2, epilogue=1))
        report(f"geglu_{tag}", ms, 2.0 * M * N * K, ref_ms=ref)

for (M, N, K, tag) in [(4096, 1280, 1280, "out1280"), (4096, 1280, 5120, "ff2_1280"), (8192, 1280, 5120, "ff2_1280_b8"),
                       (8192, 1280, 1280, "out1280_b8"), (16384, 640, 2560, "ff2_640")]:
    x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    out = torch.empty(M, N, device=dev, dtype=torch.float16)
    for cp in (1, 3):
        ms = timeit(lambda: ops.linear(x, w, out=out, block_n=160, cta_pair=cp))
        report(f"{'tall' if cp == 3 else 'single'}_bn160_{tag}", ms, 2.0 * M * N * K)

# ---- convs
for (B, H, C, N, tag) in [(4, 128, 320, 320, "res128"), (4, 64, 640, 640, "res64"), (4, 32, 1280, 1280, "res32"),
                          (4, 32, 2560, 1280, "res32_cat"), (4, 128, 960, 320, "res128_cat")]:
    x = rnd(B, H, H, C)
    w = rnd(N, C, 3, 3, scale=(9 * C) ** -0.5)
    wp = ops.pack_conv3x3_weight(w)
    out = torch.empty(B, H, H, N, device=dev, dtype=torch.float16)
    xc = x.permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    wc = w.contiguous(memory_format=torch.channels_last)
    ref = timeit(lambda: F.conv2d(xc, wc, padding=1))
    for bn in [0, 160, 256]:
        if bn == 160 and N % 160:
            continue
        ms = timeit(lambda: ops.conv3x3(x, wp, out=out, block_n=bn))
        report(f"conv3x3_{tag}_bn{bn}", ms, 2.0 * B * H * H * N * 9 * C, ref_ms=ref)
    if N % 160 == 0:
        for cp in (1, 3):
            ms = timeit(lambda: ops.conv3x3(x, wp, out=out, block_n=160, cta_pair=cp))
            report(f"conv3x3_{tag}_{'tall' if cp == 3 else 'single'}160", ms, 2.0 * B * H * H * N * 9 * C, ref_ms=ref)

# ---- attention
for (B, N, heads, tag) in [(4, 4096, 10, "self4096"), (4, 1024, 20, "self1024"), (8, 1024, 20, "self1024_b8")]:
    Cc = heads * 64
    qkv = rnd(B, N, 3 * Cc)
    out = torch.empty(B, N, Cc, device=dev, dtype=torch.float16)
    items = [(b, b, b, b) for b in range(B)]
    q, k, v = [t.reshape(B, N, heads, 64).transpose(1, 2) for t in qkv.chunk(3, dim=-1)]
    ref = timeit(lambda: F.scaled_dot_product_attention(q, k, v))
    ms = timeit(lambda: ops.attention(qkv, qkv, qkv, out, heads, N, N, items, 0, Cc, 2 * Cc))
    report(f"attn_{tag}", ms, 4.0 * B * heads * N * N * 64, ref_ms=ref)
for (B, N, heads, L, tag) in [(4, 4096, 10, 77, "cross4096"), (4, 1024, 20, 77, "cross1024")]:
    Cc = heads * 64
    qx, kv = rnd(B, N, Cc), rnd(B, L, 2 * Cc)
    out = torch.empty(B, N, Cc, device=dev, dtype=torch.float16)
    items = [(b, b, b, b) for b in range(B)]
    ms = timeit(lambda: ops.attention(qx, kv, kv, out, heads, N, L, items, 0, 0, Cc))
    report(f"attn_{tag}", ms, 4.0 * B * heads * N * L * 64, bytes_=2.0 * (2 * B * N * Cc + B * L * 2 * Cc))

# ---- norms
for (B, HW, C, tag) in [(4, 16384, 320, "gn128"), (4, 4096, 640, "gn64"), (4, 1024, 1280, "gn32"), (4, 1024, 2560, "gn32cat")]:
    x = rnd(B, HW, C)
    g, b = rnd(C), rnd(C)
    out = torch.empty_like(x)
    ws = torch.empty(B * (10240 + 64 * 256), device=dev)
    ms = timeit(lambda: ops.groupnorm(x, g, b, 1e-5, 1, out=out, stats_ws=ws))
    xn = x.transpose(1, 2).contiguous()
    ref = timeit(lambda: F.silu(F.group_norm(xn, 32, g, b, 1e-5)))
    report(f"groupnorm_{tag}", ms, bytes_=3.0 * x.numel() * 2, ref_ms=ref)
for (rows, C, tag) in [(16384, 640, "ln640"), (4096, 1280, "ln1280")]:
    x = rnd(rows, C)
    g, b = rnd(C), rnd(C)
    out = torch.empty_like(x)
    ms = timeit(lambda: ops.layernorm(x, g, b, out=out))
    ref = timeit(lambda: F.layer_norm(x, (C,), g, b))
    report(f"layernorm_{tag}", ms, bytes_=2.0 * x.numel() * 2, ref_ms=ref)

json.dump(res, open("gpurun_out/kernel_bench.json", "w"), indent=1)
