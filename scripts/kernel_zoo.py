"""One launch of every kernel variant of the hot path at its SDXL shape (after warm-ups), inside the NVTX range "zoo":
the target of ONE `ncu --set full --import-source on --nvtx --nvtx-include "zoo/"` capture
(profiles/r02_ncu_kernel_table.csv is read out of that report).  Each launch is preceded by an NVTX marker range
naming the shape, so the report rows can be told apart.
"""
import os
import sys

import torch

sys.path.insert(0, ".")
from omg_b200 import _lib as L  # noqa: E402
from omg_b200 import ops  # noqa: E402

dev = "cuda"
torch.manual_seed(0)


def rnd(*s, scale=1.0):
    return (torch.randn(*s, device=dev) * scale).half()


cases = []


def case(name):
    def deco(fn):
        cases.append((name, fn))
        return fn
    return deco


# ---- attention
def self_attn(B, N, heads):
    C = heads * 64
    qkv = rnd(B, N, 3 * C)
    out = torch.empty(B, N, C, device=dev, dtype=torch.float16)
    items = [(b, b, b, b) for b in range(B)]
    return lambda: ops.attention(qkv, qkv, qkv, out, heads, N, N, items, 0, C, 2 * C)


def cross_attn(B, N, heads, Lk):
    C = heads * 64
    q, kv = rnd(B, N, C), rnd(B, Lk, 2 * C)
    out = torch.empty(B, N, C, device=dev, dtype=torch.float16)
    items = [(b, b, b, b) for b in range(B)]
    return lambda: ops.attention(q, kv, kv, out, heads, N, Lk, items, 0, 0, C)


cases.append(("self_attn N=1024 B=4 h=20", self_attn(4, 1024, 20)))
cases.append(("self_attn N=4096 B=4 h=10", self_attn(4, 4096, 10)))
cases.append(("cross_attn N=1024 L=77 B=4 h=20", cross_attn(4, 1024, 20, 77)))
cases.append(("cross_attn N=4096 L=77 B=4 h=10", cross_attn(4, 4096, 10, 77)))
cases.append(("ip_attn N=1024 L=16 B=4 h=20", cross_attn(4, 1024, 20, 16)))


# ---- GEMMs
def lin(M, N, K, epi=L.EPI_NONE, residual=False):
    x, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    if epi == L.EPI_GEGLU:
        w, _ = ops.pack_geglu_weight(w)
    out = torch.empty(M, N // 2 if epi == L.EPI_GEGLU else N, device=dev, dtype=torch.float16)
    res = rnd(M, N) if residual else None
    bias = rnd(N)
    return lambda: ops.linear(x, w, bias=bias, residual=res, out=out, epilogue=epi)


cases.append(("ff1 GEGLU 4096x10240x1280 (128 x 256 tiles)", lin(4096, 10240, 1280, L.EPI_GEGLU)))
cases.append(("ff2 4096x1280x5120 +residual (tall tile)", lin(4096, 1280, 5120, residual=True)))
cases.append(("qkv 4096x3840x1280", lin(4096, 3840, 1280)))
cases.append(("out-proj 4096x1280x1280 +residual (tall tile)", lin(4096, 1280, 1280, residual=True)))
cases.append(("ff1 GEGLU 16384x5120x640", lin(16384, 5120, 640, L.EPI_GEGLU)))


def conv(B, H, W, Cin, N, stats=True):
    x = rnd(B, H, W, Cin)
    w = ops.pack_conv3x3_weight(rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
    out = torch.empty(B, H, W, N, device=dev, dtype=torch.float16)
    part = torch.empty(B, ops.colstats_blocks(W, H), N, 2, device=dev) if stats else None
    bias, temb = rnd(N), rnd(B, N)
    return (lambda: ops.conv3x3(x, w, bias=bias, rowvec=temb, out=out, colstats=part)), out, part


c320, y320, p320 = conv(4, 128, 128, 320, 320)
c1280, y1280, p1280 = conv(4, 32, 32, 1280, 1280)
cases.append(("conv3x3 320->320 @128x128 B=4 (+time-emb rowvec, +GroupNorm column stats)", c320))
cases.append(("conv3x3 1280->1280 @32x32 B=4 (+GroupNorm column stats)", c1280))


# ---- GroupNorm from producer statistics, LayerNorm, fused step
def gn(y, part):
    C = y.shape[-1]
    gamma, beta = rnd(C) * 0.1 + 1, rnd(C) * 0.1
    out = torch.empty_like(y)
    ws = torch.empty(y.shape[0] * (10240 + 64 * 256), device=dev)
    return lambda: ops.groupnorm_apply(y, part, gamma, beta, 1e-5, 1, out=out, stats_ws=ws)


cases.append(("GroupNorm+SiLU 320ch @128x128 B=4 (reduce + apply)", gn(y320, p320)))
cases.append(("GroupNorm+SiLU 1280ch @32x32 B=4 (reduce + apply)", gn(y1280, p1280)))

HW = 128 * 128
nm, nc = rnd(4, HW, 8), [rnd(2, HW, 8), rnd(2, HW, 8)]
masks = [(torch.rand(HW, device=dev) > 0.7).float() for _ in range(2)]
lat = torch.randn(2, 128, 128, 4, device=dev)
nxt, nxc = torch.empty(4, HW, 8, device=dev, dtype=torch.float16), torch.empty(2, HW, 8, device=dev, dtype=torch.float16)
cases.append(("fuse_step (2 concepts) @128x128", lambda: ops.fuse_step(nm, nc, masks, 7.5, 5.0, 4.2, lat, nxt, nxc)))

only = os.environ.get("OMG_ZOO_ONLY")   # substring filter: capture a subset (e.g. "self_attn") after a kernel change
if only:
    cases = [c for c in cases if only in c[0]]
for name, fn in cases:   # warm-ups (kernel attributes, caches)
    fn()
    fn()
torch.cuda.synchronize()
torch.cuda.nvtx.range_push("zoo")
for name, fn in cases:
    torch.cuda.nvtx.range_push(name)
    fn()
    torch.cuda.nvtx.range_pop()
torch.cuda.synchronize()
torch.cuda.nvtx.range_pop()
print("zoo:", len(cases), "cases")
