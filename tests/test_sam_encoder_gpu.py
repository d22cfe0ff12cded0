"""SURVEY 8f-4 on the GPU: the EfficientViT-SAM image encoder (the segmentation model the reference runs between the two
stages) executed on this repo's kernels, against golden vectors produced by the UNMODIFIED reference modules
(tests/golden/make_golden.py imports src/efficientvit: LiteMLA, EfficientViTBlock, EfficientViTLargeBackbone, SamNeck,
EfficientViTSamImageEncoder) - this row's oracle is the reference itself.  Plus the four non-GEMM kernels against torch."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden", "sam_encoder.pt")
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_golden import sam_input  # noqa: E402  (pure helper; does not import the reference)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*s, generator=g, device="cuda") * scale).half()


@pytest.mark.parametrize("k,stride,act,bias", [(3, 1, 0, True), (3, 2, 1, True), (5, 1, 0, False), (5, 2, 1, True)])
def test_depthwise_conv(k, stride, act, bias):
    from omg_b200 import ops
    B, H, W, C = 2, 22, 18, 96
    x, w = rnd(B, H, W, C, seed=1), rnd(C, 1, k, k, seed=2, scale=1.0 / k)
    b = rnd(C, seed=3) if bias else None
    y = ops.dwconv(x, w.reshape(C, k * k).t().contiguous(), b, ksize=k, stride=stride, act=act)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), None if b is None else b.float(), stride=stride, padding=k // 2, groups=C)
    if act:
        ref = F.gelu(ref, approximate="tanh")
    assert y.shape == (B, (H + stride - 1) // stride, (W + stride - 1) // stride, C)
    assert rel(y.permute(0, 3, 1, 2), ref) < 2e-3
    # strided rows: input and output are channel slices of wider tensors
    xw, yw = rnd(B, H, W, 2 * C, seed=4), torch.zeros(B, H, W, 3 * C, device="cuda", dtype=torch.float16)
    if stride == 1:
        ops.dwconv(xw[..., C:], w.reshape(C, k * k).t().contiguous(), b, out=yw[..., C:2 * C], ksize=k, stride=1, act=act)
        r2 = F.conv2d(xw[..., C:].float().permute(0, 3, 1, 2), w.float(), None if b is None else b.float(), padding=k // 2, groups=C)
        r2 = F.gelu(r2, approximate="tanh") if act else r2
        assert rel(yw[..., C:2 * C].permute(0, 3, 1, 2), r2) < 2e-3 and float(yw[..., :C].abs().sum()) == 0


def test_grouped_pointwise_conv_and_relu_linear_attention():
    from omg_b200 import ops
    B, N, heads = 2, 300, 6
    C = heads * 96
    x, w = rnd(B, N, C, seed=1), rnd(C, 32, 1, 1, seed=2, scale=32 ** -0.5)
    y = torch.empty_like(x)
    ops.group1x1(x, w.reshape(C, 32).contiguous(), y)
    ref = F.conv2d(x.float().permute(0, 2, 1)[..., None], w.float(), groups=C // 32)[..., 0].permute(0, 2, 1)
    assert rel(y, ref) < 2e-3
    # LiteMLA.relu_linear_att (src/efficientvit/models/nn/ops.py:404-440) restated on (B, N, heads, 3, 32)
    out = ops.relu_linear_attention(x, heads, 32, 1e-15)
    q, k, v = x.float().view(B, N, heads, 3, 32).permute(3, 0, 2, 1, 4)
    q, k = F.relu(q), F.relu(k)
    kv = k.transpose(-1, -2) @ F.pad(v, (0, 1), value=1.0)
    o = q @ kv
    ref = (o[..., :-1] / (o[..., -1:] + 1e-15)).permute(0, 2, 1, 3).reshape(B, N, heads * 32)
    assert rel(out, ref) < 2e-3


@pytest.mark.parametrize("hw,out", [((12, 12), 64), ((24, 20), 64), ((128, 128), 64), ((64, 64), 64), ((7, 9), 16)])
def test_bicubic_resize_matches_interpolate(hw, out):
    from omg_b200 import ops
    x = rnd(2, hw[0], hw[1], 64, seed=5)
    y = ops.resize_bicubic(x, out, out)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), size=(out, out), mode="bicubic", align_corners=False)
    assert rel(y.permute(0, 3, 1, 2), ref) < 1e-3


def test_tanh_gelu_epilogue():
    from omg_b200 import _lib as L, ops
    x, w, b = rnd(300, 128, seed=1), rnd(96, 128, seed=2, scale=128 ** -0.5), rnd(96, seed=3)
    y = ops.linear(x, w, bias=b, epilogue=L.EPI_GELU_TANH)
    assert rel(y, F.gelu(x.float() @ w.float().t() + b.float(), approximate="tanh")) < 2e-3


def test_lite_mla_and_efficientvit_block_match_the_reference_modules():
    from omg_b200.sam_encoder import efficientvit_block, lite_mla
    d = torch.load(G)
    to = lambda t: t.permute(0, 2, 3, 1).contiguous().cuda()  # noqa: E731
    y = lite_mla({"m." + k: v for k, v in d["mla_sd"].items()}, "m", to(sam_input("mla").half()))
    e1 = rel(y.permute(0, 3, 1, 2), d["mla_y"])
    y = efficientvit_block({"b." + k: v for k, v in d["blk_sd"].items()}, "b", to(sam_input("blk").half()))
    e2 = rel(y.permute(0, 3, 1, 2), d["blk_y"])
    print("LiteMLA rel err", e1, "EfficientViTBlock rel err", e2)
    assert e1 < 5e-4 and e2 < 5e-4   # measured on H100: 3.9e-4 / 3.5e-4


def test_sam_image_encoder_matches_the_reference_module():
    from omg_b200.sam_encoder import PackedSamImageEncoder
    d = torch.load(G)
    enc = PackedSamImageEncoder(d["sd"], device="cuda")
    x = sam_input().half()
    y, feats = enc(x, return_features=True)
    assert tuple(y.shape) == (1, 256, 64, 64)
    assert {f"stage{k}": tuple(v.shape) for k, v in feats.items()} == {k: v for k, v in d["stage_shapes"].items()
                                                                         if k.startswith("stage") and k != "stage_final"}
    e3, e5, e = rel(feats[3], d["stage3"]), rel(feats[5], d["stage5"]), rel(y[..., ::8, ::8], d["y_sub"])
    print("sam encoder rel err: stage3", e3, "stage5", e5, "output", e)
    assert e3 < 5.5e-4 and e5 < 6e-4 and e < 8.5e-4   # measured on H100: 4.6e-4 / 4.6e-4 / 6.4e-4
    # the call above captured a CUDA graph; a replay on another image must equal the eager launches for that image bit for bit
    x2 = x.flip(-1) * 0.5
    y2 = enc(x2, return_features=True)[0]
    eager = PackedSamImageEncoder(d["sd"], device="cuda", use_graph=False)
    assert torch.equal(y2, eager(x2)) and torch.equal(enc(x, return_features=True)[0], y) and not torch.equal(y2, y)
