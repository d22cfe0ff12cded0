"""EfficientViT-SAM image encoder on the C-ABI kernels (SURVEY section 8, row f-4: "visual comprehension on-device").

The reference segments the stage-1 image with EfficientViT-SAM between the two denoising stages
(inference_lora.py:176,262-290 -> src/efficientvit/sam_model_zoo.py -> EfficientViTSamPredictor.set_image,
src/efficientvit/models/efficientvit/sam.py:276-297); the encoder is where its time goes.  This module executes
`EfficientViTSamImageEncoder` (sam.py:176-192: EfficientViTLargeBackbone -> SamNeck -> LayerNorm2d) from the
reference's own state dict: the topology is read off the parameter names (`backbone.stages.S.op_list.I.main.*`,
`...context_module.main.*`, `neck.input_ops.*`, ...), so any of the zoo's L / XL variants loads without a config.

Mapping (reference module -> kernel):
  ConvLayer 3x3 / 1x1 (+BatchNorm, +tanh-GELU)   omg_gemm, BN folded into weights / bias, OMG_EPI_GELU_TANH, residual in the epilogue
  depthwise 3x3 / 5x5 (MBConv, LiteMLA.aggreg)    omg_dwconv
  grouped 1x1 (LiteMLA.aggreg)                    omg_group1x1
  LiteMLA.relu_linear_att                          omg_relu_linear_attention (fp32 like the reference)
  UpSampleLayer(bicubic, size 64x64)               omg_resize_bicubic
  LayerNorm2d                                      omg_layernorm over the channels-last rows
Activations are channels-last fp16 like the UNet's.  Parity: tests/golden/sam_encoder.pt holds input / output / state
dict of the UNMODIFIED reference modules (tests/golden/make_golden.py imports them), so this row is pinned."""
import re
from typing import Dict, List, Optional

import torch

from . import _lib as L
from . import ops


def _fold(sd, prefix, eps):
    """ConvLayer at `prefix` -> (weight fp32 (N, C/groups, k, k), bias fp32 (N,) or None) with BatchNorm folded."""
    w = sd[prefix + ".conv.weight"].float()
    b = sd[prefix + ".conv.bias"].float() if (prefix + ".conv.bias") in sd else None
    if (prefix + ".norm.weight") in sd:
        g, beta = sd[prefix + ".norm.weight"].float(), sd[prefix + ".norm.bias"].float()
        mean, var = sd[prefix + ".norm.running_mean"].float(), sd[prefix + ".norm.running_var"].float()
        s = g / torch.sqrt(var + eps)
        w = w * s[:, None, None, None]
        b = beta - mean * s + (b * s if b is not None else 0.0)
    return w, b


class _Conv:
    """One ConvLayer packed for the kernels."""

    def __init__(self, sd, prefix, eps, dev, stride=1, act=False):
        w, b = _fold(sd, prefix, eps)
        self.stride, self.act = stride, act
        self.n, cin_g, self.k, _ = w.shape
        self.depthwise = cin_g == 1 and self.n > 1 and sd[prefix + ".conv.weight"].shape[1] == 1
        h = lambda t: t.to(dev, torch.float16).contiguous()  # noqa: E731
        self.bias = None if b is None else h(b)
        if self.depthwise:
            self.w = h(w.reshape(self.n, self.k * self.k).t())              # tap-major [k*k, C]
        elif self.k == 3:
            pad = (-cin_g) % 8                                                # conv_in: 3 -> 8 input channels
            if pad:
                w = torch.cat([w, w.new_zeros(self.n, pad, 3, 3)], dim=1)
            self.cin = cin_g + pad
            self.w = h(ops.pack_conv3x3_weight(w))
        else:
            self.cin = cin_g
            self.w = h(w.reshape(self.n, cin_g))

    def __call__(self, x, residual=None, out=None):
        epi = L.EPI_GELU_TANH if self.act else L.EPI_NONE
        B, H, W, _ = x.shape
        if self.depthwise:
            assert residual is None
            return ops.dwconv(x, self.w, self.bias, out=out, ksize=self.k, stride=self.stride, act=int(self.act))
        if self.k == 1:
            y = out if out is not None else torch.empty((B, H, W, self.n), dtype=torch.float16, device=x.device)
            views, segs = [ops.view4(x)], [(0, 0, 0, 0, x.shape[3], 0)]
            ops.gemm(views, segs, self.w, self.n, self.w.shape[1], ops.view4(y), bias=self.bias, residual=residual,
                     residual_ld=0 if residual is None else self.n, epilogue=epi)
            return y
        if self.stride == 2:
            assert residual is None and not (H % 2 or W % 2)
            return ops.conv3x3_s2(x, self.w, bias=self.bias, out=out, epilogue=epi)
        y = out if out is not None else torch.empty((B, H, W, self.n), dtype=torch.float16, device=x.device)
        ops.gemm([ops.view4(x)], ops._taps3x3(x.shape[3]), self.w, self.n, self.w.shape[1], ops.view4(y), bias=self.bias,
                 residual=residual, residual_ld=0 if residual is None else self.n, epilogue=epi)
        return y


class _LiteMLA:
    """LiteMLA (ops.py:335-454): qkv 1x1 -> [identity | depthwise k x k + grouped 1x1 per scale] -> ReLU linear attention per
    head of 32 channels -> proj 1x1 (+BN)."""

    def __init__(self, sd, prefix, eps, dev, dim=32, att_eps=1e-15):
        self.qkv = _Conv(sd, prefix + ".qkv", eps, dev)
        self.total = self.qkv.n // 3
        self.dim, self.att_eps = dim, att_eps
        self.scales = []
        i = 0
        while f"{prefix}.aggreg.{i}.0.weight" in sd:
            wd = sd[f"{prefix}.aggreg.{i}.0.weight"].float()      # (3T, 1, k, k) depthwise, no bias in the zoo models
            k = wd.shape[-1]
            wg = sd[f"{prefix}.aggreg.{i}.1.weight"].float()      # (3T, dim, 1, 1) grouped, groups = 3 * heads
            assert wg.shape[1] == dim == 32 and f"{prefix}.aggreg.{i}.0.bias" not in sd
            self.scales.append((k, wd.reshape(-1, k * k).t().to(dev, torch.float16).contiguous(),
                                wg.reshape(-1, dim).to(dev, torch.float16).contiguous()))
            i += 1
        self.proj = _Conv(sd, prefix + ".proj", eps, dev)

    def __call__(self, x, residual):
        B, H, W, _ = x.shape
        T3, ns = 3 * self.total, len(self.scales)
        ms = torch.empty((B, H, W, (1 + ns) * T3), dtype=torch.float16, device=x.device)   # cat([qkv, aggreg(qkv)...], C)
        self.qkv(x, out=ms[..., :T3])
        for i, (k, wd, wg) in enumerate(self.scales):
            tmp = ops.dwconv(ms[..., :T3], wd, None, ksize=k, stride=1, act=0)
            ops.group1x1(tmp, wg, ms[..., (1 + i) * T3:(2 + i) * T3])
        heads = (1 + ns) * self.total // self.dim
        att = ops.relu_linear_attention(ms.view(B, H * W, -1), heads, self.dim, self.att_eps)
        return self.proj(att.view(B, H, W, heads * self.dim), residual=residual)


def efficientvit_block(sd, prefix, x, norm_eps=1e-6, dim=32):
    """One EfficientViTBlock (ops.py:457-493) at `prefix` of a state dict on a channels-last fp16 tensor."""
    dev = x.device
    mla = _LiteMLA(sd, f"{prefix}.context_module.main", norm_eps, dev, dim)
    lm = f"{prefix}.local_module.main"
    convs = [_Conv(sd, lm + ".inverted_conv", norm_eps, dev, act=True), _Conv(sd, lm + ".depth_conv", norm_eps, dev, act=True),
             _Conv(sd, lm + ".point_conv", norm_eps, dev)]
    x = mla(x, residual=x)
    return PackedSamImageEncoder._run_block(convs, x, True)


def lite_mla(sd, prefix, x, norm_eps=1e-6, dim=32):
    """One LiteMLA (ops.py:335-454) at `prefix` of a state dict on a channels-last fp16 tensor (no shortcut)."""
    return _LiteMLA(sd, prefix, norm_eps, x.device, dim)(x, residual=None)


class PackedSamImageEncoder:
    """EfficientViTSamImageEncoder executed on the kernels; built from the reference state dict (keys `backbone.*`,
    `neck.*`, `norm.*`; a full EfficientViTSam checkpoint's `image_encoder.` prefix is stripped)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", norm_eps: float = 1e-6, neck_size: int = 64,
                 use_graph: bool = True):
        sd = {k[len("image_encoder."):] if k.startswith("image_encoder.") else k: v for k, v in state_dict.items()}
        self.dev, self.eps, self.neck_size = torch.device(device), norm_eps, neck_size
        self.use_graph, self._graphs = use_graph, {}
        dev, eps = self.dev, norm_eps
        n_stages = 1 + max(int(m.group(1)) for k in sd for m in [re.match(r"backbone\.stages\.(\d+)\.", k)] if m)
        self.stages: List[List[tuple]] = []
        for s in range(n_stages):
            n_ops = 1 + max(int(m.group(1)) for k in sd for m in [re.match(rf"backbone\.stages\.{s}\.op_list\.(\d+)\.", k)] if m)
            stage = []
            for i in range(n_ops):
                p = f"backbone.stages.{s}.op_list.{i}"
                first = i == 0
                if f"{p}.conv.weight" in sd:                      # stage 0 stem: ConvLayer(3 -> w0, stride 2, BN, GELU)
                    stage.append(("conv", _Conv(sd, p, eps, dev, stride=2, act=True)))
                elif f"{p}.context_module.main.qkv.conv.weight" in sd:   # EfficientViTBlock
                    lm = f"{p}.local_module.main"
                    stage.append(("vit", _LiteMLA(sd, f"{p}.context_module.main", eps, dev),
                                  [_Conv(sd, lm + ".inverted_conv", eps, dev, act=True), _Conv(sd, lm + ".depth_conv", eps, dev, act=True),
                                   _Conv(sd, lm + ".point_conv", eps, dev)]))
                else:
                    # ResBlock (conv1, conv2) / FusedMBConv (spatial_conv, point_conv) / MBConv (inverted, depth, point):
                    # activation after every conv but the last; the stride-2 conv of a stage's first block (s >= 1) is the
                    # first spatial one; blocks other than that one carry an identity shortcut (backbone.py:223-283)
                    names = next(n for n in (("conv1", "conv2"), ("spatial_conv", "point_conv"),
                                             ("inverted_conv", "depth_conv", "point_conv")) if f"{p}.main.{n[0]}.conv.weight" in sd)
                    down = first and s >= 1
                    spatial = names[1] if len(names) == 3 else names[0]
                    convs = [_Conv(sd, f"{p}.main.{n}", eps, dev, stride=2 if (down and n == spatial) else 1, act=n != names[-1])
                             for n in names]
                    stage.append(("block", convs, not down))
            self.stages.append(stage)
        # SamNeck (sam.py:103-173): inputs (1x1 conv + BN, bicubic resize), summed; FusedMBConv / ResBlock / MBConv residual
        # blocks; 1x1 output conv with bias; then LayerNorm2d
        self.neck_in = []
        i = 0
        fids = self._neck_fids(sd, n_stages)
        while f"neck.input_ops.{i}.op_list.0.conv.weight" in sd:
            self.neck_in.append((fids[i], _Conv(sd, f"neck.input_ops.{i}.op_list.0", eps, dev)))
            i += 1
        self.neck_mid = []
        i = 0
        while any(k.startswith(f"neck.middle.op_list.{i}.") for k in sd):
            p = f"neck.middle.op_list.{i}.main"
            names = next(n for n in (("conv1", "conv2"), ("spatial_conv", "point_conv"),
                                     ("inverted_conv", "depth_conv", "point_conv")) if f"{p}.{n[0]}.conv.weight" in sd)
            self.neck_mid.append([_Conv(sd, f"{p}.{n}", eps, dev, act=n != names[-1]) for n in names])
            i += 1
        self.neck_out = _Conv(sd, "neck.output_ops.0.op_list.0", eps, dev)
        self.ln = (sd["norm.weight"].to(dev, torch.float16).contiguous(), sd["norm.bias"].to(dev, torch.float16).contiguous())

    @staticmethod
    def _neck_fids(sd, n_stages):
        """SamNeck's inputs are the last three stages, deepest first (fid_list of every zoo variant, sam.py:553-556,643-645)."""
        n = 0
        while f"neck.input_ops.{n}.op_list.0.conv.weight" in sd:
            n += 1
        return [n_stages - 1 - i for i in range(n)]

    @staticmethod
    def _run_block(convs, x, residual):
        h = x
        for c in convs[:-1]:
            h = c(h)
        return convs[-1](h, residual=x if residual else None)

    @torch.no_grad()
    def __call__(self, image: torch.Tensor, return_features: bool = False, out_dtype: Optional[torch.dtype] = None):
        """image (B, 3, H, W) normalised like SamResize / transforms.Normalize produce it -> (B, 256, 64, 64) fp16
        [, {stage index: (B, C, h, w) backbone features}].  The ~330 launches of an image are replayed as one CUDA graph per
        input shape (`use_graph`, default on: eager, the encoder is bound by the host's launch rate - 6 to 13 ms per image
        depending on the box - for ~4 ms of device time); results are copies of the graph's static buffers."""
        if not self.use_graph:
            return self._encode(image, return_features, out_dtype)
        key = (tuple(image.shape), bool(return_features), out_dtype)
        ent = self._graphs.get(key)
        if ent is None:
            static_in = torch.empty(image.shape, dtype=torch.float16, device=self.dev)
            static_in.copy_(image)
            self._encode(static_in, return_features, out_dtype)       # eager warm-up: kernel attributes, allocator pools
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = self._encode(static_in, return_features, out_dtype)
            ent = self._graphs[key] = (g, static_in, out)
        g, static_in, out = ent
        static_in.copy_(image)
        g.replay()
        if return_features:
            return out[0].clone(), {k: v.clone() for k, v in out[1].items()}
        return out.clone()

    def _encode(self, image: torch.Tensor, return_features: bool = False, out_dtype: Optional[torch.dtype] = None):
        x = image.to(self.dev, torch.float16).permute(0, 2, 3, 1)
        x = torch.cat([x, x.new_zeros(*x.shape[:3], 5)], dim=3).contiguous()
        feats = {}
        for s, stage in enumerate(self.stages):
            for op in stage:
                if op[0] == "conv":
                    x = op[1](x)
                elif op[0] == "block":
                    x = self._run_block(op[1], x, op[2])
                else:
                    x = op[1](x, residual=x)                      # context module: LiteMLA + identity
                    x = self._run_block(op[2], x, True)           # local module: MBConv + identity
            feats[s] = x
        acc = None
        for fid, conv in self.neck_in:
            f = conv(feats[fid])
            if f.shape[1] != self.neck_size or f.shape[2] != self.neck_size:
                f = ops.resize_bicubic(f, self.neck_size, self.neck_size)
            acc = f if acc is None else ops.axpy(acc, f, 1.0)
        x = acc
        for convs in self.neck_mid:
            x = self._run_block(convs, x, True)
        x = self.neck_out(x)
        B, H, W, C = x.shape
        y = ops.layernorm(x.view(B * H * W, C), self.ln[0], self.ln[1], eps=self.eps).view(B, H, W, C).permute(0, 3, 1, 2)
        if out_dtype is not None:   # the reference's prompt encoder / mask decoder run in the model's dtype (fp32 in the CLI)
            y = y.to(out_dtype)
        if return_features:
            return y, {k: v.permute(0, 3, 1, 2) for k, v in feats.items()}
        return y
