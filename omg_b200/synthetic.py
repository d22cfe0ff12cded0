"""Synthetic, seeded, SDXL-shaped weights and inputs (there is no network for checkpoints; SURVEY section 8d fixes the
recipe): every Linear/Conv ~ N(0, 1/fan_in), norms gamma=1 beta=0, LoRA rank r with A ~ N(0, 1/in),
B ~ N(0, 1/r) * 0.1.  Optional small random biases / affine jitter exercise those code paths in tests."""
import math
from typing import Dict, List, Optional, Tuple

import torch

from .config import UNetConfig, lora_conv_target_names, lora_target_names, param_shapes


def make_state_dict(cfg: UNetConfig, seed: int = 0, controlnet: bool = False, device="cpu", dtype=torch.float32,
                    bias_std: float = 0.0, affine_jitter: float = 0.0) -> Dict[str, torch.Tensor]:
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for name, shp in param_shapes(cfg, controlnet).items():
        is_norm = ".norm" in name or name.startswith("conv_norm_out")
        if name.endswith(".weight") and len(shp) > 1:
            fan_in = math.prod(shp[1:])
            t = torch.randn(shp, generator=g, device=device, dtype=torch.float32) * fan_in ** -0.5
        elif name.endswith(".weight"):  # norm gamma
            t = torch.ones(shp, device=device)
            if affine_jitter:
                t = t + affine_jitter * torch.randn(shp, generator=g, device=device)
        elif is_norm:  # norm beta
            t = torch.zeros(shp, device=device)
            if affine_jitter:
                t = affine_jitter * torch.randn(shp, generator=g, device=device)
        else:
            t = torch.zeros(shp, device=device)
            if bias_std:
                t = bias_std * torch.randn(shp, generator=g, device=device)
        sd[name] = t.to(dtype)
    return sd


def make_lora(cfg: UNetConfig, seed: int, rank: int = 32, alpha: Optional[float] = None, device="cpu",
              dtype=torch.float32, conv: bool = False) -> Dict[str, Tuple[torch.Tensor, torch.Tensor, float]]:
    """name -> (A [r, in], B [out, r], alpha/r).  Covers every transformer Linear (q,k,v,out,ff.proj,ff.out,
    proj_in,proj_out).  conv=True (a LoCon adapter) adds the ResBlock / down-sampler / up-sampler modules of
    lora_conv_target_names with A [r, in, k, k] (A [r, in] for time_emb_proj), drawn from a generator of their own so
    the Linear entries of a seed are the same either way."""
    g = torch.Generator(device=device).manual_seed(seed)
    alpha = float(rank) if alpha is None else alpha
    out = {}
    for name, i, o in lora_target_names(cfg):
        A = torch.randn((rank, i), generator=g, device=device) * i ** -0.5
        Bm = torch.randn((o, rank), generator=g, device=device) * rank ** -0.5 * 0.1
        out[name] = (A.to(dtype), Bm.to(dtype), alpha / rank)
    if conv:
        gc = torch.Generator(device=device).manual_seed(seed + (1 << 20))
        for name, kind, i, o, k in lora_conv_target_names(cfg):
            shape = (rank, i) if kind == "linear" else (rank, i, k, k)
            A = torch.randn(shape, generator=gc, device=device) * (i * k * k) ** -0.5
            Bm = torch.randn((o, rank), generator=gc, device=device) * rank ** -0.5 * 0.1
            out[name] = (A.to(dtype), Bm.to(dtype), alpha / rank)
    return out


def make_ip_adapter(cfg: UNetConfig, seed: int, device="cpu", dtype=torch.float32):
    """attn2 path -> (to_k_ip [c, ctx], to_v_ip [c, ctx]) (src/ip_adapter/attention_processor.py:107-108)."""
    from .config import transformer_names
    g = torch.Generator(device=device).manual_seed(seed)
    out = {}
    d = cfg.cross_attention_dim
    for name, ch, layers in transformer_names(cfg):
        for k in range(layers):
            wk = torch.randn((ch, d), generator=g, device=device) * d ** -0.5
            wv = torch.randn((ch, d), generator=g, device=device) * d ** -0.5
            out[f"{name}.transformer_blocks.{k}.attn2"] = (wk.to(dtype), wv.to(dtype))
    return out


def make_conditioning(cfg: UNetConfig, batch: int, seed: int, ctx_len: int = 77, size=(1024, 1024), device="cpu"):
    """Synthetic text-encoder outputs: prompt_embeds (batch, 77, D), pooled (batch, P), add_time_ids (batch, 6)."""
    g = torch.Generator(device=device).manual_seed(seed)
    pe = torch.randn((batch, ctx_len, cfg.cross_attention_dim), generator=g, device=device)
    pooled = torch.randn((batch, cfg.pooled_dim), generator=g, device=device)
    h, w = size
    tid = torch.tensor([[h, w, 0, 0, h, w]], dtype=torch.float32, device=device).repeat(batch, 1)
    return pe, pooled, tid


def rect_masks(n: int, size=(1024, 1024), device="cpu") -> List[torch.Tensor]:
    """Config-2 style masks: n disjoint vertical rectangles (x ranges spread over the width, y in [1/8, 7/8))."""
    H, W = size
    out = []
    for k in range(n):
        m = torch.zeros((H, W), device=device)
        x0 = int(W * (k + 0.09375 * (k + 1)) / (n + 0.09375 * (n + 1)))
        x1 = int(x0 + W * 0.34375 * 2 / max(n, 2))
        m[H // 8: 7 * H // 8, x0:x1] = 1.0
        out.append(m)
    return out


def make_vae_state_dict(cfg=None, seed: int = 0, device="cpu", dtype=torch.float32):
    """Random-init VAE decoder weights (diffusers AutoencoderKL keys) with O(1) activations through the stack."""
    from .vae import VaeConfig, vae_decoder_param_shapes
    cfg = cfg or VaeConfig.sdxl()
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for name, shape in vae_decoder_param_shapes(cfg).items():
        if name.endswith(".bias"):
            t = torch.randn(shape, generator=g, device=device) * 0.05
        elif len(shape) == 1:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        else:
            fan_in = shape[1] * (shape[2] * shape[3] if len(shape) == 4 else 1)
            t = torch.randn(shape, generator=g, device=device) * fan_in ** -0.5
        sd[name] = t.to(dtype)
    return sd


def make_sam_state_dict(seed: int = 0, device="cpu", dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """A full EfficientViT-SAM xl1 state dict with random weights: the image encoder's keys and shapes are those of the
    reference module (tests/golden/sam_xl1_shapes.json, prefixed `image_encoder.`), the prompt encoder's and mask
    decoder's are segment_anything's [3P] in the configuration of sam.py:520-544 (oracle.sam_decoder.decoder_shapes).
    Linear / conv weights ~ N(0, 1/fan_in); BatchNorm statistics and norm affines jittered; biases and the learned
    embeddings small (biases) or unit (token / point embeddings, the Fourier matrix) normal."""
    import json
    import os
    from oracle.sam_decoder import decoder_shapes
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, "..", "tests", "golden", "sam_xl1_shapes.json")) as f:
        enc = json.load(f)
    shapes = {"image_encoder." + k: tuple(v) for k, v in enc.items()}
    shapes.update(decoder_shapes())
    g = torch.Generator().manual_seed(seed)
    return {k: _sam_param(k, shp, g).to(device, dtype) for k, shp in shapes.items()}


def _sam_param(k, shp, g):
    """One random SAM parameter (make_sam_state_dict's initialisation rules), drawn from the CPU generator g."""
    if k.endswith("running_var"):
        return torch.rand(shp, generator=g) + 0.5
    if k.endswith("running_mean") or k.endswith(".bias"):
        return torch.randn(shp, generator=g) * 0.05
    if len(shp) == 1:                                         # norm gamma
        return 1.0 + 0.1 * torch.randn(shp, generator=g)
    if k.endswith(("embeddings.0.weight", "embeddings.1.weight", "embeddings.2.weight", "embeddings.3.weight",
                   "_embed.weight", "token.weight", "tokens.weight", "gaussian_matrix")):
        return torch.randn(shp, generator=g)
    fan_in = math.prod(shp[1:])
    if "output_upscaling" in k:                               # ConvTranspose2d weight [in, out, k, k]: fan-in = in
        fan_in = shp[0]
    return torch.randn(shp, generator=g) * fan_in ** -0.5


def make_sam_vit_state_dict(kind: str = "vit_b", seed: int = 0, device="cpu", dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """A full original-SAM state dict (`image_encoder.*` of ImageEncoderViT [3P] in build_sam's `kind` topology, plus
    the prompt encoder and mask decoder of make_sam_state_dict) with random weights that keep activations O(1) through
    the depth: linear weights ~ N(0, 1/fan_in), the two residual branches of each block scaled by depth^-0.5.  The
    rel-pos tables are NON-zero (SAM initialises them to zero, which would hide a missing bias)."""
    from .sam_vit import GRID, KINDS, OUT_CHANS, PATCH, WINDOW
    C, depth, heads, glob = KINDS[kind]
    hd = C // heads
    g = torch.Generator(device=device).manual_seed(seed)

    def rn(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g, device=device) * scale).to(dtype)

    branch = depth ** -0.5
    p = "image_encoder."
    sd = {p + "patch_embed.proj.weight": rn(C, 3, PATCH, PATCH, scale=(3 * PATCH * PATCH) ** -0.5),
          p + "patch_embed.proj.bias": rn(C, scale=0.05), p + "pos_embed": rn(1, GRID, GRID, C, scale=0.1)}
    for i in range(depth):
        b = f"{p}blocks.{i}."
        n = 2 * (GRID if i in glob else WINDOW) - 1
        for norm in ("norm1", "norm2"):
            sd[b + norm + ".weight"], sd[b + norm + ".bias"] = 1 + rn(C, scale=0.1), rn(C, scale=0.05)
        sd[b + "attn.qkv.weight"], sd[b + "attn.qkv.bias"] = rn(3 * C, C, scale=C ** -0.5), rn(3 * C, scale=0.3)
        sd[b + "attn.proj.weight"], sd[b + "attn.proj.bias"] = rn(C, C, scale=branch * C ** -0.5), rn(C, scale=0.05)
        sd[b + "attn.rel_pos_h"], sd[b + "attn.rel_pos_w"] = rn(n, hd, scale=0.1), rn(n, hd, scale=0.1)
        sd[b + "mlp.lin1.weight"], sd[b + "mlp.lin1.bias"] = rn(4 * C, C, scale=C ** -0.5), rn(4 * C, scale=0.05)
        sd[b + "mlp.lin2.weight"] = rn(C, 4 * C, scale=branch * (4 * C) ** -0.5)
        sd[b + "mlp.lin2.bias"] = rn(C, scale=0.05)
    sd[p + "neck.0.weight"] = rn(OUT_CHANS, C, 1, 1, scale=C ** -0.5)
    sd[p + "neck.2.weight"] = rn(OUT_CHANS, OUT_CHANS, 3, 3, scale=(9 * OUT_CHANS) ** -0.5)
    for k in ("neck.1", "neck.3"):
        sd[p + k + ".weight"], sd[p + k + ".bias"] = 1 + rn(OUT_CHANS, scale=0.1), rn(OUT_CHANS, scale=0.05)
    from oracle.sam_decoder import decoder_shapes
    gd = torch.Generator().manual_seed(seed + 1)
    sd.update({k: _sam_param(k, shp, gd).to(device, dtype) for k, shp in decoder_shapes().items()})
    return sd
