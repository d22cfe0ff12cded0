"""The original SAM's image encoder (segment_anything ImageEncoderViT [3P]; ViT-B / L / H) on the C-ABI kernels: the
segmenter of the reference's `--segment_type GroundingDINO` branch (inference_lora.py:91-126,191-198, SamPredictor on
`sam_vit_h_4b8939.pth`).  oracle/sam_vit.py restates the module in fp32 and lists the facts it depends on.

The topology is read off the state dict (`image_encoder.` prefix optional): embed dim from patch_embed.proj.weight, depth
from the blocks.N keys, head_dim from the rel_pos_h width, global blocks are those whose rel_pos_h has 127 rows.

Mapping (reference op -> kernel), 4096 tokens at the fixed 1024² input:
  PatchEmbed Conv2d(3, C, 16, stride 16) + pos_embed   omg_gemm, K = 768 (the patch gather is one torch permute),
                                                        pos_embed as the GEMM's residual
  norm1 / norm2 (LayerNorm, eps 1e-6)                   omg_layernorm on the fp16 copy of the trunk (not folded)
  attn.qkv                                              omg_gemm with bias
  Attention with decomposed rel-pos, window / global    omg_attention_relpos (window padding = the qkv bias)
  attn.proj / mlp.lin2 + residual                       omg_gemm; the residual trunk is kept in fp32 (residual_f32 /
                                                        out_f32 twins) so 32 blocks do not accumulate fp16 rounding
  mlp.lin1 + GELU (erf)                                 omg_gemm, OMG_EPI_GELU
  neck: conv1x1, LayerNorm2d, conv3x3, LayerNorm2d      omg_gemm, omg_layernorm over channels, omg_gemm (3x3 taps)
Activations are fp16.  The output is checked for finiteness: a non-finite embedding raises FloatingPointError instead of
becoming NaN masks.  One image's ~200 launches are replayed as one CUDA graph per input shape."""
from typing import Dict, Tuple

import torch

from . import _lib as L
from . import ops

WINDOW, PATCH, GRID, OUT_CHANS, LN_EPS = 14, 16, 64, 256, 1e-6
KINDS = {"vit_b": (768, 12, 12, (2, 5, 8, 11)), "vit_l": (1024, 24, 16, (5, 11, 17, 23)),
         "vit_h": (1280, 32, 16, (7, 15, 23, 31))}   # embed dim, depth, heads, global blocks (build_sam.py [3P])


def strip_prefix(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The image encoder's keys of a SAM state dict without the `image_encoder.` prefix."""
    pre = "image_encoder."
    if any(k.startswith(pre) for k in sd):
        return {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
    return dict(sd)


def vit_topology(sd: Dict[str, torch.Tensor]) -> Tuple[int, int, int, int, Tuple[int, ...]]:
    """(embed dim, depth, heads, head_dim, global block indices) of an image-encoder state dict; ValueError when the dict
    is not a 1024-input ImageEncoderViT."""
    sd = strip_prefix(sd)
    try:
        C = sd["patch_embed.proj.weight"].shape[0]
        depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
        hd = sd["blocks.0.attn.rel_pos_h"].shape[1]
        rows = [sd[f"blocks.{i}.attn.rel_pos_h"].shape[0] for i in range(depth)]
    except (KeyError, ValueError) as e:
        raise ValueError(f"not a SAM ViT image-encoder state dict: {e!r}") from None
    if tuple(sd["patch_embed.proj.weight"].shape[1:]) != (3, PATCH, PATCH) or C % hd or hd not in (64, 80):
        raise ValueError(f"not a SAM ViT image encoder: patch weight {tuple(sd['patch_embed.proj.weight'].shape)}, "
                         f"head_dim {hd}")
    if any(r not in (2 * GRID - 1, 2 * WINDOW - 1) for r in rows):
        raise ValueError(f"rel_pos_h rows {sorted(set(rows))}: expected 127 (global) or 27 (14 x 14 windows) at 1024²")
    glob = tuple(i for i, r in enumerate(rows) if r == 2 * GRID - 1)
    return C, depth, C // hd, hd, glob


def topology_kind(sd) -> str:
    """"vit_b" | "vit_l" | "vit_h" for a state dict with one of build_sam's topologies, else ValueError."""
    C, depth, heads, _, glob = vit_topology(sd)
    for kind, t in KINDS.items():
        if t == (C, depth, heads, glob):
            return kind
    raise ValueError(f"ViT topology (embed {C}, depth {depth}, heads {heads}, global {glob}) is none of {list(KINDS)}")


class PackedSamViTImageEncoder:
    """ImageEncoderViT on the kernels: (B, 3, 1024, 1024) normalised image -> (B, 256, 64, 64) fp16."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", use_graph: bool = True):
        sd = strip_prefix(state_dict)
        self.dev = torch.device(device)
        self.use_graph = use_graph
        self.C, self.depth, self.heads, self.hd, self.glob = vit_topology(sd)
        h = lambda t: t.to(self.dev, torch.float16).contiguous()  # noqa: E731
        C = self.C
        self.patch_w = h(sd["patch_embed.proj.weight"].reshape(C, 3 * PATCH * PATCH))
        self.patch_b = h(sd["patch_embed.proj.bias"])
        self.pos = h(sd["pos_embed"].reshape(GRID * GRID, C))
        self.blocks = []
        for i in range(self.depth):
            p = f"blocks.{i}."
            blk = {n: h(sd[p + n]) for n in ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias",
                                              "attn.proj.weight", "attn.proj.bias", "attn.rel_pos_h", "attn.rel_pos_w",
                                              "norm2.weight", "norm2.bias", "mlp.lin1.weight", "mlp.lin1.bias",
                                              "mlp.lin2.weight", "mlp.lin2.bias")}
            blk["window"] = 0 if i in self.glob else WINDOW
            blk["k_bias"] = blk["attn.qkv.bias"][C:2 * C]
            blk["v_bias"] = blk["attn.qkv.bias"][2 * C:]
            self.blocks.append(blk)
        self.neck0 = h(sd["neck.0.weight"].reshape(OUT_CHANS, C))
        self.neck1 = (h(sd["neck.1.weight"]), h(sd["neck.1.bias"]))
        self.neck2 = h(ops.pack_conv3x3_weight(sd["neck.2.weight"].float()))
        self.neck3 = (h(sd["neck.3.weight"]), h(sd["neck.3.bias"]))
        self._graphs = {}

    @torch.no_grad()
    def __call__(self, image: torch.Tensor) -> torch.Tensor:
        """Results are copies of the graph's static buffers; raises FloatingPointError on a non-finite embedding."""
        if not self.use_graph:
            y = self._encode(image)
        else:
            key = tuple(image.shape)
            ent = self._graphs.get(key)
            if ent is None:
                static_in = torch.empty(image.shape, dtype=torch.float16, device=self.dev)
                static_in.copy_(image)
                self._encode(static_in)                   # eager warm-up: kernel attributes, allocator pools
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    out = self._encode(static_in)
                ent = self._graphs[key] = (g, static_in, out)
            g, static_in, out = ent
            static_in.copy_(image)
            g.replay()
            y = out.clone()
        if not bool(torch.isfinite(y).all()):
            raise FloatingPointError("SAM ViT image embedding is not finite (fp16 range exceeded)")
        return y

    def block(self, i: int, x: torch.Tensor, x32: torch.Tensor, B: int) -> None:
        """Block i in place on the trunk: x fp16 [B * 4096, C] and its fp32 twin x32 (the residual's master copy)."""
        blk, C, T = self.blocks[i], self.C, GRID * GRID
        hN = ops.layernorm(x, blk["norm1.weight"], blk["norm1.bias"], eps=LN_EPS)
        qkv = ops.linear(hN, blk["attn.qkv.weight"], blk["attn.qkv.bias"])
        a = ops.attention_relpos(qkv.view(B, T, 3 * C), GRID, GRID, self.heads, self.hd, blk["attn.rel_pos_h"],
                                 blk["attn.rel_pos_w"], window=blk["window"], k_bias=blk["k_bias"], v_bias=blk["v_bias"])
        ops.linear(a.view(B * T, C), blk["attn.proj.weight"], blk["attn.proj.bias"], residual_f32=x32, out=x, out_f32=x32)
        hN = ops.layernorm(x, blk["norm2.weight"], blk["norm2.bias"], eps=LN_EPS)
        m = ops.linear(hN, blk["mlp.lin1.weight"], blk["mlp.lin1.bias"], epilogue=L.EPI_GELU)
        ops.linear(m, blk["mlp.lin2.weight"], blk["mlp.lin2.bias"], residual_f32=x32, out=x, out_f32=x32)

    def _encode(self, image: torch.Tensor) -> torch.Tensor:
        B = image.shape[0]
        assert tuple(image.shape[1:]) == (3, GRID * PATCH, GRID * PATCH), "the SAM ViT encoder takes 1024² inputs"
        C, T = self.C, GRID * GRID
        patches = image.to(self.dev, torch.float16).view(B, 3, GRID, PATCH, GRID, PATCH).permute(0, 2, 4, 1, 3, 5)
        patches = patches.reshape(B * T, 3 * PATCH * PATCH)
        pos = self.pos if B == 1 else self.pos.repeat(B, 1)
        x32 = torch.empty(B * T, C, dtype=torch.float32, device=self.dev)
        x = ops.linear(patches, self.patch_w, self.patch_b, residual=pos, out_f32=x32)
        for i in range(self.depth):
            self.block(i, x, x32, B)
        n = ops.linear(x, self.neck0)
        n = ops.layernorm(n, *self.neck1, eps=LN_EPS).view(B, GRID, GRID, OUT_CHANS)
        n = ops.conv3x3(n, self.neck2)
        n = ops.layernorm(n.view(B * T, OUT_CHANS), *self.neck3, eps=LN_EPS)
        return n.view(B, GRID, GRID, OUT_CHANS).permute(0, 3, 1, 2)
