"""Architecture description of the SDXL UNet / ControlNet the hot path runs (diffusers UNet2DConditionModel config of
stabilityai/stable-diffusion-xl-base-1.0, restated; the reference loads it through from_pretrained at
inference_lora.py:153-159)."""
import math
from dataclasses import dataclass
from typing import Dict, List, Tuple


@dataclass(frozen=True)
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280)
    layers_per_block: int = 2
    transformer_layers: Tuple[int, ...] = (0, 2, 10)  # 0 = block without attention
    head_dim: int = 64
    cross_attention_dim: int = 2048
    addition_time_embed_dim: int = 256
    pooled_dim: int = 1280
    norm_groups: int = 32
    cond_embed_channels: Tuple[int, ...] = (16, 32, 96, 256)

    @property
    def time_embed_dim(self) -> int:
        return self.block_out_channels[0] * 4

    @property
    def add_in_dim(self) -> int:
        return self.pooled_dim + 6 * self.addition_time_embed_dim

    @staticmethod
    def sdxl() -> "UNetConfig":
        return UNetConfig()

    @staticmethod
    def tiny() -> "UNetConfig":
        """Same topology at toy widths (CPU-oracle-sized parity tests)."""
        return UNetConfig(block_out_channels=(64, 128, 256), transformer_layers=(0, 1, 2), cross_attention_dim=256,
                          addition_time_embed_dim=64, pooled_dim=128, cond_embed_channels=(16, 32, 64, 128))


def param_shapes(cfg: UNetConfig, controlnet: bool = False) -> Dict[str, Tuple[int, ...]]:
    """Parameter name -> shape, diffusers key layout (what a real SDXL checkpoint's state dict contains)."""
    S: Dict[str, Tuple[int, ...]] = {}

    def lin(n, i, o, bias=True):
        S[n + ".weight"] = (o, i)
        if bias:
            S[n + ".bias"] = (o,)

    def cv(n, i, o, k=3):
        S[n + ".weight"] = (o, i, k, k)
        S[n + ".bias"] = (o,)

    def norm(n, ch):
        S[n + ".weight"] = (ch,)
        S[n + ".bias"] = (ch,)

    def res(n, i, o):
        norm(n + ".norm1", i)
        cv(n + ".conv1", i, o)
        lin(n + ".time_emb_proj", cfg.time_embed_dim, o)
        norm(n + ".norm2", o)
        cv(n + ".conv2", o, o)
        if i != o:
            cv(n + ".conv_shortcut", i, o, 1)

    def tr(n, ch, layers):
        norm(n + ".norm", ch)
        lin(n + ".proj_in", ch, ch)
        for k in range(layers):
            b = f"{n}.transformer_blocks.{k}"
            for a, kd in (("attn1", ch), ("attn2", cfg.cross_attention_dim)):
                lin(f"{b}.{a}.to_q", ch, ch, False)
                lin(f"{b}.{a}.to_k", kd, ch, False)
                lin(f"{b}.{a}.to_v", kd, ch, False)
                lin(f"{b}.{a}.to_out.0", ch, ch)
            for m in ("norm1", "norm2", "norm3"):
                norm(f"{b}.{m}", ch)
            lin(f"{b}.ff.net.0.proj", ch, 8 * ch)
            lin(f"{b}.ff.net.2", 4 * ch, ch)
        lin(n + ".proj_out", ch, ch)

    boc = cfg.block_out_channels
    nb = len(boc)
    cv("conv_in", cfg.in_channels, boc[0])
    lin("time_embedding.linear_1", boc[0], cfg.time_embed_dim)
    lin("time_embedding.linear_2", cfg.time_embed_dim, cfg.time_embed_dim)
    lin("add_embedding.linear_1", cfg.add_in_dim, cfg.time_embed_dim)
    lin("add_embedding.linear_2", cfg.time_embed_dim, cfg.time_embed_dim)
    skip_ch = [boc[0]]
    ch = boc[0]
    for i in range(nb):
        for j in range(cfg.layers_per_block):
            res(f"down_blocks.{i}.resnets.{j}", ch, boc[i])
            ch = boc[i]
            if cfg.transformer_layers[i] > 0:
                tr(f"down_blocks.{i}.attentions.{j}", ch, cfg.transformer_layers[i])
            skip_ch.append(ch)
        if i < nb - 1:
            cv(f"down_blocks.{i}.downsamplers.0.conv", ch, ch)
            skip_ch.append(ch)
    res("mid_block.resnets.0", ch, ch)
    tr("mid_block.attentions.0", ch, cfg.transformer_layers[-1])
    res("mid_block.resnets.1", ch, ch)
    if controlnet:
        cec = cfg.cond_embed_channels
        cv("controlnet_cond_embedding.conv_in", 3, cec[0])
        for i in range(len(cec) - 1):
            cv(f"controlnet_cond_embedding.blocks.{2 * i}", cec[i], cec[i])
            cv(f"controlnet_cond_embedding.blocks.{2 * i + 1}", cec[i], cec[i + 1])
        cv("controlnet_cond_embedding.conv_out", cec[-1], boc[0])
        for i, sc in enumerate(skip_ch):
            cv(f"controlnet_down_blocks.{i}", sc, sc, 1)
        cv("controlnet_mid_block", ch, ch, 1)
        return S
    skips = list(skip_ch)
    for i in range(nb):
        out = boc[nb - 1 - i]
        for j in range(cfg.layers_per_block + 1):
            res(f"up_blocks.{i}.resnets.{j}", ch + skips.pop(), out)
            ch = out
            if cfg.transformer_layers[nb - 1 - i] > 0:
                tr(f"up_blocks.{i}.attentions.{j}", ch, cfg.transformer_layers[nb - 1 - i])
        if i < nb - 1:
            cv(f"up_blocks.{i}.upsamplers.0.conv", ch, ch)
    norm("conv_norm_out", ch)
    cv("conv_out", ch, cfg.out_channels)
    return S


def transformer_names(cfg: UNetConfig, controlnet: bool = False) -> List[Tuple[str, int, int]]:
    """(Transformer2DModel path, channels, layers) in forward order."""
    out = []
    boc = cfg.block_out_channels
    nb = len(boc)
    for i in range(nb):
        if cfg.transformer_layers[i] > 0:
            for j in range(cfg.layers_per_block):
                out.append((f"down_blocks.{i}.attentions.{j}", boc[i], cfg.transformer_layers[i]))
    out.append(("mid_block.attentions.0", boc[-1], cfg.transformer_layers[-1]))
    if not controlnet:
        for i in range(nb):
            if cfg.transformer_layers[nb - 1 - i] > 0:
                for j in range(cfg.layers_per_block + 1):
                    out.append((f"up_blocks.{i}.attentions.{j}", boc[nb - 1 - i], cfg.transformer_layers[nb - 1 - i]))
    return out


def resnet_names(cfg: UNetConfig, controlnet: bool = False) -> List[Tuple[str, int]]:
    """(ResnetBlock2D path, out channels) in forward order."""
    out = []
    boc = cfg.block_out_channels
    nb = len(boc)
    for i in range(nb):
        for j in range(cfg.layers_per_block):
            out.append((f"down_blocks.{i}.resnets.{j}", boc[i]))
    out += [("mid_block.resnets.0", boc[-1]), ("mid_block.resnets.1", boc[-1])]
    if not controlnet:
        for i in range(nb):
            for j in range(cfg.layers_per_block + 1):
                out.append((f"up_blocks.{i}.resnets.{j}", boc[nb - 1 - i]))
    return out


def lora_target_names(cfg: UNetConfig) -> List[Tuple[str, int, int]]:
    """(Linear path, in, out) of every transformer Linear a LoRA may wrap (SURVEY section 8d coverage)."""
    out = []
    for name, ch, layers in transformer_names(cfg):
        out.append((name + ".proj_in", ch, ch))
        for k in range(layers):
            b = f"{name}.transformer_blocks.{k}"
            for a, kd in (("attn1", ch), ("attn2", cfg.cross_attention_dim)):
                out += [(f"{b}.{a}.to_q", ch, ch), (f"{b}.{a}.to_k", kd, ch), (f"{b}.{a}.to_v", kd, ch),
                        (f"{b}.{a}.to_out.0", ch, ch)]
            out += [(f"{b}.ff.net.0.proj", ch, 8 * ch), (f"{b}.ff.net.2", 4 * ch, ch)]
        out.append((name + ".proj_out", ch, ch))
    return out


def lora_conv_target_names(cfg: UNetConfig) -> List[Tuple[str, str, int, int, int]]:
    """(module path, kind, in, out, kernel) of the modules a LoCon adapter wraps besides the transformer Linears: every
    ResnetBlock2D's conv1 / conv2 (3x3), conv_shortcut (1x1, where in != out) and time_emb_proj (kind "linear",
    kernel 1), the Downsample2D conv (3x3, stride 2) and the Upsample2D conv (3x3 after nearest 2x).  conv_in, conv_out
    and the embedding MLPs are not LoRA targets (kohya never wraps them)."""
    out = []
    for key, shp in param_shapes(cfg).items():
        if not key.endswith(".weight"):
            continue
        name = key[: -len(".weight")]
        leaf = name.rsplit(".", 1)[-1]
        if leaf == "time_emb_proj":
            out.append((name, "linear", shp[1], shp[0], 1))
        elif (".resnets." in name and leaf in ("conv1", "conv2", "conv_shortcut")) or \
                name.endswith((".downsamplers.0.conv", ".upsamplers.0.conv")):
            out.append((name, "conv", shp[1], shp[0], shp[2]))
    return out


def unet_flops(cfg: UNetConfig, H: int, W: int, ctx_len: int = 77, controlnet: bool = False) -> float:
    """Algorithmic FLOPs of one sample-forward at latent H x W: 2*MAC of every conv/linear + 4*N*L*c per
    attention; norms / activations excluded (BASELINE.md section 3)."""
    S = param_shapes(cfg, controlnet)
    nb = len(cfg.block_out_channels)

    def level(name):
        p = name.split(".")
        if p[0] == "down_blocks":
            return int(p[1]) + (1 if p[2] == "downsamplers" else 0)
        if p[0] == "mid_block" or p[0] == "controlnet_mid_block":
            return nb - 1
        if p[0] == "up_blocks":
            return nb - 1 - int(p[1]) - (1 if p[2] == "upsamplers" else 0)
        return 0

    total = 0.0
    for n, shp in S.items():
        if not n.endswith(".weight") or len(shp) == 1 or n.startswith("controlnet_cond_embedding"):
            continue
        lvl = level(n)
        if n.startswith("controlnet_down_blocks"):
            idx = int(n.split(".")[1])
            lvl = [0, 0, 0, 1, 1, 1, 2, 2, 2][idx] if nb == 3 else 0
        hw = (H >> lvl) * (W >> lvl)
        macs = math.prod(shp)
        if "time_emb" in n or "time_embedding" in n or "add_embedding" in n:
            total += 2 * macs
        elif ".attn2.to_k" in n or ".attn2.to_v" in n:
            total += 2 * macs * ctx_len
        else:
            total += 2 * macs * hw
    for name, ch, layers in transformer_names(cfg, controlnet):
        hw = (H >> level(name)) * (W >> level(name))
        total += layers * (4.0 * hw * hw * ch + 4.0 * hw * ctx_len * ch)
    return total
