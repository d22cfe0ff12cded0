"""On-disk formats of the checkpoints OMG consumes, converted to what the packed executors take (SURVEY 8f-3).

* UNet / ControlNet: diffusers `diffusion_pytorch_model[.fp16].safetensors` - the key layout PackedUNet already uses.
* LoRA (`pipe.load_lora_weights(path, weight_name, adapter_name)`, inference_lora.py:163-169): the three layouts
  diffusers 0.25's loader accepts [3P, restated from the published formats]
    - kohya / Civitai with SGM block names   `lora_unet_input_blocks_4_1_transformer_blocks_0_attn1_to_q.lora_down.weight`
    - kohya with diffusers block names        `lora_unet_down_blocks_1_attentions_0_transformer_blocks_0_attn1_to_q.lora_down.weight`
    - diffusers / peft                        `unet.down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q.lora_A.weight`
                                              (also `.lora.down.weight`, `.lora_linear_layer.down.weight`,
                                               `.processor.to_q_lora.down.weight` of older diffusers)
  all become {Linear path: (A [r, in], B [out, r], alpha / r)}; text-encoder entries are returned separately.
* InstantID `ip-adapter.bin` (instantid_single_pieline.py:179-213): {"image_proj": Resampler state dict,
  "ip_adapter": {"<i>.to_k_ip.weight", "<i>.to_v_ip.weight"}} with i the position of the processor in
  `unet.attn_processors` (registration order: down blocks, up blocks, mid block; attn1 / attn2 alternating).

No tensor math happens here beyond reshapes; nothing in this module touches the GPU.
"""
import os
import re
from typing import Dict, List, Optional, Tuple

import torch

from .config import UNetConfig, lora_target_names, transformer_names

LoraDict = Dict[str, Tuple[torch.Tensor, torch.Tensor, float]]


# ------------------------------------------------------------------------------------------------ files
def load_state_dict(path: str) -> Dict[str, torch.Tensor]:
    """.safetensors, or a torch pickle (.bin / .pt / .ckpt, weights only)."""
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path)
    sd = torch.load(path, map_location="cpu", weights_only=True)
    return sd.get("state_dict", sd) if isinstance(sd, dict) else sd


def find_diffusers_weights(model_dir: str, subfolder: str = "unet", variant: Optional[str] = "fp16") -> str:
    """`<model_dir>/<subfolder>/diffusion_pytorch_model[.<variant>].safetensors` as `from_pretrained` resolves it
    (inference_lora.py:152-155: torch_dtype=float16, variant='fp16')."""
    base = os.path.join(model_dir, subfolder) if subfolder else model_dir
    names = []
    if variant:
        names.append(f"diffusion_pytorch_model.{variant}.safetensors")
    names += ["diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.bin"]
    for n in names:
        p = os.path.join(base, n)
        if os.path.isfile(p):
            return p
    raise FileNotFoundError(f"no diffusion_pytorch_model[.{variant}].safetensors|.bin under {base}")


def load_unet_weights(model_dir: str, subfolder: str = "unet", variant: Optional[str] = "fp16"):
    return load_state_dict(find_diffusers_weights(model_dir, subfolder, variant))


# ------------------------------------------------------------------------------------------------ LoRA
def _sgm_to_diffusers_block(cfg: UNetConfig, part: str, idx: int, sub: int) -> Optional[str]:
    """SGM `input_blocks.<idx>.<sub>` / `middle_block.<sub>` / `output_blocks.<idx>.<sub>` -> diffusers module path.

    SGM numbers the encoder as [conv_in, (res[,attn]) x layers_per_block, downsample, ...] and the decoder as
    (layers_per_block + 1) x (res[,attn][,upsample]) per level."""
    lpb = cfg.layers_per_block
    nb = len(cfg.block_out_channels)
    if part == "middle_block":
        return {0: "mid_block.resnets.0", 1: "mid_block.attentions.0", 2: "mid_block.resnets.1"}.get(sub)
    if part == "input_blocks":
        if idx == 0:
            return "conv_in"
        blk, pos = divmod(idx - 1, lpb + 1)
        if blk >= nb:
            return None
        if pos == lpb:
            return f"down_blocks.{blk}.downsamplers.0"
        return f"down_blocks.{blk}.{'resnets' if sub == 0 else 'attentions'}.{pos}"
    if part == "output_blocks":
        blk, pos = divmod(idx, lpb + 1)
        if blk >= nb:
            return None
        has_attn = cfg.transformer_layers[nb - 1 - blk] > 0
        if sub == 0:
            return f"up_blocks.{blk}.resnets.{pos}"
        if sub == 1 and has_attn:
            return f"up_blocks.{blk}.attentions.{pos}"
        return f"up_blocks.{blk}.upsamplers.0"
    return None


def _kohya_lookup(cfg: UNetConfig) -> Dict[str, str]:
    """kohya flattens the module path with '_' (ambiguous to split), so match against the known Linear targets."""
    table = {}
    for name, _i, _o in lora_target_names(cfg):
        table["lora_unet_" + name.replace(".", "_")] = name
    # SGM spellings of the same modules
    for tname, _ch, _layers in transformer_names(cfg):
        for part, rng in (("input_blocks", range(0, 3 * len(cfg.block_out_channels) + 1)), ("middle_block", [0]),
                          ("output_blocks", range(0, 3 * len(cfg.block_out_channels) + 3))):
            for idx in rng:
                for sub in (0, 1, 2):
                    if _sgm_to_diffusers_block(cfg, part, idx, sub) == tname:
                        sgm = f"{part}_{idx}_{sub}" if part != "middle_block" else f"middle_block_{sub}"
                        for full, name in list(table.items()):
                            if name.startswith(tname + "."):
                                tail = name[len(tname) + 1:].replace(".", "_")
                                table[f"lora_unet_{sgm}_{tail}"] = name
    return table


_PEFT_SUFFIXES = (
    (".lora_A.weight", "A"), (".lora_B.weight", "B"),
    (".lora_A.default.weight", "A"), (".lora_B.default.weight", "B"),
    (".lora.down.weight", "A"), (".lora.up.weight", "B"),
    (".lora_linear_layer.down.weight", "A"), (".lora_linear_layer.up.weight", "B"),
    (".lora_down.weight", "A"), (".lora_up.weight", "B"),
)


def convert_lora_state_dict(sd: Dict[str, torch.Tensor], cfg: Optional[UNetConfig] = None, strict: bool = False):
    """-> (unet_lora, text_encoder_lora, skipped).

    unet_lora: {diffusers Linear path: (A [r,in], B [out,r], alpha/r)} for omg_b200 `load_lora_weights`.
    text_encoder_lora: same triple keyed `te1.<path>` / `te2.<path>` (consumed by whoever owns the text encoders).
    skipped: keys of UNet modules the packed executor does not adapt (conv / time-embedding LoRA); strict=True raises.
    The rank scale follows kohya / peft: alpha / r, with alpha = r when the file stores none."""
    cfg = cfg or UNetConfig.sdxl()
    known = {name for name, _i, _o in lora_target_names(cfg)}
    kohya = _kohya_lookup(cfg)
    parts: Dict[str, Dict[str, torch.Tensor]] = {}
    te_parts: Dict[str, Dict[str, torch.Tensor]] = {}
    skipped: List[str] = []

    def slot(store, name):
        return store.setdefault(name, {})

    for key, val in sd.items():
        if key.startswith("lora_te"):  # kohya text encoders: lora_te1_text_model_encoder_layers_0_self_attn_q_proj...
            m = re.match(r"lora_(te\d?)_(.+?)\.(lora_down\.weight|lora_up\.weight|alpha)$", key)
            if m:
                name = (m.group(1) if m.group(1) != "te" else "te1") + "." + m.group(2)
                slot(te_parts, name)[{"lora_down.weight": "A", "lora_up.weight": "B", "alpha": "alpha"}[m.group(3)]] = val
            continue
        if key.startswith("text_encoder"):
            m = re.match(r"(text_encoder(?:_2)?)\.(.+?)(\.alpha|" + "|".join(re.escape(s) for s, _ in _PEFT_SUFFIXES) + ")$", key)
            if m:
                name = ("te2." if m.group(1).endswith("_2") else "te1.") + m.group(2)
                what = "alpha" if m.group(3) == ".alpha" else dict(_PEFT_SUFFIXES)[m.group(3)]
                slot(te_parts, name)[what] = val
            continue
        if key.startswith("lora_unet_"):
            stem, _, tail = key.partition(".")
            what = {"lora_down.weight": "A", "lora_up.weight": "B", "alpha": "alpha"}.get(tail)
            if what is None:
                skipped.append(key)
                continue
            name = kohya.get(stem)
            if name is None:
                skipped.append(key)
                continue
            slot(parts, name)[what] = val
            continue
        k = key[5:] if key.startswith("unet.") else key
        mp = re.match(r"(.+\.processor\.to_(?:q|k|v|out)_lora)\.(down|up)\.weight$", k)
        if mp:  # older diffusers attention-processor layout: ...attn1.processor.to_q_lora.down.weight
            name, what = mp.group(1), "A" if mp.group(2) == "down" else "B"
        elif k.endswith(".alpha"):
            name, what = k[:-6], "alpha"
        else:
            for suf, w in _PEFT_SUFFIXES:
                if k.endswith(suf):
                    name, what = k[: -len(suf)], w
                    break
            else:
                skipped.append(key)
                continue
        name = re.sub(r"\.processor\.(to_(?:q|k|v|out))_lora$", lambda m: "." + m.group(1), name)
        name = re.sub(r"\.to_out$", ".to_out.0", name)
        if name not in known:
            skipped.append(key)
            continue
        slot(parts, name)[what] = val

    def finish(store):
        out = {}
        for name, d in store.items():
            if "A" not in d or "B" not in d:
                raise ValueError(f"LoRA entry {name} lacks its {'down' if 'A' not in d else 'up'} matrix")
            A, B = d["A"], d["B"]
            if A.ndim != 2 or B.ndim != 2:
                A, B = A.flatten(1), B.flatten(1)  # 1x1-conv spelling of a Linear
            r = A.shape[0]
            if B.shape[1] != r:
                raise ValueError(f"LoRA entry {name}: down is {tuple(A.shape)}, up is {tuple(B.shape)}")
            alpha = float(d["alpha"]) if "alpha" in d else float(r)
            out[name] = (A, B, alpha / r)
        return out

    if strict and skipped:
        raise ValueError(f"{len(skipped)} LoRA tensors target modules this path does not adapt, e.g. {skipped[:3]}")
    unet_lora = finish(parts)
    shapes = {n: (i, o) for n, i, o in lora_target_names(cfg)}
    for name, (A, B, _s) in unet_lora.items():
        i, o = shapes[name]
        if A.shape[1] != i or B.shape[0] != o:
            raise ValueError(f"LoRA entry {name}: expected in={i}, out={o}, file has in={A.shape[1]}, out={B.shape[0]}")
    return unet_lora, finish(te_parts), skipped


def load_lora(path: str, cfg: Optional[UNetConfig] = None, strict: bool = False):
    """File -> (unet_lora, text_encoder_lora, skipped); see convert_lora_state_dict."""
    return convert_lora_state_dict(load_state_dict(path), cfg, strict)


# ------------------------------------------------------------------------------------------------ IP-adapter
def attn_processor_order(cfg: UNetConfig) -> List[str]:
    """Paths of `unet.attn_processors` in diffusers' registration order (down_blocks, up_blocks, mid_block - the
    ModuleLists are created before the mid block), which is the numbering of `ip_adapter` keys."""
    def block_paths(prefix):
        out = []
        for name, _ch, layers in transformer_names(cfg):
            if name.startswith(prefix):
                for k in range(layers):
                    out += [f"{name}.transformer_blocks.{k}.attn1", f"{name}.transformer_blocks.{k}.attn2"]
        return out
    return block_paths("down_blocks") + block_paths("up_blocks") + block_paths("mid_block")


def convert_ip_adapter(sd: Dict, cfg: Optional[UNetConfig] = None):
    """`ip-adapter.bin` dict -> (image_proj state dict, {attn2 path: (to_k_ip [c, ctx], to_v_ip [c, ctx])})."""
    cfg = cfg or UNetConfig.sdxl()
    ip = sd.get("ip_adapter", sd)
    order = attn_processor_order(cfg)
    out = {}
    for key, val in ip.items():
        m = re.match(r"(\d+)\.(to_k_ip|to_v_ip)\.weight$", key)
        if not m:
            raise ValueError(f"unexpected ip_adapter key {key}")
        idx = int(m.group(1))
        if idx >= len(order) or not order[idx].endswith("attn2"):
            raise ValueError(f"ip_adapter key {key} does not address a cross-attention processor of this UNet")
        out.setdefault(order[idx], {})[m.group(2)] = val
    weights = {}
    for path, d in out.items():
        if set(d) != {"to_k_ip", "to_v_ip"}:
            raise ValueError(f"ip_adapter entry for {path} is incomplete")
        weights[path] = (d["to_k_ip"], d["to_v_ip"])
    missing = [p for p in order if p.endswith("attn2") and p not in weights]
    if missing:
        raise ValueError(f"ip_adapter lacks {len(missing)} cross-attention layers, e.g. {missing[0]}")
    return sd.get("image_proj"), weights


def load_ip_adapter(path: str, cfg: Optional[UNetConfig] = None):
    return convert_ip_adapter(torch.load(path, map_location="cpu", weights_only=True), cfg)
