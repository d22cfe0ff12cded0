"""fp32 torch restatement of segment_anything v1.0's ImageEncoderViT [3P], the image encoder of the original SAM
(ViT-B/L/H) that the reference's `--segment_type GroundingDINO` branch prompts (inference_lora.py:91-126,191-198;
`sam_model_registry[...]` / `SamPredictor`).  segment_anything is neither installed here nor shipped in the reference
tree, so this module states the facts it relies on; each can be checked against segment_anything/modeling/
image_encoder.py and build_sam.py of v1.0:

  1. build_sam_vit_{h,l,b}: embed dim 1280 / 1024 / 768, depth 32 / 24 / 12, heads 16 / 16 / 12, global_attn_indexes
     (7, 15, 23, 31) / (5, 11, 17, 23) / (2, 5, 8, 11); image size 1024, patch 16, window 14, mlp_ratio 4, out_chans 256,
     qkv_bias, use_rel_pos, rel_pos_zero_init, use_abs_pos; norm_layer = LayerNorm(eps=1e-6).
  2. PatchEmbed: Conv2d(3, C, 16, stride 16) then permute to (B, H, W, C); then `x + pos_embed` with pos_embed (1, 64, 64, C).
  3. Block: shortcut = x; x = norm1(x); window_partition if window_size > 0; x = attn(x); window_unpartition;
     x = shortcut + x; x = x + mlp(norm2(x)).  MLPBlock = lin1, nn.GELU() (erf), lin2.
  4. Block i uses window_size = 0 when i is in global_attn_indexes, else 14; Attention's input_size is (64, 64) for a
     global block and (14, 14) for a windowed one, so rel_pos_h / rel_pos_w have 2 * 64 - 1 = 127 or 2 * 14 - 1 = 27 rows.
  5. Attention: qkv = Linear(C, 3C) reshaped (B, HW, 3, heads, hd), so q / k / v of head h are columns s C + h hd + d;
     attn = (q * scale) @ k^T with scale = hd^-0.5; add_decomposed_rel_pos(attn, q, ...) with the UNSCALED q;
     softmax over keys; (attn @ v) with heads concatenated; proj = Linear(C, C).
  6. add_decomposed_rel_pos: Rh = get_rel_pos(qh, kh, rel_pos_h), Rw likewise; rel_h = einsum("bhwc,hkc->bhwk", q, Rh),
     rel_w = einsum("bhwc,wkc->bhwk", q, Rw); attn[q, (kh, kw)] += rel_h[q, kh] + rel_w[q, kw].
  7. get_rel_pos with q_size == k_size == S and a table of 2S - 1 rows is the gather rel_pos[q - k + S - 1].
  8. window_partition zero-pads (B, H, W, C) at the bottom and right to multiples of the window BEFORE qkv (so padded
     tokens get q = k = v = the qkv bias) and window_unpartition crops the padding away.
  9. Neck: Conv2d(C, 256, 1, bias=False), LayerNorm2d(256), Conv2d(256, 256, 3, padding=1, bias=False), LayerNorm2d(256);
     LayerNorm2d normalises over channels with eps 1e-6.  The encoder returns (B, 256, 64, 64).

State-dict keys are the checkpoint's own (`image_encoder.` prefix stripped): patch_embed.proj.{weight,bias}, pos_embed,
blocks.N.{norm1,norm2}.{weight,bias}, blocks.N.attn.{qkv,proj}.{weight,bias}, blocks.N.attn.rel_pos_{h,w},
blocks.N.mlp.{lin1,lin2}.{weight,bias}, neck.{0,2}.weight, neck.{1,3}.{weight,bias}."""
import torch
import torch.nn.functional as F

LN_EPS, WINDOW, PATCH, OUT_CHANS = 1e-6, 14, 16, 256


def get_rel_pos(q_size, k_size, rel_pos):
    """Fact 7: equal sizes only (a 1024 input never interpolates)."""
    assert q_size == k_size and rel_pos.shape[0] == 2 * q_size - 1
    idx = torch.arange(q_size)[:, None] - torch.arange(k_size)[None, :] + (k_size - 1)
    return rel_pos[idx.to(rel_pos.device)]


def add_decomposed_rel_pos(attn, q, rel_pos_h, rel_pos_w, q_size, k_size):
    """Fact 6.  attn (B, qh*qw, kh*kw), q (B, qh*qw, hd)."""
    q_h, q_w = q_size
    k_h, k_w = k_size
    Rh = get_rel_pos(q_h, k_h, rel_pos_h)
    Rw = get_rel_pos(q_w, k_w, rel_pos_w)
    B, _, dim = q.shape
    r_q = q.reshape(B, q_h, q_w, dim)
    rel_h = torch.einsum("bhwc,hkc->bhwk", r_q, Rh)
    rel_w = torch.einsum("bhwc,wkc->bhwk", r_q, Rw)
    attn = attn.view(B, q_h, q_w, k_h, k_w) + rel_h[:, :, :, :, None] + rel_w[:, :, :, None, :]
    return attn.view(B, q_h * q_w, k_h * k_w)


def window_partition(x, ws):
    """Fact 8: (B, H, W, C) -> (B * nWin, ws, ws, C), (Hp, Wp)."""
    B, H, W, C = x.shape
    pad_h, pad_w = (ws - H % ws) % ws, (ws - W % ws) % ws
    if pad_h or pad_w:
        x = F.pad(x, (0, 0, 0, pad_w, 0, pad_h))
    Hp, Wp = H + pad_h, W + pad_w
    x = x.view(B, Hp // ws, ws, Wp // ws, ws, C)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, ws, ws, C), (Hp, Wp)


def window_unpartition(windows, ws, pad_hw, hw):
    Hp, Wp = pad_hw
    H, W = hw
    B = windows.shape[0] // (Hp * Wp // ws // ws)
    x = windows.view(B, Hp // ws, Wp // ws, ws, ws, -1)
    x = x.permute(0, 1, 3, 2, 4, 5).contiguous().view(B, Hp, Wp, -1)
    return x[:, :H, :W, :].contiguous()


def attention_core(qkv, heads, rel_pos_h, rel_pos_w, scale=None, mask_fn=None):
    """Fact 5 after the qkv Linear: qkv (B, H, W, 3C) -> (B, H, W, C) before proj.  mask_fn(attn) may edit the logits
    (tests use it to show that masking padded keys differs from the reference)."""
    B, H, W, C3 = qkv.shape
    hd = C3 // 3 // heads
    scale = hd ** -0.5 if scale is None else scale
    t = qkv.reshape(B, H * W, 3, heads, hd).permute(2, 0, 3, 1, 4).reshape(3, B * heads, H * W, hd)
    q, k, v = t.unbind(0)
    attn = (q * scale) @ k.transpose(-2, -1)
    attn = add_decomposed_rel_pos(attn, q, rel_pos_h, rel_pos_w, (H, W), (H, W))
    if mask_fn is not None:
        attn = mask_fn(attn)
    attn = attn.softmax(dim=-1)
    return (attn @ v).view(B, heads, H, W, hd).permute(0, 2, 3, 1, 4).reshape(B, H, W, -1)


def attention_block_attn(x, sd, p, heads, window, mask_fn=None):
    """Facts 3, 5 and 8 for the attention half of a block: x = norm1(shortcut), (B, H, W, C) -> attn output (B, H, W, C)."""
    H, W = x.shape[1], x.shape[2]
    if window > 0:
        x, pad_hw = window_partition(x, window)
    qkv = F.linear(x, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
    y = attention_core(qkv, heads, sd[p + "attn.rel_pos_h"], sd[p + "attn.rel_pos_w"], mask_fn=mask_fn)
    y = F.linear(y, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    if window > 0:
        y = window_unpartition(y, window, pad_hw, (H, W))
    return y


def block(x, sd, p, heads, window):
    """Fact 3: one Block on (B, H, W, C)."""
    C = x.shape[-1]
    h = F.layer_norm(x, (C,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], LN_EPS)
    x = x + attention_block_attn(h, sd, p, heads, window)
    h = F.layer_norm(x, (C,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], LN_EPS)
    h = F.gelu(F.linear(h, sd[p + "mlp.lin1.weight"], sd[p + "mlp.lin1.bias"]))
    return x + F.linear(h, sd[p + "mlp.lin2.weight"], sd[p + "mlp.lin2.bias"])


def layernorm2d(x, w, b, eps=LN_EPS):
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return w[:, None, None] * x + b[:, None, None]


def topology(sd):
    """(embed dim, depth, heads, head_dim, global block indices) read off an image-encoder state dict (facts 1, 4)."""
    C = sd["patch_embed.proj.weight"].shape[0]
    depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
    hd = sd["blocks.0.attn.rel_pos_h"].shape[1]
    glob = tuple(i for i in range(depth) if sd[f"blocks.{i}.attn.rel_pos_h"].shape[0] == 2 * 64 - 1)
    return C, depth, C // hd, hd, glob


def image_encoder(x, sd):
    """Facts 2-4 and 9: normalised (B, 3, 1024, 1024) -> (B, 256, 64, 64), fp32 throughout."""
    C, depth, heads, _, glob = topology(sd)
    x = F.conv2d(x, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=PATCH).permute(0, 2, 3, 1)
    x = x + sd["pos_embed"]
    for i in range(depth):
        x = block(x, sd, f"blocks.{i}.", heads, 0 if i in glob else WINDOW)
    x = F.conv2d(x.permute(0, 3, 1, 2), sd["neck.0.weight"])
    x = layernorm2d(x, sd["neck.1.weight"], sd["neck.1.bias"])
    x = F.conv2d(x, sd["neck.2.weight"], padding=1)
    return layernorm2d(x, sd["neck.3.weight"], sd["neck.3.bias"])


class OracleImageEncoderViT:
    """image_encoder(x, sd) as the callable OraclePredictor takes (sd: `image_encoder.*` keys, prefix optional)."""

    def __init__(self, sd, device="cpu"):
        pre = "image_encoder."
        self.sd = {(k[len(pre):] if k.startswith(pre) else k): v.float().to(device) for k, v in sd.items()
                   if k.startswith(pre) or not k.startswith(("prompt_encoder.", "mask_decoder."))}

    @torch.no_grad()
    def __call__(self, x):
        return image_encoder(x.float(), self.sd)
