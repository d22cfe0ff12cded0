"""fp32 torch restatement of the EfficientViT-SAM prompt-to-mask path: segment_anything v1.0 PromptEncoder, MaskDecoder and
TwoWayTransformer [3P] (the reference imports them from segment_anything, which it does not ship) in the configuration of
reference src/efficientvit/models/efficientvit/sam.py:520-544, and the predictor plumbing of EfficientViTSamPredictor /
EfficientViTSam.postprocess_masks / SamResize (sam.py:64-98,197-459), which tests/golden/sam_predictor.pt pins.

Every function reads a state dict with the reference's key names (`prompt_encoder.*`, `mask_decoder.*`).  LayerNorm eps
is 1e-6 everywhere (create_sam_model calls set_norm_eps(model, 1e-6), sam_model_zoo.py:44)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

EMBED, IMG_EMB, IMG_SIZE, NUM_MASK_TOKENS, HEADS, LN_EPS = 256, 64, 1024, 4, 8, 1e-6
PIXEL_MEAN = [123.675 / 255, 116.28 / 255, 103.53 / 255]
PIXEL_STD = [58.395 / 255, 57.12 / 255, 57.375 / 255]


def decoder_shapes():
    """Parameter shapes of PromptEncoder(256, (64, 64), (1024, 1024), 16) and MaskDecoder(TwoWayTransformer(2, 256, 2048,
    8), 3 multimask outputs, IoU head 3 x 256) [3P], keyed as in an EfficientViT-SAM state dict."""
    s = {"prompt_encoder.pe_layer.positional_encoding_gaussian_matrix": (2, 128)}
    for i in range(4):
        s[f"prompt_encoder.point_embeddings.{i}.weight"] = (1, EMBED)
    s["prompt_encoder.not_a_point_embed.weight"] = (1, EMBED)
    s.update({"prompt_encoder.mask_downscaling.0.weight": (4, 1, 2, 2), "prompt_encoder.mask_downscaling.0.bias": (4,),
              "prompt_encoder.mask_downscaling.1.weight": (4,), "prompt_encoder.mask_downscaling.1.bias": (4,),
              "prompt_encoder.mask_downscaling.3.weight": (16, 4, 2, 2), "prompt_encoder.mask_downscaling.3.bias": (16,),
              "prompt_encoder.mask_downscaling.4.weight": (16,), "prompt_encoder.mask_downscaling.4.bias": (16,),
              "prompt_encoder.mask_downscaling.6.weight": (EMBED, 16, 1, 1), "prompt_encoder.mask_downscaling.6.bias": (EMBED,),
              "prompt_encoder.no_mask_embed.weight": (1, EMBED)})

    def attn(p, internal):
        for n in "qkv":
            s[f"{p}.{n}_proj.weight"], s[f"{p}.{n}_proj.bias"] = (internal, EMBED), (internal,)
        s[f"{p}.out_proj.weight"], s[f"{p}.out_proj.bias"] = (EMBED, internal), (EMBED,)

    def norm(p):
        s[f"{p}.weight"], s[f"{p}.bias"] = (EMBED,), (EMBED,)

    t = "mask_decoder.transformer"
    for i in range(2):
        p = f"{t}.layers.{i}"
        attn(p + ".self_attn", EMBED)
        norm(p + ".norm1")
        attn(p + ".cross_attn_token_to_image", EMBED // 2)
        norm(p + ".norm2")
        s[p + ".mlp.lin1.weight"], s[p + ".mlp.lin1.bias"] = (2048, EMBED), (2048,)
        s[p + ".mlp.lin2.weight"], s[p + ".mlp.lin2.bias"] = (EMBED, 2048), (EMBED,)
        norm(p + ".norm3")
        norm(p + ".norm4")
        attn(p + ".cross_attn_image_to_token", EMBED // 2)
    attn(t + ".final_attn_token_to_image", EMBED // 2)
    norm(t + ".norm_final_attn")
    s["mask_decoder.iou_token.weight"] = (1, EMBED)
    s["mask_decoder.mask_tokens.weight"] = (NUM_MASK_TOKENS, EMBED)
    s.update({"mask_decoder.output_upscaling.0.weight": (EMBED, 64, 2, 2), "mask_decoder.output_upscaling.0.bias": (64,),
              "mask_decoder.output_upscaling.1.weight": (64,), "mask_decoder.output_upscaling.1.bias": (64,),
              "mask_decoder.output_upscaling.3.weight": (64, 32, 2, 2), "mask_decoder.output_upscaling.3.bias": (32,)})
    for i in range(NUM_MASK_TOKENS):
        for j, (o, k) in enumerate(((EMBED, EMBED), (EMBED, EMBED), (32, EMBED))):
            s[f"mask_decoder.output_hypernetworks_mlps.{i}.layers.{j}.weight"] = (o, k)
            s[f"mask_decoder.output_hypernetworks_mlps.{i}.layers.{j}.bias"] = (o,)
    for j, (o, k) in enumerate(((EMBED, EMBED), (EMBED, EMBED), (NUM_MASK_TOKENS, EMBED))):
        s[f"mask_decoder.iou_prediction_head.layers.{j}.weight"] = (o, k)
        s[f"mask_decoder.iou_prediction_head.layers.{j}.bias"] = (o,)
    return s


# ------------------------------------------------------------------------------------------------ prompt encoder [3P]
def pe_encoding(sd, coords):
    """PositionEmbeddingRandom._pe_encoding: coords in [0, 1] -> [sin, cos](2 pi (2c - 1) @ G)."""
    g = sd["prompt_encoder.pe_layer.positional_encoding_gaussian_matrix"].float()
    c = (2 * coords - 1) @ g.to(coords.device)
    c = 2 * math.pi * c
    return torch.cat([torch.sin(c), torch.cos(c)], dim=-1)


def dense_pe(sd):
    """PromptEncoder.get_dense_pe(): (1, 256, 64, 64)."""
    h = w = IMG_EMB
    grid = torch.ones((h, w))
    y = (grid.cumsum(dim=0) - 0.5) / h
    x = (grid.cumsum(dim=1) - 0.5) / w
    return pe_encoding(sd, torch.stack([x, y], dim=-1)).permute(2, 0, 1).unsqueeze(0)


def _with_coords(sd, coords):
    coords = coords.clone().float()
    coords[..., 0] = coords[..., 0] / IMG_SIZE
    coords[..., 1] = coords[..., 1] / IMG_SIZE
    return pe_encoding(sd, coords)


def prompt_encoder(sd, points=None, boxes=None, masks=None):
    """PromptEncoder.forward: ((B, N, 2) coords, (B, N) labels) / (B, 4) boxes in the 1024 input frame ->
    sparse (B, S, 256), dense (B, 256, 64, 64)."""
    if masks is not None:
        raise ValueError("mask prompts are not supported")
    pe = lambda i: sd[f"prompt_encoder.point_embeddings.{i}.weight"].float()  # noqa: E731
    bs = points[0].shape[0] if points is not None else (boxes.shape[0] if boxes is not None else 1)
    sparse = torch.empty((bs, 0, EMBED))
    if points is not None:
        coords, labels = points
        coords = coords.float() + 0.5
        labels = labels.clone()
        if boxes is None:
            coords = torch.cat([coords, torch.zeros((coords.shape[0], 1, 2))], dim=1)
            labels = torch.cat([labels, -torch.ones((labels.shape[0], 1), dtype=labels.dtype)], dim=1)
        emb = _with_coords(sd, coords)
        emb[labels == -1] = 0.0
        emb[labels == -1] += sd["prompt_encoder.not_a_point_embed.weight"].float()
        emb[labels == 0] += pe(0)
        emb[labels == 1] += pe(1)
        sparse = torch.cat([sparse, emb], dim=1)
    if boxes is not None:
        corners = _with_coords(sd, (boxes.float() + 0.5).reshape(-1, 2, 2))
        corners[:, 0, :] += pe(2)
        corners[:, 1, :] += pe(3)
        sparse = torch.cat([sparse, corners], dim=1)
    dense = sd["prompt_encoder.no_mask_embed.weight"].float().reshape(1, -1, 1, 1).expand(bs, -1, IMG_EMB, IMG_EMB)
    return sparse, dense


# ------------------------------------------------------------------------------------------------ mask decoder [3P]
def _lin(sd, p, x):
    return F.linear(x, sd[p + ".weight"].float(), sd[p + ".bias"].float())


def _ln(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"].float(), sd[p + ".bias"].float(), LN_EPS)


def _attention(sd, p, q, k, v):
    q, k, v = _lin(sd, p + ".q_proj", q), _lin(sd, p + ".k_proj", k), _lin(sd, p + ".v_proj", v)
    b, nq, c = q.shape
    sep = lambda t: t.reshape(b, t.shape[1], HEADS, c // HEADS).transpose(1, 2)  # noqa: E731
    q, k, v = sep(q), sep(k), sep(v)
    attn = torch.softmax(q @ k.permute(0, 1, 3, 2) / math.sqrt(c // HEADS), dim=-1)
    out = (attn @ v).transpose(1, 2).reshape(b, nq, c)
    return _lin(sd, p + ".out_proj", out)


def two_way_transformer(sd, image_embedding, image_pe, point_embedding):
    t = "mask_decoder.transformer"
    keys = image_embedding.flatten(2).permute(0, 2, 1)
    key_pe = image_pe.flatten(2).permute(0, 2, 1)
    queries = point_embedding
    for i in range(2):
        p = f"{t}.layers.{i}"
        if i == 0:   # skip_first_layer_pe
            queries = _attention(sd, p + ".self_attn", queries, queries, queries)
        else:
            q = queries + point_embedding
            queries = queries + _attention(sd, p + ".self_attn", q, q, queries)
        queries = _ln(sd, p + ".norm1", queries)
        q, k = queries + point_embedding, keys + key_pe
        queries = _ln(sd, p + ".norm2", queries + _attention(sd, p + ".cross_attn_token_to_image", q, k, keys))
        mlp = _lin(sd, p + ".mlp.lin2", torch.relu(_lin(sd, p + ".mlp.lin1", queries)))
        queries = _ln(sd, p + ".norm3", queries + mlp)
        q, k = queries + point_embedding, keys + key_pe
        keys = _ln(sd, p + ".norm4", keys + _attention(sd, p + ".cross_attn_image_to_token", k, q, queries))
    q, k = queries + point_embedding, keys + key_pe
    queries = _ln(sd, t + ".norm_final_attn", queries + _attention(sd, t + ".final_attn_token_to_image", q, k, keys))
    return queries, keys


def _mlp(sd, p, x, n=3):
    for i in range(n):
        x = _lin(sd, f"{p}.layers.{i}", x)
        if i < n - 1:
            x = torch.relu(x)
    return x


def _layernorm2d(x, w, b, eps=LN_EPS):
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return w[:, None, None] * x + b[:, None, None]


def output_upscaling(sd, src):
    m = "mask_decoder.output_upscaling"
    x = F.conv_transpose2d(src, sd[m + ".0.weight"].float(), sd[m + ".0.bias"].float(), stride=2)
    x = F.gelu(_layernorm2d(x, sd[m + ".1.weight"].float(), sd[m + ".1.bias"].float()))
    return F.gelu(F.conv_transpose2d(x, sd[m + ".3.weight"].float(), sd[m + ".3.bias"].float(), stride=2))


def mask_decoder(sd, image_embeddings, image_pe, sparse_prompt_embeddings, dense_prompt_embeddings, multimask_output):
    """MaskDecoder.forward -> (low-res logits (B, 1 | 3, 256, 256), iou predictions (B, 1 | 3))."""
    md = "mask_decoder"
    out_tokens = torch.cat([sd[md + ".iou_token.weight"].float(), sd[md + ".mask_tokens.weight"].float()], dim=0)
    out_tokens = out_tokens.unsqueeze(0).expand(sparse_prompt_embeddings.size(0), -1, -1)
    tokens = torch.cat((out_tokens, sparse_prompt_embeddings.float()), dim=1)
    src = torch.repeat_interleave(image_embeddings.float(), tokens.shape[0], dim=0) + dense_prompt_embeddings.float()
    pos = torch.repeat_interleave(image_pe.float(), tokens.shape[0], dim=0)
    b, c, h, w = src.shape
    hs, src = two_way_transformer(sd, src, pos, tokens)
    iou_out, mask_out = hs[:, 0, :], hs[:, 1:1 + NUM_MASK_TOKENS, :]
    up = output_upscaling(sd, src.transpose(1, 2).reshape(b, c, h, w))
    hyper_in = torch.stack([_mlp(sd, f"{md}.output_hypernetworks_mlps.{i}", mask_out[:, i, :]) for i in range(NUM_MASK_TOKENS)],
                           dim=1)
    b, c, h, w = up.shape
    masks = (hyper_in @ up.view(b, c, h * w)).view(b, -1, h, w)
    iou = _mlp(sd, md + ".iou_prediction_head", iou_out)
    sl = slice(1, None) if multimask_output else slice(0, 1)
    return masks[:, sl], iou[:, sl]


# ------------------------------------------------------------------------------------------------ predictor plumbing
def preprocess_shape(oldh, oldw, long_side=IMG_SIZE):
    """SamResize.get_preprocess_shape / ResizeLongestSide.get_preprocess_shape."""
    scale = long_side * 1.0 / max(oldh, oldw)
    return int(oldh * scale + 0.5), int(oldw * scale + 0.5)


def preprocess(image: np.ndarray, size=IMG_SIZE) -> torch.Tensor:
    """EfficientViTSam.transform: SamResize (PIL bilinear, only when the long side != size) -> ToTensor -> Normalize ->
    SamPad (corner) -> (1, 3, size, size) fp32."""
    from PIL import Image
    h, w = image.shape[:2]
    if max(h, w) != size:
        nh, nw = preprocess_shape(h, w, size)
        image = np.array(Image.fromarray(image).resize((nw, nh), Image.BILINEAR))
    x = torch.from_numpy(np.ascontiguousarray(image)).permute(2, 0, 1).float() / 255.0
    x = (x - torch.tensor(PIXEL_MEAN)[:, None, None]) / torch.tensor(PIXEL_STD)[:, None, None]
    x = F.pad(x, (0, size - x.shape[2], 0, size - x.shape[1]))
    return x.unsqueeze(0)


def postprocess_masks(masks, input_size, original_size, size=IMG_SIZE):
    masks = F.interpolate(masks, (size, size), mode="bilinear", align_corners=False)
    masks = masks[..., :input_size[0], :input_size[1]]
    return F.interpolate(masks, tuple(original_size), mode="bilinear", align_corners=False)


def apply_coords(coords, original_size, input_size):
    coords = np.array(coords, dtype=float, copy=True)
    coords[..., 0] = coords[..., 0] * (input_size[1] / original_size[1])
    coords[..., 1] = coords[..., 1] * (input_size[0] / original_size[0])
    return coords


def apply_boxes(boxes, original_size, input_size):
    return apply_coords(np.asarray(boxes).reshape(-1, 2, 2), original_size, input_size).reshape(-1, 4)


class OraclePredictor:
    """EfficientViTSamPredictor restated on the functions above (fp32, CPU or GPU); `image_encoder` maps the
    (1, 3, 1024, 1024) normalised image to the (1, 256, 64, 64) embedding."""

    def __init__(self, sd, image_encoder, image_format="RGB", device="cpu"):
        self.sd = {k: v.float().to(device) for k, v in sd.items() if k.startswith(("prompt_encoder.", "mask_decoder."))}
        self.image_encoder, self.image_format, self.device = image_encoder, image_format, device
        self.dense_pe = dense_pe({k: v.cpu() for k, v in self.sd.items() if k.startswith("prompt_encoder.pe")}).to(device)
        self.reset_image()

    def reset_image(self):
        self.is_image_set, self.features, self.original_size, self.input_size = False, None, None, None

    @torch.no_grad()
    def set_image(self, image, image_format="RGB"):
        if image_format != self.image_format:
            image = image[..., ::-1]
        self.reset_image()
        self.original_size = image.shape[:2]
        self.input_size = preprocess_shape(*self.original_size)
        self.features = self.image_encoder(preprocess(image).to(self.device))
        self.is_image_set = True

    @torch.no_grad()
    def predict_torch(self, point_coords=None, point_labels=None, boxes=None, multimask_output=True, return_logits=False):
        dev = self.device
        with torch.device("cpu"):
            points = None if point_coords is None else (point_coords.cpu(), point_labels.cpu())
            sd_pe = {k: v.cpu() for k, v in self.sd.items() if k.startswith("prompt_encoder.")}
            sparse, dense = prompt_encoder(sd_pe, points, None if boxes is None else boxes.cpu())
        low, iou = mask_decoder(self.sd, self.features, self.dense_pe, sparse.to(dev), dense.to(dev), multimask_output)
        masks = postprocess_masks(low, self.input_size, self.original_size)
        if not return_logits:
            masks = masks > 0.0
        return masks, iou, low

    def predict(self, point_coords=None, point_labels=None, box=None, multimask_output=True, return_logits=False):
        ct = lt = bt = None
        if point_coords is not None:
            ct = torch.as_tensor(apply_coords(point_coords, self.original_size, self.input_size), dtype=torch.float)[None]
            lt = torch.as_tensor(point_labels, dtype=torch.int)[None]
        if box is not None:
            bt = torch.as_tensor(apply_boxes(box, self.original_size, self.input_size), dtype=torch.float)[None]
        masks, iou, low = self.predict_torch(ct, lt, bt, multimask_output, return_logits)
        return masks[0].cpu().numpy(), iou[0].cpu().numpy(), low[0].cpu().numpy()
