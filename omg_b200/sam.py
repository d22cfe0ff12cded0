"""EfficientViT-SAM box / point prompts -> masks on the kernels: prompt encoder, mask decoder and predictor (SURVEY
section 8, row f-4: "visual comprehension on-device").

Between its two stages the reference turns the stage-1 image into one mask per concept: a detector box prompts
EfficientViT-SAM xl1 (inference_lora.py:91-126 -> EfficientViTSamPredictor.set_image / .predict(box=...,
multimask_output=False), src/efficientvit/models/efficientvit/sam.py:244-459).  The image encoder runs on
omg_b200.sam_encoder; this module adds the rest of the model with the reference's surface.  The prompt encoder,
MaskDecoder and TwoWayTransformer are segment_anything v1.0 [3P] (the reference imports them; configuration
sam.py:520-544: embed 256, 64 x 64 image embedding, 1024 input, TwoWayTransformer(depth 2, mlp 2048, 8 heads),
3 multimask outputs, IoU head 3 x 256), restated in fp32 torch by oracle/sam_decoder.py.

Mapping (reference op -> kernel), B prompts x T = 5 + sparse tokens, 4096 image tokens per prompt:
  q / k / v / out projections, MLP (ReLU), hypernetworks, IoU head   omg_gemm (OMG_EPI_RELU); "+ PE" inputs are a second
                                                                       K-segment against the same weights, the image-side
                                                                       PE projections are constants folded in at load
  residual adds                                                        omg_gemm epilogue residual
  LayerNorm (eps 1e-6)                                                 omg_layernorm
  attention (head dim 32 self, 16 cross)                               omg_attention_small
  ConvTranspose2d #1                                                   omg_gemm, weight rows (dy, dx, channel)
  LayerNorm2d, GELU, ConvTranspose2d #2, GELU, hyper_in @ upscaled     omg_sam_mask_head
  postprocess_masks + threshold                                        omg_sam_postprocess
Torch is plumbing: the positional encoding of <= 64 prompt tokens, buffer allocation, and one CUDA graph per prompt
shape.  Mask prompts (`mask_input`) are not supported: OMG never passes them."""
import math
import os
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _lib as L
from . import ops
from .sam_encoder import PackedSamImageEncoder

EMBED, IMG_EMB, IMG_SIZE, NUM_MASK_TOKENS, HEADS, LN_EPS = 256, 64, 1024, 4, 8, 1e-6
PIXEL_MEAN = (123.675 / 255, 116.28 / 255, 103.53 / 255)
PIXEL_STD = (58.395 / 255, 57.12 / 255, 57.375 / 255)
MAX_TOKENS = 64   # omg_attention_small: the short side of every attention is the prompt's token count


def _pe_encoding(g, coords):
    """PositionEmbeddingRandom._pe_encoding [3P]: coords in [0, 1] -> [sin, cos](2 pi (2c - 1) @ G)."""
    c = 2 * math.pi * ((2 * coords - 1) @ g)
    return torch.cat([torch.sin(c), torch.cos(c)], dim=-1)


class PackedSamPromptEncoder:
    """segment_anything PromptEncoder [3P] for point and box prompts, from the `prompt_encoder.*` keys."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda"):
        sd = {k[len("prompt_encoder."):]: v for k, v in state_dict.items() if k.startswith("prompt_encoder.")}
        self.dev = torch.device(device)
        f = lambda k: sd[k].float().to(self.dev)  # noqa: E731
        self.gauss = f("pe_layer.positional_encoding_gaussian_matrix")
        self.point_embeddings = [f(f"point_embeddings.{i}.weight")[0] for i in range(4)]
        self.not_a_point_embed = f("not_a_point_embed.weight")[0]
        self.no_mask_embed = f("no_mask_embed.weight")[0]
        grid = torch.ones((IMG_EMB, IMG_EMB), device=self.dev)
        y, x = (grid.cumsum(0) - 0.5) / IMG_EMB, (grid.cumsum(1) - 0.5) / IMG_EMB
        self.dense_pe_cl = _pe_encoding(self.gauss, torch.stack([x, y], dim=-1))    # (64, 64, 256) fp32, once per model

    def get_dense_pe(self) -> torch.Tensor:
        return self.dense_pe_cl.permute(2, 0, 1).unsqueeze(0)

    def _coords_pe(self, coords):
        return _pe_encoding(self.gauss, coords / IMG_SIZE)      # input_image_size (1024, 1024): x / W, y / H

    def __call__(self, points: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, boxes: Optional[torch.Tensor] = None,
                 masks: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """((B, N, 2) coords, (B, N) labels) and / or (B, 4) boxes, in the 1024 input frame -> sparse (B, S, 256) fp32,
        dense (B, 256, 64, 64) (the broadcast no_mask_embed).  Written without data-dependent indexing so that it can be
        captured in a CUDA graph."""
        if masks is not None:
            raise ValueError("mask prompts (mask_input) are not supported")
        parts = []
        if points is not None:
            coords, labels = points
            coords = coords.to(self.dev, torch.float32) + 0.5
            labels = labels.to(self.dev)
            if boxes is None:   # pad point (label -1) when there is no box
                coords = torch.cat([coords, coords.new_zeros(coords.shape[0], 1, 2)], dim=1)
                labels = torch.cat([labels, -labels.new_ones(labels.shape[0], 1)], dim=1)
            emb = self._coords_pe(coords)
            lab = labels[..., None]
            emb = emb + (lab == 0) * self.point_embeddings[0] + (lab == 1) * self.point_embeddings[1]
            parts.append(torch.where(lab == -1, self.not_a_point_embed.expand_as(emb), emb))
        if boxes is not None:
            corners = self._coords_pe(boxes.to(self.dev, torch.float32).reshape(-1, 2, 2) + 0.5)
            parts.append(corners + torch.stack(self.point_embeddings[2:4])[None])
        if not parts:
            raise ValueError("give point and / or box prompts")
        sparse = torch.cat(parts, dim=1)
        dense = self.no_mask_embed.reshape(1, -1, 1, 1).expand(sparse.shape[0], -1, IMG_EMB, IMG_EMB)
        return sparse, dense


def _h(t, dev):
    return t.to(dev, torch.float16).contiguous()


class PackedSamMaskDecoder:
    """segment_anything MaskDecoder + TwoWayTransformer [3P] on the kernels, from the `mask_decoder.*` keys (and the
    prompt encoder's dense PE, whose projections are constants per model)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], dense_pe_cl: torch.Tensor, device="cuda"):
        sd = {k[len("mask_decoder."):]: v.float() for k, v in state_dict.items() if k.startswith("mask_decoder.")}
        dev = self.dev = torch.device(device)
        pe = dense_pe_cl.reshape(IMG_EMB * IMG_EMB, EMBED).float().cpu()
        W = lambda p: sd[p + ".weight"]  # noqa: E731
        Bv = lambda p: sd[p + ".bias"]  # noqa: E731
        z = lambda t: torch.zeros_like(t)  # noqa: E731
        self.layers = []
        t = "transformer"
        for i in range(2):
            p = f"{t}.layers.{i}"
            sa, ti, it = p + ".self_attn", p + ".cross_attn_token_to_image", p + ".cross_attn_image_to_token"
            L_ = {}
            if i == 0:   # skip_first_layer_pe: q = k = v = queries
                L_["sa_w"] = _h(torch.cat([W(sa + ".q_proj"), W(sa + ".k_proj"), W(sa + ".v_proj")]), dev)
            else:        # [queries | query_pe] against [[Wq | Wq]; [Wk | Wk]; [Wv | 0]]
                wq, wk, wv = W(sa + ".q_proj"), W(sa + ".k_proj"), W(sa + ".v_proj")
                L_["sa_w"] = _h(torch.cat([torch.cat([wq, wq], 1), torch.cat([wk, wk], 1), torch.cat([wv, z(wv)], 1)]), dev)
            L_["sa_b"] = _h(torch.cat([Bv(sa + ".q_proj"), Bv(sa + ".k_proj"), Bv(sa + ".v_proj")]), dev)
            L_["sa_o"] = (_h(W(sa + ".out_proj"), dev), _h(Bv(sa + ".out_proj"), dev))
            wq = W(ti + ".q_proj")
            L_["ti_q"] = (_h(torch.cat([wq, wq], 1), dev), _h(Bv(ti + ".q_proj"), dev))
            # image side of both cross-attentions: keys @ [Wk_t2i; Wv_t2i; Wq_i2t]^T, + key_pe projected once here
            wk, wv, wq2 = W(ti + ".k_proj"), W(ti + ".v_proj"), W(it + ".q_proj")
            L_["img_w"] = _h(torch.cat([wk, wv, wq2]), dev)
            L_["img_b"] = _h(torch.cat([Bv(ti + ".k_proj"), Bv(ti + ".v_proj"), Bv(it + ".q_proj")]), dev)
            L_["img_pe"] = _h(torch.cat([pe @ wk.t(), torch.zeros(pe.shape[0], wv.shape[0]), pe @ wq2.t()], 1), dev)
            L_["ti_o"] = (_h(W(ti + ".out_proj"), dev), _h(Bv(ti + ".out_proj"), dev))
            L_["mlp1"] = (_h(W(p + ".mlp.lin1"), dev), _h(Bv(p + ".mlp.lin1"), dev))
            L_["mlp2"] = (_h(W(p + ".mlp.lin2"), dev), _h(Bv(p + ".mlp.lin2"), dev))
            wk, wv = W(it + ".k_proj"), W(it + ".v_proj")
            L_["it_kv"] = (_h(torch.cat([torch.cat([wk, wk], 1), torch.cat([wv, z(wv)], 1)]), dev),
                           _h(torch.cat([Bv(it + ".k_proj"), Bv(it + ".v_proj")]), dev))
            L_["it_o"] = (_h(W(it + ".out_proj"), dev), _h(Bv(it + ".out_proj"), dev))
            for n in range(1, 5):
                L_[f"norm{n}"] = (_h(W(f"{p}.norm{n}"), dev), _h(Bv(f"{p}.norm{n}"), dev))
            self.layers.append(L_)
        fa = t + ".final_attn_token_to_image"
        wq, wk, wv = W(fa + ".q_proj"), W(fa + ".k_proj"), W(fa + ".v_proj")
        self.fin_q = (_h(torch.cat([wq, wq], 1), dev), _h(Bv(fa + ".q_proj"), dev))
        self.fin_img = (_h(torch.cat([wk, wv]), dev), _h(torch.cat([Bv(fa + ".k_proj"), Bv(fa + ".v_proj")]), dev))
        self.fin_pe = _h(torch.cat([pe @ wk.t(), torch.zeros(pe.shape[0], wv.shape[0])], 1), dev)
        self.fin_o = (_h(W(fa + ".out_proj"), dev), _h(Bv(fa + ".out_proj"), dev))
        self.norm_final = (_h(W(t + ".norm_final_attn"), dev), _h(Bv(t + ".norm_final_attn"), dev))
        self.out_tokens = torch.cat([sd["iou_token.weight"], sd["mask_tokens.weight"]]).to(dev)       # (5, 256) fp32
        # heads on every token row: layer 1 of the 4 hypernetworks and the IoU head side by side, layers 2 / 3
        # block-diagonal; output columns [hyper_0 | .. | hyper_3 | iou (4) | 0 (4)]
        hp = [f"output_hypernetworks_mlps.{i}.layers" for i in range(NUM_MASK_TOKENS)] + ["iou_prediction_head.layers"]
        self.head1 = (_h(torch.cat([W(f"{q}.0") for q in hp]), dev), _h(torch.cat([Bv(f"{q}.0") for q in hp]), dev))
        self.head2 = (_h(torch.block_diag(*[W(f"{q}.1") for q in hp]), dev), _h(torch.cat([Bv(f"{q}.1") for q in hp]), dev))
        w3 = torch.block_diag(*[W(f"{q}.2") for q in hp])
        b3 = torch.cat([Bv(f"{q}.2") for q in hp])
        pad = (-w3.shape[0]) % 8
        self.head3 = (_h(torch.cat([w3, w3.new_zeros(pad, w3.shape[1])]), dev), _h(torch.cat([b3, b3.new_zeros(pad)]), dev))
        self.head_n = self.head3[0].shape[0]
        self.iou_col = 32 * NUM_MASK_TOKENS
        u0 = sd["output_upscaling.0.weight"]                                     # [256 in, 64 out, 2, 2]
        self.up1 = (_h(u0.permute(2, 3, 1, 0).reshape(4 * 64, EMBED), dev), _h(sd["output_upscaling.0.bias"].repeat(4), dev))
        self.ln2d = (sd["output_upscaling.1.weight"].to(dev).contiguous(), sd["output_upscaling.1.bias"].to(dev).contiguous())
        self.up2 = (sd["output_upscaling.3.weight"].permute(2, 3, 0, 1).contiguous().to(dev),     # [ey, ex, c, o]
                    sd["output_upscaling.3.bias"].to(dev).contiguous())
        self._rep = {}

    def _repeat(self, name, t, B):
        """t [4096, N] repeated for B prompts (the per-pixel residual of a GEMM over B images), cached per B."""
        if B == 1:
            return t
        key = (name, B)
        if key not in self._rep:
            self._rep[key] = t.repeat(B, 1).contiguous()
        return self._rep[key]

    @staticmethod
    def _ln(x, wb):
        return ops.layernorm(x, wb[0], wb[1], eps=LN_EPS)

    def __call__(self, src: torch.Tensor, tokens_in: torch.Tensor, multimask_output: bool):
        """src (1, 4096, 256) fp16: image embedding + dense prompt embedding (channels-last); tokens_in (B, S, 256)
        fp32 sparse prompt embeddings -> (low-res logits (B, 3 | 1, 256, 256) fp32, iou (B, 3 | 1) fp32)."""
        dev = self.dev
        B = tokens_in.shape[0]
        T = NUM_MASK_TOKENS + 1 + tokens_in.shape[1]
        if T > MAX_TOKENS:
            raise ValueError(f"at most {MAX_TOKENS - 5} sparse prompt tokens per prompt")
        HW = IMG_EMB * IMG_EMB
        pe_tok = torch.cat([self.out_tokens[None].expand(B, -1, -1), tokens_in], dim=1).half().reshape(B * T, EMBED).contiguous()
        q = pe_tok
        keys = None                     # layer 0: src, shared by all prompts
        keys0 = src.expand(B, HW, EMBED).reshape(B * HW, EMBED)   # residual of layer 0's image-to-token update
        ws = ops.attention_small_ws(B, HEADS, T, HW, dev)
        bcast = [(b, b, 0, 0) for b in range(B)]
        for i, Lw in enumerate(self.layers):
            # self-attention (layer 0: no PE, queries replaced)
            if i == 0:
                qkv = ops.linear(q, Lw["sa_w"], bias=Lw["sa_b"])
            else:
                qkv = ops.linear(q, Lw["sa_w"], bias=Lw["sa_b"], extra=[(pe_tok, EMBED)])
            a = torch.empty((B * T, EMBED), dtype=torch.float16, device=dev)
            v3 = qkv.view(B, T, 3 * EMBED)
            ops.attention_small(v3, v3, v3, a.view(B, T, EMBED), HEADS, 32, T, T, 0, EMBED, 2 * EMBED, 0)
            q = ops.linear(a, *Lw["sa_o"], residual=None if i == 0 else q)
            q = self._ln(q, Lw["norm1"])
            # image-side projections of this block: [k_t2i | v_t2i | q_i2t] of keys + key_pe
            Bk = 1 if keys is None else B
            img = ops.linear(src.reshape(HW, EMBED) if keys is None else keys, Lw["img_w"], bias=Lw["img_b"],
                             residual=self._repeat(("img", i), Lw["img_pe"], Bk))
            img3 = img.view(Bk, HW, 3 * 128)
            # token -> image
            tq = ops.linear(q, Lw["ti_q"][0], bias=Lw["ti_q"][1], extra=[(pe_tok, EMBED)])
            a = torch.empty((B, T, 128), dtype=torch.float16, device=dev)
            ops.attention_small(tq.view(B, T, 128), img3, img3, a, HEADS, 16, T, HW, 0, 0, 128, 0, ws=ws,
                                items=bcast if keys is None else None)
            q = self._ln(ops.linear(a.view(B * T, 128), *Lw["ti_o"], residual=q), Lw["norm2"])
            # MLP
            h = ops.linear(q, *Lw["mlp1"], epilogue=L.EPI_RELU)
            q = self._ln(ops.linear(h, *Lw["mlp2"], residual=q), Lw["norm3"])
            # image -> token: queries = image tokens (short side: the prompt's T tokens)
            kv = ops.linear(q, Lw["it_kv"][0], bias=Lw["it_kv"][1], extra=[(pe_tok, EMBED)]).view(B, T, 256)
            a = torch.empty((B, HW, 128), dtype=torch.float16, device=dev)
            ops.attention_small(img3, kv, kv, a, HEADS, 16, HW, T, 256, 0, 128, 0,
                                items=[(b, 0, b, b) for b in range(B)] if keys is None else None)
            keys = self._ln(ops.linear(a.view(B * HW, 128), *Lw["it_o"], residual=keys0 if i == 0 else keys), Lw["norm4"])
        # final token -> image attention
        img = ops.linear(keys, *self.fin_img, residual=self._repeat("fin", self.fin_pe, B)).view(B, HW, 256)
        tq = ops.linear(q, self.fin_q[0], bias=self.fin_q[1], extra=[(pe_tok, EMBED)])
        a = torch.empty((B, T, 128), dtype=torch.float16, device=dev)
        ops.attention_small(tq.view(B, T, 128), img, img, a, HEADS, 16, T, HW, 0, 0, 128, 0, ws=ws)
        q = self._ln(ops.linear(a.view(B * T, 128), *self.fin_o, residual=q), self.norm_final)
        # hypernetworks + IoU head on every token row (rows 1..4 / 0 are read)
        h = ops.linear(q, *self.head1, epilogue=L.EPI_RELU)
        h = ops.linear(h, *self.head2, epilogue=L.EPI_RELU)
        heads = ops.linear(h, *self.head3)                                          # (B * T, head_n)
        m0, M = (1, 3) if multimask_output else (0, 1)
        n = self.head_n
        hyper = torch.as_strided(heads, (B, M, 32), (T * n, n + 32, 1), heads.storage_offset() + (1 + m0) * n + m0 * 32)
        iou = heads.view(B, T, n)[:, 0, self.iou_col + m0:self.iou_col + m0 + M].float()
        up1 = ops.linear(keys, *self.up1)                                             # (B * 4096, (dy, dx, 64))
        low = ops.sam_mask_head(up1, self.ln2d[0], self.ln2d[1], self.up2[0], self.up2[1], hyper, M, eps=LN_EPS)
        return low, iou


class PackedEfficientViTSam:
    """EfficientViTSam (sam.py:195-241) on the kernels: image encoder, prompt encoder, mask decoder, postprocess."""
    mask_threshold: float = 0.0
    image_format: str = "RGB"

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", use_graph: bool = True):
        self.device = torch.device(device)
        enc_sd = {k: v for k, v in state_dict.items() if not k.startswith(("prompt_encoder.", "mask_decoder."))}
        self.image_encoder = PackedSamImageEncoder(enc_sd, device=device, use_graph=use_graph)
        self.prompt_encoder = PackedSamPromptEncoder(state_dict, device=device)
        self.mask_decoder = PackedSamMaskDecoder(state_dict, self.prompt_encoder.dense_pe_cl, device=device)
        self.image_size = (IMG_SIZE, IMG_SIZE)
        self.use_graph = use_graph
        self._no_mask = self.prompt_encoder.no_mask_embed.half().expand(1, IMG_EMB, IMG_EMB, EMBED).contiguous()

    def to(self, device):
        assert torch.device(device) == self.device or torch.device(device).type == self.device.type, "built for one device"
        return self

    def eval(self):
        return self

    def image_src(self, features: torch.Tensor) -> torch.Tensor:
        """(1, 256, 64, 64) image embedding -> (1, 4096, 256) fp16 decoder input src = embedding + dense prompt embedding
        (no_mask_embed: the same for every prompt without a mask)."""
        f = features.to(self.device, torch.float16).permute(0, 2, 3, 1).contiguous()
        return ops.axpy(f, self._no_mask, 1.0).view(1, IMG_EMB * IMG_EMB, EMBED)

    def postprocess_masks(self, masks, input_size, original_size, return_logits=True, return_mask=False):
        mask, logits = ops.sam_postprocess(masks.contiguous(), input_size, original_size, mid=self.image_size[0],
                                           threshold=self.mask_threshold, return_mask=return_mask,
                                           return_logits=return_logits)
        return logits if return_logits and not return_mask else (mask, logits)


REGISTERED_SAM_MODEL = {"xl0": "assets/checkpoints/sam/xl0.pt", "xl1": "assets/checkpoints/sam/xl1.pt"}


def load_state_dict_from_file(file: str) -> Dict[str, torch.Tensor]:
    """Like the reference's (src/efficientvit/models/utils/network.py:70-77): torch.load on CPU, unwrap "state_dict"."""
    ckpt = torch.load(os.path.realpath(os.path.expanduser(file)), map_location="cpu")
    return ckpt["state_dict"] if "state_dict" in ckpt else ckpt


def create_sam_model(name: str = "xl1", pretrained: bool = True, weight_url: Optional[str] = None,
                     state_dict: Optional[Dict[str, torch.Tensor]] = None, device="cuda") -> PackedEfficientViTSam:
    """sam_model_zoo.create_sam_model for the 1024-input zoo models (xl0, xl1; the image encoder's topology is read off the
    state dict).  `state_dict` short-circuits loading (synthetic weights)."""
    if name.split("-")[0] not in REGISTERED_SAM_MODEL:
        raise ValueError(f"Do not find {name} in the model zoo. List of models: {list(REGISTERED_SAM_MODEL)}")
    if state_dict is None:
        if not pretrained:
            raise ValueError("the packed model is built from weights: pretrained=False has nothing to pack")
        weight_url = weight_url or REGISTERED_SAM_MODEL.get(name)
        state_dict = load_state_dict_from_file(weight_url)
    return PackedEfficientViTSam(state_dict, device=device)


class EfficientViTSamPredictor:
    """EfficientViTSamPredictor (sam.py:244-459) on the packed model.  predict_torch replays one CUDA graph per prompt
    shape (prompt count, point count, box or not, multimask, return_logits, image size)."""

    def __init__(self, sam_model: PackedEfficientViTSam) -> None:
        self.model = sam_model
        self._graphs = {}
        self._src = None
        self.reset_image()

    @property
    def transform(self):
        return self

    @property
    def device(self):
        return self.model.device

    def reset_image(self) -> None:
        self.is_image_set = False
        self.features = None
        self.original_size = None
        self.input_size = None

    def apply_coords(self, coords: np.ndarray, im_size=None) -> np.ndarray:
        old_h, old_w = self.original_size
        new_h, new_w = self.input_size
        coords = np.array(coords, dtype=float, copy=True)
        coords[..., 0] = coords[..., 0] * (new_w / old_w)
        coords[..., 1] = coords[..., 1] * (new_h / old_h)
        return coords

    def apply_boxes(self, boxes: np.ndarray, im_size=None) -> np.ndarray:
        return self.apply_coords(np.asarray(boxes).reshape(-1, 2, 2)).reshape(-1, 4)

    def apply_boxes_torch(self, boxes: torch.Tensor, im_size=None) -> torch.Tensor:
        old_h, old_w = self.original_size
        new_h, new_w = self.input_size
        scale = torch.tensor([new_w / old_w, new_h / old_h] * 2, dtype=torch.float32, device=boxes.device)
        return boxes.float().reshape(-1, 4) * scale

    @staticmethod
    def get_preprocess_shape(oldh: int, oldw: int, long_side_length: int) -> Tuple[int, int]:
        scale = long_side_length * 1.0 / max(oldh, oldw)
        return int(oldh * scale + 0.5), int(oldw * scale + 0.5)

    def preprocess(self, image: np.ndarray) -> torch.Tensor:
        """SamResize (PIL bilinear - what torchvision's resize does on a PIL image - only when the long side != 1024),
        ToTensor, Normalize, SamPad (corner) -> (1, 3, 1024, 1024) fp32 on the device."""
        from PIL import Image
        size = self.model.image_size[1]
        h, w = image.shape[:2]
        if max(h, w) != size:
            nh, nw = self.get_preprocess_shape(h, w, size)
            image = np.array(Image.fromarray(np.ascontiguousarray(image)).resize((nw, nh), Image.BILINEAR))
        x = torch.from_numpy(np.array(image)).to(self.device).permute(2, 0, 1).float() / 255.0
        x = (x - torch.tensor(PIXEL_MEAN, device=self.device)[:, None, None]) / torch.tensor(PIXEL_STD, device=self.device)[:, None, None]
        return torch.nn.functional.pad(x, (0, size - x.shape[2], 0, size - x.shape[1])).unsqueeze(0)

    @torch.inference_mode()
    def set_image(self, image: np.ndarray, image_format: str = "RGB") -> None:
        assert image_format in ["RGB", "BGR"], f"image_format must be in ['RGB', 'BGR'], is {image_format}."
        if image_format != self.model.image_format:
            image = image[..., ::-1]
        self.reset_image()
        self.original_size = tuple(image.shape[:2])
        self.input_size = self.get_preprocess_shape(*self.original_size, long_side_length=self.model.image_size[0])
        self.features = self.model.image_encoder(self.preprocess(image))
        src = self.model.image_src(self.features)
        if self._src is None:
            self._src = torch.empty_like(src)
        self._src.copy_(src)     # a fixed buffer: the recorded CUDA graphs read the current image from here
        self.is_image_set = True

    def predict(self, point_coords=None, point_labels=None, box=None, mask_input=None, multimask_output: bool = True,
                return_logits: bool = False):
        """Masks for one prompt (points and / or a box in original-image pixels) -> numpy (masks (C, H, W),
        iou (C,), low-res logits (C, 256, 256))."""
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) before mask prediction.")
        if mask_input is not None:
            raise ValueError("mask_input is not supported")
        coords_t = labels_t = box_t = None
        if point_coords is not None:
            assert point_labels is not None, "point_labels must be supplied if point_coords is supplied."
            coords_t = torch.as_tensor(self.apply_coords(point_coords), dtype=torch.float, device=self.device)[None]
            labels_t = torch.as_tensor(point_labels, dtype=torch.int, device=self.device)[None]
        if box is not None:
            box_t = torch.as_tensor(self.apply_boxes(box), dtype=torch.float, device=self.device)[None]
        masks, iou, low = self.predict_torch(coords_t, labels_t, box_t, None, multimask_output, return_logits)
        return masks[0].cpu().numpy(), iou[0].cpu().numpy(), low[0].cpu().numpy()

    def _run(self, coords, labels, boxes, multimask_output, return_logits):
        sparse, _ = self.model.prompt_encoder(None if coords is None else (coords, labels), boxes)
        low, iou = self.model.mask_decoder(self._src, sparse, multimask_output)
        mask, logits = ops.sam_postprocess(low, self.input_size, self.original_size, mid=self.model.image_size[0],
                                           threshold=self.model.mask_threshold, return_mask=not return_logits,
                                           return_logits=return_logits)
        return (logits if return_logits else mask), iou, low

    @torch.inference_mode()
    def predict_torch(self, point_coords=None, point_labels=None, boxes=None, mask_input=None, multimask_output: bool = True,
                      return_logits: bool = False):
        """Batched prompts already in the 1024 input frame: point_coords (B, N, 2), point_labels (B, N), boxes (B, 4) ->
        device tensors (masks (B, C, H, W) bool, or fp32 logits with return_logits; iou (B, C); low-res (B, C, 256, 256))."""
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) before mask prediction.")
        if mask_input is not None:
            raise ValueError("mask_input is not supported")
        if point_coords is None and boxes is None:
            raise ValueError("give point and / or box prompts")
        dev = self.device
        coords = None if point_coords is None else point_coords.to(dev, torch.float32).reshape(-1, point_coords.shape[-2], 2)
        labels = None if point_labels is None else point_labels.to(dev, torch.int32).reshape(coords.shape[0], -1)
        boxes = None if boxes is None else boxes.to(dev, torch.float32).reshape(-1, 4)
        if not self.model.use_graph:
            return self._run(coords, labels, boxes, multimask_output, return_logits)
        key = (None if coords is None else tuple(coords.shape), None if boxes is None else tuple(boxes.shape),
               bool(multimask_output), bool(return_logits), self.original_size, self.input_size)
        ent = self._graphs.get(key)
        if ent is None:
            st = [None if t is None else t.clone() for t in (coords, labels, boxes)]
            self._run(*st, multimask_output, return_logits)          # eager warm-up: kernel attributes, allocator pools
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = self._run(*st, multimask_output, return_logits)
            ent = self._graphs[key] = (g, st, out)
        g, st, out = ent
        for s, t in zip(st, (coords, labels, boxes)):
            if s is not None:
                s.copy_(t)
        g.replay()
        return tuple(t.clone() for t in out)


# ------------------------------------------------------------------------------- original SAM (ViT-B / L / H)
# The segmenter of the reference's `--segment_type GroundingDINO` branch: segment_anything's `sam_model_registry` /
# `SamPredictor` on `sam_vit_h_4b8939.pth` (inference_lora.py:105,191-198).  The image encoder is omg_b200.sam_vit; the
# prompt encoder and mask decoder are the same segment_anything modules the EfficientViT-SAM path runs, with the same
# keys (`prompt_encoder.*`, `mask_decoder.*`).
class PackedSam(PackedEfficientViTSam):
    """segment_anything Sam (image encoder ViT, prompt encoder, mask decoder, postprocess) on the kernels.  Its
    pixel_mean / pixel_std are SAM's (0-255 scale) - the same normalisation as EfficientViT-SAM's ToTensor + Normalize."""

    pixel_mean = (123.675, 116.28, 103.53)
    pixel_std = (58.395, 57.12, 57.375)

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", use_graph: bool = True):
        from .sam_vit import PackedSamViTImageEncoder
        self.device = torch.device(device)
        self.image_encoder = PackedSamViTImageEncoder(state_dict, device=device, use_graph=use_graph)
        dec = {k: v.cpu() for k, v in state_dict.items() if k.startswith(("prompt_encoder.", "mask_decoder."))}
        self.prompt_encoder = PackedSamPromptEncoder(dec, device=device)      # packs from CPU tensors
        self.mask_decoder = PackedSamMaskDecoder(dec, self.prompt_encoder.dense_pe_cl, device=device)
        self.image_size = (IMG_SIZE, IMG_SIZE)
        self.use_graph = use_graph
        self._no_mask = self.prompt_encoder.no_mask_embed.half().expand(1, IMG_EMB, IMG_EMB, EMBED).contiguous()


def _build_sam(kind: str, checkpoint: Optional[str] = None, state_dict: Optional[Dict[str, torch.Tensor]] = None,
               device="cuda", use_graph: bool = True) -> PackedSam:
    from .sam_vit import topology_kind
    if state_dict is None:
        if checkpoint is None:
            raise ValueError("the packed model is built from weights: give checkpoint= (or state_dict=)")
        with open(checkpoint, "rb") as f:
            state_dict = torch.load(f, map_location="cpu")
    got = topology_kind(state_dict)
    if got != kind:
        raise ValueError(f"checkpoint is a SAM {got} image encoder, not the requested {kind}")
    return PackedSam(state_dict, device=device, use_graph=use_graph)


def build_sam_vit_h(checkpoint=None, **kw) -> PackedSam:
    return _build_sam("vit_h", checkpoint, **kw)


def build_sam_vit_l(checkpoint=None, **kw) -> PackedSam:
    return _build_sam("vit_l", checkpoint, **kw)


def build_sam_vit_b(checkpoint=None, **kw) -> PackedSam:
    return _build_sam("vit_b", checkpoint, **kw)


build_sam = build_sam_vit_h
sam_model_registry = {"default": build_sam_vit_h, "vit_h": build_sam_vit_h, "vit_l": build_sam_vit_l,
                      "vit_b": build_sam_vit_b}


class ResizeLongestSide:
    """segment_anything.utils.transforms.ResizeLongestSide [3P]: resize so the long side is target_length (PIL bilinear on
    uint8 HWC arrays), and map coordinates / boxes from the original frame into that frame."""

    def __init__(self, target_length: int) -> None:
        self.target_length = target_length

    @staticmethod
    def get_preprocess_shape(oldh: int, oldw: int, long_side_length: int) -> Tuple[int, int]:
        return EfficientViTSamPredictor.get_preprocess_shape(oldh, oldw, long_side_length)

    def apply_image(self, image: np.ndarray) -> np.ndarray:
        from PIL import Image
        h, w = self.get_preprocess_shape(image.shape[0], image.shape[1], self.target_length)
        return np.array(Image.fromarray(np.ascontiguousarray(image)).resize((w, h), Image.BILINEAR))

    def apply_coords(self, coords: np.ndarray, original_size) -> np.ndarray:
        old_h, old_w = original_size
        new_h, new_w = self.get_preprocess_shape(old_h, old_w, self.target_length)
        coords = np.array(coords, dtype=float, copy=True)
        coords[..., 0] = coords[..., 0] * (new_w / old_w)
        coords[..., 1] = coords[..., 1] * (new_h / old_h)
        return coords

    def apply_boxes(self, boxes: np.ndarray, original_size) -> np.ndarray:
        return self.apply_coords(np.asarray(boxes).reshape(-1, 2, 2), original_size).reshape(-1, 4)

    def apply_coords_torch(self, coords: torch.Tensor, original_size) -> torch.Tensor:
        old_h, old_w = original_size
        new_h, new_w = self.get_preprocess_shape(old_h, old_w, self.target_length)
        coords = coords.clone().float()
        coords[..., 0] = coords[..., 0] * (new_w / old_w)
        coords[..., 1] = coords[..., 1] * (new_h / old_h)
        return coords

    def apply_boxes_torch(self, boxes: torch.Tensor, original_size) -> torch.Tensor:
        return self.apply_coords_torch(boxes.reshape(-1, 2, 2), original_size).reshape(-1, 4)


class SamPredictor(EfficientViTSamPredictor):
    """segment_anything SamPredictor [3P] on the packed model: set_image / set_torch_image / predict / predict_torch /
    get_image_embedding / reset_image, with `transform` a ResizeLongestSide.  The machinery (prompt graphs,
    postprocess) is the EfficientViT-SAM predictor's; only segment_anything's surface differs."""

    def __init__(self, sam_model: PackedSam) -> None:
        super().__init__(sam_model)
        self._transform = ResizeLongestSide(sam_model.image_size[0])

    @property
    def transform(self):
        return self._transform

    def apply_coords(self, coords, im_size=None):
        return self.transform.apply_coords(coords, self.original_size if im_size is None else im_size)

    def apply_boxes(self, boxes, im_size=None):
        return self.transform.apply_boxes(boxes, self.original_size if im_size is None else im_size)

    def apply_boxes_torch(self, boxes, im_size=None):
        return self.transform.apply_boxes_torch(boxes, self.original_size if im_size is None else im_size)

    @torch.inference_mode()
    def set_image(self, image: np.ndarray, image_format: str = "RGB") -> None:
        assert image_format in ["RGB", "BGR"], f"image_format must be in ['RGB', 'BGR'], is {image_format}."
        if image_format != self.model.image_format:
            image = image[..., ::-1]
        input_image = self.transform.apply_image(image)
        x = torch.as_tensor(input_image, device=self.device).permute(2, 0, 1).contiguous()[None, :, :, :]
        self.set_torch_image(x, image.shape[:2])

    @torch.inference_mode()
    def set_torch_image(self, transformed_image: torch.Tensor, original_image_size) -> None:
        """(1, 3, H, W) image already resized so its long side is 1024 (0-255 values) -> normalise, pad, encode."""
        assert (len(transformed_image.shape) == 4 and transformed_image.shape[1] == 3
                and max(*transformed_image.shape[2:]) == self.model.image_size[0]), \
            f"set_torch_image input must be BCHW with long side {self.model.image_size[0]}."
        self.reset_image()
        self.original_size = tuple(original_image_size)
        self.input_size = tuple(transformed_image.shape[-2:])
        x = transformed_image.to(self.device, torch.float32)
        mean = torch.tensor(self.model.pixel_mean, device=self.device)[None, :, None, None]
        std = torch.tensor(self.model.pixel_std, device=self.device)[None, :, None, None]
        x = (x - mean) / std
        size = self.model.image_size[0]
        x = torch.nn.functional.pad(x, (0, size - x.shape[-1], 0, size - x.shape[-2]))
        self.features = self.model.image_encoder(x)
        src = self.model.image_src(self.features)
        if self._src is None:
            self._src = torch.empty_like(src)
        self._src.copy_(src)
        self.is_image_set = True

    def get_image_embedding(self) -> torch.Tensor:
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) to generate an embedding.")
        return self.features


def uses_original_sam(segment_type: str) -> bool:
    """`--segment_type GroundingDINO` prompts the original SAM (ViT-H); any other value keeps EfficientViT-SAM, as the
    reference's `else` branch does (inference_lora.py:191-198,276-283)."""
    return segment_type == "GroundingDINO"


def make_segmenter(segment_type: str, synthetic: bool, tiny: bool, efficientvit_checkpoint: str, sam_checkpoint: str):
    """The predictor the CLIs' --sam_boxes prompt: SamPredictor(build_sam(sam_checkpoint)) for GroundingDINO, else
    EfficientViTSamPredictor(xl1).  --synthetic: random-init weights (ViT-H-shaped, ViT-B-shaped with --tiny)."""
    from . import synthetic as syn
    if uses_original_sam(segment_type):
        if synthetic:
            kind = "vit_b" if tiny else "vit_h"
            model = sam_model_registry[kind](state_dict=syn.make_sam_vit_state_dict(kind, 0, device="cuda",
                                                                                     dtype=torch.float16))
        else:
            model = build_sam(checkpoint=sam_checkpoint)
        return SamPredictor(model)
    if synthetic:
        model = create_sam_model("xl1", state_dict=syn.make_sam_state_dict(0))
    else:
        model = create_sam_model("xl1", weight_url=efficientvit_checkpoint)
    return EfficientViTSamPredictor(model)


# ------------------------------------------------------------------------------------------------ CLI helpers
def parse_sam_boxes(spec: str) -> List[Optional[Tuple[float, float, float, float]]]:
    """--sam_boxes "x0,y0,x1,y1|...": one box per concept in stage-1 image pixels; an empty entry is None (that concept
    is skipped, as an empty detection is in the reference, inference_lora.py:117-125)."""
    out: List[Optional[Tuple[float, float, float, float]]] = []
    for entry in spec.split("|"):
        entry = entry.strip()
        if not entry:
            out.append(None)
            continue
        vals = [float(v) for v in entry.split(",")]
        if len(vals) != 4 or vals[2] <= vals[0] or vals[3] <= vals[1]:
            raise ValueError(f"--sam_boxes entry {entry!r}: expected x0,y0,x1,y1 with x1 > x0 and y1 > y0")
        out.append((vals[0], vals[1], vals[2], vals[3]))
    return out


def check_sam_flags(sam_boxes: str, mask_boxes: str, decoded: bool) -> None:
    """--sam_boxes prompts SAM on the decoded stage-1 image: it excludes --mask_boxes and needs a decoder."""
    if not sam_boxes:
        return
    if mask_boxes:
        raise SystemExit("--sam_boxes and --mask_boxes are exclusive: SAM masks from boxes, or the boxes as rectangles")
    if not decoded:
        raise SystemExit("--sam_boxes segments the decoded stage-1 image: pass --decode (with --synthetic: a "
                         "random-init VAE) or, for the LoRA CLI, --vae_fp16_safe")


def sam_region_masks(predictor, image, boxes) -> List[Optional[torch.Tensor]]:
    """One device bool mask (H, W) per box (None stays None) of the RGB image (PIL or HWC uint8): set_image once, then
    predict_torch(boxes, multimask_output=False) - the reference's predict_mask (inference_lora.py:91-126) for boxes."""
    predictor.set_image(np.asarray(image), image_format="RGB")
    idx = [i for i, b in enumerate(boxes) if b is not None]
    out: List[Optional[torch.Tensor]] = [None] * len(boxes)
    if idx:
        bt = torch.tensor([boxes[i] for i in idx], dtype=torch.float32, device=predictor.device)
        masks, _, _ = predictor.predict_torch(boxes=predictor.transform.apply_boxes_torch(bt, predictor.original_size),
                                              multimask_output=False)
        for j, i in enumerate(idx):
            out[i] = masks[j, 0]
    return out
