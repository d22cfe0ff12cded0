"""SDXL UNet / ControlNet executor over the C-ABI kernels.

Replaces `self.unet(...)`, `concept_models.unet(...)` and `self.controlnet(...)` of the reference loops
(src/pipelines/lora_pipeline.py:520-529,546-566,592-599; src/pipelines/instantid_pipeline.py:580-616,639-674).

Layout: activations channels-last fp16, (B,H,W,C) == (B*H*W tokens, C); latents enter/leave as (B,H,W,8) with
channels 4..7 zero.  Per UNet call the launch sequence is static, so it is captured once per variant in a CUDA graph
and replayed (no host work, no syncs inside a step).

What is hoisted out of the per-step path (all step-invariant in the reference too):
  * time / added-cond embeddings and every ResBlock's time_emb_proj: one GEMM table for all timesteps per call;
  * cross-attention K/V of the text (and IP-adapter image) tokens: once per call per context / LoRA set;
  * the ControlNet conditioning embedding of the (constant) condition image: once per call.
"""
import math
import os
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib as L
from . import ops
from .config import UNetConfig, lora_conv_target_names, lora_target_names, resnet_names, transformer_names


def _f16(t, dev):
    return t.to(device=dev, dtype=torch.float16).contiguous()


def timestep_embedding(t: torch.Tensor, dim: int) -> torch.Tensor:
    """diffusers Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0): [cos | sin], fp32."""
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    ang = t.float()[:, None] * freqs[None, :]
    return torch.cat([torch.cos(ang), torch.sin(ang)], dim=-1)


# (weight key suffix, LayerNorm) pairs whose LayerNorm is folded into the GEMM
LN_CONSUMERS = (("attn1.qkv", "norm1"), ("attn2.q", "norm2"), ("ff1", "norm3"))

# kernels executed through CUDA-graph replays (the C-ABI launch counter only sees direct launches; a capture counts
# once there and is not executed)
REPLAYED_LAUNCHES = [0]
CAPTURED_LAUNCHES = [0]


def total_kernel_launches() -> int:
    """Kernels of this library executed so far: direct launches + launches inside replayed graphs."""
    return L.launch_count() - CAPTURED_LAUNCHES[0] + REPLAYED_LAUNCHES[0]


def pack_conv_lora(cfg: UNetConfig, adapters, global_scale: float = 1.0, temb_off: Optional[Dict[str, int]] = None,
                   device=None) -> Dict[str, List[Tuple[torch.Tensor, torch.Tensor, int, int]]]:
    """The conv / time-embedding part of a LoRA set (a LoCon adapter: config.lora_conv_target_names), keyed by the
    packed weight it changes: `<resnet>.w1`, `<resnet>.w2` (conv2 and, behind its 9 * out columns, conv_shortcut),
    `down<i>.w`, `up<i>.w` and `temb_all.w` (every time_emb_proj, at its rows of the concatenation).

    adapters: list of (lora, adapter_weight), lora[path] = (A [r, in, k, k] | [r, in], B [out, r], alpha / r).
    Entry: (A [R, K] fp32 in the packed (ky, kx, c) column order, B [n, R] fp32 with  alpha / r * adapter_weight *
    global_scale  folded in, first row, first column) - the adapters of the set concatenated along R, so that
    dW[row0 : row0 + n, col0 : col0 + K] = B A  is their sum."""
    if temb_off is None:
        temb_off, off = {}, 0
        for name, cout in resnet_names(cfg):
            temb_off[name] = off
            off += cout
    out: Dict[str, List[Tuple[torch.Tensor, torch.Tensor, int, int]]] = {}
    for path, kind, _cin, cout, _k in lora_conv_target_names(cfg):
        As, Bs = [], []
        for lora, wgt in adapters:
            if path in lora:
                A, Bm, s = lora[path]
                A = A.to(device=device, dtype=torch.float32)
                As.append(ops.pack_conv3x3_weight(A) if A.dim() == 4 and A.shape[2] == 3 else A.flatten(1))
                Bs.append(Bm.to(device=device, dtype=torch.float32) * (s * wgt * global_scale))
        if not As:
            continue
        mod, leaf = path.rsplit(".", 1)
        p = path.split(".")
        if leaf == "time_emb_proj":
            key, row0, col0 = "temb_all.w", temb_off[mod], 0
        elif leaf == "conv":
            key, row0, col0 = ("down" if p[2] == "downsamplers" else "up") + p[1] + ".w", 0, 0
        else:
            key, row0, col0 = mod + (".w1" if leaf == "conv1" else ".w2"), 0, 9 * cout if leaf == "conv_shortcut" else 0
        out.setdefault(key, []).append((torch.cat(As, dim=0), torch.cat(Bs, dim=1), row0, col0))
    return out


def merge_conv_lora(w: torch.Tensor, entries) -> torch.Tensor:
    """Packed base weight [N, K] + the deltas of pack_conv_lora entries, summed in fp32 and rounded once."""
    wf = w.float().clone()
    for A, Bm, row0, col0 in entries:
        wf[row0:row0 + Bm.shape[0], col0:col0 + A.shape[1]] += Bm @ A
    return wf.to(w.dtype)


class PackedUNet:
    """Weights of one UNet (or ControlNet trunk) repacked for the kernels, resident in HBM as fp16."""

    def __init__(self, cfg: UNetConfig, state_dict: Dict[str, torch.Tensor], device="cuda", controlnet: bool = False):
        self.cfg, self.device, self.controlnet = cfg, torch.device(device), controlnet
        sd = state_dict
        dev = self.device
        self.p: Dict[str, torch.Tensor] = {}
        P = self.p

        def conv_w(name, pad_in=0, pad_out=0):
            w = sd[name + ".weight"].to(dev, torch.float16)
            b = sd[name + ".bias"].to(dev, torch.float16)
            if pad_in:
                w = torch.cat([w, w.new_zeros(w.shape[0], pad_in, *w.shape[2:])], dim=1)
            if pad_out:
                w = torch.cat([w, w.new_zeros(pad_out, *w.shape[1:])], dim=0)
                b = torch.cat([b, b.new_zeros(pad_out)])
            if w.shape[2] == 3:
                w = ops.pack_conv3x3_weight(w)
            else:
                w = w.reshape(w.shape[0], w.shape[1]).contiguous()
            return w, b.contiguous()

        boc = cfg.block_out_channels
        P["conv_in.w"], P["conv_in.b"] = conv_w("conv_in", pad_in=8 - cfg.in_channels)
        for n in ("time_embedding.linear_1", "time_embedding.linear_2", "add_embedding.linear_1",
                  "add_embedding.linear_2"):
            P[n + ".w"], P[n + ".b"] = _f16(sd[n + ".weight"], dev), _f16(sd[n + ".bias"], dev)
        # every ResBlock's time_emb_proj concatenated: one GEMM produces all of them for all timesteps
        self.res_names = resnet_names(cfg, controlnet)
        self.temb_off: Dict[str, int] = {}
        tw, tb, off = [], [], 0
        for name, cout in self.res_names:
            self.temb_off[name] = off
            tw.append(sd[name + ".time_emb_proj.weight"])
            tb.append(sd[name + ".time_emb_proj.bias"])
            off += cout
        self.temb_cols = off
        P["temb_all.w"] = _f16(torch.cat(tw, dim=0), dev)
        P["temb_all.b"] = _f16(torch.cat(tb, dim=0), dev)
        for name, cout in self.res_names:
            cin = sd[name + ".conv1.weight"].shape[1]
            P[name + ".g1"], P[name + ".b1"] = _f16(sd[name + ".norm1.weight"], dev), _f16(sd[name + ".norm1.bias"], dev)
            P[name + ".g2"], P[name + ".b2"] = _f16(sd[name + ".norm2.weight"], dev), _f16(sd[name + ".norm2.bias"], dev)
            P[name + ".w1"], P[name + ".bias1"] = conv_w(name + ".conv1")
            w2, b2 = conv_w(name + ".conv2")
            if (name + ".conv_shortcut.weight") in sd:
                ws, bs = conv_w(name + ".conv_shortcut")
                w2 = torch.cat([w2, ws], dim=1).contiguous()
                b2 = (b2.float() + bs.float()).half()
            P[name + ".w2"], P[name + ".bias2"] = w2, b2
        self.tr_names = transformer_names(cfg, controlnet)
        for name, ch, layers in self.tr_names:
            P[name + ".norm.g"], P[name + ".norm.b"] = _f16(sd[name + ".norm.weight"], dev), _f16(sd[name + ".norm.bias"], dev)
            for lin in ("proj_in", "proj_out"):
                P[f"{name}.{lin}.w"], P[f"{name}.{lin}.b"] = _f16(sd[f"{name}.{lin}.weight"], dev), _f16(sd[f"{name}.{lin}.bias"], dev)
            for k in range(layers):
                b = f"{name}.transformer_blocks.{k}"
                for m in ("norm1", "norm2", "norm3"):
                    P[f"{b}.{m}.g"], P[f"{b}.{m}.b"] = _f16(sd[f"{b}.{m}.weight"], dev), _f16(sd[f"{b}.{m}.bias"], dev)
                P[f"{b}.attn1.qkv.w"] = _f16(torch.cat([sd[f"{b}.attn1.to_q.weight"], sd[f"{b}.attn1.to_k.weight"],
                                                        sd[f"{b}.attn1.to_v.weight"]], dim=0), dev)
                P[f"{b}.attn2.q.w"] = _f16(sd[f"{b}.attn2.to_q.weight"], dev)
                P[f"{b}.attn2.kv.w"] = _f16(torch.cat([sd[f"{b}.attn2.to_k.weight"], sd[f"{b}.attn2.to_v.weight"]],
                                                      dim=0), dev)
                for a in ("attn1", "attn2"):
                    P[f"{b}.{a}.out.w"], P[f"{b}.{a}.out.b"] = _f16(sd[f"{b}.{a}.to_out.0.weight"], dev), _f16(sd[f"{b}.{a}.to_out.0.bias"], dev)
                wi, bi = ops.pack_geglu_weight(sd[f"{b}.ff.net.0.proj.weight"], sd[f"{b}.ff.net.0.proj.bias"])
                P[f"{b}.ff1.w"], P[f"{b}.ff1.b"] = _f16(wi, dev), _f16(bi, dev)
                P[f"{b}.ff2.w"], P[f"{b}.ff2.b"] = _f16(sd[f"{b}.ff.net.2.weight"], dev), _f16(sd[f"{b}.ff.net.2.bias"], dev)
                # LayerNorm folded into the consuming GEMM: W' = W diag(gamma) (fp16), c1 = row sums of the ROUNDED
                # W' (so that the mean term cancels exactly in fp32), c2 = W beta + bias
                for key, norm in LN_CONSUMERS:
                    w = P[f"{b}.{key}.w"].float()
                    gam, bet = P[f"{b}.{norm}.g"].float(), P[f"{b}.{norm}.b"].float()
                    wl = (w * gam[None, :]).half()
                    P[f"{b}.{key}.lnw"] = wl
                    P[f"{b}.{key}.c1"] = wl.float().sum(dim=1).contiguous()
                    c2 = w @ bet
                    if f"{b}.{key}.b" in P:
                        c2 = c2 + P[f"{b}.{key}.b"].float()
                    P[f"{b}.{key}.c2"] = c2.contiguous()
        nb = len(boc)
        for i in range(nb - 1):
            P[f"down{i}.w"], P[f"down{i}.b"] = conv_w(f"down_blocks.{i}.downsamplers.0.conv")
        if controlnet:
            cec = cfg.cond_embed_channels
            P["cond.conv_in.w"], P["cond.conv_in.b"] = conv_w("controlnet_cond_embedding.conv_in", pad_in=5)
            for i in range(2 * (len(cec) - 1)):
                P[f"cond.{i}.w"], P[f"cond.{i}.b"] = conv_w(f"controlnet_cond_embedding.blocks.{i}")
            P["cond.conv_out.w"], P["cond.conv_out.b"] = conv_w("controlnet_cond_embedding.conv_out")
            self.n_skips = 1 + nb * cfg.layers_per_block + (nb - 1)
            for i in range(self.n_skips):
                P[f"zero{i}.w"], P[f"zero{i}.b"] = conv_w(f"controlnet_down_blocks.{i}")
            P["zero_mid.w"], P["zero_mid.b"] = conv_w("controlnet_mid_block")
        else:
            for i in range(nb - 1):
                P[f"up{i}.w"], P[f"up{i}.b"] = conv_w(f"up_blocks.{i}.upsamplers.0.conv")
            P["norm_out.g"], P["norm_out.b"] = _f16(sd["conv_norm_out.weight"], dev), _f16(sd["conv_norm_out.bias"], dev)
            P["conv_out.w"], P["conv_out.b"] = conv_w("conv_out", pad_out=8 - cfg.out_channels)
        # LoRA sets: key -> {linear key -> (A_cat [R, in], B2 [N, R])}; IP-adapter weights
        self.lora_sets: Dict[str, Dict[str, Tuple[torch.Tensor, torch.Tensor]]] = {}
        self.ip: Optional[Dict[str, torch.Tensor]] = None
        self.ip_scale, self.ip_tokens = 1.0, 16
        # bumped whenever something a captured CUDA graph may have baked in changes (LoRA sets, IP-adapter weights,
        # the IP scale scalar): runners drop their graphs when they see a new version
        self.adapter_version = 0
        # bumped when a LoRA set is added or replaced: runners drop their merged weight planes
        self.lora_version = 0

    # ------------------------------------------------------------------------------------------- adapters
    def add_lora_set(self, key: str, adapters, global_scale: float = 1.0):
        """Register a set of simultaneously active adapters (peft `set_adapters(names, adapter_weights)` +
        `cross_attention_kwargs={'scale': s}`; src/pipelines/lora_pipeline.py:588-596).

        adapters: list of (lora, adapter_weight); lora maps the diffusers Linear path to (A [r,in], B [out,r],
        alpha/r).  The delta stays un-merged: t = A_cat x is one skinny GEMM, s*B is a second weight matrix whose
        columns become extra K-segments of the main GEMM.  The conv / time-embedding modules of a LoCon adapter
        (pack_conv_lora) are kept beside them under the key of the packed weight they change; runners always merge
        those into per-stream weights."""
        dev = self.device
        packed: Dict[str, Tuple[torch.Tensor, torch.Tensor]] = {}

        def cat_adapters(name):
            As, Bs = [], []
            for lora, wgt in adapters:
                if name in lora:
                    A, Bm, s = lora[name]
                    As.append(A.float())
                    Bs.append(Bm.float() * (s * wgt * global_scale))
            if not As:
                return None
            return torch.cat(As, dim=0), torch.cat(Bs, dim=1)

        def put(key_out, parts, geglu=False):
            """parts: list of (A_cat [R_i,in], B [N_i,R_i]) for row blocks of a fused weight.  The summed rank is padded
            to a multiple of 8 with zero rows of A and zero columns of B2 (exact): t = A x is a GEMM output with r_tot
            channels and B2 a weight matrix with r_tot columns, and omg_gemm takes both only in multiples of 8."""
            if all(p is None for p in parts["ab"]):
                return
            As, rows = [], []
            r_off = 0
            r_sum = sum(0 if ab is None else ab[0].shape[0] for ab in parts["ab"])
            r_tot = (r_sum + 7) // 8 * 8
            dev0 = next(ab[0].device for ab in parts["ab"] if ab is not None)
            for ab, n_rows in zip(parts["ab"], parts["rows"]):
                blk = torch.zeros(n_rows, r_tot, device=dev0)
                if ab is not None:
                    A, Bm = ab
                    As.append(A)
                    blk[:, r_off:r_off + A.shape[0]] = Bm
                    r_off += A.shape[0]
                rows.append(blk)
            if r_tot > r_sum:
                As.append(As[0].new_zeros(r_tot - r_sum, As[0].shape[1]))
            B2 = torch.cat(rows, dim=0)
            if geglu:
                B2, _ = ops.pack_geglu_weight(B2)
            a_cat = torch.cat(As, dim=0)
            entry = [_f16(a_cat, dev), _f16(B2, dev), None, None, None]
            norm = next((n for k, n in LN_CONSUMERS if key_out.endswith("." + k)), None)
            if norm is not None:  # A' = A diag(gamma); c1_A = row sums of rounded A'; c2_A = A beta
                blk = key_out[: key_out.rfind(".transformer_blocks.")] + key_out[key_out.rfind(".transformer_blocks."):].split(".attn")[0].split(".ff1")[0]
                gam, bet = self.p[f"{blk}.{norm}.g"].float(), self.p[f"{blk}.{norm}.b"].float()
                a_ln = (a_cat.to(dev).float() * gam[None, :]).half()
                entry[2] = a_ln.contiguous()
                entry[3] = a_ln.float().sum(dim=1)
                entry[4] = a_cat.to(dev).float() @ bet
            packed[key_out] = tuple(entry)

        for name, ch, layers in self.tr_names:
            for lin in ("proj_in", "proj_out"):
                put(f"{name}.{lin}", {"ab": [cat_adapters(f"{name}.{lin}")], "rows": [ch]})
            for k in range(layers):
                b = f"{name}.transformer_blocks.{k}"
                put(f"{b}.attn1.qkv", {"ab": [cat_adapters(f"{b}.attn1.to_{x}") for x in "qkv"], "rows": [ch] * 3})
                put(f"{b}.attn2.q", {"ab": [cat_adapters(f"{b}.attn2.to_q")], "rows": [ch]})
                put(f"{b}.attn2.kv", {"ab": [cat_adapters(f"{b}.attn2.to_{x}") for x in "kv"], "rows": [ch] * 2})
                for a in ("attn1", "attn2"):
                    put(f"{b}.{a}.out", {"ab": [cat_adapters(f"{b}.{a}.to_out.0")], "rows": [ch]})
                put(f"{b}.ff1", {"ab": [cat_adapters(f"{b}.ff.net.0.proj")], "rows": [8 * ch]}, geglu=True)
                put(f"{b}.ff2", {"ab": [cat_adapters(f"{b}.ff.net.2")], "rows": [ch]})
        known = set()
        for lora, _ in adapters:
            known |= set(lora.keys())
        conv_names = set() if self.controlnet else {t[0] for t in lora_conv_target_names(self.cfg)}
        unsupported = known - {n for n, _, _ in lora_target_names(self.cfg)} - conv_names
        if unsupported:
            raise ValueError("LoRA targets outside the UNet's transformer Linears, ResBlocks and down- / up-samplers are "
                             f"not supported: {sorted(unsupported)[:4]}…")
        packed.update(pack_conv_lora(self.cfg, adapters, global_scale, self.temb_off, dev))
        self.lora_sets[key] = packed
        self.adapter_version += 1
        self.lora_version += 1

    def set_ip_adapter(self, ip_weights: Dict[str, Tuple[torch.Tensor, torch.Tensor]], scale: float = 1.0,
                       num_tokens: int = 16):
        """IPAttnProcessor weights (src/ip_adapter/attention_processor.py:107-108): attn2 path -> (to_k_ip, to_v_ip)."""
        self.ip = {k: _f16(torch.cat([wk, wv], dim=0), self.device) for k, (wk, wv) in ip_weights.items()}
        self.ip_scale, self.ip_tokens = float(scale), int(num_tokens)
        self.adapter_version += 1

    def set_ip_adapter_scale(self, scale: float):
        if float(scale) != self.ip_scale:
            self.ip_scale = float(scale)
            self.adapter_version += 1

    def num_attention_layers(self) -> int:
        return 2 * sum(layers for _, _, layers in self.tr_names)


class RowGroup:
    """A contiguous range of batch rows that shares one adapter configuration ("stream").  Several streams - the
    main UNet rows and every concept's rows - run through ONE launch sequence: the base weights are shared, each
    stream contributes its own LoRA K-segment (its block of t = A x is non-zero only on its rows), its own IP-adapter
    attention term and its own ControlNet residuals.  This is the parity-exact form of "one kernel computes every
    concept" (SURVEY section 7, step 8)."""

    def __init__(self, start: int, stop: int, lora_key: Optional[str] = None, ip: bool = False):
        self.start, self.stop, self.lora_key, self.ip = start, stop, lora_key, ip


class UNetRunner:
    """One (model, batch, latent size) execution context: preallocated activations, hoisted per-call tables,
    CUDA graphs per variant."""

    def __init__(self, model: PackedUNet, batch: int, H: int, W: int, lora_key: Optional[str] = None,
                 use_graphs: bool = True, groups: Optional[List[RowGroup]] = None, use_plans: bool = False):
        self.m, self.B, self.H, self.W = model, batch, H, W
        self.groups = groups or [RowGroup(0, batch, lora_key, model.ip is not None)]
        self._b2_cache: Dict[str, object] = {}
        # LayerNorm folded into the GEMM pairs (OMG_LN_FOLD=0: standalone LayerNorm kernel)
        self.ln_fold = os.environ.get("OMG_LN_FOLD", "1") != "0"
        # LoRA streams of a grouped launch use per-stream merged weight planes (OMG_LORA=unmerged: K-segment path)
        self.merge_lora = os.environ.get("OMG_LORA", "merged") != "unmerged"
        # GroupNorm statistics come out of the producing conv / GEMM epilogue (OMG_GN_FUSE=0: statistics pass per norm)
        self.gn_fuse = os.environ.get("OMG_GN_FUSE", "1") != "0"
        # fp32 master copy of the residual trunk (every tensor that is later a residual addend has an fp32 twin, written
        # by the GEMM that produces it): rounding to fp16 no longer accumulates over the ~70 blocks.  Opt-in
        # (OMG_TRUNK_F32=1 / pipe.trunk_f32 = True): final latents of config 2 move from 1.53e-3 to 1.17e-3 of the fp32
        # oracle, the forward gets 10 % slower (per-thread 128 B fp32 rows in the epilogues of the 210 residual GEMMs)
        self.trunk_f32 = os.environ.get("OMG_TRUNK_F32", "0") == "1"
        self.dev = model.device
        self.ws: Dict[str, torch.Tensor] = {}
        self.use_graphs = use_graphs
        # use_plans (with use_graphs=False): every forward variant is recorded once as a C-ABI launch plan (omg_plan) and
        # replayed from C - the executor a host without CUDA-graph plumbing (or without Python) drives
        self.use_plans = use_plans and not use_graphs
        self.plans: Dict[tuple, "ops.LaunchPlan"] = {}
        self.graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self.graph_launches: Dict[tuple, int] = {}
        self.warm: set = set()
        self._out: Dict[tuple, object] = {}
        self._graph_version = model.adapter_version
        self._lora_version = model.lora_version
        self.temb_table = None
        self.kv: Dict[str, torch.Tensor] = {}
        self.kv_ip: Dict[str, torch.Tensor] = {}
        self.ctx_rows = batch
        self.sample_in = self.buf("sample_in", (batch, H, W, 8))
        self.sample_in.zero_()
        self.temb_step = self.buf("temb_step", (batch, model.temb_cols))
        self.cross_items: List[List[tuple]] = []
        self.cross_weights: List[float] = []
        self.cond_emb = None
        # one slot, or a list of slots, (9 skip residual tensors, mid residual, scale[, row0]) produced by ControlNet
        # runners; a slot is added to the batch rows [row0, row0 + residual batch)
        self.residuals_in = None
        self.stats_ws = torch.empty(batch * (10240 + 64 * 256), dtype=torch.float32, device=self.dev)

    # ------------------------------------------------------------------------------------------- buffers
    def drop_graphs(self):
        """Forget every captured graph / recorded launch plan (they hold raw device pointers and launch-time scalars)."""
        self.plans.clear()
        self.graphs.clear()
        self.graph_launches.clear()
        self.warm.clear()
        self._out.clear()

    def _alloc(self, name, shape, dtype, zero) -> torch.Tensor:
        t = self.ws.get(name)
        if t is None or tuple(t.shape) != tuple(shape):
            if t is not None and self.graphs:
                # a buffer a captured graph may point at is being replaced (e.g. the K/V rows change when a
                # controller is added to / removed from the same runner): the old graphs are stale
                self.drop_graphs()
            t = (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=self.dev)
            self.ws[name] = t
        return t

    def buf(self, name, shape) -> torch.Tensor:
        return self._alloc(name, shape, torch.float16, False)

    def zbuf(self, name, shape) -> torch.Tensor:
        return self._alloc(name, shape, torch.float16, True)

    def fbuf(self, name, shape) -> torch.Tensor:
        return self._alloc(name, shape, torch.float32, True)

    def _cs(self, t: torch.Tensor, W: int, H: int, launches: int = 1):
        """Column-statistics partials buffer for the GEMM output `t` over a per-image grid (W, H): the producing launch
        fills it, the consuming GroupNorm finds it as `t._cs` (no statistics pass over t)."""
        if not self.gn_fuse:
            return None
        rb = ops.colstats_blocks(W, H) * launches
        part = self._alloc(f"cs.{t.data_ptr()}", (t.shape[0], rb, t.shape[-1], 2), torch.float32, False)
        t._cs = part
        return part

    def _twin(self, t: torch.Tensor):
        """fp32 twin [pixels, C] of the trunk tensor `t`, found later as `t._f32`."""
        if not self.trunk_f32:
            return None
        tw = self._alloc(f"f32.{t.data_ptr()}", (t.numel() // t.shape[-1], t.shape[-1]), torch.float32, False)
        t._f32 = tw
        return tw

    def _res(self, x):
        """(fp16 residual, fp32 residual) arguments for a GEMM that adds the trunk tensor x."""
        tw = getattr(x, "_f32", None) if self.trunk_f32 else None
        return (None, tw) if tw is not None else (x, None)

    def _gn(self, x, gamma, beta, eps, silu, out, x2=None):
        p1 = getattr(x, "_cs", None)
        p2 = None if x2 is None else getattr(x2, "_cs", None)
        if self.gn_fuse and p1 is not None and (x2 is None or p2 is not None):
            return ops.groupnorm_apply(x, p1, gamma, beta, eps, silu, x2=x2, part2=p2, out=out, stats_ws=self.stats_ws)
        return ops.groupnorm(x, gamma, beta, eps, silu, x2=x2, out=out, stats_ws=self.stats_ws)

    def _ln_vectors(self, key, groups, n, active):
        """c1 / c2 planes of the folded LayerNorm for every row group: the LoRA delta  s B (A' x)  is linear in the
        raw input too, so a stream's LoRA simply shifts its plane by  B2 c1_A  /  B2 c2_A."""
        P = self.m.p
        sig = key + "|" + ",".join(f"{g.start}-{g.stop}:{g.lora_key}" for g in groups) + f"|{n}"
        hit = self._b2_cache.get("ln|" + sig)
        if hit is not None:
            return hit
        base = groups[0].start
        if not active:
            res = (P[key + ".c1"], P[key + ".c2"], [(groups[-1].stop - base) * n])
        else:
            lo = {id(g): e for g, e in active}
            c1s, c2s = [], []
            for g in groups:
                c1, c2 = P[key + ".c1"], P[key + ".c2"]
                e = lo.get(id(g))
                if e is not None:
                    c1 = c1 + e[1].float() @ e[3]
                    c2 = c2 + e[1].float() @ e[4]
                c1s.append(c1)
                c2s.append(c2)
            res = (torch.stack(c1s).contiguous(), torch.stack(c2s).contiguous(), [(g.stop - base) * n for g in groups])
        self._b2_cache["ln|" + sig] = res
        return res

    def _merged_planes(self, key, groups, active, folded):
        """[G*N, K] fp16 stack of per-stream weights (W, or W + s B_g A_g for LoRA streams) and, for LayerNorm
        consumers, the matching c1/c2 planes (gamma folded AFTER the merge, c1 from the rounded weights)."""
        P = self.m.p
        ck = "merged|" + key + "|" + ",".join(f"{g.start}-{g.stop}:{g.lora_key}" for g in groups) + f"|{folded}"
        hit = self._b2_cache.get(ck)
        if hit is not None:
            return hit
        lo = {id(g): e for g, e in active}
        w = P[key + ".w"].float()
        gam = bet = None
        if folded:
            norm = next(nm for k, nm in LN_CONSUMERS if key.endswith("." + k))
            blk = key[: -(len(next(k for k, nm in LN_CONSUMERS if key.endswith("." + k))) + 1)]
            gam, bet = P[f"{blk}.{norm}.g"].float(), P[f"{blk}.{norm}.b"].float()
        ws, c1s, c2s = [], [], []
        for g in groups:
            e = lo.get(id(g))
            wg = w if e is None else w + e[1].float() @ e[0].float()
            if folded:
                wl = (wg * gam[None, :]).half()
                c2 = wg @ bet
                if (key + ".b") in P:
                    c2 = c2 + P[key + ".b"].float()
                ws.append(wl)
                c1s.append(wl.float().sum(dim=1))
                c2s.append(c2)
            else:
                ws.append(wg.half())
        res = (torch.cat(ws, dim=0).contiguous(), torch.stack(c1s).contiguous() if folded else None,
               torch.stack(c2s).contiguous() if folded else None)
        self._b2_cache[ck] = res
        return res

    def _sync_lora(self):
        """A LoRA set was added or replaced since the merged weight planes were built: forget them."""
        if self._lora_version != self.m.lora_version:
            self._b2_cache.clear()
            self._lora_version = self.m.lora_version

    def _conv_planes(self, key):
        """Per-stream weights of the conv (or temb_all) weight `key` for this runner's row groups: None when no group's
        LoRA set changes it (the launch is then the plain one), else ([G * N, K] fp16 stack - plane g = W + dW_g merged in
        fp32 and rounded once, the base weight for streams without a delta - and the cumulative image counts)."""
        sets = self.m.lora_sets
        if not any(g.lora_key and key in sets[g.lora_key] for g in self.groups):
            return None
        ck = "conv|" + key + "|" + ",".join(f"{g.start}-{g.stop}:{g.lora_key}" for g in self.groups)
        hit = self._b2_cache.get(ck)
        if hit is None:
            w = self.m.p[key]
            planes = [merge_conv_lora(w, sets[g.lora_key][key]) if g.lora_key and key in sets[g.lora_key] else w
                      for g in self.groups]
            hit = (torch.cat(planes, dim=0).contiguous(), [g.stop - self.groups[0].start for g in self.groups])
            self._b2_cache[ck] = hit
        return hit

    def _conv(self, fn, key, x, shortcut=None, **kw):
        """fn = ops.conv3x3 | conv3x3_s2 | upsample2x_conv3x3 with the weight `key`.  Streams whose LoRA set has a conv
        delta for it get their own weight plane in the same launch; where planes are not used (OMG_LORA=unmerged, more
        than 8 streams) the conv runs once per stream over that stream's images with that stream's merged weight -
        images are independent in a conv and every other operand is a slice by image."""
        planes = self._conv_planes(key)
        if shortcut is not None:
            kw["shortcut"] = shortcut
        if planes is None:
            return fn(x, self.m.p[key], **kw)
        w, ends = planes
        if self.merge_lora and len(ends) <= 8:
            return fn(x, w, row_groups=ends, **kw)
        B, N = x.shape[0], w.shape[0] // len(ends)

        def rows(t, i0, i1):  # per-image (B, ...) or per-pixel [B * HW, C] operand -> the images [i0, i1)
            return t[i0 * (t.shape[0] // B):i1 * (t.shape[0] // B)]

        for gi, i1 in enumerate(ends):
            i0 = ends[gi - 1] if gi else 0
            kg = {k: (v if k == "bias" or not torch.is_tensor(v) else rows(v, i0, i1)) for k, v in kw.items()}
            if shortcut is not None:
                kg["shortcut"] = [(t[i0:i1], off) for t, off in shortcut]
            fn(x[i0:i1], w[gi * N:(gi + 1) * N], **kg)
        return kw["out"]

    def _lin(self, key, x2d, out, bias=None, residual=None, epilogue=L.EPI_NONE, groups=None, rows_per_item=None,
             stats_out=None, ln=None, colstats=None, residual_f32=None, out_f32=None):
        """Linear with the un-merged LoRA deltas of every row group: t[rows_g, cols_g] = x[rows_g] A_g^T (skinny
        GEMMs, the other blocks of t stay zero), then ONE GEMM over all rows whose extra K-segment is t against
        [s B_1 | s B_2 | ...].  ln = (row statistics, parts, channels): the input's LayerNorm is folded into this
        GEMM (weights pre-multiplied by gamma, mean / rstd applied in the epilogue); stats_out: emit the row statistics
        of this GEMM's output for the next folded LayerNorm."""
        P = self.m.p
        groups = self.groups if groups is None else groups
        active = [(g, self.m.lora_sets[g.lora_key][key]) for g in groups
                  if g.lora_key and key in self.m.lora_sets[g.lora_key]]
        M = x2d.shape[0]
        n = rows_per_item if rows_per_item is not None else M // (groups[-1].stop - groups[0].start)
        w, ln_arg = P[key + ".w"], None
        if ln is not None:
            stats, parts, dim = ln
            c1, c2, ends = self._ln_vectors(key, groups, n, active)
            w, bias = P[key + ".lnw"], None
            ln_arg = (stats, parts, M, 0, dim, 1e-5, c1, c2, ends)
        if not active:
            return ops.linear(x2d, w, bias=bias, residual=residual, out=out, epilogue=epilogue, stats_out=stats_out,
                              ln=ln_arg, colstats=colstats, residual_f32=residual_f32, out_f32=out_f32)
        base = groups[0].start
        ends = [(g.stop - base) * n for g in groups]
        if self.merge_lora and groups is self.groups and len(groups) <= 8 and all(e % 128 == 0 for e in ends[:-1]):
            # per-stream weight planes W_g = W + s B_g A_g (built once, resident in HBM): the grouped launch picks the
            # plane of the stream a tile belongs to, so the per-step path has no LoRA GEMMs or K-segments at all
            wm, c1m, c2m = self._merged_planes(key, groups, active, ln is not None)
            if ln is not None:
                ln_arg = (ln[0], ln[1], M, 0, ln[2], 1e-5, c1m, c2m, ends)
            return ops.linear(x2d, wm, bias=bias, residual=residual, out=out, epilogue=epilogue, stats_out=stats_out,
                              ln=ln_arg, row_groups=ends, colstats=colstats, residual_f32=residual_f32, out_f32=out_f32)
        a_idx = 2 if ln is not None else 0   # gamma-folded A for LayerNorm consumers
        r_tot = sum(e[0].shape[0] for _, e in active)
        sig = ",".join(f"{g.start}-{g.stop}:{e[0].shape[0]}" for g, e in active)
        t = self.zbuf(f"lora_t.{M}.{sig}", (M, r_tot))
        ck = key + "|" + sig + "|" + ",".join(g.lora_key for g, _ in active)
        b2 = self._b2_cache.get(ck)
        if b2 is None:
            b2 = torch.cat([e[1] for _, e in active], dim=1).contiguous() if len(active) > 1 else active[0][1][1]
            self._b2_cache[ck] = b2
        c0 = 0
        base = groups[0].start
        for g, e in active:
            r0, r1 = (g.start - base) * n, (g.stop - base) * n
            ops.linear(x2d[r0:r1], e[a_idx], out=t[r0:r1, c0:c0 + e[0].shape[0]])
            c0 += e[0].shape[0]
        return ops.linear(x2d, w, bias=bias, residual=residual, out=out, epilogue=epilogue, lora=(t, b2),
                          stats_out=stats_out, ln=ln_arg, colstats=colstats, residual_f32=residual_f32, out_f32=out_f32)

    # ------------------------------------------------------------------------------------------- per-call setup
    def set_conditioning(self, timesteps, ctx, text_embeds: torch.Tensor, time_ids: torch.Tensor,
                         extra_ctx: Optional[torch.Tensor] = None):
        """Hoisted, step-invariant work (see module docstring).  text_embeds / time_ids: one row per batch row.
        ctx: (rows, L, D) [text tokens, then IP tokens for IP streams], or a list of (ctx, lora_key, has_ip) segments
        (one per stream; K/V rows are numbered in list order); extra_ctx: further text rows of the FIRST segment
        (prompt-to-prompt mixed contexts)."""
        m, cfg, P, B = self.m, self.m.cfg, self.m.p, self.B
        dev = self.dev
        ts = torch.as_tensor(timesteps, dtype=torch.float32, device=dev).reshape(-1)
        T = ts.numel()
        t_sin = timestep_embedding(ts, cfg.block_out_channels[0]).half()
        e = ops.linear(t_sin, P["time_embedding.linear_1.w"], bias=P["time_embedding.linear_1.b"], epilogue=L.EPI_SILU)
        t_emb = ops.linear(e, P["time_embedding.linear_2.w"], bias=P["time_embedding.linear_2.b"])
        tid = timestep_embedding(time_ids.to(dev).reshape(-1), cfg.addition_time_embed_dim).reshape(B, -1)
        add_in = torch.cat([text_embeds.to(dev).float(), tid], dim=-1).half().contiguous()
        a = ops.linear(add_in, P["add_embedding.linear_1.w"], bias=P["add_embedding.linear_1.b"], epilogue=L.EPI_SILU)
        aug = ops.linear(a, P["add_embedding.linear_2.w"], bias=P["add_embedding.linear_2.b"])
        emb = t_emb.float()[:, None, :] + aug.float()[None, :, :]               # (T, B, 1280)
        act = torch.nn.functional.silu(emb).half().reshape(T * B, -1).contiguous()
        self._sync_lora()
        self.temb_table = ops.linear(act, P["temb_all.w"], bias=P["temb_all.b"]).reshape(T, B, m.temb_cols)
        planes = self._conv_planes("temb_all.w")
        if planes is not None:  # time_emb_proj LoRA: the rows of such a stream come from its merged temb_all plane
            act3 = act.view(T, B, -1)
            for gi, g in enumerate(self.groups):
                if g.lora_key and "temb_all.w" in m.lora_sets[g.lora_key]:
                    a_g = act3[:, g.start:g.stop].reshape(T * (g.stop - g.start), -1).contiguous()
                    t_g = ops.linear(a_g, planes[0][gi * m.temb_cols:(gi + 1) * m.temb_cols], bias=P["temb_all.b"])
                    self.temb_table[:, g.start:g.stop] = t_g.view(T, g.stop - g.start, m.temb_cols)
        self.set_context(ctx, extra_ctx)

    def set_context(self, ctx, extra_ctx: Optional[torch.Tensor] = None):
        """Project the cross-attention K/V of every attn2 layer once per call (they are step-invariant): text rows
        of every stream with that stream's LoRA [+ mixed rows]; IP-adapter image tokens of the IP streams."""
        m = self.m
        if torch.is_tensor(ctx):
            g0 = self.groups[0]
            ctx = [(ctx, g0.lora_key, g0.ip)]
        txts, segs, ips = [], [], []
        row = 0
        for i, (c, lora_key, has_ip) in enumerate(ctx):
            c = c.to(self.dev, torch.float16)
            n_ip = m.ip_tokens if has_ip else 0
            t = c[:, : c.shape[1] - n_ip]
            if i == 0 and extra_ctx is not None:
                t = torch.cat([t, extra_ctx.to(self.dev, torch.float16)], dim=0)
            txts.append(t)
            segs.append(RowGroup(row, row + t.shape[0], lora_key))
            if n_ip:
                ips.append(c[:, c.shape[1] - n_ip:])
            row += t.shape[0]
        txt = torch.cat(txts, dim=0).contiguous()
        self.ctx_txt, self.ctx_segs = txt, segs
        self.ctx_rows, self.ctx_len = txt.shape[0], txt.shape[1]
        txt2d = txt.reshape(-1, txt.shape[-1])
        ip = torch.cat(ips, dim=0).contiguous() if ips else None
        for name, ch, layers in m.tr_names:
            for k in range(layers):
                b = f"{name}.transformer_blocks.{k}"
                kv = self.buf(b + ".kv", (self.ctx_rows, self.ctx_len, 2 * ch))
                self._lin(b + ".attn2.kv", txt2d, kv.view(-1, 2 * ch), groups=segs, rows_per_item=self.ctx_len)
                self.kv[b] = kv
                if ip is not None:
                    kvi = self.buf(b + ".kv_ip", (ip.shape[0], ip.shape[1], 2 * ch))
                    ops.linear(ip.reshape(-1, ip.shape[-1]), m.ip[b + ".attn2"], out=kvi.view(-1, 2 * ch))
                    self.kv_ip[b] = kvi

    def update_context_rows(self, row0: int, rows: torch.Tensor):
        """Re-project K/V for the text context rows [row0, row0+n) of the first segment only (prompt-to-prompt mixed
        contexts that change with the step's alpha)."""
        m = self.m
        n = rows.shape[0]
        self.ctx_txt[row0:row0 + n].copy_(rows)
        x2d = self.ctx_txt[row0:row0 + n].reshape(-1, rows.shape[-1])
        seg = [RowGroup(0, n, self.ctx_segs[0].lora_key)]
        for name, ch, layers in m.tr_names:
            for k in range(layers):
                b = f"{name}.transformer_blocks.{k}"
                self._lin(b + ".attn2.kv", x2d, self.kv[b][row0:row0 + n].view(-1, 2 * ch), groups=seg,
                          rows_per_item=self.ctx_len)

    def set_controlnet_cond(self, cond: torch.Tensor):
        """ControlNet conditioning embedding of the (constant) condition image (B,3,Himg,Wimg) in [0,1]: conv stack
        of controlnet_cond_embedding [3P], run once per call."""
        m, P, cfg = self.m, self.m.p, self.m.cfg
        x = cond.to(self.dev, torch.float16).permute(0, 2, 3, 1)
        x = torch.cat([x, x.new_zeros(*x.shape[:3], 5)], dim=3).contiguous()
        h = self._silu(ops.conv3x3(x, P["cond.conv_in.w"], bias=P["cond.conv_in.b"]))
        for i in range(2 * (len(cfg.cond_embed_channels) - 1)):
            f = ops.conv3x3_s2 if i % 2 == 1 else ops.conv3x3
            h = self._silu(f(h, P[f"cond.{i}.w"], bias=P[f"cond.{i}.b"]))
        # persistent buffer: the captured ControlNet graph reads it through a raw pointer (conv_in's residual), so a
        # new condition image must land in the SAME memory
        Bc, Hc, Wc, _ = h.shape
        self.cond_emb = ops.conv3x3(h, P["cond.conv_out.w"], bias=P["cond.conv_out.b"],
                                    out=self.buf("cond_emb", (Bc, Hc, Wc, P["cond.conv_out.b"].shape[0])))

    @staticmethod
    def _silu(t):
        # once-per-call prologue (not on the per-step path)
        return torch.nn.functional.silu(t.float()).half()

    # ------------------------------------------------------------------------------------------- blocks
    def _resblock(self, name, x, skip=None):
        P, m = self.m.p, self.m
        B, H, W, C1 = x.shape
        C2 = 0 if skip is None else skip.shape[3]
        cout = P[name + ".bias1"].shape[0]
        a1 = self._gn(x, P[name + ".g1"], P[name + ".b1"], 1e-5, 1, self.buf(name + ".a1", (B, H, W, C1 + C2)), x2=skip)
        off = m.temb_off[name]
        h = self.buf(name + ".h", (B, H, W, cout))
        self._conv(ops.conv3x3, name + ".w1", a1, bias=P[name + ".bias1"], rowvec=self.temb_step[:, off:off + cout], out=h,
                   colstats=self._cs(h, W, H))
        a2 = self._gn(h, P[name + ".g2"], P[name + ".b2"], 1e-5, 1, self.buf(name + ".a2", (B, H, W, cout)))
        out = self.buf(name + ".out", (B, H, W, cout))
        cs = self._cs(out, W, H)
        if P[name + ".w2"].shape[1] > 9 * cout:
            sc = [(x, 9 * cout)] + ([(skip, 9 * cout + C1)] if skip is not None else [])
            return self._conv(ops.conv3x3, name + ".w2", a2, bias=P[name + ".bias2"], shortcut=sc, out=out, colstats=cs,
                              out_f32=self._twin(out))
        r16, r32 = self._res(x)
        return self._conv(ops.conv3x3, name + ".w2", a2, bias=P[name + ".bias2"], residual=r16, out=out, colstats=cs,
                          residual_f32=r32, out_f32=self._twin(out))

    def _transformer(self, name, ch, layers, x, variant):
        P, m = self.m.p, self.m
        B, H, W, _ = x.shape
        N = H * W
        M = B * N
        heads = ch // m.cfg.head_dim
        scale = m.cfg.head_dim ** -0.5
        n = self._gn(x, P[name + ".norm.g"], P[name + ".norm.b"], 1e-6, 0, self.buf(f"tr.n.{ch}.{N}", (B, H, W, ch)))
        h = self.buf(f"tr.h.{ch}.{N}", (M, ch))
        # LayerNorm fold: every GEMM that produces h also emits h's row statistics; the GEMMs that consume
        # LayerNorm(h) run on raw h.  Needs 128-row-aligned stream boundaries (tiles must not straddle streams).
        fold = self.ln_fold and (len(self.groups) == 1 or all(((g.stop - g.start) * N) % 128 == 0 for g in self.groups))
        stats = lnS = None
        if fold:
            parts = ops.gemm_plan(ch, L.EPI_NONE, M)[1]
            stats = self.fbuf(f"tr.rowstats.{ch}.{N}", (parts, M, 2))
            lnS = (stats, parts, ch)
        h32 = self._alloc(f"tr.h32.{ch}.{N}", (M, ch), torch.float32, False) if self.trunk_f32 else None
        hres = dict(residual=h) if h32 is None else dict(residual_f32=h32, out_f32=h32)   # h <- h + f(h), in place
        self._lin(name + ".proj_in", n.view(M, ch), h, bias=P[name + ".proj_in.b"], stats_out=stats, out_f32=h32)
        ln = self.buf(f"tr.ln.{ch}.{N}", (M, ch))
        qkv = self.buf(f"tr.qkv.{ch}.{N}", (B, N, 3 * ch))
        q = self.buf(f"tr.q.{ch}.{N}", (B, N, ch))
        o = self.buf(f"tr.o.{ch}.{N}", (B, N, ch))
        g = self.buf(f"tr.g.{ch}.{N}", (M, 4 * ch))
        self_replace = variant.get("self_replace", False) and N <= variant.get("self_threshold", 0)
        ident = [(b, b, b, b) for b in range(B)]
        self_items = variant["self_items"] if self_replace else ident

        def normed(b, norm):  # unfused path: materialise LayerNorm(h)
            if fold:
                return h
            return ops.layernorm(h, P[f"{b}.{norm}.g"], P[f"{b}.{norm}.b"], out=ln)

        for k in range(layers):
            b = f"{name}.transformer_blocks.{k}"
            self._lin(b + ".attn1.qkv", normed(b, "norm1"), qkv.view(M, 3 * ch), ln=lnS)
            ops.attention(qkv, qkv, qkv, o, heads, N, N, self_items, 0, ch, 2 * ch, scale=scale)
            self._lin(b + ".attn1.out", o.view(M, ch), h, bias=P[b + ".attn1.out.b"], stats_out=stats, **hres)
            self._lin(b + ".attn2.q", normed(b, "norm2"), q.view(M, ch), ln=lnS)
            kv = self.kv[b]
            for ti, (items, wgt) in enumerate(zip(variant["cross_items"], variant["cross_weights"])):
                ops.attention(q, kv, kv, o, heads, N, self.ctx_len, items, 0, 0, ch, scale=scale, out_weight=wgt,
                              accumulate=ti > 0)
            if variant.get("ip_items"):
                kvi = self.kv_ip[b]
                ops.attention(q, kvi, kvi, o, heads, N, m.ip_tokens, variant["ip_items"], 0, 0, ch, scale=scale,
                              out_weight=m.ip_scale, accumulate=True)
            self._lin(b + ".attn2.out", o.view(M, ch), h, bias=P[b + ".attn2.out.b"], stats_out=stats, **hres)
            self._lin(b + ".ff1", normed(b, "norm3"), g, bias=P[b + ".ff1.b"], epilogue=L.EPI_GEGLU, ln=lnS)
            self._lin(b + ".ff2", g, h, bias=P[b + ".ff2.b"], stats_out=stats, **hres)
        out = self.buf(name + ".out", (B, H, W, ch))
        # the [M, ch] GEMM walks 128-token tiles: its per-32-row partials are per-image partials iff N % 128 == 0
        cs = self._cs(out, N, 1) if N % 128 == 0 else None
        r16, r32 = self._res(x)
        self._lin(name + ".proj_out", h, out.view(M, ch), bias=P[name + ".proj_out.b"], residual=None if r16 is None else r16.view(M, ch),
                  colstats=cs, residual_f32=r32, out_f32=self._twin(out))
        return out

    def _encoder(self, h, variant):
        m, cfg, P = self.m, self.m.cfg, self.m.p
        skips = [h]
        nb = len(cfg.block_out_channels)
        for i in range(nb):
            ch, layers = cfg.block_out_channels[i], cfg.transformer_layers[i]
            for j in range(cfg.layers_per_block):
                h = self._resblock(f"down_blocks.{i}.resnets.{j}", h)
                if layers > 0:
                    h = self._transformer(f"down_blocks.{i}.attentions.{j}", ch, layers, h, variant)
                skips.append(h)
            if i < nb - 1:
                B, H, W, _ = h.shape
                d = self.buf(f"down{i}.out", (B, H // 2, W // 2, ch))
                h = self._conv(ops.conv3x3_s2, f"down{i}.w", h, bias=P[f"down{i}.b"], out=d, colstats=self._cs(d, W // 2, H // 2))
                skips.append(h)
        ch = cfg.block_out_channels[-1]
        h = self._resblock("mid_block.resnets.0", h)
        h = self._transformer("mid_block.attentions.0", ch, cfg.transformer_layers[-1], h, variant)
        h = self._resblock("mid_block.resnets.1", h)
        return h, skips

    def _forward_unet(self, variant):
        m, cfg, P = self.m, self.m.cfg, self.m.p
        B, H, W = self.B, self.H, self.W
        h = self.buf("conv_in.out", (B, H, W, cfg.block_out_channels[0]))
        ops.conv3x3(self.sample_in, P["conv_in.w"], bias=P["conv_in.b"], out=h, colstats=self._cs(h, W, H), out_f32=self._twin(h))
        h, skips = self._encoder(h, variant)
        if variant.get("residuals", False):
            # ControlNet outputs * conditioning_scale, added in place to the rows of the stream they belong to.  Several
            # slots may be active in one grouped forward: the main-pass ControlNet on rows 0-3 and the IdentityNet on
            # the concept rows (instantid_pipeline.py:574-616 and :639-674 run in the same step).
            slots = self.residuals_in if isinstance(self.residuals_in, list) else [self.residuals_in]
            for slot in slots:
                down_r, mid_r, r_scale = slot[:3]
                r0 = slot[3] if len(slot) > 3 else 0
                for sk, r in zip(skips + [h], list(down_r) + [mid_r]):
                    dst = sk[r0:r0 + r.shape[0]]
                    ops.axpy(dst, r, r_scale, out=dst)
                    sk._f32 = None   # the fp32 twin no longer matches (no later residual add reads these tensors)
                    part = getattr(sk, "_cs", None)
                    if part is not None:  # the producer's statistics no longer describe these images: recompute them
                        hw = sk.shape[1] * sk.shape[2]
                        if part.shape[1] == (hw + 31) // 32:
                            ops.colstats(dst, out=part[r0:r0 + r.shape[0]])
                        else:
                            sk._cs = None
        nb = len(cfg.block_out_channels)
        for i in range(nb):
            ch, layers = cfg.block_out_channels[nb - 1 - i], cfg.transformer_layers[nb - 1 - i]
            for j in range(cfg.layers_per_block + 1):
                h = self._resblock(f"up_blocks.{i}.resnets.{j}", h, skips.pop())
                if layers > 0:
                    h = self._transformer(f"up_blocks.{i}.attentions.{j}", ch, layers, h, variant)
            if i < nb - 1:
                Bh, Hh, Wh, _ = h.shape
                u = self.buf(f"up{i}.out", (Bh, 2 * Hh, 2 * Wh, ch))
                h = self._conv(ops.upsample2x_conv3x3, f"up{i}.w", h, bias=P[f"up{i}.b"], out=u, colstats=self._cs(u, Wh, Hh, launches=4))
        a = self._gn(h, P["norm_out.g"], P["norm_out.b"], 1e-5, 1, self.buf("norm_out", tuple(h.shape)))
        return ops.conv3x3(a, P["conv_out.w"], bias=P["conv_out.b"], out=self.buf("noise", (B, H, W, 8)))

    def _forward_controlnet(self, variant):
        m, cfg, P = self.m, self.m.cfg, self.m.p
        B, H, W = self.B, self.H, self.W
        c0 = cfg.block_out_channels[0]
        # sample = conv_in(sample) + cond_embedding: the embedding is the GEMM epilogue residual
        h = self.buf("conv_in.out", (B, H, W, c0))
        ops.conv3x3(self.sample_in, P["conv_in.w"], bias=P["conv_in.b"], residual=self.cond_emb, out=h,
                    colstats=self._cs(h, W, H), out_f32=self._twin(h))
        h, skips = self._encoder(h, variant)
        outs = []
        for i, s in enumerate(skips):
            Bs, Hs, Ws, Cs = s.shape
            o = self.buf(f"zero{i}.out", (Bs, Hs, Ws, Cs))
            ops.linear(s.view(-1, Cs), P[f"zero{i}.w"], bias=P[f"zero{i}.b"], out=o.view(-1, Cs))
            outs.append(o)
        Bs, Hs, Ws, Cs = h.shape
        mid = self.buf("zero_mid.out", (Bs, Hs, Ws, Cs))
        ops.linear(h.view(-1, Cs), P["zero_mid.w"], bias=P["zero_mid.b"], out=mid.view(-1, Cs))
        return outs, mid

    # ------------------------------------------------------------------------------------------- public
    def default_variant(self) -> dict:
        """Identity attention routing: K/V row == batch row; IP term for the rows of IP streams (IP K/V rows are
        numbered in stream order)."""
        ident = [(b, b, b, b) for b in range(self.B)]
        ip_items, n = [], 0
        for g in self.groups:
            if g.ip:
                for b in range(g.start, g.stop):
                    ip_items.append((b, b, n, n))
                    n += 1
        return {"self_replace": False, "self_threshold": 0, "self_items": ident, "cross_items": [ident],
                "cross_weights": [1.0], "residuals": False, "ip_items": ip_items}

    def forward(self, step_index: int, variant: Optional[dict] = None, key: Optional[tuple] = None):
        """Run one forward for the timestep `step_index` of the schedule given to set_conditioning.  The input is
        whatever self.sample_in holds; returns the (persistent) output buffer(s)."""
        variant = variant or self.default_variant()
        self._sync_lora()
        self.temb_step.copy_(self.temb_table[step_index])
        fn = self._forward_controlnet if self.m.controlnet else self._forward_unet
        if self.use_plans and key is not None:
            if self._graph_version != self.m.adapter_version:
                self.drop_graphs()
                self._graph_version = self.m.adapter_version
            if key in self.plans:
                self.plans[key].run()
                return self._out[key]
            if key not in self.warm:
                self.warm.add(key)
                self._out[key] = fn(variant)  # eager run: allocates the persistent buffers, builds the weight caches
                return self._out[key]
            plan = ops.LaunchPlan()
            with plan:
                self._out[key] = fn(variant)  # launches AND records
            self.plans[key] = plan
            return self._out[key]
        if not self.use_graphs or key is None:
            return fn(variant)
        if self._graph_version != self.m.adapter_version:  # adapters / IP scale changed since the graphs were captured
            self.drop_graphs()
            self._graph_version = self.m.adapter_version
        if key in self.graphs:
            self.graphs[key].replay()
            REPLAYED_LAUNCHES[0] += self.graph_launches[key]
            return self._out[key]
        if key not in self.warm:
            self.warm.add(key)
            self._out[key] = fn(variant)  # eager run: allocates buffers, sets kernel attributes
            return self._out[key]
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        n0 = L.launch_count()
        with torch.cuda.graph(g):
            self._out[key] = fn(variant)
        self.graph_launches[key] = L.launch_count() - n0
        CAPTURED_LAUNCHES[0] += self.graph_launches[key]
        self.graphs[key] = g
        g.replay()
        REPLAYED_LAUNCHES[0] += self.graph_launches[key]
        return self._out[key]
