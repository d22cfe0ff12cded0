"""The two-stage OMG denoising pipelines on the H100 kernels, behind the reference call surface.

  LoraMultiConceptPipeline        <- src/pipelines/lora_pipeline.py:154-681
  InstantidMultiConceptPipeline   <- src/pipelines/instantid_pipeline.py:157-767
  ConceptModels                   <- the `concept_models` object the reference passes in (a diffusers
                                     StableDiffusionXLPipeline with LoRA adapters, inference_lora.py:159-170, or
                                     InstantidSingleConceptPipeline with IP-adapter, instantid_single_pieline.py:159-243)

`__call__` keeps the reference keyword arguments (prompt=[[global, global], [(region, region_neg[, ref]), ...]],
negative_prompt, generator, guidance_scale, num_inference_steps, cross_attention_kwargs, controller,
concept_models, stage, region_masks, lora_list, styleL, image, height, width, output_type, ...).  Text encoders,
VAE, segmentation and face analysis sit outside the hot path (SURVEY section 8): prompts are turned into embeddings
by a pluggable `prompt_encoder`, `output_type="latent"` is native and image output needs a `vae_decoder`.

Per step (one iteration of lora_pipeline.py:485-632) the device executes: main UNet (CUDA graph) -> [concept
UNets (CUDA graphs)] -> omg_fuse_step (Euler on epsilon) or omg_solver_step (every other schedule of
omg_b200.scheduler).  No host sync happens inside the loop.  `pipe.scheduler` is any schedule of omg_b200.scheduler;
`from_pretrained` reads the checkpoint's scheduler/scheduler_config.json.
"""
import hashlib
import os
import sys
from dataclasses import dataclass
from typing import Callable, Dict, Optional, Tuple

import torch

from . import ops
from .config import UNetConfig
from .prompt_attention import AttentionReplace
from .scheduler import EulerDiscreteSchedule, _Schedule, load_scheduler
from .unet import PackedUNet, UNetRunner

FUSION_AFTER_STEP = 15  # `if i > 15 and stage == 2` (lora_pipeline.py:568)


@dataclass
class PipelineOutput:
    images: object


class SyntheticPromptEncoder:
    """Deterministic stand-in for the two CLIP text encoders (out of the hot path; no checkpoints offline):
    a prompt string maps to seeded N(0,1) (77, D) hidden states and a (P,) pooled vector."""

    def __init__(self, cfg: UNetConfig, ctx_len: int = 77):
        self.cfg, self.ctx_len = cfg, ctx_len

    def __call__(self, prompt: str, lora_scale=None):
        seed = int.from_bytes(hashlib.sha256(prompt.encode("utf-8")).digest()[:4], "little")
        g = torch.Generator().manual_seed(seed)
        return (torch.randn(self.ctx_len, self.cfg.cross_attention_dim, generator=g),
                torch.randn(self.cfg.pooled_dim, generator=g))


class ConceptModels:
    """Concept UNet + its adapters (what the reference reaches through `concept_models.unet`, `.set_adapters`,
    `.encode_prompt`, `._execution_device`, `.set_ip_adapter_scale`, `._encode_prompt_image_emb`)."""

    def __init__(self, unet: PackedUNet, prompt_encoder: Optional[Callable] = None):
        self.unet = unet
        self.prompt_encoder = prompt_encoder or SyntheticPromptEncoder(unet.cfg)
        self._loras: Dict[str, dict] = {}
        self._active: Tuple[Tuple[str, ...], Tuple[float, ...]] = ((), ())
        self.image_proj = None  # (state dict, heads, dim_head) of the Resampler

    @classmethod
    def from_pretrained(cls, pretrained_model, unet: Optional[PackedUNet] = None, prompt_encoder=None,
                        torch_dtype=torch.float16, variant: Optional[str] = "fp16", device="cuda", **_):
        """`StableDiffusionXLPipeline.from_pretrained(pretrained_model, torch_dtype=float16, variant="fp16")` /
        `InstantidSingleConceptPipeline.from_pretrained(...)` as the reference builds its concept pipeline
        (inference_lora.py:159, inference_instantid.py:206-210).  `unet=` shares already packed base weights (the
        reference loads the same checkpoint twice; the packed weights are immutable, so one copy serves both)."""
        unet, prompt_encoder = _load_base(pretrained_model, unet, prompt_encoder, torch_dtype, variant, device)
        return cls(unet, prompt_encoder=prompt_encoder)

    def to(self, device=None, *_, **__):
        return self

    @property
    def _execution_device(self):
        return self.unet.device

    def load_lora_weights(self, lora, adapter_name: str, weight_name: Optional[str] = None, **_):
        """lora: a checkpoint path (file, or directory + weight_name; kohya / SGM / diffusers key layouts, see
        omg_b200.checkpoints) as in inference_lora.py:163-169, or the converted dict Linear path -> (A [r,in],
        B [out,r], alpha/r)."""
        self._loras[adapter_name] = _resolve_lora(self, lora, adapter_name, weight_name)

    def set_adapters(self, adapter_names, adapter_weights=None):
        names = (adapter_names,) if isinstance(adapter_names, str) else tuple(adapter_names)
        weights = tuple(1.0 for _ in names) if adapter_weights is None else tuple(float(w) for w in adapter_weights)
        for n in names:
            if n not in self._loras:
                raise ValueError(f"Adapter name {n} not found")
        self._active = (names, weights)

    def active_lora_key(self, global_scale: float) -> str:
        names, weights = self._active
        key = "|".join(f"{n}:{w:g}" for n, w in zip(names, weights)) + f"@{global_scale:g}"
        if key not in self.unet.lora_sets:
            self.unet.add_lora_set(key, [(self._loras[n], w) for n, w in zip(names, weights)], global_scale)
        return key

    def encode_prompt(self, prompt, negative_prompt=None, lora_scale=None, **_):
        kw = {}
        if getattr(self.prompt_encoder, "supports_adapters", False):  # text-encoder LoRA of the active adapters
            kw["adapters"] = (*self._active, getattr(self, "text_encoder_loras", {}))
        pe, pp = self.prompt_encoder(prompt, lora_scale, **kw)
        if negative_prompt is None:  # SDXL force_zeros_for_empty_prompt [3P encode_prompt]: zeros, not encode("")
            ne, np_ = torch.zeros_like(pe), torch.zeros_like(pp)
        else:
            ne, np_ = self.prompt_encoder(negative_prompt, lora_scale, **kw)
        return pe[None], ne[None], pp[None], np_[None]

    # --- InstantID pieces (instantid_single_pieline.py:159-243) --------------------------------------------
    def load_ip_adapter_instantid(self, image_proj_sd, ip_weights: Optional[dict] = None, heads: int = 20,
                                  dim_head: int = 64, num_tokens: int = 16, scale: float = 0.5):
        """`load_ip_adapter_instantid(model_ckpt)` with the path of InstantID's ip-adapter.bin as in the reference
        (instantid_single_pieline.py:159-161), or the two converted dicts."""
        if isinstance(image_proj_sd, (str, os.PathLike)):
            from .checkpoints import load_ip_adapter
            image_proj_sd, ip_weights = load_ip_adapter(os.fspath(image_proj_sd), self.unet.cfg)
            image_proj_sd = {k: v.float().to(self.unet.device) for k, v in image_proj_sd.items()}
        self.image_proj = (image_proj_sd, heads, dim_head)
        self.unet.set_ip_adapter(ip_weights, scale, num_tokens)

    def set_ip_adapter_scale(self, scale: float):
        self.unet.set_ip_adapter_scale(scale)

    def _encode_prompt_image_emb(self, prompt_image_emb, device=None, dtype=None, do_classifier_free_guidance=True):
        from .resampler import resampler_forward
        emb = torch.as_tensor(prompt_image_emb, dtype=torch.float32).reshape(1, -1, 512)
        if do_classifier_free_guidance:
            emb = torch.cat([torch.zeros_like(emb), emb], dim=0)
        sd, heads, dim_head = self.image_proj
        return resampler_forward(sd, emb.to(next(iter(sd.values())).device), heads, dim_head)


def _load_base(pretrained_model, unet, prompt_encoder, torch_dtype, variant, device):
    """UNet weights (`<dir>/unet/diffusion_pytorch_model[.fp16].safetensors`) and the two CLIP towers of an SDXL
    diffusers checkout."""
    from . import checkpoints as ck
    if unet is None:
        unet = PackedUNet(UNetConfig.sdxl(), ck.load_unet_weights(os.fspath(pretrained_model), "unet", variant), device=device)
    if prompt_encoder is None:
        from .text import ClipPromptEncoder
        prompt_encoder = ClipPromptEncoder.from_pretrained(os.fspath(pretrained_model), device, torch_dtype)
    return unet, prompt_encoder


def load_controlnet(path, device="cuda", variant: Optional[str] = None) -> PackedUNet:
    """`ControlNetModel.from_pretrained(path, torch_dtype=float16)` (inference_lora.py:153,
    inference_instantid.py:196,205,219): a directory holding diffusion_pytorch_model[.fp16].safetensors."""
    from . import checkpoints as ck
    return PackedUNet(UNetConfig.sdxl(), ck.load_unet_weights(os.fspath(path), "", variant), device=device, controlnet=True)


def _resolve_lora(owner, lora, adapter_name: str, weight_name: Optional[str]):
    """Path -> converted UNet LoRA dict (the text-encoder part is kept on the owner for its prompt encoder)."""
    if not isinstance(lora, (str, os.PathLike)):
        return lora
    from .checkpoints import load_lora
    path = os.fspath(lora)
    if os.path.isdir(path):
        path = os.path.join(path, weight_name or "pytorch_lora_weights.safetensors")
    unet_lora, te_lora, skipped = load_lora(path, owner.unet.cfg, conv=True)
    if skipped:
        print(f"{adapter_name}: {len(skipped)} LoRA tensors of {path} target modules that are not adapted and are "
              f"ignored, e.g. {skipped[:3]}", file=sys.stderr)
    if not hasattr(owner, "text_encoder_loras"):
        owner.text_encoder_loras = {}
    owner.text_encoder_loras[adapter_name] = te_lora
    owner.skipped_lora_keys = skipped
    return unet_lora


def _binary_latent_mask(mask: Optional[torch.Tensor], h: int, w: int, device) -> Optional[torch.Tensor]:
    """mask.float() -> nearest resize to (h, w) -> (== 1) (lora_pipeline.py:350,578-580,602,674-681)."""
    if mask is None:
        return None
    m = torch.nn.functional.interpolate(mask[None, None].float(), size=(h, w), mode="nearest")[0, 0]
    return (m == 1).float().reshape(-1).contiguous().to(device)


class _BasePipeline:
    vae_scale_factor = 8

    def __init__(self, unet: PackedUNet, controlnet: Optional[PackedUNet] = None,
                 prompt_encoder: Optional[Callable] = None, vae_decoder: Optional[Callable] = None,
                 use_graphs: bool = True):
        self.unet, self.controlnet = unet, controlnet
        self.controlnet2: Optional[PackedUNet] = None
        self.prompt_encoder = prompt_encoder or SyntheticPromptEncoder(unet.cfg)
        self.vae_decoder = vae_decoder
        self.scheduler = EulerDiscreteSchedule()
        self.use_graphs = use_graphs
        # how a UNet forward is issued: "graph" (CUDA graphs, the default), "plan" (C-ABI launch plans, omg_plan: recorded
        # once, replayed from C - the executor for hosts without graph plumbing) or "eager"; OMG_EXECUTOR overrides
        self.executor = (os.environ.get("OMG_EXECUTOR") or "graph") if use_graphs else "eager"
        if self.executor not in ("graph", "plan", "eager"):
            raise ValueError(f"unknown executor {self.executor!r} (graph | plan | eager)")
        self.controller: Optional[AttentionReplace] = None
        self.main_lora_key: Optional[str] = None
        self._runners: Dict[tuple, UNetRunner] = {}
        self.timings: Dict[str, float] = {}
        # opt-in exact work de-duplication (SURVEY 8d "legal algebraic dedup"), off by default = as the reference executes
        self.dedup = False
        self._prefix: Optional[dict] = None
        self.sample_forwards = 0  # UNet sample-forwards executed by the last call (296 per image as-executed)
        # accuracy / speed switch: fp32 master copy of the UNet's residual trunk (see UNetRunner.trunk_f32); None = the
        # runner's default (OMG_TRUNK_F32)
        self.trunk_f32: Optional[bool] = None

    @classmethod
    def from_pretrained(cls, pretrained_model, controlnet=None, torch_dtype=torch.float16, variant: Optional[str] = "fp16",
                        device="cuda", unet: Optional[PackedUNet] = None, prompt_encoder=None, vae_decoder=None,
                        use_graphs: bool = True, **_):
        """`LoraMultiConceptPipeline.from_pretrained(pretrained_model, controlnet=controlnet, torch_dtype=float16,
        variant="fp16")` (inference_lora.py:154-155, inference_instantid.py:197-198).  controlnet: a PackedUNet, a
        checkpoint directory, or None.  The VAE is not loaded here: image output is opt-in through `vae_decoder=`
        (default output is latents), e.g. `PackedVaeDecoder.from_pretrained(pretrained_model)`, which decodes the
        checkpoint's own VAE in bf16 (the original SDXL VAE weights overflow fp16 activations)."""
        unet, prompt_encoder = _load_base(pretrained_model, unet, prompt_encoder, torch_dtype, variant, device)
        if isinstance(controlnet, (str, os.PathLike)):
            controlnet = load_controlnet(controlnet, device)
        pipe = cls(unet, controlnet=controlnet, prompt_encoder=prompt_encoder, vae_decoder=vae_decoder, use_graphs=use_graphs)
        pipe.scheduler = load_scheduler(pretrained_model)
        return pipe

    def to(self, device=None, *_, **__):
        return self

    @property
    def tokenizer(self):
        """`pipe.tokenizer` as the CLIs use it (inference_lora.py:156,277): the first CLIP tokenizer."""
        tok = getattr(self.prompt_encoder, "tokenizer", None)
        if tok is None:
            raise AttributeError("this pipeline's prompt encoder has no tokenizer (synthetic encoder)")
        return tok

    @property
    def _execution_device(self):
        return self.unet.device

    # ---------------------------------------------------------------------------------------------- helpers
    def _runner(self, tag, model: PackedUNet, batch, h, w, lora_key=None, groups=None, tag_extra=None) -> UNetRunner:
        key = (tag, id(model), batch, h, w, lora_key, tag_extra, self.trunk_f32)
        r = self._runners.get(key)
        if r is None:
            r = UNetRunner(model, batch, h, w, lora_key=lora_key, use_graphs=self.executor == "graph", groups=groups,
                           use_plans=self.executor == "plan")
            if self.trunk_f32 is not None:
                r.trunk_f32 = bool(self.trunk_f32)
            self._runners[key] = r
        return r

    def load_lora_weights(self, lora, adapter_name: str = "style", scale: float = 0.8,
                          weight_name: Optional[str] = None, **_):
        """Style LoRA on the main UNet (inference_lora.py:163; applied with cross_attention_kwargs scale 0.8); a
        checkpoint path or a converted dict."""
        lora = _resolve_lora(self, lora, adapter_name, weight_name)
        key = f"main:{adapter_name}@{scale:g}"
        self.unet.add_lora_set(key, [(lora, 1.0)], scale)
        self.main_lora_key = key

    def encode_prompt(self, prompt, negative_prompt, lora_scale=None):
        """-> prompt_embeds (n,77,D), negative (n,77,D), pooled (n,P), negative pooled (n,P) for a list of prompts."""
        prompts = [prompt] if isinstance(prompt, str) else list(prompt)
        negs = [negative_prompt] * len(prompts) if isinstance(negative_prompt, (str, type(None))) else list(negative_prompt)
        pe, pp, ne, np_ = [], [], [], []
        kw = {}
        if getattr(self.prompt_encoder, "supports_adapters", False) and getattr(self, "text_encoder_loras", None):
            names = tuple(self.text_encoder_loras)  # the style adapter's text-encoder part (inference_lora.py:163)
            kw["adapters"] = (names, tuple(1.0 for _ in names), self.text_encoder_loras)
        for p, n in zip(prompts, negs):
            e, pooled = self.prompt_encoder(p, lora_scale, **kw)
            if n is None:  # force_zeros_for_empty_prompt [3P]: a missing negative prompt is zeros, not encode("")
                e2, pooled2 = torch.zeros_like(e), torch.zeros_like(pooled)
            else:
                e2, pooled2 = self.prompt_encoder(n, lora_scale, **kw)
            pe.append(e), pp.append(pooled), ne.append(e2), np_.append(pooled2)
        return torch.stack(pe), torch.stack(ne), torch.stack(pp), torch.stack(np_)

    def prepare_latents(self, h, w, generator, latents, dtype=torch.float16):
        """randn((1,4,h,w), generator) * init_noise_sigma, then cat([l, l.clone()]) (lora_pipeline.py:397-409)."""
        dev = self._execution_device
        if latents is None:
            gdev = generator.device if generator is not None else dev
            latents = torch.randn((1, 4, h, w), generator=generator, device=gdev, dtype=dtype).to(dev)
        lat = latents.to(dev).float() * self.scheduler.init_noise_sigma
        lat = torch.cat([lat, lat.clone()])
        return lat.permute(0, 2, 3, 1).contiguous()  # (2, h, w, 4) fp32 channels-last state

    def _p2p_variant(self, runner: UNetRunner, controller: Optional[AttentionReplace], residuals: bool):
        """Edit specification of the main UNet (rows u0,u1,c0,c1) for the controller's current step."""
        v = runner.default_variant()
        v["residuals"] = residuals
        key = ("main", residuals)
        if controller is None:
            return v, key + (False,)
        v["self_replace"] = controller.self_window_active()
        v["self_threshold"] = controller.width * controller.height
        v["self_items"] = [(0, 0, 0, 0), (1, 1, 1, 1), (2, 2, 2, 2), (3, 2, 2, 3)]
        # cross: c1 = P(c0) . V(row 4 = M diag(alpha) ctx_1)  [+ P(c1) . V(row 5 = diag(1-alpha) ctx_1)]
        items0 = [(0, 0, 0, 0), (1, 1, 1, 1), (2, 2, 2, 2), (3, 2, 2, 4)]
        v["cross_items"], v["cross_weights"] = [items0], [1.0]
        two = self._cross_two_terms
        if two:
            v["cross_items"].append([(3, 3, 3, 5)])
            v["cross_weights"].append(1.0)
        return v, key + (True, v["self_replace"], two)

    def _update_p2p_context(self, runners, controller: AttentionReplace, ctx4: torch.Tensor, first: bool):
        """(Re)build the mixed context rows 4,5 when the step's alpha row differs from the previous step's."""
        if isinstance(runners, UNetRunner):
            runners = [runners]
        coef_base, coef_keep = controller.cross_edit()
        sig = (coef_base.numpy().tobytes(), None if coef_keep is None else coef_keep.numpy().tobytes())
        if not first and sig == self._p2p_sig:
            return
        self._p2p_sig = sig
        dev = self._execution_device
        c1 = ctx4[3:4].to(dev, torch.float16).contiguous()
        mix_a = ops.ctx_mix(c1, coef_base.to(dev).contiguous())
        if coef_keep is not None:
            mix_b = ops.ctx_mix(c1, coef_keep.to(dev).contiguous())
        else:
            mix_b = torch.zeros_like(c1)
        self._cross_two_terms = coef_keep is not None
        rows = torch.cat([mix_a, mix_b], dim=0)
        if first:
            self._p2p_rows = rows
        else:
            for r in runners:
                r.update_context_rows(4, rows)

    def _set_timesteps(self, num_inference_steps: int):
        if not isinstance(self.scheduler, _Schedule):
            raise ValueError(f"pipe.scheduler: {type(self.scheduler).__name__} is not supported; use a schedule of "
                             "omg_b200.scheduler (EulerDiscreteScheduler, EulerAncestralDiscreteScheduler, "
                             "DPMSolverMultistepScheduler)")
        return self.scheduler.set_timesteps(num_inference_steps)

    def _step_end(self, callback, i, t, lat, main, cbuf):
        """`callback_on_step_end(self, i, t, {"latents": latents})` (lora_pipeline.py:617-625): the callback sees the
        latents after the scheduler step as (2,4,h,w) and may return {"latents": replacement}.  A multistep schedule's
        history (the previous x0) is left as it is, as diffusers' scheduler keeps its own."""
        view = lat.permute(0, 3, 1, 2)
        given = view.clone()
        out = callback(self, i, t, {"latents": given})
        new = (out or {}).get("latents", given)
        if new is not given:
            lat.copy_(new.to(lat.device, lat.dtype).permute(0, 2, 3, 1))
            if i + 1 < len(self.scheduler.timesteps):  # next step's scaled inputs (the step wrote them from the old latents)
                x = (lat * self.scheduler.input_scale(i + 1)).half()
                main.sample_in[..., :4] = torch.cat([x, x], dim=0)
                cbuf[..., :4] = torch.cat([x[1:2], x[1:2]], dim=0)

    def _denoise(self, *, ts, lat, ctx4, pooled4, tid, concepts, masks, stage, guidance_scale, h, w, concept_unet,
                 main_cn=None, identity=None, callback=None, generator=None):
        """The step loop (lora_pipeline.py:485-632 / instantid_pipeline.py:540-690).

        concepts: list of dicts {ctx (2, L, D) [text tokens (+ IP tokens)], pooled (2, P), lora_key, ip (bool)};
        main_cn:  None or (ControlNet PackedUNet, condition image (4,3,H,W), scale, keep(i) -> 0/1) for the main rows;
        identity: None or (IdentityNet PackedUNet, condition image (2,3,H,W), scale, [face tokens (2,16,D) per concept]);
        generator: the call's generator; a stochastic schedule draws its per-step noise from it as diffusers'
                   randn_tensor does (on the generator's device; torch's global CUDA RNG when None).

        Steps without fusion run the main UNet alone (B=4).  Fusion steps (index > 15, stage 2) run ONE grouped
        forward: rows 0-3 = main stream, then two rows per active concept, every stream with its own LoRA segment /
        IP term / IdentityNet residuals - when the concept UNet shares the packed base weights with the main UNet
        (the reference's two pipelines load the same checkpoint, inference_lora.py:153-159); otherwise the concept
        streams run as separate forwards."""
        dev = self._execution_device
        sch = self.scheduler
        sig = sch.sigmas
        controller = self.controller
        active = [k for k in range(len(concepts)) if stage == 2 and masks[k] is not None]
        n_act = len(active)
        grouped = n_act > 0 and concept_unet is self.unet
        from .unet import RowGroup
        main = self._runner("main", self.unet, 4, h, w, groups=[RowGroup(0, 4, self.main_lora_key, False)])
        extra = None
        if controller is not None:
            self._update_p2p_context([], controller, ctx4, first=True)
            extra = self._p2p_rows
        main.set_conditioning(ts, ctx4, pooled4, tid.repeat(4, 1), extra_ctx=extra)
        p2p_runners = [main]
        fused, crun = None, []
        if grouped:
            groups = [RowGroup(0, 4, self.main_lora_key, False)]
            ctx_list = [(ctx4, self.main_lora_key, False)]
            for j, k in enumerate(active):
                c = concepts[k]
                groups.append(RowGroup(4 + 2 * j, 6 + 2 * j, c["lora_key"], c["ip"]))
                ctx_list.append((c["ctx"], c["lora_key"], c["ip"]))
            fused = self._runner("fused", self.unet, 4 + 2 * n_act, h, w, groups=groups,
                                 tag_extra=tuple((g.lora_key, g.ip) for g in groups))
            fused.set_conditioning(ts, ctx_list, torch.cat([pooled4.to(dev)] + [concepts[k]["pooled"].to(dev) for k in active]),
                                   tid.repeat(4 + 2 * n_act, 1), extra_ctx=extra)
            p2p_runners.append(fused)
        else:
            for k in active:
                c = concepts[k]
                r = self._runner(f"concept{k}", concept_unet, 2, h, w,
                                 groups=[RowGroup(0, 2, c["lora_key"], c["ip"])], tag_extra=(c["lora_key"], c["ip"]))
                r.set_conditioning(ts, c["ctx"], c["pooled"], tid.repeat(2, 1))
                crun.append(r)
        cn = None
        if main_cn is not None:
            cn_model, cn_cond, cn_scale, cn_keep = main_cn
            cn = self._runner("cn", cn_model, 4, h, w, groups=[RowGroup(0, 4, None, False)])
            cn.set_conditioning(ts, ctx4, pooled4, tid.repeat(4, 1))
            cn.set_controlnet_cond(cn_cond)
        idr = None
        if identity is not None and n_act > 0:
            id_model, id_cond, id_scale, id_tokens = identity
            idr = self._runner("identity", id_model, 2 * n_act, h, w, groups=[RowGroup(0, 2 * n_act, None, False)])
            idr.set_conditioning(ts, torch.cat([id_tokens[k].to(dev) for k in active]),
                                 torch.cat([concepts[k]["pooled"].to(dev) for k in active]), tid.repeat(2 * n_act, 1))
            idr.set_controlnet_cond(id_cond.repeat(n_act, 1, 1, 1))
        # initial model inputs: scale_model_input(cat([latents]*2), t0)  (:491-492)
        x0 = (lat * self.scheduler.input_scale(0)).half()
        main.sample_in[..., :4] = torch.cat([x0, x0], dim=0)
        cbuf = torch.zeros((2, h, w, 8), dtype=torch.float16, device=dev)  # scaled image-1 latent twice (:583-585)
        cbuf[..., :4] = torch.cat([x0[1:2], x0[1:2]], dim=0)
        lat = lat.contiguous()
        n_att = self.unet.num_attention_layers()
        self.sample_forwards = 0
        # ---- opt-in de-duplication of bitwise-identical work (results unchanged; bench reports it as "effective")
        #  * twin rows: until the first fusion step image 1 IS image 0 (same latents, same prompt, and the
        #    prompt-to-prompt edit of identical rows is the identity), so the main UNet runs B=2 [uncond, cond];
        #  * stage-2 prefix: steps 0..15 of stage 2 repeat stage 1 on the same inputs, so stage 2 resumes from the
        #    latents stage 1 had after step 15 (and the solver history and generator state it had then).  A stochastic
        #    schedule gives the two images different noise (no twins), and without a generator its noise comes from
        #    the global RNG, which cannot be replayed (no prefix).
        hist = torch.zeros((2, h, w, 4), dtype=torch.float32, device=dev) if sch.uses_history else None
        gdev = generator.device if generator is not None else dev

        def step(noise_main, noises, fmasks, i):
            if sch.uses_fuse_step:
                ops.fuse_step(noise_main, noises, fmasks, guidance_scale, float(sig[i]), float(sig[i + 1]), lat,
                              main.sample_in, cbuf)
                return
            z = None
            if sch.stochastic:  # randn_tensor(model_output.shape, generator, device, fp16)
                z = torch.randn((2, 4, h, w), generator=generator, device=gdev, dtype=torch.float16).to(dev)
            ops.solver_step(noise_main, noises, fmasks, guidance_scale, sch.step_coeffs(i), lat, main.sample_in, cbuf,
                            history=hist, store_x0=hist is not None, noise=z)

        dd = self.dedup and cn is None
        prefix_ok = dd and not (sch.stochastic and generator is None)
        gen0 = generator.get_state() if (sch.stochastic and generator is not None) else None
        twin = dd and not sch.stochastic and bool(torch.equal(lat[0], lat[1]) and torch.equal(ctx4[0], ctx4[1]) and torch.equal(ctx4[2], ctx4[3])
                           and torch.equal(pooled4[0], pooled4[1]) and torch.equal(pooled4[2], pooled4[3]))
        i0 = 0
        sig_key = (tuple(float(t) for t in ts), float(guidance_scale), self.main_lora_key, h, w, sch.scheduler_key())
        if prefix_ok and stage == 2 and n_act > 0 and len(ts) > FUSION_AFTER_STEP + 1 and self._prefix is not None:
            pf = self._prefix
            if (pf["key"] == sig_key and torch.equal(pf["lat0"], lat) and torch.equal(pf["ctx4"], ctx4.to(dev))
                    and torch.equal(pf["pooled4"], pooled4.to(dev))
                    and (gen0 is None or (pf["gen0"] is not None and torch.equal(pf["gen0"], gen0)))):
                i0 = FUSION_AFTER_STEP + 1
                lat.copy_(pf["lat"])
                main.sample_in.copy_(pf["sample_in"])
                cbuf.copy_(pf["cbuf"])
                if hist is not None:
                    hist.copy_(pf["hist"])
                if gen0 is not None:
                    generator.set_state(pf["gen"])
                if controller is not None:
                    for _ in range(i0):
                        controller.advance(n_att)
        twin = twin and (n_act == 0 or i0 <= FUSION_AFTER_STEP)  # any step left that runs without fusion?
        main2 = noise4 = None
        if twin:
            main2 = self._runner("main2", self.unet, 2, h, w, groups=[RowGroup(0, 2, self.main_lora_key, False)])
            main2.set_conditioning(ts, ctx4[[0, 2]], pooled4[[0, 2]], tid.repeat(2, 1))
            noise4 = torch.empty((4, h, w, 8), dtype=torch.float16, device=dev)
        lat0_keep = lat.clone() if (prefix_ok and stage == 1) else None

        def keep_prefix():
            self._prefix = {"key": sig_key, "lat0": lat0_keep, "ctx4": ctx4.to(dev).clone(),
                            "pooled4": pooled4.to(dev).clone(), "lat": lat.clone(),
                            "sample_in": main.sample_in.clone(), "cbuf": cbuf.clone(),
                            "hist": None if hist is None else hist.clone(), "gen0": gen0,
                            "gen": None if gen0 is None else generator.get_state()}

        for i in range(i0, len(ts)):
            fuse = i > FUSION_AFTER_STEP and n_act > 0
            if twin and not fuse:
                main2.sample_in.copy_(main.sample_in.view(2, 2, h, w, 8)[:, 0])
                n2 = main2.forward(i, main2.default_variant(), key=("twin",))
                noise4.view(2, 2, h, w, 8).copy_(n2[:, None])
                if controller is not None:
                    controller.advance(n_att)
                self.sample_forwards += 2
                step(noise4, [], [], i)
                if callback is not None:
                    self._step_end(callback, i, ts[i], lat, main, cbuf)
                if lat0_keep is not None and i == FUSION_AFTER_STEP:
                    keep_prefix()
                continue
            twin = False  # from the first fusion step on the two images differ
            if controller is not None:
                self._update_p2p_context(p2p_runners, controller, ctx4, first=False)
            run = fused if (fuse and grouped) else main
            variant, key = self._p2p_variant(run, controller, cn is not None)
            if run is fused:
                run.sample_in[0:4].copy_(main.sample_in)
                for j in range(n_act):
                    run.sample_in[4 + 2 * j:6 + 2 * j].copy_(cbuf)
                # concept streams: plain attention on their own K/V rows (after the main 4 text rows + 2 P2P rows)
                kv0 = 4 + (2 if controller is not None else 0)
                ident_c = [(4 + r, 4 + r, kv0 + r, kv0 + r) for r in range(2 * n_act)]
                variant["self_items"] = variant["self_items"][:4] + [(4 + r, 4 + r, 4 + r, 4 + r) for r in range(2 * n_act)]
                variant["cross_items"] = [variant["cross_items"][0][:4] + ident_c] + variant["cross_items"][1:]
                variant["ip_items"], n_ip = [], 0
                for j, k in enumerate(active):
                    if concepts[k]["ip"]:
                        for r in (4 + 2 * j, 5 + 2 * j):
                            variant["ip_items"].append((r, r, n_ip, n_ip))
                            n_ip += 1
            slots = []
            if cn is not None:
                cn.sample_in.copy_(main.sample_in)
                down, mid = cn.forward(i, key=("cn",))
                sc = cn_scale * cn_keep(i)
                slots.append((down, mid, sc, 0))
                key = key + (sc,)
            if fuse and idr is not None:
                for j in range(n_act):
                    idr.sample_in[2 * j:2 * j + 2].copy_(cbuf)
                id_down, id_mid = idr.forward(i, key=("identity",))
            if run is fused and idr is not None:
                # IdentityNet residuals go to the concept rows (4 ..), a main-pass ControlNet's to rows 0-3: two
                # residual slots of the same grouped forward
                slots.append((id_down, id_mid, id_scale, 4))
                variant["residuals"] = True
                key = key + ("id", id_scale)
            run.residuals_in = slots
            noise = run.forward(i, variant, key=key)
            if controller is not None:
                controller.advance(n_att)
            noises, fmasks = [], []
            if fuse:
                if grouped:
                    noises = [noise[4 + 2 * j:6 + 2 * j] for j in range(n_act)]
                else:
                    for j, r in enumerate(crun):
                        r.sample_in.copy_(cbuf)
                        v = r.default_variant()
                        ckey = ("concept",)
                        if idr is not None:
                            r.residuals_in = ([d[2 * j:2 * j + 2] for d in id_down], id_mid[2 * j:2 * j + 2], id_scale, 0)
                            v["residuals"] = True
                            ckey = ("concept", "id", id_scale)
                        noises.append(r.forward(i, v, key=ckey))
                fmasks = [masks[k] for k in active]
            self.sample_forwards += 4 + (2 * n_act if fuse else 0)
            step(noise[0:4] if run is fused else noise, noises, fmasks, i)
            if callback is not None:
                self._step_end(callback, i, ts[i], lat, main, cbuf)
            if lat0_keep is not None and i == FUSION_AFTER_STEP:
                keep_prefix()
        return lat

    def _finish(self, latents_nhwc: torch.Tensor, output_type: str, return_dict: bool):
        lat = latents_nhwc.permute(0, 3, 1, 2).contiguous().half()  # (2,4,h,w) like the reference's fp16 latents
        if output_type == "latent":
            image = lat
        else:
            if self.vae_decoder is None:
                raise RuntimeError("image output needs a vae_decoder (the VAE is outside the accelerated hot path); "
                                   "use output_type='latent'")
            image = self.vae_decoder(lat, output_type)
        return PipelineOutput(images=image) if return_dict else (image,)


class LoraMultiConceptPipeline(_BasePipeline):
    """src/pipelines/lora_pipeline.py:154-681."""

    def __call__(self, prompt=None, prompt_2=None, image=None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: int = 50, guidance_scale: float = 5.0,
                 negative_prompt=None, negative_prompt_2=None, num_images_per_prompt: int = 1, eta: float = 0.0,
                 generator=None, latents=None, prompt_embeds=None, negative_prompt_embeds=None,
                 pooled_prompt_embeds=None, negative_pooled_prompt_embeds=None, output_type: str = "pil",
                 return_dict: bool = True, cross_attention_kwargs=None, controlnet_conditioning_scale=1.0,
                 guess_mode: bool = False, control_guidance_start=0.0, control_guidance_end=1.0, original_size=None,
                 crops_coords_top_left=(0, 0), target_size=None, controller=None, concept_models: ConceptModels = None,
                 stage=None, region_masks=None, lora_list=None, styleL=None, region_prompt_embeds=None,
                 callback_on_step_end=None, **kwargs):
        dev = self._execution_device
        scale = (cross_attention_kwargs or {}).get("scale", 1.0)
        # 3.1 prompts: prompt = [[global, global], [(region, region_neg), ...]]  (lora_pipeline.py:310-347)
        global_prompt = prompt[0]
        region_prompts = [pt[0] for pt in prompt[1]]
        region_negs = [pt[1] for pt in prompt[1]]
        lora_list = list(lora_list or [])
        if prompt_embeds is None:
            prompt_embeds, negative_prompt_embeds, pooled_prompt_embeds, negative_pooled_prompt_embeds = \
                self.encode_prompt(global_prompt, negative_prompt, scale)
        height = height or 128 * self.vae_scale_factor
        width = width or 128 * self.vae_scale_factor
        h, w = height // self.vae_scale_factor, width // self.vae_scale_factor
        concepts = []
        for k, (lp, rp, rn) in enumerate(zip(lora_list, region_prompts, region_negs)):
            if styleL:
                concept_models.set_adapters([lp, "style"], adapter_weights=[0.7, 0.5])
            else:
                concept_models.set_adapters(lp)
            if region_prompt_embeds is not None:
                pe, ne, pp, np_ = region_prompt_embeds[k]
            else:
                pe, ne, pp, np_ = concept_models.encode_prompt(rp, negative_prompt=rn, lora_scale=scale)
            concepts.append({"ctx": torch.cat([ne, pe], dim=0), "pooled": torch.cat([np_, pp], dim=0),
                             "lora_key": concept_models.active_lora_key(0.8)})  # {'scale': 0.8} (:596)
        masks = [None] * len(concepts)
        if stage == 2:
            masks = [_binary_latent_mask(m, h, w, dev) for m in region_masks]
        # 5/6 timesteps + latents
        ts = self._set_timesteps(num_inference_steps)
        lat = self.prepare_latents(h, w, generator, latents)
        # 7.2 added conditioning
        original_size = original_size or (height, width)
        target_size = target_size or (height, width)
        tid = torch.tensor([list(original_size) + list(crops_coords_top_left) + list(target_size)], dtype=torch.float32)
        ctx4 = torch.cat([negative_prompt_embeds, prompt_embeds], dim=0)          # rows [neg0, neg1, pos0, pos1]
        pooled4 = torch.cat([negative_pooled_prompt_embeds, pooled_prompt_embeds], dim=0)
        # the controller acts through self.controller (installed by revise_regionally_controlnet_forward); the
        # `controller=` kwarg is accepted and ignored exactly like the reference (:248)
        main_cn = None
        if image is not None and self.controlnet is not None:
            cn_scale = controlnet_conditioning_scale[0] if isinstance(controlnet_conditioning_scale, list) else controlnet_conditioning_scale
            n_ts = len(ts)
            s0 = control_guidance_start[0] if isinstance(control_guidance_start, list) else control_guidance_start
            e0 = control_guidance_end[0] if isinstance(control_guidance_end, list) else control_guidance_end
            main_cn = (self.controlnet, self._prepare_image(image, width, height, 4), cn_scale,
                       lambda i: 1.0 - float(i / n_ts < s0 or (i + 1) / n_ts > e0))      # controlnet_keep (:421-427)
        for c in concepts:
            c["ip"] = False
        lat = self._denoise(ts=ts, lat=lat, ctx4=ctx4, pooled4=pooled4, tid=tid, concepts=concepts, masks=masks,
                            stage=stage, guidance_scale=guidance_scale, h=h, w=w, concept_unet=concept_models.unet
                            if concept_models is not None else self.unet, main_cn=main_cn, callback=callback_on_step_end,
                            generator=generator)
        return self._finish(lat, output_type, return_dict)

    def _prepare_image(self, image, width, height, batch):
        """ControlNet condition: list/tensor/PIL -> (batch, 3, H, W) in [0,1] (diffusers prepare_image [3P])."""
        img = image[0] if isinstance(image, (list, tuple)) else image
        if not torch.is_tensor(img):
            import numpy as np
            img = torch.from_numpy(np.asarray(img.convert("RGB").resize((width, height)), dtype="float32") / 255.0)
            img = img.permute(2, 0, 1)
        if img.dim() == 3:
            img = img[None]
        return img.float().repeat(batch // img.shape[0], 1, 1, 1)


def revise_regionally_controlnet_forward(pipe_or_unet, controller: AttentionReplace):
    """src/pipelines/lora_pipeline.py:136-152: hook the controller into every attention layer of the main UNet and
    set controller.num_att_layers = 2 * (#cross-attention layers).  Here the "processors" are the fused kernels, so
    installing means handing the pipeline the controller."""
    pipe = pipe_or_unet
    unet = pipe.unet if hasattr(pipe, "unet") else pipe
    count = unet.num_attention_layers() // 2
    print(f"Number of attention layer registered {count}")
    controller.num_att_layers = count * 2
    if hasattr(pipe, "controller"):
        pipe.controller = controller
    return controller


class InstantidMultiConceptPipeline(_BasePipeline):
    """src/pipelines/instantid_pipeline.py:157-767.  `self.controlnet` is the IdentityNet (used only in the concept
    pass, :638-648), `self.controlnet2` an optional spatial ControlNet for the main pass (:574-616)."""

    def __call__(self, prompt=None, image=None, height=None, width=None, num_inference_steps: int = 50,
                 guidance_scale: float = 5.0, negative_prompt=None, generator=None, latents=None,
                 output_type: str = "pil", return_dict: bool = True, cross_attention_kwargs=None,
                 controlnet_conditioning_scale=1.0, original_size=None, crops_coords_top_left=(0, 0), target_size=None,
                 controller=None, concept_models: ConceptModels = None, stage=None, region_masks=None, face_app=None,
                 t2i_image=None, t2i_controlnet_conditioning_scale=1.0, face_embeds=None, prompt_embeds=None,
                 negative_prompt_embeds=None, pooled_prompt_embeds=None, negative_pooled_prompt_embeds=None,
                 region_prompt_embeds=None, callback_on_step_end=None, **kwargs):
        dev = self._execution_device
        scale = (cross_attention_kwargs or {}).get("scale", 1.0)
        global_prompt = prompt[0]
        regions = prompt[1]
        if prompt_embeds is None:
            prompt_embeds, negative_prompt_embeds, pooled_prompt_embeds, negative_pooled_prompt_embeds = \
                self.encode_prompt(global_prompt, negative_prompt, scale)
        height = height or 128 * self.vae_scale_factor
        width = width or 128 * self.vae_scale_factor
        h, w = height // self.vae_scale_factor, width // self.vae_scale_factor
        concepts = []
        for k, reg in enumerate(regions):
            if region_prompt_embeds is not None:
                pe, ne, pp, np_ = region_prompt_embeds[k]
            else:
                pe, ne, pp, np_ = self.encode_prompt(reg[0], reg[1], scale)
            c = {"ctx": torch.cat([ne, pe], dim=0), "pooled": torch.cat([np_, pp], dim=0), "tokens": None}
            if stage == 2:
                if face_embeds is not None:
                    emb = face_embeds[k]
                else:
                    emb = self.get_face_embedding(face_app, reg[2])
                c["tokens"] = concept_models._encode_prompt_image_emb(emb, dev, torch.float16, True)  # (2,16,D)
            concepts.append(c)
        masks = [None] * len(concepts)
        if stage == 2:
            masks = [_binary_latent_mask(m, h, w, dev) for m in region_masks]
        ts = self._set_timesteps(num_inference_steps)
        lat = self.prepare_latents(h, w, generator, latents)
        original_size = original_size or (height, width)
        target_size = target_size or (height, width)
        tid = torch.tensor([list(original_size) + list(crops_coords_top_left) + list(target_size)], dtype=torch.float32)
        ctx4 = torch.cat([negative_prompt_embeds, prompt_embeds], dim=0)
        pooled4 = torch.cat([negative_pooled_prompt_embeds, pooled_prompt_embeds], dim=0)
        main_cn = None
        if t2i_image is not None and self.controlnet2 is not None:
            t2i_scale = t2i_controlnet_conditioning_scale[0] if isinstance(t2i_controlnet_conditioning_scale, list) else t2i_controlnet_conditioning_scale
            main_cn = (self.controlnet2, LoraMultiConceptPipeline._prepare_image(self, t2i_image, width, height, 4),
                       t2i_scale, lambda i: 1.0)
        identity = None
        cn_scale = controlnet_conditioning_scale[0] if isinstance(controlnet_conditioning_scale, list) else controlnet_conditioning_scale
        for c in concepts:
            c["lora_key"] = None
            c["ip"] = c["tokens"] is not None
            if c["ip"]:
                c["ctx"] = torch.cat([c["ctx"].to(dev), c["tokens"].to(dev).to(c["ctx"].dtype)], dim=1)  # (:663)
        if stage == 2 and image is not None and self.controlnet is not None:
            identity = (self.controlnet, LoraMultiConceptPipeline._prepare_image(self, image, width, height, 2), cn_scale,
                        [c["tokens"] for c in concepts])
        lat = self._denoise(ts=ts, lat=lat, ctx4=ctx4, pooled4=pooled4, tid=tid, concepts=concepts, masks=masks,
                            stage=stage, guidance_scale=guidance_scale, h=h, w=w, concept_unet=concept_models.unet
                            if concept_models is not None else self.unet, main_cn=main_cn, identity=identity,
                            callback=callback_on_step_end, generator=generator)
        return self._finish(lat, output_type, return_dict)

    def get_face_embedding(self, face_app, ref_image):
        """instantid_pipeline.py:757-767: the reference sorts detections by (x2-x0)*y2 - y1 ascending and takes the
        first (documented quirk); kept as is.  A photo without a face raises ValueError naming it (the reference fails
        with an IndexError)."""
        import cv2
        import numpy as np
        from PIL import Image
        info = face_app.get(cv2.cvtColor(np.array(Image.open(ref_image).convert("RGB")), cv2.COLOR_RGB2BGR))
        if len(info) == 0:
            raise ValueError(f"no face detected in the reference photo {ref_image}")
        info = sorted(info, key=lambda x: (x["bbox"][2] - x["bbox"][0]) * x["bbox"][3] - x["bbox"][1])[0]
        return info["embedding"]
