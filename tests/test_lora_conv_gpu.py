"""GPU tests of LoCon adapters: per-stream conv weight planes at the op level (every conv form of the UNet, three row
groups of 4 + 2 + 2 images), the UNet executor against the fp32 oracle per stream, the three executors, and the
pipelines with adapters loaded from kohya files written here.  No real LoCon checkpoint is used (none is available
offline): the adapters are synthetic, drawn like synthetic.make_lora draws them.

Op-level outputs sit between NaN-filled guard images and the weight planes between NaN-filled planes, inside memory the
test owns: a store outside the output or a tile that reads the wrong plane changes values, it cannot fault."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from util_locon import locon_oracle  # noqa: E402,F401  (autouse: the oracle's conv applies LoCon entries)
from util_models import from_nhwc, ocfg, oracle_lora, r16, rel, to_nhwc8, weights  # noqa: E402

TOL = 1.9e-3   # the bound of tests/test_unet_gpu.py
ENDS = [4, 6, 8]


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _guarded(B, H, W, N):
    big = torch.full((B + 2, H, W, N), float("nan"), dtype=torch.float16, device="cuda")
    return big, big[1:-1]


def _planes(ws):
    """Stack of weight planes between two NaN planes."""
    N = ws[0].shape[0]
    big = torch.full(((len(ws) + 2) * N, ws[0].shape[1]), float("nan"), dtype=torch.float16, device="cuda")
    big[N:-N] = torch.cat(ws, dim=0)
    return big[N:-N]


def _rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def _conv_ref(x, w4, stride=1, up=False):
    xf = x.float().permute(0, 3, 1, 2)
    if up:
        xf = F.interpolate(xf, scale_factor=2.0, mode="nearest")
    return F.conv2d(xf, w4.float(), stride=stride, padding=1).permute(0, 2, 3, 1)


def _groups_of(B):
    return [(0 if i == 0 else ENDS[i - 1], e) for i, e in enumerate(ENDS)]


@pytest.mark.parametrize("C,HW", [(320, 64), (640, 32), (1280, 16), (64, 8)])
def test_conv3x3_planes(C, HW):
    """ResBlock conv1 form: rowvec, column statistics and the fp32 twin; planes vs one launch per group, bit for bit
    (block_n pinned: the automatic choice depends on the number of m-tiles, which differs between the two)."""
    from omg_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator().manual_seed(C + HW)
    B, H, W = 8, HW, HW
    x = _rand(g, B, H, W, C)
    w4 = [_rand(g, C, C, 3, 3, scale=(9 * C) ** -0.5) for _ in ENDS]
    ws = [ops.pack_conv3x3_weight(w) for w in w4]
    bias, rowvec = _rand(g, C, scale=0.1), _rand(g, B, C, scale=0.5)
    res = _rand(g, B, H, W, C)
    rb = ops.colstats_blocks(W, H)
    bn = 128 if C % 128 == 0 else 64
    outs = []
    for mode in ("planes", "per_group", "planes_again"):
        big, out = _guarded(B, H, W, C)
        cs = torch.zeros(B, rb, C, 2, dtype=torch.float32, device="cuda")
        twin = torch.zeros(B * H * W, C, dtype=torch.float32, device="cuda")
        if mode == "per_group":
            for (i0, i1), w in zip(_groups_of(B), ws):
                ops.conv3x3(x[i0:i1], w, bias=bias, rowvec=rowvec[i0:i1], residual=res[i0:i1], out=out[i0:i1], block_n=bn,
                            colstats=cs[i0:i1], out_f32=twin[i0 * H * W:i1 * H * W])
        else:
            ops.conv3x3(x, _planes(ws), bias=bias, rowvec=rowvec, residual=res, out=out, block_n=bn, colstats=cs,
                        out_f32=twin, row_groups=ENDS)
        torch.cuda.synchronize()
        assert torch.isnan(big[0]).all() and torch.isnan(big[-1]).all()
        outs.append((out.clone(), cs, twin))
    for o, cs, twin in outs[1:]:
        assert torch.equal(_bits(o), _bits(outs[0][0])) and torch.equal(cs, outs[0][1]) and torch.equal(twin, outs[0][2])
    out, cs, twin = outs[0]
    for (i0, i1), w in zip(_groups_of(B), w4):
        ref = _conv_ref(x[i0:i1], w) + bias.float() + rowvec[i0:i1].float()[:, None, None, :] + res[i0:i1].float()
        assert rel(out[i0:i1], ref) < 1e-3 and rel(twin.view(B, H, W, C)[i0:i1], ref) < 1e-4
    # the statistics are those of the stored (rounded) output, per image
    s = cs.sum(dim=1)
    of = out.float().reshape(B, H * W, C)
    assert torch.allclose(s[..., 0], of.sum(1), rtol=1e-4, atol=1e-2) and torch.allclose(s[..., 1], of.pow(2).sum(1), rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize("split", [[4, 6, 8], [3, 6, 8]])
def test_conv3x3_planes_tall_tiles(split):
    """Tall tiles pair two consecutive m-tiles.  On an 8 x 8 grid an image is one m-tile: with boundaries at images 4 and
    6 the pairs stay inside a group and tall tiles run; with a boundary at image 3 a pair would straddle two groups and
    the launch uses single tiles.  Either way the result equals the single-tile launch bit for bit."""
    from omg_b200 import ops
    g = torch.Generator().manual_seed(7)
    B, H, W, C, N = 8, 8, 8, 1280, 160
    x = _rand(g, B, H, W, C)
    ws = [ops.pack_conv3x3_weight(_rand(g, N, C, 3, 3, scale=(9 * C) ** -0.5)) for _ in split]
    outs = []
    for cta_pair in (1, 3):
        big, out = _guarded(B, H, W, N)
        ops.conv3x3(x, _planes(ws), out=out, block_n=160, cta_pair=cta_pair, row_groups=split)
        torch.cuda.synchronize()
        assert torch.isnan(big[0]).all() and torch.isnan(big[-1]).all()
        outs.append(out.clone())
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))
    for gi, i1 in enumerate(split):
        i0 = split[gi - 1] if gi else 0
        ref = ops.conv3x3(x[i0:i1].contiguous(), ws[gi], block_n=160, cta_pair=1)
        assert torch.equal(_bits(outs[0][i0:i1]), _bits(ref))


def test_conv3x3_shortcut_planes():
    """ResBlock conv2 of an up block at SDXL width: nine taps over 1280 channels plus the two K-segments of the 1x1
    shortcut (x and the skip, 2560 channels behind the 9 * 1280 columns), 11 segments in all."""
    from omg_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator().manual_seed(3)
    B, H, W, C = 8, 16, 16, 1280
    a2, x, skip = _rand(g, B, H, W, C), _rand(g, B, H, W, C), _rand(g, B, H, W, C)
    w4 = [_rand(g, C, C, 3, 3, scale=(9 * C) ** -0.5) for _ in ENDS]
    wsc = [_rand(g, C, 2 * C, scale=(2 * C) ** -0.5) for _ in ENDS]
    ws = [torch.cat([ops.pack_conv3x3_weight(a), b], dim=1).contiguous() for a, b in zip(w4, wsc)]
    bias = _rand(g, C, scale=0.1)
    outs = []
    for mode in ("planes", "per_group"):
        big, out = _guarded(B, H, W, C)
        if mode == "planes":
            ops.conv3x3(a2, _planes(ws), bias=bias, shortcut=[(x, 9 * C), (skip, 10 * C)], out=out, block_n=128, row_groups=ENDS)
        else:
            for (i0, i1), w in zip(_groups_of(B), ws):
                ops.conv3x3(a2[i0:i1], w, bias=bias, shortcut=[(x[i0:i1], 9 * C), (skip[i0:i1], 10 * C)], out=out[i0:i1], block_n=128)
        torch.cuda.synchronize()
        assert torch.isnan(big[0]).all() and torch.isnan(big[-1]).all()
        outs.append(out.clone())
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))
    for (i0, i1), w, wsk in zip(_groups_of(B), w4, wsc):
        ref = _conv_ref(a2[i0:i1], w) + torch.cat([x[i0:i1], skip[i0:i1]], dim=-1).float() @ wsk.float().t() + bias.float()
        assert rel(outs[0][i0:i1], ref) < 1e-3


@pytest.mark.parametrize("form", ["s2", "up"])
@pytest.mark.parametrize("C,HW", [(640, 32), (64, 16)])
def test_resampler_planes(form, C, HW):
    """Down-sampler (stride-2 phase views; output grid HW/2) and up-sampler (four phase launches through strided
    output views; each counts the HW x HW input grid per image), with column statistics; the 16 x 16 case runs the
    stride-2 conv on an 8 x 8 output grid."""
    from omg_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator().manual_seed(C + HW + len(form))
    B, H, W = 8, HW, HW
    fn = ops.conv3x3_s2 if form == "s2" else ops.upsample2x_conv3x3
    Ho = H // 2 if form == "s2" else 2 * H
    rb = ops.colstats_blocks(Ho, Ho) if form == "s2" else 4 * ops.colstats_blocks(W, H)
    x = _rand(g, B, H, W, C)
    w4 = [_rand(g, C, C, 3, 3, scale=(9 * C) ** -0.5) for _ in ENDS]
    ws = [ops.pack_conv3x3_weight(w) for w in w4]
    bias = _rand(g, C, scale=0.1)
    bn = 128 if C % 128 == 0 else 64
    outs = []
    for mode in ("planes", "per_group"):
        big, out = _guarded(B, Ho, Ho, C)
        cs = torch.zeros(B, rb, C, 2, dtype=torch.float32, device="cuda")
        if mode == "planes":
            fn(x, _planes(ws), bias=bias, out=out, block_n=bn, colstats=cs, row_groups=ENDS)
        else:
            for (i0, i1), w in zip(_groups_of(B), ws):
                fn(x[i0:i1], w, bias=bias, out=out[i0:i1], block_n=bn, colstats=cs[i0:i1])
        torch.cuda.synchronize()
        assert torch.isnan(big[0]).all() and torch.isnan(big[-1]).all()
        outs.append((out.clone(), cs))
    assert torch.equal(_bits(outs[0][0]), _bits(outs[1][0])) and torch.equal(outs[0][1], outs[1][1])
    out, cs = outs[0]
    for (i0, i1), w in zip(_groups_of(B), w4):
        ref = _conv_ref(x[i0:i1], w, stride=2 if form == "s2" else 1, up=form == "up") + bias.float()
        assert rel(out[i0:i1], ref) < 1e-3
    of = out.float().reshape(B, Ho * Ho, C)
    assert torch.allclose(cs.sum(dim=1)[..., 0], of.sum(1), rtol=1e-4, atol=1e-2)


# ------------------------------------------------------------------------------------------------ UNet
def _locon(cfg, seed, rank=8):
    from omg_b200 import synthetic
    return {k: (r16(a), r16(b), s) for k, (a, b, s) in synthetic.make_lora(cfg, seed, rank=rank, conv=True).items()}


def _inputs(cfg, B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = r16(torch.randn(B, 4, H, W, generator=g))
    ctx = r16(torch.randn(B, 77, cfg.cross_attention_dim, generator=g))
    pooled = r16(torch.randn(B, cfg.pooled_dim, generator=g))
    tid = torch.tensor([[H * 8, W * 8, 0, 0, H * 8, W * 8]], dtype=torch.float32).repeat(B, 1)
    return x, ctx, pooled, tid


@pytest.fixture(scope="module")
def env():
    from omg_b200.config import UNetConfig
    from omg_b200.unet import PackedUNet
    cfg = UNetConfig.tiny()
    sd = weights(cfg, 0)
    la, lb, ls = _locon(cfg, 11), _locon(cfg, 12), _locon(cfg, 13)
    model = PackedUNet(cfg, sd)
    model.add_lora_set("A", [(la, 1.0)], 0.8)
    model.add_lora_set("B+style", [(lb, 0.7), (ls, 0.5)], 0.8)
    return {"cfg": cfg, "sd": sd, "model": model, "sets": {None: [], "A": [(la, 1.0)], "B+style": [(lb, 0.7), (ls, 0.5)]}}


def _grouped(env, B=4, H=32, W=32, seed=5, **kw):
    from omg_b200.unet import RowGroup, UNetRunner
    groups = [RowGroup(0, 2, None), RowGroup(2, 3, "A"), RowGroup(3, 4, "B+style")]
    x, ctx, pooled, tid = _inputs(env["cfg"], B, H, W, seed)
    r = UNetRunner(kw.pop("model", env["model"]), B, H, W, groups=groups, **kw)
    r.set_conditioning([250.0, 33.0], [(ctx[g.start:g.stop], g.lora_key, False) for g in groups], pooled, tid)
    r.sample_in.copy_(to_nhwc8(x))
    return r, groups, (x, ctx, pooled, tid)


@pytest.mark.parametrize("merged", [True, False], ids=["planes", "per_group"])
def test_grouped_unet_locon_vs_oracle(env, merged):
    """main rows + concept A (LoCon) + concept B (LoCon + style, weights 0.7 / 0.5) in one launch sequence, each stream
    against the fp32 oracle with that stream's un-merged adapters; 32 x 32 latents, so the mid block runs on 8 x 8
    images.  per_group: the conv-per-stream path taken when weight planes are not used."""
    from oracle import unet as ou
    cfg = env["cfg"]
    r, groups, (x, ctx, pooled, tid) = _grouped(env, use_graphs=False)
    r.merge_lora = merged
    for step, t in enumerate([250.0, 33.0]):
        out = from_nhwc(r.forward(step))
        for g in groups:
            sl = slice(g.start, g.stop)
            c = ou.Ctx(env["sd"], ocfg(cfg), lora=oracle_lora(env["sets"][g.lora_key], 0.8))
            ref = ou.unet_forward(c, x[sl], t, ctx[sl], pooled[sl], tid[sl])
            base = ou.unet_forward(ou.Ctx(env["sd"], ocfg(cfg)), x[sl], t, ctx[sl], pooled[sl], tid[sl])
            e = rel(out[sl], ref)
            print(f"locon stream {g.lora_key} t={t} rel err {e:.3e}, adapter effect {rel(ref, base):.3e}")
            assert e < TOL and (g.lora_key is None or rel(ref, base) > 5 * e)


def test_conv_modules_take_effect_and_zero_up_is_exact(env):
    """The conv / time-embedding part of the adapter moves the output well beyond the parity error; an adapter whose conv
    up matrices are zero gives exactly the transformer-only result."""
    from omg_b200.config import lora_conv_target_names
    from omg_b200.unet import PackedUNet
    cfg = env["cfg"]
    conv_names = {t[0] for t in lora_conv_target_names(cfg)}
    la = env["sets"]["A"][0][0]
    lb, ls = (s[0] for s in env["sets"]["B+style"])
    outs = {}
    for kind in ("full", "linear_only", "zero_up"):
        def cut(lo):
            if kind == "full":
                return lo
            if kind == "linear_only":
                return {k: v for k, v in lo.items() if k not in conv_names}
            return {k: (a, torch.zeros_like(b) if k in conv_names else b, s) for k, (a, b, s) in lo.items()}
        model = PackedUNet(cfg, env["sd"])
        model.add_lora_set("A", [(cut(la), 1.0)], 0.8)
        model.add_lora_set("B+style", [(cut(lb), 0.7), (cut(ls), 0.5)], 0.8)
        r, groups, _ = _grouped(env, use_graphs=False, model=model)
        outs[kind] = r.forward(0).clone()
    assert torch.equal(outs["zero_up"], outs["linear_only"])
    assert torch.equal(outs["full"][:2], outs["linear_only"][:2])          # the main rows have no adapter
    assert rel(outs["full"][2:], outs["linear_only"][2:]) > 20 * TOL


def test_executors_agree_and_a_replaced_set_is_used(env):
    from omg_b200.unet import PackedUNet
    cfg = env["cfg"]
    model = PackedUNet(cfg, env["sd"])
    model.add_lora_set("A", env["sets"]["A"], 0.8)
    model.add_lora_set("B+style", env["sets"]["B+style"], 0.8)
    eager, _, _ = _grouped(env, use_graphs=False, model=model)
    graph, _, _ = _grouped(env, use_graphs=True, model=model)
    plan, _, _ = _grouped(env, use_graphs=False, use_plans=True, model=model)
    ref = eager.forward(0).clone()
    for r in (graph, plan):
        for _ in range(3):     # eager warm-up, capture / recording, replay
            assert torch.equal(r.forward(0, key=("k",)), ref)
    assert ("k",) in graph.graphs and ("k",) in plan.plans
    v0 = model.adapter_version
    model.add_lora_set("A", [(_locon(cfg, 99), 1.0)], 0.8)
    assert model.adapter_version == v0 + 1
    fresh = PackedUNet(cfg, env["sd"])
    fresh.add_lora_set("A", [(_locon(cfg, 99), 1.0)], 0.8)
    fresh.add_lora_set("B+style", env["sets"]["B+style"], 0.8)
    new, _, (x, ctx, pooled, tid) = _grouped(env, use_graphs=False, model=fresh)
    ref2 = new.forward(0).clone()
    assert not torch.equal(ref2[2:3], ref[2:3]) and torch.equal(ref2[3:], ref[3:]) and torch.equal(ref2[:2], ref[:2])
    for r in (eager, graph, plan):
        r.set_conditioning([250.0, 33.0], [(ctx[0:2], None, False), (ctx[2:3], "A", False), (ctx[3:4], "B+style", False)], pooled, tid)
        for _ in range(3):
            out = r.forward(0, key=("k",))
        assert torch.equal(out, ref2)


# ------------------------------------------------------------------------------------------------ files and pipelines
def _kohya_sgm_file(cfg, lo, path):
    """Write `lo` as a kohya LoCon file with SGM block names (what a Civitai SDXL LoCon uses)."""
    from safetensors.torch import save_file
    from omg_b200 import checkpoints as ck
    sgm = ("lora_unet_input_blocks_", "lora_unet_middle_block_", "lora_unet_output_blocks_")
    stems = {v: k for table in (ck._kohya_lookup(cfg), ck._kohya_conv_lookup(cfg)) for k, v in table.items() if k.startswith(sgm)}
    sd = {}
    for name, (A, B, s) in lo.items():
        stem = stems[name]
        sd[stem + ".lora_down.weight"] = A.contiguous()
        sd[stem + ".lora_up.weight"] = (B[:, :, None, None] if A.dim() == 4 else B).contiguous()
        sd[stem + ".alpha"] = torch.tensor(s * A.shape[0])
    save_file(sd, path)


def test_pipeline_with_locon_files(tmp_path):
    """The two-stage loop at the tiny topology (as the smoke run: main UNet under prompt-to-prompt control, two concept
    UNets, region fusion, CFG, Euler; fusion from step 15) with both concepts loaded from kohya SGM LoCon files,
    against the oracle pipeline; and the same files without their conv entries give a different image."""
    from omg_b200 import synthetic
    from omg_b200.config import UNetConfig, lora_conv_target_names
    from omg_b200.pipelines import ConceptModels, LoraMultiConceptPipeline, revise_regionally_controlnet_forward
    from omg_b200.prompt_attention import AttentionReplace
    from omg_b200.unet import PackedUNet
    from oracle import p2p as op2p
    from oracle import unet as ou
    from oracle.pipeline import Concept, denoise
    cfg = UNetConfig.tiny()
    sd = weights(cfg, 0)
    loras = [_locon(cfg, 100 + i) for i in range(2)]
    conv_names = {t[0] for t in lora_conv_target_names(cfg)}
    size, steps = 128, 17
    prompts = ["a man and a woman"] * 2
    regions = [("a man", "bad"), ("a woman", "bad")]
    masks = synthetic.rect_masks(2, (size, size))
    lat0 = torch.randn(1, 4, size // 8, size // 8, generator=torch.Generator().manual_seed(14)).half()
    outs = {}
    for kind in ("locon", "linear_only"):
        pipe = LoraMultiConceptPipeline(PackedUNet(cfg, sd))
        ctrl = AttentionReplace(prompts, 50, {"default_": 1.0}, 0.4, width=4, height=4)
        revise_regionally_controlnet_forward(pipe, ctrl)
        cm = ConceptModels(PackedUNet(cfg, sd))
        for i, lo in enumerate(loras):
            path = str(tmp_path / f"{kind}{i}.safetensors")
            _kohya_sgm_file(cfg, lo if kind == "locon" else {k: v for k, v in lo.items() if k not in conv_names}, path)
            cm.load_lora_weights(path, adapter_name=f"c{i}")
            assert cm.skipped_lora_keys == [] and set(cm._loras[f"c{i}"]) == (set(lo) if kind == "locon" else set(lo) - conv_names)
        outs[kind] = pipe(prompt=[prompts, regions], negative_prompt=["noisy"] * 2, guidance_scale=7.5, num_inference_steps=steps,
                          cross_attention_kwargs={"scale": 0.8}, concept_models=cm, lora_list=["c0", "c1"], styleL=False, stage=2,
                          region_masks=masks, height=size, width=size, output_type="latent", latents=lat0).images.float().cpu()
    oc = ocfg(cfg)
    pe, ne, pp, np_ = pipe.encode_prompt(prompts, ["noisy"] * 2)
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32)
    concepts = []
    for k, (rp, rn) in enumerate(regions):
        e, n_, p_, np2 = cm.encode_prompt(rp, negative_prompt=rn)
        concepts.append(Concept(r16(torch.cat([n_, e])), r16(torch.cat([np2, p_])), tid.repeat(2, 1), masks[k]))
    refs = {}
    for kind in ("locon", "linear_only"):
        octrl = op2p.AttentionReplaceOracle(prompts, 50, {"default_": 1.0}, 0.4, 4, 4)
        octrl.num_att_layers = len(ou.attention_names(oc))
        for k, c in enumerate(concepts):
            lo = loras[k] if kind == "locon" else {n: v for n, v in loras[k].items() if n not in conv_names}
            c.unet = ou.Ctx(sd, oc, lora=oracle_lora([(lo, 1.0)], 0.8))
        refs[kind] = denoise(ou.Ctx(sd, oc, attn_core=ou.make_p2p_attn_core(octrl)), lat0.float(), r16(torch.cat([ne, pe])),
                             r16(torch.cat([np_, pp])), tid.repeat(4, 1), concepts, 2, steps, 7.5)
    e = rel(outs["locon"], refs["locon"])
    # the concepts enter after step 15 only, so the conv entries move the final latents by less (1.5e-4) than the error
    # the 17 chained steps have accumulated; the change itself still points the way the oracle's does
    d_gpu, d_ref = outs["locon"] - outs["linear_only"], refs["locon"] - refs["linear_only"]
    cos = ((d_gpu * d_ref).sum() / (d_gpu.norm() * d_ref.norm())).item()
    print(f"locon pipeline: final-latent rel err {e:.3e}; the conv entries move the latents by "
          f"{rel(refs['locon'], refs['linear_only']):.3e} (oracle) {rel(outs['locon'], outs['linear_only']):.3e} (cuda), "
          f"cosine of the two changes {cos:.3f}")
    assert e < 3e-3 and cos > 0.4   # measured on an H100 (700 W): 2.35e-3 and 0.69


def test_sdxl_width_fusion_step_with_locon_files(tmp_path):
    """Config-1 shape at full SDXL widths: stage-2 step 16 at 64 x 64 latents, main rows (B = 4) and two LoCon concepts
    (B = 2 each, loaded from kohya SGM files) as ONE grouped forward on weight planes, then omg_fuse_step; against the
    oracle run in fp32 (TF32 off) on the same device.  Bounds: those of tests/test_config1_gpu.py for the main rows and
    the latents; 1.25 x measured for the concept rows (2.95e-3 and 2.23e-3 on an H100 at 700 W - the adapters here change
    the concept noise by a third, and the merged weights are rounded to fp16 once more than the base weights)."""
    from omg_b200 import ops, synthetic
    from omg_b200.config import UNetConfig
    from omg_b200.pipelines import ConceptModels
    from omg_b200.unet import PackedUNet, RowGroup, UNetRunner
    from oracle import unet as ou
    from oracle.pipeline import fuse_noise
    from oracle.scheduler import EulerDiscrete
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda"
    cfg = UNetConfig.sdxl()
    sd = synthetic.make_state_dict(cfg, seed=0, device=dev, dtype=torch.float16)
    H = W = 64
    size = H * 8
    unet = PackedUNet(cfg, sd, device=dev)
    cm = ConceptModels(unet)
    loras, keys = [], []
    for k in range(2):
        lo = {n: (a.half().float().cpu(), b.half().float().cpu(), s)
              for n, (a, b, s) in synthetic.make_lora(cfg, seed=1000 + k, rank=16, device=dev, conv=True).items()}
        path = str(tmp_path / f"c{k}.safetensors")
        _kohya_sgm_file(cfg, lo, path)
        cm.load_lora_weights(path, adapter_name=f"c{k}")
        assert cm.skipped_lora_keys == []
        cm.set_adapters([f"c{k}"])
        keys.append(cm.active_lora_key(0.8))
        loras.append(lo)
    g = torch.Generator().manual_seed(0)
    ctx = torch.randn(8, 77, 2048, generator=g).half().float()
    pooled = torch.randn(8, 1280, generator=g).half().float()
    tid = torch.tensor([[size, size, 0, 0, size, size]], dtype=torch.float32).repeat(8, 1)
    sched = EulerDiscrete()
    ts = sched.set_timesteps(30)
    i = 16
    lat = (torch.randn(2, 4, H, W, generator=g) * float(sched.sigmas[i])).half().float()
    lmi = sched.scale_model_input(torch.cat([lat] * 2), i).half().float()
    xin = torch.cat([lmi, lmi[3:4], lmi[3:4], lmi[3:4], lmi[3:4]])
    masks = []
    for k in range(2):
        m = torch.zeros(size, size)
        m[:, k * size // 2:(k + 1) * size // 2 - 32] = 1
        masks.append(m)
    groups = [RowGroup(0, 4, None), RowGroup(4, 6, keys[0]), RowGroup(6, 8, keys[1])]
    r = UNetRunner(unet, 8, H, W, use_graphs=False, groups=groups)
    r.set_conditioning([float(ts[i])], [(ctx[g_.start:g_.stop], g_.lora_key, False) for g_ in groups], pooled, tid)
    r.sample_in.copy_(to_nhwc8(xin))
    assert r._conv_planes("down0.w")[0].shape == (3 * 320, 9 * 320)
    noise = r.forward(0)
    lat_dev = lat.permute(0, 2, 3, 1).contiguous().to(dev)
    m_lat = [(F.interpolate(m[None, None], size=(H, W), mode="nearest")[0, 0] == 1).float().reshape(-1).to(dev) for m in masks]
    ops.fuse_step(noise[0:4], [noise[4:6], noise[6:8]], m_lat, 7.5, float(sched.sigmas[i]), float(sched.sigmas[i + 1]), lat_dev)
    torch.cuda.synchronize()
    noise_gpu = from_nhwc(noise)
    sd32 = {k: v.float() for k, v in sd.items()}
    oc = ou.UNetConfig()
    d = lambda t: t.to(dev)  # noqa: E731
    effects = []
    with torch.no_grad():
        refs = [ou.unet_forward(ou.Ctx(sd32, oc), d(xin[:4]), float(ts[i]), d(ctx[:4]), d(pooled[:4]), d(tid[:4]))]
        for k in range(2):
            olo = {n: [(d(a), d(b), s * 0.8)] for n, (a, b, s) in loras[k].items()}
            sl = slice(4 + 2 * k, 6 + 2 * k)
            refs.append(ou.unet_forward(ou.Ctx(sd32, oc, lora=olo), d(xin[sl]), float(ts[i]), d(ctx[sl]), d(pooled[sl]), d(tid[sl])))
            lin = {n: v for n, v in olo.items() if v[0][0].dim() == 2 and not n.endswith("time_emb_proj")}
            nolocon = ou.unet_forward(ou.Ctx(sd32, oc, lora=lin), d(xin[sl]), float(ts[i]), d(ctx[sl]), d(pooled[sl]), d(tid[sl]))
            effects.append(rel(refs[-1], nolocon))
    refs = [t.cpu() for t in refs]
    fused = fuse_noise(refs[0], refs[1:], masks)
    nu, nt = fused.chunk(2)
    ref_lat = sched.step(nu + 7.5 * (nt - nu), i, lat)
    errs = [rel(noise_gpu[:4], refs[0]), rel(noise_gpu[4:6], refs[1]), rel(noise_gpu[6:8], refs[2])]
    e_lat = rel(lat_dev.permute(0, 3, 1, 2), ref_lat)
    print(f"sdxl-width locon step: noise rel err main {errs[0]:.3e}, concepts {errs[1]:.3e} {errs[2]:.3e}; latents {e_lat:.3e}; "
          f"the conv / time-embedding entries move the concept noise by {effects[0]:.3e} {effects[1]:.3e}")
    assert errs[0] < 2.2e-3 and max(errs[1:]) < 3.7e-3 and e_lat < 1.4e-3
    assert min(effects) > 5 * max(errs)
