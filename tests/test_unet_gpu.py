"""GPU parity of the UNet / ControlNet executor and of both pipelines against the fp32 CPU oracle, tiny topology
(same code paths as SDXL: conv tails, GroupNorm over concatenated skips, P2P remaps, LoRA K-segments, IP-adapter,
ControlNet residuals).  Tolerance: relative L2 <= 1.9e-3 per UNet call (the largest error is the general
P2P two-term step; fp16 storage vs the fp32 oracle fed the same fp16-rounded weights)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from util_models import from_nhwc, lora, ocfg, oracle_lora, r16, rel, to_nhwc8, weights  # noqa: E402

TOL = 1.9e-3


@pytest.fixture(scope="module")
def env():
    from omg_b200.config import UNetConfig
    from omg_b200.unet import PackedUNet
    cfg = UNetConfig.tiny()
    sd = weights(cfg, 0)
    return {"cfg": cfg, "sd": sd, "model": PackedUNet(cfg, sd)}


def _inputs(cfg, B, H, W, seed, L=77):
    g = torch.Generator().manual_seed(seed)
    x = r16(torch.randn(B, 4, H, W, generator=g))
    ctx = r16(torch.randn(B, L, cfg.cross_attention_dim, generator=g))
    pooled = r16(torch.randn(B, cfg.pooled_dim, generator=g))
    tid = torch.tensor([[H * 8, W * 8, 0, 0, H * 8, W * 8]], dtype=torch.float32).repeat(B, 1)
    return x, ctx, pooled, tid


def test_plain_unet(env):
    from omg_b200.unet import UNetRunner
    from oracle import unet as ou
    cfg = env["cfg"]
    B, H, W = 2, 32, 32
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 1)
    r = UNetRunner(env["model"], B, H, W, use_graphs=False)
    r.set_conditioning([501.0, 7.0], ctx, pooled, tid)
    r.sample_in.copy_(to_nhwc8(x))
    for i, t in enumerate([501.0, 7.0]):
        out = from_nhwc(r.forward(i))
        ref = ou.unet_forward(ou.Ctx(env["sd"], ocfg(cfg)), x, t, ctx, pooled, tid)
        e = rel(out, ref)
        print("plain unet rel err", e)
        assert e < TOL


def test_fp32_trunk_twins(env):
    """Opt-in fp32 master copy of the residual trunk (UNetRunner.trunk_f32): the residual GEMMs read / write fp32 twins.
    Same bound as the default path on the tiny topology (the gain shows at SDXL depth, over many chained residual adds),
    and the twins are really used (results differ bitwise)."""
    from omg_b200.unet import UNetRunner
    from oracle import unet as ou
    cfg = env["cfg"]
    B, H, W = 2, 32, 32
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 1)
    outs = []
    for twin in (False, True):
        r = UNetRunner(env["model"], B, H, W, use_graphs=False)
        r.trunk_f32 = twin
        r.set_conditioning([501.0], ctx, pooled, tid)
        r.sample_in.copy_(to_nhwc8(x))
        outs.append(from_nhwc(r.forward(0)))
    ref = ou.unet_forward(ou.Ctx(env["sd"], ocfg(cfg)), x, 501.0, ctx, pooled, tid)
    e0, e1 = rel(outs[0], ref), rel(outs[1], ref)
    print("fp16 trunk rel err", e0, "fp32 twins rel err", e1)
    assert e0 < TOL and e1 < TOL and not torch.equal(outs[0], outs[1])


def test_graph_replay_matches_eager(env):
    from omg_b200.unet import UNetRunner
    cfg = env["cfg"]
    B, H, W = 2, 32, 32
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 2)
    r = UNetRunner(env["model"], B, H, W, use_graphs=True)
    r.set_conditioning([333.0], ctx, pooled, tid)
    r.sample_in.copy_(to_nhwc8(x))
    a = r.forward(0, key=("k",)).clone()     # eager warm-up
    b = r.forward(0, key=("k",)).clone()     # capture + replay
    c = r.forward(0, key=("k",)).clone()     # replay
    assert torch.equal(a, b) and torch.equal(b, c)


def test_launch_plan_replay_matches_eager(env):
    """The forward as a C-ABI handle (omg_plan): recorded once, replayed from C.  Bit-identical to the eager launches, one
    plan step per entry-point call (omg_groupnorm_apply is two kernels), no pointer into freed memory (the allocator is churned between recording and replay),
    and a replay recomputes (a new input gives the eager result for that input)."""
    from omg_b200 import _lib as L
    from omg_b200.unet import UNetRunner
    cfg = env["cfg"]
    B, H, W = 2, 32, 32
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 2)
    x2 = _inputs(cfg, B, H, W, 3)[0]
    e = UNetRunner(env["model"], B, H, W, use_graphs=False)
    e.set_conditioning([333.0], ctx, pooled, tid)
    e.sample_in.copy_(to_nhwc8(x))
    n0 = L.launch_count()
    ref1 = e.forward(0).clone()
    launches = L.launch_count() - n0
    e.sample_in.copy_(to_nhwc8(x2))
    ref2 = e.forward(0).clone()
    r = UNetRunner(env["model"], B, H, W, use_graphs=False, use_plans=True)
    r.set_conditioning([333.0], ctx, pooled, tid)
    r.sample_in.copy_(to_nhwc8(x))
    a = r.forward(0, key=("k",)).clone()     # eager warm-up
    b = r.forward(0, key=("k",)).clone()     # eager + recording
    assert 0 < len(r.plans[("k",)]) <= launches
    junk = [torch.randn(1 << 20, device="cuda") for _ in range(16)]   # churn the caching allocator
    del junk
    junk = [torch.full((3 << 18,), float("nan"), device="cuda") for _ in range(24)]
    n1 = L.launch_count()
    c = r.forward(0, key=("k",)).clone()     # replay from C
    assert L.launch_count() - n1 == launches
    assert torch.equal(a, ref1) and torch.equal(b, ref1) and torch.equal(c, ref1)
    r.sample_in.copy_(to_nhwc8(x2))
    d = r.forward(0, key=("k",)).clone()
    assert torch.equal(d, ref2) and not torch.equal(d, ref1)
    del junk


def test_main_unet_p2p(env):
    """B=4 rows (u0,u1,c0,c1) under AttentionReplace: self-replace window on (step 0) and off (step 25)."""
    from omg_b200.prompt_attention import AttentionReplace
    from omg_b200.pipelines import LoraMultiConceptPipeline, revise_regionally_controlnet_forward
    from oracle import p2p as op2p
    from oracle import unet as ou
    cfg = env["cfg"]
    H = W = 32
    x1, ctx2, pooled2, tid = _inputs(cfg, 2, H, W, 3)
    x = torch.cat([x1[:1], x1[1:2], x1[:1], x1[1:2]])
    ctx = torch.cat([ctx2[:1], ctx2[:1], ctx2[1:], ctx2[1:]])        # [neg, neg, pos, pos]
    pooled = torch.cat([pooled2[:1], pooled2[:1], pooled2[1:], pooled2[1:]])
    tid = tid[:1].repeat(4, 1)
    prompts = ["a b c"] * 2
    for step in (0, 25):
        pipe = LoraMultiConceptPipeline(env["model"], use_graphs=False)
        ctrl = AttentionReplace(prompts, 50, {"default_": 1.0}, 0.4, 8, 8)
        revise_regionally_controlnet_forward(pipe, ctrl)
        ctrl.cur_step = step
        main = pipe._runner("main", env["model"], 4, H, W)
        pipe._update_p2p_context(main, ctrl, ctx, first=True)
        main.set_conditioning([400.0], ctx, pooled, tid, extra_ctx=pipe._p2p_rows)
        main.sample_in.copy_(to_nhwc8(x))
        variant, _ = pipe._p2p_variant(main, ctrl, False)
        out = from_nhwc(main.forward(0, variant))
        octrl = op2p.AttentionReplaceOracle(prompts, 50, {"default_": 1.0}, 0.4, 8, 8)
        octrl.num_att_layers = len(ou.attention_names(ocfg(cfg)))
        octrl.cur_step = step
        c = ou.Ctx(env["sd"], ocfg(cfg), attn_core=ou.make_p2p_attn_core(octrl))
        ref = ou.unet_forward(c, x, 400.0, ctx, pooled, tid)
        e = rel(out, ref)
        print(f"p2p main unet step {step} rel err", e)
        assert e < TOL
        assert octrl.cur_step == step + 1
        # shipped config: image-1 cond row equals image-0 cond row while self-replace is on for all layers? no:
        # only layers with <= 64 tokens are replaced, so rows differ; the uncond half is never touched
        assert rel(out[0], ref[0]) < TOL and rel(out[3], ref[3]) < TOL


def test_p2p_general_cross_edit(env):
    """alpha < 1 for some tokens and a non-identity mapper: two-term cross-attention path."""
    from omg_b200.prompt_attention import AttentionReplace
    from omg_b200.pipelines import LoraMultiConceptPipeline, revise_regionally_controlnet_forward
    from oracle import p2p as op2p
    from oracle import unet as ou
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_golden import ToyTokenizer
    cfg = env["cfg"]
    H = W = 16
    g = torch.Generator().manual_seed(5)
    x = r16(torch.randn(4, 4, H, W, generator=g))
    ctx = r16(torch.randn(4, 77, cfg.cross_attention_dim, generator=g))
    pooled = r16(torch.randn(4, cfg.pooled_dim, generator=g))
    tid = torch.tensor([[128, 128, 0, 0, 128, 128]], dtype=torch.float32).repeat(4, 1)
    prompts = ["a photo of a man on the beach", "a photo of a dog on the beach"]
    cross = {"default_": 0.6, "dog": (0.2, 0.9)}
    for step in (1, 7):
        pipe = LoraMultiConceptPipeline(env["model"], use_graphs=False)
        ctrl = AttentionReplace(prompts, 10, dict(cross), 0.3, 4, 4, tokenizer=ToyTokenizer())
        revise_regionally_controlnet_forward(pipe, ctrl)
        ctrl.cur_step = step
        main = pipe._runner("main", env["model"], 4, H, W)
        pipe._update_p2p_context(main, ctrl, ctx, first=True)
        main.set_conditioning([400.0], ctx, pooled, tid, extra_ctx=pipe._p2p_rows)
        main.sample_in.copy_(to_nhwc8(x))
        variant, _ = pipe._p2p_variant(main, ctrl, False)
        out = from_nhwc(main.forward(0, variant))
        octrl = op2p.AttentionReplaceOracle(prompts, 10, dict(cross), 0.3, 4, 4, tokenizer=ToyTokenizer())
        octrl.num_att_layers = len(ou.attention_names(ocfg(cfg)))
        octrl.cur_step = step
        c = ou.Ctx(env["sd"], ocfg(cfg), attn_core=ou.make_p2p_attn_core(octrl))
        ref = ou.unet_forward(c, x, 400.0, ctx, pooled, tid)
        e = rel(out, ref)
        print(f"general p2p step {step} two_terms={pipe._cross_two_terms} rel err", e)
        assert e < TOL


def test_concept_unet_lora(env):
    from omg_b200.unet import PackedUNet, UNetRunner
    from oracle import unet as ou
    cfg = env["cfg"]
    B, H, W = 2, 32, 32
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 7)
    la, ls = lora(cfg, 11), lora(cfg, 12)
    model = PackedUNet(cfg, env["sd"])
    model.add_lora_set("c", [(la, 0.7), (ls, 0.5)], 0.8)
    c = ou.Ctx(env["sd"], ocfg(cfg), lora=oracle_lora([(la, 0.7), (ls, 0.5)], 0.8))
    ref = ou.unet_forward(c, x, 250.0, ctx, pooled, tid)
    base = ou.unet_forward(ou.Ctx(env["sd"], ocfg(cfg)), x, 250.0, ctx, pooled, tid)
    for merged in (True, False):   # per-stream merged weight planes / un-merged K-segment path
        r = UNetRunner(model, B, H, W, lora_key="c", use_graphs=False)
        r.merge_lora = merged
        r.set_conditioning([250.0], ctx, pooled, tid)
        r.sample_in.copy_(to_nhwc8(x))
        out = from_nhwc(r.forward(0))
        e = rel(out, ref)
        print("lora unet rel err", e, "merged" if merged else "unmerged", "lora effect", rel(ref, base))
        assert e < TOL and rel(ref, base) > 5 * e


def test_controlnet_and_residuals(env):
    from omg_b200.unet import PackedUNet, UNetRunner
    from oracle import unet as ou
    cfg = env["cfg"]
    B, H, W = 2, 16, 16
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 8)
    csd = weights(cfg, 21, controlnet=True)
    g = torch.Generator().manual_seed(9)
    cond = r16(torch.rand(B, 3, H * 8, W * 8, generator=g))
    cn = UNetRunner(PackedUNet(cfg, csd, controlnet=True), B, H, W, use_graphs=False)
    cn.set_conditioning([600.0], ctx, pooled, tid)
    cn.set_controlnet_cond(cond)
    cn.sample_in.copy_(to_nhwc8(x))
    down, mid = cn.forward(0)
    rd, rm = ou.controlnet_forward(ou.Ctx(csd, ocfg(cfg)), x, 600.0, ctx, cond, 0.8, pooled, tid)
    for a, b in zip(down + [mid], rd + [rm]):
        assert rel(from_nhwc(a, a.shape[-1]) * 0.8, b) < TOL
    r = UNetRunner(env["model"], B, H, W, use_graphs=False)
    r.set_conditioning([600.0], ctx, pooled, tid)
    r.sample_in.copy_(to_nhwc8(x))
    r.residuals_in = (down, mid, 0.8)
    v = r.default_variant()
    v["residuals"] = True
    out = from_nhwc(r.forward(0, v))
    ref = ou.unet_forward(ou.Ctx(env["sd"], ocfg(cfg)), x, 600.0, ctx, pooled, tid, rd, rm)
    e = rel(out, ref)
    print("controlnet+unet rel err", e)
    assert e < TOL


def test_ip_adapter_unet(env):
    from omg_b200 import synthetic
    from omg_b200.unet import PackedUNet, UNetRunner
    from oracle import unet as ou
    cfg = env["cfg"]
    B, H, W = 2, 16, 16
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 10, L=77 + 16)
    ipw = {k: (r16(a), r16(b)) for k, (a, b) in synthetic.make_ip_adapter(cfg, 31).items()}
    model = PackedUNet(cfg, env["sd"])
    model.set_ip_adapter(ipw, 0.8, 16)
    r = UNetRunner(model, B, H, W, use_graphs=False)
    r.set_conditioning([120.0], ctx, pooled, tid)
    r.sample_in.copy_(to_nhwc8(x))
    out = from_nhwc(r.forward(0))
    c = ou.Ctx(env["sd"], ocfg(cfg), ip_weights=ipw, ip_tokens=16, ip_scale=0.8)
    ref = ou.unet_forward(c, x, 120.0, ctx, pooled, tid)
    e = rel(out, ref)
    print("ip-adapter unet rel err", e)
    assert e < TOL
