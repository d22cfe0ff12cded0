"""CPU: the oracle restatements against golden vectors produced by the UNMODIFIED reference modules
(tests/golden/make_golden.py; the reference tree does not travel to the GPU box)."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_golden import ToyTokenizer, sha256_of  # noqa: E402  (pure helper; does not import the reference)

from oracle import p2p, unet  # noqa: E402
from oracle.resampler import resampler_forward  # noqa: E402
from oracle.scheduler import EulerDiscrete  # noqa: E402

G = os.path.join(os.path.dirname(__file__), "golden")


def _replay(ctrl, layers, steps, bh, seed):
    g = torch.Generator().manual_seed(seed)
    ctrl.num_att_layers = len(layers)
    rec = []
    for s in range(steps):
        for (is_cross, n, l) in layers:
            p = torch.softmax(torch.randn(bh, n, l, generator=g), dim=-1)
            out = ctrl(p.clone(), is_cross, "mid")
            rec.append((s, is_cross, p, out, ctrl.cur_step, ctrl.cur_att_layer))
    return rec


def test_p2p_shipped_config_matches_reference():
    d = torch.load(os.path.join(G, "p2p_same.pt"))
    ctrl = p2p.AttentionReplaceOracle(d["prompts"], 50, {"default_": 1.0}, 0.4, d["width"], d["height"],
                                      tokenizer=ToyTokenizer())
    assert torch.equal(ctrl.cross_replace_alpha, d["alpha"])
    assert torch.equal(ctrl.mapper, d["mapper"])
    assert tuple(ctrl.num_self_replace) == tuple(d["num_self_replace"]) == (0, 20)
    assert torch.equal(ctrl.mapper[0], torch.eye(77))            # SURVEY section 9.3
    assert ctrl.cross_replace_alpha.unique().tolist() == [1.0]
    rec = _replay(ctrl, d["layers"], 22, 4, seed=0)
    by_key = {(s, i % len(d["layers"])): r for i, r in enumerate(rec) for s in [r[0]]}
    n = 0
    for j, r in enumerate(d["records"]):
        li = j % len(d["layers"])
        mine = by_key[(r["step"], li)]
        assert torch.equal(mine[2], r["in"])
        assert torch.allclose(mine[3], r["out"], atol=1e-7)
        assert mine[4] == r["cur_step"] and mine[5] == r["cur_att_layer"]
        n += 1
    assert n == 16


def test_p2p_word_edit_matches_reference():
    d = torch.load(os.path.join(G, "p2p_edit.pt"))
    ctrl = p2p.AttentionReplaceOracle(d["prompts"], d["num_steps"], dict(d["cross"]), d["self"], d["width"],
                                      d["height"], tokenizer=ToyTokenizer())
    assert torch.equal(ctrl.cross_replace_alpha, d["alpha"])
    assert torch.equal(ctrl.mapper, d["mapper"])
    rec = _replay(ctrl, d["layers"], 10, 4, seed=1)
    assert len(rec) == len(d["records"])
    for mine, r in zip(rec, d["records"]):
        assert sha256_of(mine[2]) == r["in_sha256"]
        assert torch.allclose(mine[3], r["out"], atol=1e-6)
        assert mine[4] == r["cur_step"]


def test_p2p_length_mismatch_raises():
    with pytest.raises(ValueError):
        p2p.replacement_mapper(["a b c", "a b"], ToyTokenizer())


def test_ip_attention_matches_reference():
    d = torch.load(os.path.join(G, "ip_attn.pt"))
    cfg = unet.UNetConfig(head_dim=d["dim"] // d["heads"])
    sd = {"a." + k: v for k, v in d["attn"].items()}
    c = unet.Ctx(sd, cfg, ip_weights={"a": (d["ip"]["to_k_ip.weight"], d["ip"]["to_v_ip.weight"])},
                 ip_tokens=d["num_tokens"], ip_scale=d["scale"])
    y = unet.attention(c, "a", d["x"], d["ctx"])
    assert torch.allclose(y, d["y_ip"], atol=2e-6)
    assert torch.allclose(y, d["y_ip2"], atol=2e-6)
    c2 = unet.Ctx({"a." + k: v for k, v in d["attn_self"].items()}, cfg)
    assert torch.allclose(unet.attention(c2, "a", d["x"]), d["y_self"], atol=2e-6)


def test_resampler_matches_reference():
    d = torch.load(os.path.join(G, "resampler.pt"))
    d["sd"] = {k: v.float() for k, v in d["sd"].items()}  # stored as fp16 (fp16-representable values)
    y = resampler_forward(d["sd"], d["x"], d["heads"], d["dim_head"])
    assert torch.allclose(y, d["y"], atol=2e-6)


def test_sdxl_topology_counts():
    cfg = unet.UNetConfig.sdxl()
    n = sum(math.prod(s) for s in unet.param_shapes(cfg).values())
    assert n == 2_567_463_684                                   # SDXL-base UNet parameter count
    nc = sum(math.prod(s) for s in unet.param_shapes(cfg, controlnet=True).values())
    assert nc == 1_251_014_160                                  # SDXL ControlNet
    names = unet.attention_names(cfg)
    assert len(names) == 140 and sum(n_.endswith("attn2") for n_ in names) == 70
    assert abs(unet.unet_flops(cfg, 128, 128) / 1e12 - 6.761) < 2e-3
    assert abs(unet.unet_flops(cfg, 64, 64) / 1e12 - 1.589) < 2e-3


def test_euler_schedule_known_values():
    s = EulerDiscrete()
    sig_all = ((1 - s.alphas_cumprod) / s.alphas_cumprod) ** 0.5
    assert abs(float(sig_all[-1]) - 14.6146) < 1e-3             # the published SD/SDXL sigma_max
    ts = s.set_timesteps(30)
    assert ts[0].item() == 958.0 and ts[-1].item() == 1.0 and len(ts) == 30   # leading spacing, offset 1
    assert s.sigmas[-1].item() == 0.0 and len(s.sigmas) == 31
    assert abs(s.init_noise_sigma - math.sqrt(float(s.sigmas[0]) ** 2 + 1)) < 1e-6
    ts50 = s.set_timesteps(50)
    assert ts50[0].item() == 981.0
    x = torch.randn(2, 4, 8, 8)
    eps = torch.randn(2, 4, 8, 8)
    y = s.step(eps, 3, x)
    assert torch.allclose(y, x + eps * (s.sigmas[4] - s.sigmas[3]), atol=1e-5)


def test_draw_kps_multi_matches_the_reference_function():
    """IdentityNet condition image (inference_instantid.py:127-156): the CLI's renderer vs the golden image produced
    by the reference's own function on three faces (truncation to uint8 after each face included)."""
    import importlib.util
    import numpy as np
    pytest.importorskip("cv2")
    spec = importlib.util.spec_from_file_location(
        "omg_cli_instantid", os.path.join(os.path.dirname(__file__), "..", "inference_instantid.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "kps.npz"))
    got = cli.draw_kps_multi((256, 256), d["kps"].tolist())
    assert got.dtype == np.uint8 and got.shape == (256, 256, 3)
    assert np.array_equal(got, d["image"])


def _load_cli(name):
    import importlib.util
    spec = importlib.util.spec_from_file_location("omg_cli_" + name, os.path.join(os.path.dirname(__file__), "..", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_cli_prepare_text_and_region_mask_match_the_reference_functions():
    """prepare_text of both CLIs and the union-of-regions mask (lora_pipeline.py:673-681) against the outputs of the
    reference's own functions; the product computes the union from the per-concept binary latent masks."""
    from omg_b200.pipelines import _binary_latent_mask
    gold = torch.load(os.path.join(os.path.dirname(__file__), "golden", "cli.pt"))
    lora_cli, iid_cli = _load_cli("inference_lora"), _load_cli("inference_instantid")
    for s, want in gold["lora_prepare_text"]:
        assert lora_cli.prepare_text("P", s) == want
    for s, want in gold["instantid_prepare_text"]:
        assert iid_cli.prepare_text("P", s) == want
    for case in gold["region_mask"]:
        union = torch.zeros(case["h"], case["w"])
        for m in case["masks"]:
            b = _binary_latent_mask(m, case["h"], case["w"], "cpu")
            if b is not None:
                union = torch.maximum(union, b.reshape(case["h"], case["w"]).float())
        assert torch.equal(union, case["out"].float())
    # the oracle's own restatement of the same function
    from oracle.pipeline import get_region_mask as oracle_region_mask
    for case in gold["region_mask"]:
        assert torch.equal(oracle_region_mask(case["masks"], case["h"], case["w"]).float(), case["out"].float())


def test_noise_fusion_matches_the_reference_statements():
    """oracle.pipeline.fuse_noise + CFG against the output of the reference's own fusion / guidance statements
    (lora_pipeline.py:568-612, executed from the method's AST by make_golden.py): a concept without a mask is skipped,
    overlapping masks add up, non-binary mask values are outside the region."""
    from oracle.pipeline import fuse_noise
    d = torch.load(os.path.join(os.path.dirname(__file__), "golden", "fusion.pt"))
    fused = fuse_noise(d["noise_pred_in"], d["region_noise"], d["masks"])
    assert torch.equal(fused[[1, 3]], d["new_noise_pred"])
    nu, nt = fused.chunk(2)
    assert torch.allclose(nu + d["guidance_scale"] * (nt - nu), d["noise_after_cfg"], rtol=0, atol=1e-6)
    # what the concept UNets were fed: image 1's scaled latent twice, adapters [concept, style] at [0.7, 0.5]
    for sample, t, kw in d["unet_inputs"]:
        assert torch.equal(sample, torch.cat([d["latent_model_input"][3:4]] * 2)) and kw == {"scale": 0.8}
    assert [a[0][0] for a in d["adapters"]] == [["A", "style"], ["C", "style"]]


def test_region_processor_restatement_matches_the_reference_class():
    """RegionControlNet_AttnProcessor (lora_pipeline.py:61-133) + the reference's AttentionReplace, run from the
    reference source (tests/golden/region_attn.pt), against the fp32 restatement that the GPU test of
    omg_b200.processors.FusedRegionAttnProcessor uses as its expectation (materialised probabilities through the oracle
    controller).  Closes the chain reference class == restatement (here) ~= fused CUDA processor (test_processors_gpu)."""
    from make_golden import REGION_CASES, ShimAttention, region_case_inputs, region_case_setup
    d = torch.load(os.path.join(os.path.dirname(__file__), "golden", "region_attn.pt"))
    assert len(d["cases"]) == len(REGION_CASES)
    for idx, case in enumerate(d["cases"]):
        edit, is_cross, step = case["edit"], case["is_cross"], case["step"]
        assert (edit, is_cross, step) == REGION_CASES[idx]
        prompts, cross = region_case_setup(edit)
        x, ctx = region_case_inputs(idx, is_cross, d["dim"], d["ctx_dim"])
        a = ShimAttention(d["dim"], d["ctx_dim"] if is_cross else d["dim"], d["heads"])
        a.load_state_dict(d["attn_cross"] if is_cross else d["attn_self"])
        oc = p2p.AttentionReplaceOracle(prompts, 10, dict(cross), 0.3, 4, 4, tokenizer=ToyTokenizer())
        oc.num_att_layers, oc.cur_step = 2, step
        src = ctx if is_cross else x
        with torch.no_grad():
            q, k, v = a.to_q(x), a.to_k(src), a.to_v(src)
            pr = a.get_attention_scores(a.head_to_batch_dim(q), a.head_to_batch_dim(k))
            pr = oc(pr, is_cross, "mid")
            y = a.to_out[0](a.batch_to_head_dim(torch.bmm(pr, a.head_to_batch_dim(v))))
        assert oc.cur_att_layer == case["cur_att_layer"]
        assert torch.allclose(y, case["y"], rtol=0, atol=2e-6), (idx, float((y - case["y"]).abs().max()))


def test_instantid_concept_pass_matches_the_reference_statements(monkeypatch):
    """oracle.pipeline.concept_noises + fuse_noise + CFG against the reference's InstantID statements
    (instantid_pipeline.py:618-686, executed from the method's AST): what the IdentityNet and the concept UNet are
    called with - image 1's scaled latent twice, face tokens alone for the IdentityNet, [text | face] tokens for the
    UNet, the shared condition image and scale, the residual hand-over - and the fused, guided noise."""
    from oracle import pipeline as opipe
    d = torch.load(os.path.join(os.path.dirname(__file__), "golden", "fusion_iid.pt"))
    calls = {"cn": [], "un": []}
    cn_it, un_it = iter(d["controlnet_out"]), iter(d["unet_out"])

    def fake_controlnet(c, sample, t, ctx, cond, scale, text_embeds, time_ids):
        calls["cn"].append(dict(c=c, sample=sample, t=float(t), ctx=ctx, cond=cond, scale=scale, text_embeds=text_embeds,
                                time_ids=time_ids))
        down, mid = next(cn_it)
        return down, mid

    def fake_unet(c, sample, t, ctx, text_embeds, time_ids, down=None, mid=None):
        calls["un"].append(dict(c=c, sample=sample, t=float(t), ctx=ctx, text_embeds=text_embeds, time_ids=time_ids,
                                down=down, mid=mid))
        return next(un_it)

    monkeypatch.setattr(opipe, "controlnet_forward", fake_controlnet)
    monkeypatch.setattr(opipe, "unet_forward", fake_unet)
    concepts = [opipe.Concept(prompt_embeds=d["text"][k], add_text_embeds=d["pooled"][k], add_time_ids=d["time_ids"][k],
                              mask=d["masks"][k], unet=f"concept{k}", image_tokens=d["face"][k]) for k in range(3)]
    noises = opipe.concept_noises(d["latent_model_input"], d["t"], concepts, identitynet="identitynet",
                                  identity_cond=d["cond"], identity_scale=d["cond_scale"])
    assert noises[1] is None and len(calls["cn"]) == len(d["controlnet_calls"]) == 2
    for mine, ref in zip(calls["cn"], d["controlnet_calls"]):
        assert mine["c"] == "identitynet" and mine["t"] == ref["t"] and mine["scale"] == ref["scale"]
        for key in ("sample", "ctx", "cond", "text_embeds", "time_ids"):
            assert torch.equal(mine[key], ref[key]), key
    for k, (mine, ref) in enumerate(zip(calls["un"], d["unet_calls"])):
        assert mine["c"] == ("concept0", "concept2")[k] and mine["t"] == ref["t"] and ref["cross_attention_kwargs"] is None
        for key in ("sample", "ctx", "text_embeds", "time_ids", "mid"):
            assert torch.equal(mine[key], ref[key]), key
        assert all(torch.equal(a, b) for a, b in zip(mine["down"], ref["down"]))
    fused = opipe.fuse_noise(d["noise_pred_in"], noises, d["masks"])
    nu, nt = fused.chunk(2)
    assert torch.allclose(nu + d["guidance_scale"] * (nt - nu), d["noise_after_cfg"], rtol=0, atol=1e-6)
