"""CPU tests of LoCon adapters (LoRA on the ResBlock convs, time_emb_proj and the down- / up-sampler convs): target
table, the three key layouts of the loader, the un-merged conv LoRA of the oracle (tests/util_locon.py) against the merged weight, the packed
weight planes, and the row-group rule of omg_gemm on spatial grids (validated before any CUDA call, fake pointers)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from omg_b200 import checkpoints as ck
from omg_b200 import ops, synthetic
from omg_b200.config import UNetConfig, lora_conv_target_names, lora_target_names, param_shapes, resnet_names
from omg_b200.unet import merge_conv_lora, pack_conv_lora
from oracle import unet as ou
from util_locon import locon_oracle  # noqa: F401  (autouse: the oracle's conv applies LoCon entries)

_TAILS = {"conv1": "in_layers_2", "time_emb_proj": "emb_layers_1", "conv2": "out_layers_3",
          "conv_shortcut": "skip_connection"}


def _sgm_stem(cfg, path):
    """kohya stem with SGM block names of a LoCon module path, derived from the block structure independently of the
    loader's table."""
    p = path.split(".")
    lpb = cfg.layers_per_block
    nb = len(cfg.block_out_channels)
    if p[0] == "mid_block":
        return f"lora_unet_middle_block_{2 * int(p[2])}_{_TAILS[p[3]]}"
    blk = int(p[1])
    if p[0] == "down_blocks":
        if p[2] == "downsamplers":
            return f"lora_unet_input_blocks_{(blk + 1) * (lpb + 1)}_0_op"
        return f"lora_unet_input_blocks_{1 + blk * (lpb + 1) + int(p[3])}_0_{_TAILS[p[4]]}"
    if p[2] == "upsamplers":
        sub = 2 if cfg.transformer_layers[nb - 1 - blk] > 0 else 1
        return f"lora_unet_output_blocks_{blk * (lpb + 1) + lpb}_{sub}_conv"
    return f"lora_unet_output_blocks_{blk * (lpb + 1) + int(p[3])}_0_{_TAILS[p[4]]}"


def _file(cfg, lo, layout):
    linears = {n for n, _i, _o in lora_target_names(cfg)}
    sd = {}
    for name, (A, B, s) in lo.items():
        conv = A.dim() == 4
        up = B[:, :, None, None] if conv else B  # kohya / peft store a conv's up matrix as a 1x1 conv
        alpha = torch.tensor(s * A.shape[0])
        if layout == "peft":
            sd[f"unet.{name}.lora_A.weight"], sd[f"unet.{name}.lora_B.weight"], sd[f"unet.{name}.alpha"] = A, up, alpha
            continue
        if layout == "diffusers_old":
            sd[f"unet.{name}.lora.down.weight"], sd[f"unet.{name}.lora.up.weight"], sd[f"unet.{name}.alpha"] = A, up, alpha
            continue
        stem = "lora_unet_" + name.replace(".", "_")
        if layout == "kohya_sgm" and name not in linears:
            stem = _sgm_stem(cfg, name)
        sd[stem + ".lora_down.weight"], sd[stem + ".lora_up.weight"], sd[stem + ".alpha"] = A, up, alpha
    return sd


def test_target_table_sdxl():
    cfg = UNetConfig.sdxl()
    S = param_shapes(cfg)
    table = lora_conv_target_names(cfg)
    names = [t[0] for t in table]
    assert len(names) == len(set(names))
    n_res = len(resnet_names(cfg))
    n_sc = sum(1 for k in S if k.endswith("conv_shortcut.weight"))
    assert len(table) == 3 * n_res + n_sc + 4 and n_res == 17
    for name, kind, i, o, k in table:
        shp = S[name + ".weight"]
        assert (shp[1], shp[0]) == (i, o) and (kind == "linear") == (len(shp) == 2) and k == (1 if len(shp) == 2 else shp[2])
    assert not any(n.startswith(("conv_in", "conv_out", "time_embedding", "add_embedding")) for n in names)
    assert ("up_blocks.0.resnets.0.conv_shortcut", "conv", 2560, 1280, 1) in table
    assert ("down_blocks.1.downsamplers.0.conv", "conv", 640, 640, 3) in table
    assert not set(names) & {n for n, _i, _o in lora_target_names(cfg)}


def test_sgm_names_resolve_for_every_module_of_sdxl():
    cfg = UNetConfig.sdxl()
    table = ck._kohya_conv_lookup(cfg)
    for name, *_ in lora_conv_target_names(cfg):
        assert table[_sgm_stem(cfg, name)] == name
        assert table["lora_unet_" + name.replace(".", "_")] == name
    # the spellings a kohya SDXL file uses
    assert table["lora_unet_input_blocks_4_0_in_layers_2"] == "down_blocks.1.resnets.0.conv1"
    assert table["lora_unet_input_blocks_4_0_emb_layers_1"] == "down_blocks.1.resnets.0.time_emb_proj"
    assert table["lora_unet_input_blocks_4_0_out_layers_3"] == "down_blocks.1.resnets.0.conv2"
    assert table["lora_unet_input_blocks_4_0_skip_connection"] == "down_blocks.1.resnets.0.conv_shortcut"
    assert table["lora_unet_input_blocks_3_0_op"] == "down_blocks.0.downsamplers.0.conv"
    assert table["lora_unet_output_blocks_2_2_conv"] == "up_blocks.0.upsamplers.0.conv"
    assert table["lora_unet_output_blocks_5_2_conv"] == "up_blocks.1.upsamplers.0.conv"
    assert table["lora_unet_middle_block_2_in_layers_2"] == "mid_block.resnets.1.conv1"
    assert "lora_unet_input_blocks_1_0_skip_connection" not in table   # 320 -> 320: no shortcut conv


@pytest.mark.parametrize("cfg", [UNetConfig.sdxl(), UNetConfig.tiny()], ids=["sdxl", "tiny"])
def test_layouts_convert_to_the_same_dict(cfg):
    lo = synthetic.make_lora(cfg, 3, rank=2, alpha=1.0, conv=True)
    assert set(lo) == {n for n, _i, _o in lora_target_names(cfg)} | {t[0] for t in lora_conv_target_names(cfg)}
    for layout in ("kohya_diffusers", "kohya_sgm", "peft", "diffusers_old"):
        got, te, skipped = ck.convert_lora_state_dict(_file(cfg, lo, layout), cfg, conv=True)
        assert not skipped and not te and set(got) == set(lo), layout
        for name, (A, B, s) in lo.items():
            a, b, sc = got[name]
            assert torch.equal(a, A) and torch.equal(b, B) and sc == pytest.approx(s), (layout, name)
        # without conv=True the same file gives the transformer Linears and skips the rest, as before
        got0, _te, skipped0 = ck.convert_lora_state_dict(_file(cfg, lo, layout), cfg)
        assert set(got0) == {n for n, _i, _o in lora_target_names(cfg)}
        assert len(skipped0) == 3 * len(lora_conv_target_names(cfg))
        with pytest.raises(ValueError):
            ck.convert_lora_state_dict(_file(cfg, lo, layout), cfg, strict=True)


def test_make_lora_conv_keeps_the_linear_entries():
    cfg = UNetConfig.tiny()
    a, b = synthetic.make_lora(cfg, 5, rank=4), synthetic.make_lora(cfg, 5, rank=4, conv=True)
    assert all(torch.equal(a[k][0], b[k][0]) and torch.equal(a[k][1], b[k][1]) for k in a)
    A, Bm, s = b["down_blocks.1.resnets.0.conv1"]
    assert A.shape == (4, 64, 3, 3) and Bm.shape == (128, 4) and s == 1.0
    assert b["down_blocks.1.resnets.0.time_emb_proj"][0].shape == (4, cfg.time_embed_dim)
    assert b["down_blocks.1.resnets.0.conv_shortcut"][0].shape == (4, 64, 1, 1)


def test_malformed_conv_entries_are_rejected():
    cfg = UNetConfig.tiny()
    stem = "lora_unet_down_blocks_1_resnets_0_conv1"   # 64 -> 128, 3x3
    good = {stem + ".lora_down.weight": torch.zeros(4, 64, 3, 3), stem + ".lora_up.weight": torch.zeros(128, 4, 1, 1)}
    assert set(ck.convert_lora_state_dict(good, cfg, conv=True)[0]) == {"down_blocks.1.resnets.0.conv1"}
    with pytest.raises(ValueError, match="up kernel is \\(3, 3\\)"):
        ck.convert_lora_state_dict({**good, stem + ".lora_up.weight": torch.zeros(128, 4, 3, 3)}, cfg, conv=True)
    with pytest.raises(ValueError, match="expected in=64, out=128"):
        ck.convert_lora_state_dict({**good, stem + ".lora_down.weight": torch.zeros(4, 32, 3, 3)}, cfg, conv=True)
    with pytest.raises(ValueError, match="expected in=64, out=128"):
        ck.convert_lora_state_dict({**good, stem + ".lora_up.weight": torch.zeros(64, 4, 1, 1)}, cfg, conv=True)
    with pytest.raises(ValueError, match="3x3 down kernel"):
        ck.convert_lora_state_dict({**good, stem + ".lora_down.weight": torch.zeros(4, 64, 1, 1)}, cfg, conv=True)
    with pytest.raises(ValueError, match="lacks its up matrix"):
        ck.convert_lora_state_dict({stem + ".lora_down.weight": torch.zeros(4, 64, 3, 3)}, cfg, conv=True)
    # conv_in is not a target: skipped, and an error under strict
    other = {"lora_unet_conv_in.lora_down.weight": torch.zeros(4, 4, 3, 3), "lora_unet_conv_in.lora_up.weight": torch.zeros(64, 4, 1, 1)}
    assert len(ck.convert_lora_state_dict(other, cfg, conv=True)[2]) == 2
    with pytest.raises(ValueError):
        ck.convert_lora_state_dict(other, cfg, strict=True, conv=True)


def test_resolve_lora_reports_what_it_ignores(tmp_path, capsys):
    from safetensors.torch import save_file
    from omg_b200.pipelines import _resolve_lora
    cfg = UNetConfig.tiny()
    lo = synthetic.make_lora(cfg, 1, rank=2, conv=True)
    sd = _file(cfg, lo, "kohya_sgm")
    path = str(tmp_path / "locon.safetensors")
    save_file({k: v.contiguous() for k, v in sd.items()}, path)

    class Owner:
        class unet:
            pass
    Owner.unet.cfg = cfg
    o = Owner()
    got = _resolve_lora(o, path, "c0", None)
    assert set(got) == set(lo) and o.skipped_lora_keys == [] and capsys.readouterr().err == ""
    sd["lora_unet_conv_in.lora_down.weight"] = torch.zeros(2, 4, 3, 3)
    sd["lora_unet_conv_in.lora_up.weight"] = torch.zeros(64, 2, 1, 1)
    save_file({k: v.contiguous() for k, v in sd.items()}, path)
    _resolve_lora(o, path, "c0", None)
    err = capsys.readouterr().err
    assert len(o.skipped_lora_keys) == 2 and "2 LoRA tensors" in err and "lora_unet_conv_in" in err


# ------------------------------------------------------------------------------------------------ oracle
def _merged(W, loras):
    """W + sum s B A as a conv weight: A [r, in, k, k], B [out, r]."""
    return W + sum(s * torch.einsum("or,rikl->oikl", Bm, A) for A, Bm, s in loras)


@pytest.mark.parametrize("case", ["stride1", "stride2", "shortcut1x1", "upsample"])
def test_oracle_unmerged_conv_lora_equals_merged_weight(case):
    g = torch.Generator().manual_seed(0)
    cin, cout, k = 12, 20, 1 if case == "shortcut1x1" else 3
    W = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64)
    bias = torch.randn(cout, generator=g, dtype=torch.float64)
    x = torch.randn(2, cin, 10, 10, generator=g, dtype=torch.float64)
    loras = [(torch.randn(r, cin, k, k, generator=g, dtype=torch.float64), torch.randn(cout, r, generator=g, dtype=torch.float64), s)
             for r, s in ((3, 0.7 * 0.8), (5, 0.5 * 0.8))]     # two adapters, weights [0.7, 0.5], scale 0.8
    stride, padding = (2 if case == "stride2" else 1), k // 2
    if case == "upsample":
        x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    c = ou.Ctx({"m.weight": W, "m.bias": bias}, ou.UNetConfig.tiny(), lora={"m": loras})
    got = ou.conv(c, "m", x, stride=stride, padding=padding)
    ref = F.conv2d(x, _merged(W, loras), bias, stride=stride, padding=padding)
    plain = F.conv2d(x, W, bias, stride=stride, padding=padding)
    assert got.shape == ref.shape
    assert (got - ref).abs().max() < 1e-11 * ref.abs().max() and (ref - plain).abs().max() > 0.1
    c32 = ou.Ctx({"m.weight": W.float(), "m.bias": bias.float()}, ou.UNetConfig.tiny(),
                 lora={"m": [(A.float(), Bm.float(), s) for A, Bm, s in loras]})
    got32 = ou.conv(c32, "m", x.float(), stride=stride, padding=padding)
    assert ((got32 - ref).norm() / ref.norm()).item() < 2e-6   # fp32 round-off


def test_oracle_resnet_uses_every_locon_module():
    """Each of conv1 / conv2 / conv_shortcut / time_emb_proj of a ResBlock moves the oracle's output."""
    cfg = UNetConfig.tiny()
    sd = synthetic.make_state_dict(cfg, 0)
    lo = synthetic.make_lora(cfg, 2, rank=4, conv=True)
    name = "down_blocks.1.resnets.0"
    g = torch.Generator().manual_seed(1)
    x, emb = torch.randn(1, 64, 8, 8, generator=g), torch.randn(1, cfg.time_embed_dim, generator=g)
    base = ou.resnet(ou.Ctx(sd, ou.UNetConfig.tiny()), name, x, emb)
    for leaf in ("conv1", "conv2", "conv_shortcut", "time_emb_proj"):
        A, Bm, s = lo[f"{name}.{leaf}"]
        y = ou.resnet(ou.Ctx(sd, ou.UNetConfig.tiny(), lora={f"{name}.{leaf}": [(A, Bm, s)]}), name, x, emb)
        assert ((y - base).norm() / base.norm()).item() > 1e-3, leaf


# ------------------------------------------------------------------------------------------------ packing
def test_merged_planes_equal_the_packed_merged_weight():
    cfg = UNetConfig.tiny()
    sd = synthetic.make_state_dict(cfg, 0)
    la, ls = synthetic.make_lora(cfg, 11, rank=4, conv=True), synthetic.make_lora(cfg, 12, rank=3, conv=True)
    adapters, gs = [(la, 0.7), (ls, 0.5)], 0.8
    packed = pack_conv_lora(cfg, adapters, gs)

    def merged(path):
        return _merged(sd[path + ".weight"], [(lo[path][0], lo[path][1], lo[path][2] * w * gs) for lo, w in adapters])

    res = [n for n, _c in resnet_names(cfg)]
    assert set(packed) == {f"{n}.w1" for n in res} | {f"{n}.w2" for n in res} | {"down0.w", "down1.w", "up0.w", "up1.w", "temb_all.w"}
    for key, path in (("down_blocks.1.resnets.0.w1", "down_blocks.1.resnets.0.conv1"), ("down1.w", "down_blocks.1.downsamplers.0.conv"),
                      ("up0.w", "up_blocks.0.upsamplers.0.conv"), ("up_blocks.1.resnets.2.w1", "up_blocks.1.resnets.2.conv1")):
        got = merge_conv_lora(ops.pack_conv3x3_weight(sd[path + ".weight"]), packed[key])
        assert torch.allclose(got, ops.pack_conv3x3_weight(merged(path)), rtol=1e-5, atol=1e-6), key
    # conv2 with the conv_shortcut behind its columns (up block: the shortcut sees cat([h, skip]))
    for n in ("down_blocks.1.resnets.0", "up_blocks.0.resnets.1"):
        w2 = torch.cat([ops.pack_conv3x3_weight(sd[n + ".conv2.weight"]), sd[n + ".conv_shortcut.weight"].flatten(1)], dim=1)
        ref = torch.cat([ops.pack_conv3x3_weight(merged(n + ".conv2")), merged(n + ".conv_shortcut").flatten(1)], dim=1)
        got = merge_conv_lora(w2, packed[n + ".w2"])
        assert torch.allclose(got, ref, rtol=1e-5, atol=1e-6) and not torch.allclose(got[:, -8:], w2[:, -8:])
    # a ResBlock without shortcut has the conv2 entry only
    assert len(packed["down_blocks.0.resnets.0.w2"]) == 1 and len(packed["down_blocks.1.resnets.0.w2"]) == 2
    # time_emb_proj: every ResBlock's rows of the concatenation
    temb = torch.cat([sd[n + ".time_emb_proj.weight"] for n in res], dim=0)
    ref = torch.cat([sd[n + ".time_emb_proj.weight"] + sum(lo[n + ".time_emb_proj"][2] * w * gs * lo[n + ".time_emb_proj"][1] @ lo[n + ".time_emb_proj"][0]
                                                           for lo, w in adapters) for n in res], dim=0)
    assert torch.allclose(merge_conv_lora(temb, packed["temb_all.w"]), ref, rtol=1e-5, atol=1e-6)
    # fp16 base: merged in fp32, rounded once
    w16 = ops.pack_conv3x3_weight(sd["down_blocks.1.downsamplers.0.conv.weight"]).half()
    got16 = merge_conv_lora(w16, packed["down1.w"])
    dW = sum(Bm @ A for A, Bm, _r, _c in packed["down1.w"])
    assert got16.dtype == torch.float16 and torch.equal(got16, (w16.float() + dW).half())
    # a transformer-only adapter packs to nothing
    assert pack_conv_lora(cfg, [(synthetic.make_lora(cfg, 11, rank=4), 1.0)]) == {}


# ------------------------------------------------------------------------------------------------ descriptor
def _desc(L, W, H, B):
    """A conv-like descriptor over a (W, H, B) output grid that passes every check up to the fp32-twin stride check,
    which comes after the row-group rule and before any CUDA call: with out_f32_ld = 6 a descriptor whose groups are
    accepted still ends there, so nothing is ever launched on the fake pointers."""
    d = L.GemmDesc()
    d.n_a, d.n_segs = 1, 1
    d.a[0] = L.View4(0x1000, 64, W, H, B, 64, 64 * W, 64 * W * H)
    d.segs[0] = L.Seg(0, 0, 0, 0, 64, 0, 0)
    d.w, d.N, d.Ktot = 0x2000, 64, 64
    d.d = L.View4(0x3000, 64, W, H, B, 64, 64 * W, 64 * W * H)
    d.out_f32, d.out_f32_ld = 0x4000, 6
    return d


def _err(lib, d):
    assert lib.omg_gemm(C.byref(d), None) == 1
    return lib.omg_last_error().decode()


def test_row_groups_on_a_spatial_grid_are_whole_images():
    from omg_b200 import _lib as L
    lib = L.load()
    d = _desc(L, 8, 8, 8)                      # 8 x 8 images: 64 pixels each, 4 + 2 + 2 images
    d.w_group_planes = d.n_col_groups = 3
    d.col_group_end[0], d.col_group_end[1], d.col_group_end[2] = 4 * 64, 6 * 64, 8 * 64
    assert "fp32 twin row strides" in _err(lib, d)          # 192 + 64 k is no multiple of 128, and legal here
    d.col_group_end[0] = 3 * 64
    assert "fp32 twin row strides" in _err(lib, d)
    d.col_group_end[1] = 6 * 64 - 32
    e = _err(lib, d)
    assert "row-group boundary 352 is inside an image of the 8 x 8 output grid" in e and "multiples of 64 pixels" in e
    d2 = _desc(L, 16, 16, 4)                   # a multiple of the 128-row tile is not enough on a 16 x 16 grid
    d2.w_group_planes = d2.n_col_groups = 2
    d2.col_group_end[0], d2.col_group_end[1] = 128, 1024
    assert "row-group boundary 128 is inside an image of the 16 x 16 output grid" in _err(lib, d2)
    d2.col_group_end[0] = 512
    assert "fp32 twin row strides" in _err(lib, d2)


def test_row_groups_on_a_token_grid_keep_the_128_row_rule():
    from omg_b200 import _lib as L
    lib = L.load()
    d = _desc(L, 512, 1, 1)
    d.w_group_planes = d.n_col_groups = 2
    d.col_group_end[0], d.col_group_end[1] = 192, 512
    assert "row-group boundary 192 is not a multiple of the 128-row tile" in _err(lib, d)
    d.col_group_end[0] = 128
    assert "fp32 twin row strides" in _err(lib, d)
    d.w2, d.K2tot = 0x5000, 64
    assert "weight planes do not extend to the second weight matrix" in _err(lib, d)
    d.w2, d.K2tot = None, 0
    d.w_group_planes = 3
    assert "w_group_planes must equal n_col_groups" in _err(lib, d)
