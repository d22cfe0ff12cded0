"""CPU checks of the original-SAM model layer: topology inference of the packed encoder, the registry's ValueErrors,
ResizeLongestSide's coordinate transforms, and the CLIs' --segment_type dispatch."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _shape_sd(kind):
    """`image_encoder.*` keys and shapes of build_sam's `kind` (meta tensors: no memory)."""
    from omg_b200.sam_vit import KINDS
    C, depth, heads, glob = KINDS[kind]
    hd = C // heads
    e = lambda *s: torch.empty(*s, device="meta")  # noqa: E731
    sd = {"image_encoder.patch_embed.proj.weight": e(C, 3, 16, 16), "image_encoder.pos_embed": e(1, 64, 64, C)}
    for i in range(depth):
        n = 127 if i in glob else 27
        sd[f"image_encoder.blocks.{i}.attn.rel_pos_h"] = e(n, hd)
        sd[f"image_encoder.blocks.{i}.attn.rel_pos_w"] = e(n, hd)
    return sd


@pytest.mark.parametrize("kind,want", [("vit_b", (768, 12, 12, 64, (2, 5, 8, 11))),
                                       ("vit_l", (1024, 24, 16, 64, (5, 11, 17, 23))),
                                       ("vit_h", (1280, 32, 16, 80, (7, 15, 23, 31)))])
def test_packed_encoder_reads_the_topology_off_the_state_dict(kind, want):
    from omg_b200.sam_vit import topology_kind, vit_topology
    sd = _shape_sd(kind)
    assert vit_topology(sd) == want
    assert topology_kind(sd) == kind
    assert vit_topology({k[len("image_encoder."):]: v for k, v in sd.items()}) == want   # prefix optional


def test_malformed_state_dicts_raise_value_error():
    from omg_b200.sam_vit import topology_kind, vit_topology
    sd = _shape_sd("vit_b")
    with pytest.raises(ValueError, match="not a SAM ViT"):
        vit_topology({k: v for k, v in sd.items() if "blocks.3." not in k})           # a missing block
    with pytest.raises(ValueError, match="not a SAM ViT"):
        vit_topology({"prompt_encoder.x": torch.empty(1, device="meta")})            # no image encoder at all
    bad = dict(sd)
    bad["image_encoder.blocks.4.attn.rel_pos_h"] = torch.empty(31, 64, device="meta")  # interpolated table
    with pytest.raises(ValueError, match="rel_pos_h rows"):
        vit_topology(bad)
    odd = dict(sd)
    odd["image_encoder.blocks.3.attn.rel_pos_h"] = torch.empty(127, 64, device="meta")  # an extra global block
    with pytest.raises(ValueError, match="none of"):
        topology_kind(odd)


@pytest.mark.parametrize("builder,kind", [("build_sam_vit_b", "vit_h"), ("build_sam_vit_h", "vit_l"),
                                          ("build_sam", "vit_b"), ("build_sam_vit_l", "vit_b")])
def test_registry_rejects_a_checkpoint_of_another_kind(builder, kind):
    from omg_b200 import sam
    with pytest.raises(ValueError, match=f"is a SAM {kind} image encoder"):
        getattr(sam, builder)(state_dict=_shape_sd(kind))


def test_registry_names():
    from omg_b200 import sam
    assert set(sam.sam_model_registry) == {"default", "vit_h", "vit_l", "vit_b"}
    assert sam.sam_model_registry["default"] is sam.build_sam_vit_h and sam.build_sam is sam.build_sam_vit_h
    with pytest.raises(ValueError, match="checkpoint="):
        sam.build_sam()


def test_resize_longest_side_transforms():
    from omg_b200.sam import ResizeLongestSide
    t = ResizeLongestSide(1024)
    assert t.get_preprocess_shape(640, 896, 1024) == (731, 1024)
    img = np.zeros((640, 896, 3), dtype=np.uint8)
    assert t.apply_image(img).shape == (731, 1024, 3)
    s = (1024 / 896, 731 / 640)
    pts = np.array([[100.0, 200.0], [896.0, 640.0]])
    assert np.allclose(t.apply_coords(pts, (640, 896)), pts * np.array(s))
    box = np.array([10.0, 20.0, 300.0, 400.0])
    assert np.allclose(t.apply_boxes(box, (640, 896)), box * np.array(s * 2))
    bt = torch.tensor([[10.0, 20.0, 300.0, 400.0], [0.0, 0.0, 896.0, 640.0]])
    assert torch.allclose(t.apply_boxes_torch(bt, (640, 896)), bt * torch.tensor(s * 2, dtype=torch.float32))
    assert torch.equal(bt, torch.tensor([[10.0, 20.0, 300.0, 400.0], [0.0, 0.0, 896.0, 640.0]]))   # not in place


def test_segment_type_selects_the_segmenter(monkeypatch):
    """GroundingDINO -> SamPredictor(build_sam(--sam_checkpoint)); anything else -> EfficientViT-SAM xl1, as the
    reference's else branch.  --synthetic builds ViT-H-shaped weights, ViT-B-shaped with --tiny."""
    from omg_b200 import sam, synthetic
    calls = []
    monkeypatch.setattr(sam, "build_sam", lambda checkpoint: calls.append(("build_sam", checkpoint)) or "vit")
    monkeypatch.setitem(sam.sam_model_registry, "vit_h", lambda state_dict: calls.append(("vit_h", state_dict)) or "vit")
    monkeypatch.setitem(sam.sam_model_registry, "vit_b", lambda state_dict: calls.append(("vit_b", state_dict)) or "vit")
    monkeypatch.setattr(synthetic, "make_sam_vit_state_dict", lambda kind, seed, **kw: f"sd-{kind}")
    monkeypatch.setattr(sam, "SamPredictor", lambda m: ("SamPredictor", m))
    monkeypatch.setattr(sam, "create_sam_model", lambda name, **kw: calls.append(("xl1", kw)) or "evit")
    monkeypatch.setattr(sam, "EfficientViTSamPredictor", lambda m: ("EfficientViTSamPredictor", m))
    monkeypatch.setattr(synthetic, "make_sam_state_dict", lambda seed: "sd-xl1")
    assert sam.make_segmenter("GroundingDINO", False, False, "xl1.pt", "vit_h.pth") == ("SamPredictor", "vit")
    assert calls.pop() == ("build_sam", "vit_h.pth")
    assert sam.make_segmenter("GroundingDINO", True, False, "xl1.pt", "vit_h.pth") == ("SamPredictor", "vit")
    assert calls.pop() == ("vit_h", "sd-vit_h")
    assert sam.make_segmenter("GroundingDINO", True, True, "xl1.pt", "vit_h.pth") == ("SamPredictor", "vit")
    assert calls.pop() == ("vit_b", "sd-vit_b")
    for kind in ("yoloworld", "groundingdino", ""):
        assert sam.make_segmenter(kind, False, False, "xl1.pt", "vit_h.pth") == ("EfficientViTSamPredictor", "evit")
        assert calls.pop() == ("xl1", {"weight_url": "xl1.pt"})


@pytest.mark.parametrize("fname", ["inference_lora.py", "inference_instantid.py"])
def test_both_clis_route_segment_type_to_the_segmenter(fname):
    """The flags parse with the reference's names and defaults, and each CLI hands them to make_segmenter."""
    spec = importlib.util.spec_from_file_location("cli_vit_" + fname[:-3], os.path.join(ROOT, fname))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    argv, sys.argv = sys.argv, [fname, "--segment_type", "GroundingDINO", "--sam_boxes", "1,2,3,4|"]
    try:
        ns = mod.parse_args()
    finally:
        sys.argv = argv
    assert ns.segment_type == "GroundingDINO" and ns.sam_checkpoint == "./checkpoint/sam/sam_vit_h_4b8939.pth"
    src = open(os.path.join(ROOT, fname)).read()
    assert "make_segmenter(args.segment_type, args.synthetic, args.tiny, args.efficientViT_checkpoint," in src
    assert "args.sam_checkpoint)" in src
