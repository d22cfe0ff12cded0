"""CPU tests of the YOLO-World host code: the restricted checkpoint loader, the v1 / v2 layouts at every scale against
the oracle's modules, letterbox / scale_boxes geometry, the NMS restatements and supervision's with_nms."""
import math
import os
import pickle
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from omg_b200 import yolo_world as Y


def _fake_ultralytics_classes():
    """Classes at ultralytics' module paths, as a checkpoint pickles them (removed again by the caller)."""
    mods = {}
    for name in ("ultralytics", "ultralytics.nn", "ultralytics.nn.tasks", "ultralytics.nn.modules",
                 "ultralytics.nn.modules.conv"):
        mods[name] = types.ModuleType(name)

    class WorldModel(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.model = torch.nn.ModuleList([Conv()])
            self.yaml = {"nc": 80}

    class Conv(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.conv = torch.nn.Conv2d(3, 16, 3, bias=False)
            self.bn = torch.nn.BatchNorm2d(16)

    WorldModel.__module__, WorldModel.__qualname__ = "ultralytics.nn.tasks", "WorldModel"
    Conv.__module__, Conv.__qualname__ = "ultralytics.nn.modules.conv", "Conv"
    mods["ultralytics.nn.tasks"].WorldModel = WorldModel
    mods["ultralytics.nn.modules.conv"].Conv = Conv
    return mods, WorldModel


def test_loader_reads_an_ultralytics_checkpoint_without_ultralytics(tmp_path):
    mods, WorldModel = _fake_ultralytics_classes()
    sys.modules.update(mods)
    try:
        torch.manual_seed(0)
        ema, model = WorldModel().half(), WorldModel().half()
        ema.model[0].bn.running_mean.normal_()
        path = tmp_path / "yolo-world.pt"
        torch.save({"date": "2024", "model": model, "ema": ema, "train_args": {"imgsz": 640}}, path)
        want = {k: v.float() for k, v in ema.state_dict().items() if not k.endswith("num_batches_tracked")}
    finally:
        for name in mods:
            sys.modules.pop(name, None)
    sd, yaml = Y.load_checkpoint(str(path))
    assert set(sd) == set(want)
    for k in want:
        assert torch.equal(sd[k], want[k]), k
    assert yaml is None   # the checkpoint's yaml has no backbone / head: the built-in layouts apply
    # a plain state dict and a safetensors file load too
    torch.save(want, tmp_path / "sd.pt")
    assert all(torch.equal(Y.load_checkpoint(str(tmp_path / "sd.pt"))[0][k], want[k]) for k in want)
    from safetensors.torch import save_file
    save_file({k: v.contiguous() for k, v in want.items()}, str(tmp_path / "sd.safetensors"))
    assert all(torch.equal(Y.load_checkpoint(str(tmp_path / "sd.safetensors"))[0][k], want[k]) for k in want)


class _Evil:
    def __init__(self, target):
        self.target = target

    def __reduce__(self):
        return self.target


@pytest.mark.parametrize("reduce", [lambda f: (os.system, (f"touch {f}",)),
                                    lambda f: (eval, (f"open({str(f)!r}, 'w')",)),
                                    lambda f: (subprocess.call, (["touch", str(f)],))])
def test_loader_refuses_callables_and_runs_nothing(tmp_path, reduce):
    marker = tmp_path / "pwned"
    path = tmp_path / "evil.pt"
    torch.save({"model": _Evil(reduce(marker))}, path)
    with pytest.raises(pickle.UnpicklingError):
        Y.load_checkpoint(str(path))
    assert not marker.exists()


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("scale", ["s", "m", "l", "x"])
def test_layouts_pack_the_oracle_state_dict(variant, scale):
    """Every tensor the packer reads has the shape the layout predicts, and every tensor of the oracle's state dict
    is read (PackedYoloWorld raises on either mismatch)."""
    from oracle.yolo_world import WorldModel
    sd = WorldModel(variant, scale).state_dict()
    assert Y.variant_and_scale(sd) == (variant, scale)
    p = Y.PackedYoloWorld(sd, device="cpu")
    attn = [(s["ec"], s["nh"]) for s in p.layers if s["type"] == "C2fAttn"]
    assert all(ec // nh == 32 for ec, nh in attn)   # the 32-channel heads omg_text_gate and attention_small take
    if scale == "l":
        assert attn == [(256, 8), (128, 4), (256, 8), (256, 8)]
        n = sum(t.numel() for t in sd.values() if t.dtype.is_floating_point and t.dim() > 0)
        assert abs(n / 1e6 - (47.6 if variant == 1 else 46.9)) < 0.1


@pytest.mark.parametrize("shape", [(480, 720), (720, 480), (640, 640), (333, 1000), (1024, 1024)])
def test_letterbox_and_scale_boxes_geometry(shape):
    h, w = shape
    img = np.full((h, w, 3), 7, np.uint8)
    out = Y.letterbox(img, 640)
    H, W = out.shape[:2]
    assert max(H, W) == 640 and H % 32 == 0 and W % 32 == 0
    gain, (px, py) = Y.box_rescale((H, W), (h, w))
    # the resized image sits centred in grey padding; scale_boxes' pad is ultralytics' own rounding of the unrounded
    # border, which may be one pixel off the border LetterBox drew
    assert gain == min(640 / h, 640 / w)
    nh, nw = int(round(h * gain)), int(round(w * gain))
    rows, cols = np.nonzero(out[..., 0] == 7)
    top, left = rows.min(), cols.min()
    assert (out[top:top + nh, left:left + nw] == 7).all() and (out == 114).sum() == 3 * (H * W - nh * nw)
    assert abs(top - py) <= 1 and abs(left - px) <= 1 and abs((H - nh - top) - top) <= 1
    # a box of the original image maps to the letterbox and back
    box = np.array([[10.0, 20.0, w - 30.0, h - 5.0]])
    lb = box * gain + [px, py, px, py]
    assert np.allclose(Y.scale_boxes((H, W), lb, (h, w)), box, atol=1e-3)
    # clipping to the image
    assert np.allclose(Y.scale_boxes((H, W), np.array([[-50.0, -50.0, 5000.0, 5000.0]]), (h, w)), [[0, 0, w, h]])


@pytest.mark.parametrize("seed", range(4))
def test_oracle_nms_equals_torchvision(seed):
    import torchvision
    from oracle.yolo_world import nms
    g = np.random.default_rng(seed)
    xy = g.random((300, 2)) * 500
    boxes = np.concatenate([xy, xy + g.random((300, 2)) * 120 + 1], 1)
    scores = g.random(300)
    tv = torchvision.ops.nms(torch.from_numpy(boxes), torch.from_numpy(scores), 0.7).numpy()
    assert np.array_equal(nms(boxes, scores, 0.7), tv)


def test_supervision_with_nms_restatement():
    d = Y.Detections([[0, 0, 10, 10], [1, 1, 11, 11], [50, 50, 60, 60], [0, 0, 10, 9]], [0.5, 0.9, 0.3, 0.8],
                     [0, 1, 0, 0])
    agn = d.with_nms(threshold=0.5, class_agnostic=True)
    # 0.9 suppresses 0.5 (IoU 0.68) and 0.8 (IoU 0.61 > 0.5); order of the survivors is the original one
    assert np.array_equal(agn.confidence, np.float32([0.9, 0.3]))
    per = d.with_nms(threshold=0.5)
    # per class: class 1 keeps its box; class 0: 0.8 suppresses 0.5 (IoU 0.9)
    assert np.array_equal(per.confidence, np.float32([0.9, 0.3, 0.8]))
    assert len(Y.Detections(np.zeros((0, 4)), [], []).with_nms()) == 0


def test_loader_accepts_numpy_numbers_in_the_training_metadata(tmp_path):
    """ultralytics stores train_metrics / fitness computed with numpy: numpy scalars (and their dtypes) load inertly."""
    w = {"model.0.conv.weight": torch.randn(16, 3, 3, 3)}
    path = tmp_path / "meta.pt"
    torch.save({"model": None, "ema": None, "state": w, "train_metrics": {"fitness": np.float64(0.5)},
                "best_fitness": np.float32(0.25), "dtype": np.dtype("float64")}, path)
    obj = torch.load(path, map_location="cpu", pickle_module=Y.restricted_pickle, weights_only=False)
    assert torch.equal(obj["state"]["model.0.conv.weight"], w["model.0.conv.weight"])
    assert obj["train_metrics"]["fitness"] is None
    with pytest.raises(ValueError, match="neither"):   # no model in it: refused as a checkpoint, not as a pickle
        Y.load_checkpoint(str(path))


def test_input_channel_order_is_what_preprocess_feeds(monkeypatch):
    from oracle.yolo_world import WorldModel
    det = Y.YOLOWorld(state_dict=WorldModel(2, "s").state_dict(), device="cpu")
    img = np.zeros((64, 64, 3), np.uint8)
    img[..., 0], img[..., 2] = 255, 51
    x, _ = det.preprocess(img)
    assert float(x[0, 20, 20, 0]) == 1.0 and abs(float(x[0, 20, 20, 2]) - 0.2) < 1e-3
    monkeypatch.setattr(Y, "INPUT_CHANNEL_ORDER", "BGR")
    x, _ = det.preprocess(img)
    assert float(x[0, 20, 20, 2]) == 1.0 and abs(float(x[0, 20, 20, 0]) - 0.2) < 1e-3


# ultralytics parse_model by hand: c2 = make_divisible(min(c, max_channels) * width, 8), C2f / C2fAttn repeats
# max(round(n * depth), 1), C2fAttn ec = min(ec, max_channels // 2) * width, nh = round(min(nh, max_channels // 64)) * width
EXPECTED = {
    "s": {"backbone": [32, 64, 64, 128, 128, 256, 256, 512, 512, 512], "repeats": [1, 2, 2, 1],
          "attn": [(256, 128, 4), (128, 64, 2), (256, 128, 4), (512, 256, 8)]},
    "m": {"backbone": [48, 96, 96, 192, 192, 384, 384, 576, 576, 576], "repeats": [2, 4, 4, 2],
          "attn": [(384, 192, 6), (192, 96, 3), (384, 192, 6), (576, 288, 9)]},
    "l": {"backbone": [64, 128, 128, 256, 256, 512, 512, 512, 512, 512], "repeats": [3, 6, 6, 3],
          "attn": [(512, 256, 8), (256, 128, 4), (512, 256, 8), (512, 256, 8)]},
    "x": {"backbone": [80, 160, 160, 320, 320, 640, 640, 640, 640, 640], "repeats": [3, 6, 6, 3],
          "attn": [(640, 320, 10), (320, 160, 5), (640, 320, 10), (640, 320, 10)]},
}


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("scale", ["s", "m", "l", "x"])
def test_layout_channels_match_hand_computed_parse_model(variant, scale):
    layers = Y.parse_layout(Y.layout_yaml(variant, scale))
    e = EXPECTED[scale]
    assert [s["c2"] for s in layers[:10]] == e["backbone"]
    assert [s["n"] for s in layers[:10] if s["type"] == "C2f"] == e["repeats"]
    assert [(s["c2"], s["ec"], s["nh"]) for s in layers if s["type"] == "C2fAttn"] == e["attn"]
    assert all(s["n"] == e["repeats"][-1] for s in layers if s["type"] == "C2fAttn")
    head = layers[-1]
    assert head["type"] == "WorldDetect" and head["with_bn"] == (variant == 2)
    assert head["ch"] == [e["attn"][1][0], e["attn"][2][0], e["attn"][3][0]]
    assert (layers[16]["type"] == "ImagePoolingAttn") == (variant == 1)


def test_random_weights_pack_for_synthetic_runs():
    sd = Y.RandomWeights(0, cls_bias=0.0)
    p = Y.PackedYoloWorld(sd, Y.layout_yaml(2, "s"), device="cpu")
    assert p.variant == 2 and all(h["bias"] == 0.0 and abs(h["scale"] - math.exp(-1)) < 1e-12
                                  for h in p.packs[-1]["levels"])


def _openai_text_sd(width=128, layers=2, vocab=300, ctx=77, proj=96, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g) * 0.2  # noqa: E731
    sd = {"token_embedding.weight": r(vocab, width), "positional_embedding": r(ctx, width),
          "ln_final.weight": 1 + r(width), "ln_final.bias": r(width), "text_projection": r(width, proj),
          "visual.proj": r(4, 4), "logit_scale": torch.tensor(4.6)}
    for i in range(layers):
        o = f"transformer.resblocks.{i}."
        sd.update({o + "attn.in_proj_weight": r(3 * width, width), o + "attn.in_proj_bias": r(3 * width),
                   o + "attn.out_proj.weight": r(width, width), o + "attn.out_proj.bias": r(width),
                   o + "ln_1.weight": 1 + r(width), o + "ln_1.bias": r(width), o + "ln_2.weight": 1 + r(width),
                   o + "ln_2.bias": r(width), o + "mlp.c_fc.weight": r(4 * width, width), o + "mlp.c_fc.bias": r(4 * width),
                   o + "mlp.c_proj.weight": r(width, 4 * width), o + "mlp.c_proj.bias": r(width)})
    return sd


def _encode_text(sd, ids):
    """OpenAI CLIP's encode_text in fp32: causal pre-LN transformer, quick-GELU, EOT (argmax id) pooling, projection."""
    F = torch.nn.functional
    width = sd["token_embedding.weight"].shape[1]
    heads = width // 64
    x = sd["token_embedding.weight"][ids] + sd["positional_embedding"]
    T = ids.shape[1]
    mask = torch.full((T, T), float("-inf")).triu(1)
    i = 0
    while f"transformer.resblocks.{i}.ln_1.weight" in sd:
        o = f"transformer.resblocks.{i}."
        h = F.layer_norm(x, (width,), sd[o + "ln_1.weight"], sd[o + "ln_1.bias"])
        q, k, v = (h @ sd[o + "attn.in_proj_weight"].t() + sd[o + "attn.in_proj_bias"]).chunk(3, -1)
        sp = lambda t: t.view(t.shape[0], T, heads, 64).transpose(1, 2)  # noqa: E731
        a = torch.softmax(sp(q) @ sp(k).transpose(-1, -2) / 8.0 + mask, -1) @ sp(v)
        x = x + a.transpose(1, 2).reshape(-1, T, width) @ sd[o + "attn.out_proj.weight"].t() + sd[o + "attn.out_proj.bias"]
        h = F.layer_norm(x, (width,), sd[o + "ln_2.weight"], sd[o + "ln_2.bias"])
        h = h @ sd[o + "mlp.c_fc.weight"].t() + sd[o + "mlp.c_fc.bias"]
        x = x + (h * torch.sigmoid(1.702 * h)) @ sd[o + "mlp.c_proj.weight"].t() + sd[o + "mlp.c_proj.bias"]
        i += 1
    x = F.layer_norm(x, (width,), sd["ln_final.weight"], sd["ln_final.bias"])
    return x[torch.arange(x.shape[0]), ids.argmax(-1)] @ sd["text_projection"]


def test_openai_clip_text_conversion_equals_encode_text(tmp_path):
    sd = _openai_text_sd()
    ids = torch.tensor([[298, 5, 17, 299] + [299] * 73, [298, 40, 299] + [299] * 74])   # EOT-padded like the tokenizer
    want = _encode_text(sd, ids)
    torch.save(sd, tmp_path / "clip.pt")
    model = Y.load_clip_text(str(tmp_path / "clip.pt"))
    with torch.no_grad():
        got = model(input_ids=ids).text_embeds
    assert torch.allclose(got, want, atol=1e-4, rtol=1e-4)


def test_word_presence_and_detect_flag_validation():
    tok = Y.WordTokenizer()
    p = "Close-up photo of the cool man and beautiful woman as they discover an island"
    assert Y.word_in_prompt(tok, "man", p) and Y.word_in_prompt(tok, "woman", p)
    assert not Y.word_in_prompt(tok, "man", "a woman on a beach") and Y.word_in_prompt(tok, "woman", "a woman on a beach")
    assert tok(["man", "a dog"], padding="max_length", max_length=77, return_tensors="pt").input_ids.shape == (2, 77)
    Y.check_detect_flags(False, "GroundingDINO", "1,2,3,4", "", False)      # without --detect nothing is checked
    Y.check_detect_flags(True, "yoloworld", "", "", True)
    with pytest.raises(SystemExit, match="GroundingDINO detector is not built"):
        Y.check_detect_flags(True, "GroundingDINO", "", "", True)
    with pytest.raises(SystemExit, match="excludes --mask_boxes and --sam_boxes"):
        Y.check_detect_flags(True, "yoloworld", "1,2,3,4", "", True)
    with pytest.raises(SystemExit, match="excludes --mask_boxes and --sam_boxes"):
        Y.check_detect_flags(True, "yoloworld", "", "1,2,3,4|", True)
    with pytest.raises(SystemExit, match="decoded stage-1 image"):
        Y.check_detect_flags(True, "yoloworld", "", "", False)


@pytest.mark.parametrize("fname", ["inference_lora.py", "inference_instantid.py"])
def test_both_clis_take_the_detect_flags(fname):
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("cli_yolo_" + fname[:-3], os.path.join(root, fname))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    argv, sys.argv = sys.argv, [fname]
    try:
        ns = mod.parse_args()
        sys.argv = [fname, "--detect", "--clip_checkpoint", "hf-clip"]
        on = mod.parse_args()
    finally:
        sys.argv = argv
    assert not ns.detect and ns.yoloworld_checkpoint == "./checkpoint/yolo_world/l/yolo-world.pt"
    assert ns.clip_checkpoint == "./checkpoint/clip/ViT-B-32.pt" and on.detect and on.clip_checkpoint == "hf-clip"
    src = open(os.path.join(root, fname)).read()
    assert "yolo_world.check_detect_flags(args.detect, args.segment_type, args.mask_boxes, args.sam_boxes, decoded)" in src
