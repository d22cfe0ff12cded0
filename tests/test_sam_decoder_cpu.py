"""CPU checks of the EfficientViT-SAM prompt-to-mask path: the fp32 oracle predictor against the unmodified reference
predictor (tests/golden/sam_predictor.pt), the synthetic xl1 state dict's key set, and the --sam_boxes flag."""
import importlib.util
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_sam_golden import SAM_DECODER_CASES, sam_decoder_case, sam_decoder_weights, sam_patch_encoder  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden", "sam_predictor.pt")


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.fixture(scope="module")
def oracle_predictor():
    from oracle.sam_decoder import OraclePredictor
    return OraclePredictor(sam_decoder_weights(0), sam_patch_encoder(1))


@pytest.mark.parametrize("case", range(len(SAM_DECODER_CASES)))
def test_oracle_predictor_matches_the_reference_predictor(oracle_predictor, case):
    d = torch.load(GOLD)["cases"][case]
    img, kw = sam_decoder_case(case)
    p = oracle_predictor
    p.set_image(img)
    assert tuple(p.input_size) == d["input_size"] and tuple(p.original_size) == d["original_size"]
    if "box" in kw:
        from oracle.sam_decoder import apply_boxes
        assert np.allclose(apply_boxes(kw["box"], p.original_size, p.input_size), d["box_t"].numpy())
    masks, iou, low = p.predict(**kw)
    logits, _, _ = p.predict(**kw, return_logits=True)
    assert masks.shape[1:] == img.shape[:2] and masks.dtype == bool
    assert rel(torch.from_numpy(np.ascontiguousarray(logits[:, ::8, ::8])), d["logits_sub"]) < 1e-4
    assert rel(torch.from_numpy(np.ascontiguousarray(low[:, ::4, ::4])), d["low_sub"]) < 1e-4
    assert rel(torch.from_numpy(iou), d["iou"]) < 1e-4
    ref = d["logits_sub"]
    confident = ref.abs() > 1e-3 * ref.std()
    assert torch.equal(torch.from_numpy(np.ascontiguousarray(masks[:, ::8, ::8]))[confident], d["masks_sub"][confident])
    assert 0.1 < d["mask_fraction"] < 0.9


def test_synthetic_sam_state_dict_has_the_xl1_key_set():
    from omg_b200.synthetic import make_sam_state_dict
    from oracle.sam_decoder import decoder_shapes
    sd = make_sam_state_dict(0)
    enc = json.load(open(os.path.join(ROOT, "tests", "golden", "sam_xl1_shapes.json")))
    want = {"image_encoder." + k: tuple(v) for k, v in enc.items()}
    want.update(decoder_shapes())
    assert {k: tuple(v.shape) for k, v in sd.items()} == want
    # segment_anything v1.0's module tree [3P]: the counts a real xl1 checkpoint has
    dec = [k for k in sd if k.startswith("mask_decoder.")]
    assert len([k for k in sd if k.startswith("prompt_encoder.")]) == 17
    assert len([k for k in dec if k.startswith("mask_decoder.transformer.")]) == 2 * 36 + 10
    assert len([k for k in dec if "output_hypernetworks_mlps" in k]) == 24
    assert all(torch.isfinite(v).all() for v in sd.values())


def test_sam_box_parsing():
    from omg_b200.sam import parse_sam_boxes
    assert parse_sam_boxes("96,128,448,896|576,128,928,896") == [(96, 128, 448, 896), (576, 128, 928, 896)]
    assert parse_sam_boxes("1,2,3,4|") == [(1, 2, 3, 4), None]
    assert parse_sam_boxes("|5.5,6,7,8") == [None, (5.5, 6, 7, 8)]
    for bad in ("1,2,3", "5,5,4,9", "1,2,a,4"):
        with pytest.raises(ValueError):
            parse_sam_boxes(bad)


def test_sam_boxes_flag_exclusivity_and_decoded_image():
    from omg_b200.sam import check_sam_flags
    check_sam_flags("", "1,2,3,4", decoded=False)          # --mask_boxes keeps its meaning
    check_sam_flags("1,2,3,4", "", decoded=True)
    with pytest.raises(SystemExit, match="exclusive"):
        check_sam_flags("1,2,3,4", "1,2,3,4", decoded=True)
    with pytest.raises(SystemExit, match="decoded"):
        check_sam_flags("1,2,3,4", "", decoded=False)


@pytest.mark.parametrize("fname", ["inference_lora.py", "inference_instantid.py"])
def test_both_clis_take_sam_boxes(fname):
    spec = importlib.util.spec_from_file_location("cli_sam_" + fname[:-3], os.path.join(ROOT, fname))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    argv, sys.argv = sys.argv, [fname, "--sam_boxes", "1,2,3,4|"]
    try:
        ns = mod.parse_args()
    finally:
        sys.argv = argv
    assert ns.sam_boxes == "1,2,3,4|" and ns.mask_boxes == ""
