"""The original SAM (ViT) on the kernels against the fp32 oracle (oracle/sam_vit.py, oracle/sam_decoder.py) on the GPU:
single ViT-H blocks, the full ViT-B and ViT-H encoders, SamPredictor with box and point prompts, CUDA-graph replay, the
finiteness guard and the `--segment_type GroundingDINO` CLI path.  Weights are synthetic (make_sam_vit_state_dict) and
fp16-representable, so the oracle and the kernels hold the same values."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_sam_golden import SAM_DECODER_CASES, sam_decoder_case  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _model(kind):
    from omg_b200 import synthetic
    from omg_b200.sam_vit import PackedSamViTImageEncoder
    sd = synthetic.make_sam_vit_state_dict(kind, 0, device="cuda", dtype=torch.float16)
    osd = {k[len("image_encoder."):]: v.float() for k, v in sd.items() if k.startswith("image_encoder.")}
    return sd, osd, PackedSamViTImageEncoder(sd)


@pytest.fixture(scope="module")
def vit_h():
    m = _model("vit_h")
    yield m
    del m
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def vit_b():
    return _model("vit_b")


def _image(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(1, 3, 1024, 1024, generator=g, device="cuda")


@pytest.mark.parametrize("block", [0, 7])
def test_vit_h_block_matches_the_oracle(vit_h, block):
    """Block 0 (14 x 14 windows, padding 6) and block 7 (global) of ViT-H on the fp32 trunk twin."""
    from oracle.sam_vit import block as oracle_block
    _, osd, enc = vit_h
    g = torch.Generator(device="cuda").manual_seed(block)
    x16 = torch.randn(4096, enc.C, generator=g, device="cuda").half()
    x32 = x16.float()
    x = x16.clone()
    enc.block(block, x, x32, 1)
    ref = oracle_block(x16.float().view(1, 64, 64, enc.C), osd, f"blocks.{block}.", enc.heads,
                       0 if block in enc.glob else 14).view(4096, enc.C)
    e = rel(x32, ref)
    print(f"ViT-H block {block}: rel-L2 {e:.3e}")
    # measured on an H100 80GB HBM3 at a 400 W power limit: 4.96e-5 (block 0), 4.42e-5 (block 7)
    assert torch.isfinite(x32).all() and e < 2e-4
    assert rel(x, ref) < 1e-3                     # the fp16 copy adds its rounding (u = 4.9e-4)


@pytest.mark.parametrize("kind", ["vit_b", "vit_h"])
def test_full_encoder_matches_the_oracle(kind, vit_b, vit_h):
    from oracle.sam_vit import image_encoder
    _, osd, enc = {"vit_b": vit_b, "vit_h": vit_h}[kind]
    img = _image(1)
    out = enc(img)
    with torch.no_grad():
        ref = image_encoder(img, osd)
    e = rel(out, ref)
    print(f"{kind} encoder: rel-L2 {e:.3e}, |ref| max {ref.abs().max().item():.1f}")
    assert out.shape == (1, 256, 64, 64) and out.dtype == torch.float16
    # measured on an H100 80GB HBM3 at a 400 W power limit: 5.55e-4 (ViT-B), 5.56e-4 (ViT-H)
    assert e < 2e-3


def test_graph_replay_on_a_second_image_equals_eager_launches(vit_b):
    _, _, enc = vit_b
    enc(_image(2))                       # captures the graph on the first image
    replay = enc(_image(3))
    with torch.no_grad():
        eager = enc._encode(_image(3).half())
    assert torch.equal(replay, eager)


def test_non_finite_embedding_raises(vit_b):
    from omg_b200 import synthetic
    from omg_b200.sam_vit import PackedSamViTImageEncoder
    sd = synthetic.make_sam_vit_state_dict("vit_b", 5, device="cuda", dtype=torch.float16)
    enc = PackedSamViTImageEncoder(sd, use_graph=False)
    enc.neck0.fill_(1e4)                 # the neck's 1x1 conv overflows fp16
    with pytest.raises(FloatingPointError):
        enc(_image(4))


@pytest.fixture(scope="module")
def predictors(vit_b):
    from omg_b200.sam import PackedSam, SamPredictor, build_sam_vit_b
    from oracle.sam_decoder import OraclePredictor
    from oracle.sam_vit import OracleImageEncoderViT
    sd, _, _ = vit_b
    model = build_sam_vit_b(state_dict=sd)
    assert isinstance(model, PackedSam)
    fsd = {k: v.float() for k, v in sd.items()}
    return SamPredictor(model), OraclePredictor(fsd, OracleImageEncoderViT(fsd, device="cuda"), device="cuda")


@pytest.mark.parametrize("case", range(len(SAM_DECODER_CASES)))
def test_sam_predictor_matches_the_oracle_predictor(predictors, case):
    """Box and point prompts on a 1024² and a 640 x 896 image: low-res logits and IoU by rel-L2; the masks differ from the
    oracle's only where |oracle logit| is small."""
    pred, oracle = predictors
    img, kw = sam_decoder_case(case)
    pred.set_image(img)
    oracle.set_image(img)
    assert tuple(pred.input_size) == tuple(oracle.input_size) and tuple(pred.original_size) == img.shape[:2]
    emb = pred.get_image_embedding()
    e_emb = rel(emb, oracle.features)
    masks, iou, low = pred.predict(**kw)
    logits, _, _ = pred.predict(**kw, return_logits=True)
    r_logits, r_iou, r_low = oracle.predict(**kw, return_logits=True)
    e_low, e_iou = rel(low, r_low), rel(iou, r_iou)
    print(f"case {case}: embedding {e_emb:.3e}, low-res logits {e_low:.3e}, iou {e_iou:.3e}")
    assert masks.shape[1:] == img.shape[:2] and masks.dtype == bool
    # measured on an H100 80GB HBM3 at a 400 W power limit: embedding 5.7e-4, low-res logits 1.29e-3, iou 8.5e-3 (worst)
    assert e_emb < 2e-3 and e_low < 5e-3 and e_iou < 2e-2
    ref = torch.from_numpy(np.ascontiguousarray(r_logits))
    confident = ref.abs() > 0.05 * ref.std()
    assert torch.equal(torch.from_numpy(masks)[confident], (ref > 0)[confident])
    assert np.allclose(pred.transform.apply_boxes(np.array([1.0, 2.0, 3.0, 4.0]), pred.original_size),
                       pred.apply_boxes(np.array([1.0, 2.0, 3.0, 4.0])))


def test_set_torch_image_and_reset(predictors):
    pred, _ = predictors
    img, _ = sam_decoder_case(3)
    pred.set_image(img)
    a = pred.get_image_embedding().clone()
    x = torch.as_tensor(pred.transform.apply_image(img), device="cuda").permute(2, 0, 1)[None]
    pred.set_torch_image(x, img.shape[:2])
    assert torch.equal(pred.get_image_embedding(), a)
    pred.reset_image()
    with pytest.raises(RuntimeError):
        pred.get_image_embedding()


def test_lora_cli_segments_with_the_original_sam(tmp_path):
    """inference_lora.py --segment_type GroundingDINO: stage 2 runs from ViT-B (synthetic, --tiny) masks."""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "inference_lora.py"), "--synthetic", "--tiny", "--decode",
                        "--num_inference_steps", "3", "--segment_type", "GroundingDINO",
                        "--sam_boxes", "96,128,448,896|576,128,928,896", "--save_dir", str(tmp_path)],
                       cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("SAM mask")]
    assert len(lines) == 2 and all("pixels" in l for l in lines), r.stdout[-2000:]
