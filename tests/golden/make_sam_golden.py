"""Generate tests/golden/sam_predictor.pt from the UNMODIFIED reference EfficientViT-SAM predictor (the tests run without
the reference project, hence a committed fixture).  Run:  python tests/golden/make_sam_golden.py <reference checkout>

  sam_predictor.pt the reference's EfficientViTSamPredictor (set_image / predict), EfficientViTSam (transform,
                   postprocess_masks) and SamResize.get_preprocess_shape (sam.py:64-98,195-459) driven with the fp32
                   prompt encoder / mask decoder of oracle/sam_decoder.py injected and a seeded patch-projection image
                   encoder (sam_patch_encoder): box, point and point + box prompts on a 1024 x 1024 and a 640 x 896 image
                   (resize / pad / crop path).  Weights, images and encoder are rebuilt from seeds by the pure helpers
                   below; kept: input sizes, transformed prompts, every 8th row / column of the logits and masks, low-res
                   logits every 4th, IoU predictions.

The reference modules are imported through make_golden._import_efficientvit (packages they do not need are stubbed);
the real torchvision is imported first because SamResize resizes through it, and segment_anything's
ResizeLongestSide.get_preprocess_shape [3P] - stubbed - gets SamResize's identical formula."""
import os
import sys

import torch

OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, OUT)
from make_golden import _import_efficientvit  # noqa: E402


def sam_decoder_weights(seed=0):
    """Decoder / prompt-encoder state dict of sam_predictor.pt: segment_anything shapes (oracle.sam_decoder), weights
    ~ N(0, 1/fan_in), biases N(0, 0.05^2), norm gammas 1 + N(0, 0.1^2), embeddings and the Fourier matrix N(0, 1), all
    rounded to fp16 values.  With random weights the decoder amplifies perturbations strongly (rounding these weights to
    fp16 after the fact moves the logits by ~30 %), so the fixture uses exactly the values the kernels can hold."""
    import math
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    from oracle.sam_decoder import decoder_shapes
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in decoder_shapes().items():
        if k.endswith(".bias"):
            t = torch.randn(shp, generator=g) * 0.05
        elif len(shp) == 1:
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif "embed" in k or "token" in k or "gaussian" in k:
            t = torch.randn(shp, generator=g)
        else:
            t = torch.randn(shp, generator=g) * (shp[0] if "output_upscaling" in k else math.prod(shp[1:])) ** -0.5
        sd[k] = t.half().float()            # fp16-representable: the kernels store fp16
    return sd


def sam_patch_encoder(seed=1):
    """Image encoder stand-in of sam_predictor.pt: 16 x 16 average pooling of the normalised, padded (1, 3, 1024, 1024)
    image, then a seeded 3 -> 256 projection and tanh -> (1, 256, 64, 64).  Cheap on a CPU, and every input pixel that
    the resize / normalise / pad path produces reaches the masks."""
    g = torch.Generator().manual_seed(seed)
    w, b = torch.randn(256, 3, generator=g) * 2.0, torch.randn(256, generator=g) * 0.5

    def enc(x):
        p = torch.nn.functional.avg_pool2d(x.float(), 16)
        y = torch.tanh(torch.einsum("oc,bchw->bohw", w.to(x.device), p) + b.to(x.device)[:, None, None])
        return y.half().float()             # fp16-representable, like the packed image encoder's output
    return enc


SAM_DECODER_CASES = [  # (image (H, W), image seed, prompt)
    ((1024, 1024), 10, {"box": [96, 128, 448, 896]}),
    ((1024, 1024), 10, {"box": [576, 128, 928, 896]}),
    ((1024, 1024), 10, {"point_coords": [[300, 400], [700, 500]], "point_labels": [1, 0], "multimask_output": True}),
    ((640, 896), 11, {"box": [100, 80, 500, 600]}),
    ((640, 896), 11, {"point_coords": [[450, 320]], "point_labels": [1], "box": [300, 100, 700, 620]}),
]


def sam_decoder_case(i):
    """(uint8 HWC image, predict kwargs) of case i of sam_predictor.pt."""
    import numpy as np
    (h, w), seed, prompt = SAM_DECODER_CASES[i]
    g = torch.Generator().manual_seed(seed)
    img = (torch.rand(h // 32 + 1, w // 32 + 1, 3, generator=g) * 255).numpy().astype(np.uint8)   # smooth-ish blobs
    img = np.kron(img, np.ones((32, 32, 1), dtype=np.uint8))[:h, :w]
    img = np.clip(img.astype(np.int16) + (torch.randint(-20, 21, (h, w, 3), generator=g).numpy()), 0, 255).astype(np.uint8)
    kw = {k: (np.array(v, dtype=float if k != "point_labels" else int) if isinstance(v, list) else v) for k, v in prompt.items()}
    kw.setdefault("multimask_output", False)
    return img, kw


def make_sam_decoder():
    import numpy as np
    import torchvision.transforms.functional  # noqa: F401  (the real one: SamResize resizes through it)
    sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))
    from oracle import sam_decoder as OD
    S, _, _, _ = _import_efficientvit()
    # segment_anything's ResizeLongestSide.get_preprocess_shape [3P] is SamResize's formula (sam.py:85-98)
    S.ResizeLongestSide.get_preprocess_shape = staticmethod(S.SamResize.get_preprocess_shape)
    sd = sam_decoder_weights(0)
    enc_fn = sam_patch_encoder(1)

    class Enc(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.anchor = torch.nn.Parameter(torch.zeros(1))    # get_device(model) reads the first parameter

        def forward(self, x):
            return enc_fn(x)

    class PromptEnc(torch.nn.Module):
        def forward(self, points=None, boxes=None, masks=None):
            return OD.prompt_encoder(sd, points, boxes, masks)

        def get_dense_pe(self):
            return OD.dense_pe(sd)

    class MaskDec(torch.nn.Module):
        def forward(self, image_embeddings, image_pe, sparse_prompt_embeddings, dense_prompt_embeddings, multimask_output):
            return OD.mask_decoder(sd, image_embeddings, image_pe, sparse_prompt_embeddings, dense_prompt_embeddings,
                                   multimask_output)

    model = S.EfficientViTSam(Enc(), PromptEnc(), MaskDec(), image_size=(1024, 1024)).eval()
    pred = S.EfficientViTSamPredictor(model)
    out = {"cases": []}
    for i in range(len(SAM_DECODER_CASES)):
        img, kw = sam_decoder_case(i)
        pred.set_image(img)
        masks, iou, low = pred.predict(**kw)
        logits, _, _ = pred.predict(**kw, return_logits=True)
        rec = {"input_size": tuple(int(v) for v in pred.input_size), "original_size": tuple(int(v) for v in pred.original_size),
               "masks_sub": torch.from_numpy(np.ascontiguousarray(masks[:, ::8, ::8])),
               "logits_sub": torch.from_numpy(np.ascontiguousarray(logits[:, ::8, ::8])).float(),
               "low_sub": torch.from_numpy(np.ascontiguousarray(low[:, ::4, ::4])).float(), "iou": torch.from_numpy(iou).float(),
               "mask_fraction": float(masks.mean())}
        if "box" in kw:
            rec["box_t"] = torch.from_numpy(pred.apply_boxes(kw["box"])).float()
        if "point_coords" in kw:
            rec["points_t"] = torch.from_numpy(pred.apply_coords(kw["point_coords"])).float()
        out["cases"].append(rec)
    torch.save(out, os.path.join(OUT, "sam_predictor.pt"))


if __name__ == "__main__":
    sys.path.insert(0, sys.argv[1])
    make_sam_decoder()
    print("sam_predictor.pt", os.path.getsize(os.path.join(OUT, "sam_predictor.pt")))
