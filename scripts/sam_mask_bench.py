"""Box-prompted EfficientViT-SAM xl1 masks on the kernels (omg_b200/sam.py): a 1024 x 1024 image, 2 boxes, synthetic
weights of the reference's shapes (omg_b200.synthetic.make_sam_state_dict).  CUDA events, one JSON line:
  set_image_ms          preprocess + image encoder (graph replay) + decoder input, per image
  predict_ms_graph      predict_torch(boxes, multimask_output=False) replayed as one CUDA graph
  predict_ms_eager      the same launches issued from Python
  oracle_predict_ms     the same predict through the fp32 torch restatement (oracle/sam_decoder.py) on the GPU, for scale
  library_launches      omg_* kernel launches of one eager predict
with the card's name and power limit."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from omg_b200 import _lib, synthetic  # noqa: E402
from omg_b200.sam import EfficientViTSamPredictor, PackedEfficientViTSam  # noqa: E402
from oracle import sam_decoder as OD  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        name, watts = [x.strip() for x in r.stdout.strip().split(",")]
        return name, float(watts)
    except Exception:
        return torch.cuda.get_device_name(0), None


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    sd = synthetic.make_sam_state_dict(0)
    model = PackedEfficientViTSam(sd, device="cuda")
    pred = EfficientViTSamPredictor(model)
    g = torch.Generator().manual_seed(0)
    img = (torch.rand(1024, 1024, 3, generator=g) * 255).numpy().astype(np.uint8)
    boxes = torch.tensor([[96., 128., 448., 896.], [576., 128., 928., 896.]], device="cuda")
    set_ms = timed(lambda: pred.set_image(img), 10)
    run = lambda: pred.predict_torch(boxes=boxes, multimask_output=False)  # noqa: E731
    graph_ms = timed(run, 50)
    model.use_graph = False
    eager_ms = timed(run, 20)
    n0 = _lib.launch_count()
    masks, iou, low = run()
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    model.use_graph = True
    # fp32 torch restatement on the same device, same image embedding
    osd = {k: v.cuda() for k, v in sd.items() if k.startswith(("prompt_encoder.", "mask_decoder."))}
    dpe = OD.dense_pe({k: v.cpu() for k, v in osd.items()}).cuda()
    feats = pred.features.float()

    def oracle():
        with torch.no_grad():
            sp, dense = OD.prompt_encoder({k: v.cpu() for k, v in osd.items() if k.startswith("prompt_encoder.")}, None,
                                          boxes.cpu())
            lo, _ = OD.mask_decoder(osd, feats, dpe, sp.cuda(), dense.cuda(), False)
            return OD.postprocess_masks(lo, pred.input_size, pred.original_size) > 0
    oracle_ms = timed(oracle, 10)
    ref = oracle()
    name, watts = card()
    print(json.dumps({"workload": "EfficientViT-SAM xl1, 1024x1024 image, 2 box prompts, multimask_output=False",
                      "gpu": name, "power_limit_w": watts, "set_image_ms": round(set_ms, 3),
                      "predict_ms_graph": round(graph_ms, 3), "predict_ms_eager": round(eager_ms, 3),
                      "oracle_predict_ms": round(oracle_ms, 3), "library_launches": int(launches),
                      "mask_pixels": [int(m.sum()) for m in masks[:, 0]],
                      "mask_agreement_vs_oracle": round(float((masks == ref).float().mean()), 5),
                      "finite": bool(torch.isfinite(low).all() and torch.isfinite(iou).all())}))


if __name__ == "__main__":
    main()
