"""YOLO-World timing: YOLOWorld.infer() on a 1024 x 1024 image (letterboxed to 640 x 640, l scale, v1 and v2, random
weights, one class as best_box uses it) on the kernels (omg_b200/yolo_world.py) against fp16 torch eager (cuDNN) of
the oracle module on the same letterboxed input and GPU.  CUDA events after warm-up; each figure is the median over
alternating windows of the two paths.  Also reports the library launches per infer.  Prints one JSON line with the
card name and power limit read in the same run.

    python scripts/yolo_world_bench.py [--windows 7] [--iters 10]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]

from face_bench import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("yolo_world_bench needs a CUDA device")
    from omg_b200 import _lib as L
    from omg_b200.yolo_world import YOLOWorld
    from oracle import yolo_world as O
    torch.backends.cudnn.benchmark = True
    img = (np.random.default_rng(0).random((1024, 1024, 3)) * 255).astype(np.uint8)
    emb = torch.nn.functional.normalize(torch.randn(1, 512, generator=torch.Generator().manual_seed(1)), dim=-1)
    res = {}
    for variant in (1, 2):
        ref = O.randomize_(O.WorldModel(variant, "l"), seed=variant, bias=0.0 if variant == 1 else -1.0)
        det = YOLOWorld(state_dict=ref.state_dict())
        det.set_class_embeddings(["man"], emb)
        eager = ref.half().cuda().to(memory_format=torch.channels_last)
        x, _ = det.preprocess(img)
        xe = x[..., :3].permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
        te = emb[None].half().cuda()
        ours = lambda: det.infer(img, confidence=0.1)  # noqa: E731
        theirs = lambda: eager(xe, te)  # noqa: E731
        with torch.no_grad():
            for f in (ours, theirs):
                for _ in range(3):
                    f()
            n0 = L.launch_count()
            n_det = len(ours())
            launches = L.launch_count() - n0
            o, e = [], []
            for _ in range(args.windows):
                o.append(timed(ours, args.iters))
                e.append(timed(theirs, args.iters))
        res[f"v{variant}_l_1024"] = {"kernels_infer_ms": float(np.median(o)), "torch_fp16_eager_forward_ms": float(np.median(e)),
                                     "launches_per_infer": int(launches), "detections": n_det}
    name, pl = card()
    print(json.dumps({"gpu": name, "power_limit": pl, **res}))


if __name__ == "__main__":
    main()
