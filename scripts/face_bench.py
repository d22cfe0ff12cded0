"""Face analysis timing: FaceAnalysis.get() on a 1024 x 1024 image, the SCRFD-style detector at 640 x 640 and the
IResNet-100 recogniser at batch 1 and 2, on the kernels (omg_b200/face.py) against fp16 torch eager (cuDNN) of the same
oracle modules on the same GPU.  Full-size synthetic graphs exported to ONNX in a temporary directory.  CUDA events
after warm-up; each figure is the median over alternating windows of the two paths.  Prints one JSON line with the card
name and power limit read in the same run.

    python scripts/face_bench.py [--windows 7] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return name, pl
    except Exception as e:  # noqa: BLE001
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("face_bench needs a CUDA device")
    from omg_b200 import face as ff
    from oracle import face as of
    from util_face import face_image, write_antelopev2
    det_net = of.randomize_(of.ScrfdNet(), 5, score_bias=-2.0)
    rec_net = of.randomize_(of.IResNet(), 11)
    img = face_image(1024, 1024, 7)
    with tempfile.TemporaryDirectory() as tmp:
        app = ff.FaceAnalysis(root=write_antelopev2(tmp, det_net, rec_net))
    app.prepare(ctx_id=0, det_size=(640, 640))
    det_img, det_scale = ff.det_preprocess(img, (640, 640))
    kps = [of.ARCFACE_DST * 2.0 + np.float32(o) for o in (100, 400)]   # two faces' key-points
    crops = [ff.norm_crop(img, k) for k in kps]
    det16 = det_net.half().cuda().to(memory_format=torch.channels_last)
    rec16 = rec_net.half().cuda().to(memory_format=torch.channels_last)
    xd = torch.from_numpy(of.det_blob(det_img)).half().cuda().to(memory_format=torch.channels_last)
    xr = torch.from_numpy(of.rec_blob(crops)).half().cuda().to(memory_format=torch.channels_last)
    torch.backends.cudnn.benchmark = True
    cases = {
        "get_1024": (lambda: app.get(img), None),
        "detector_640": (lambda: app.det_model.detect_raw(app.det_model.forward_raw(det_img), 640, 640, det_scale),
                         lambda: det16(xd)),
        "recogniser_b1": (lambda: app.rec_model.get_feat(crops[:1]), lambda: rec16(xr[:1])),
        "recogniser_b2": (lambda: app.rec_model.get_feat(crops), lambda: rec16(xr)),
    }
    res = {}
    with torch.no_grad():
        for name, (ours, eager) in cases.items():
            for f in (ours, eager):
                if f is not None:
                    for _ in range(3):
                        f()
            o, e = [], []
            for _ in range(args.windows):
                o.append(timed(ours, args.iters))
                if eager is not None:
                    e.append(timed(eager, args.iters))
            res[name] = {"kernels_ms": float(np.median(o))}
            if e:
                res[name]["torch_fp16_eager_ms"] = float(np.median(e))
    res["faces_in_get"] = len(app.get(img))
    name, pl = card()
    print(json.dumps({"gpu": name, "power_limit": pl, **res}))


if __name__ == "__main__":
    main()
