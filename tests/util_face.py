"""Helpers of the face-analysis tests: ONNX files of the oracle modules from torch's TorchScript exporter (an
independent producer of the graphs the reader and the executor take), and test images."""
import io

import numpy as np
import torch

from oracle import face as of


def export(model, x, preserve_bn=True, dynamic_hw=False, opset=11):
    """ONNX bytes of `model` on example input x.  The exporter's onnxscript post-pass (which would need the `onnx`
    package) is bypassed through a private hook - acceptable in test code only.  preserve_bn keeps BatchNormalization
    nodes (TrainingMode.PRESERVE on an eval model) instead of letting the exporter fold them into the convs."""
    import torch.onnx._internal.torchscript_exporter.onnx_proto_utils as u
    saved = u._add_onnxscript_fn
    u._add_onnxscript_fn = lambda b, _: b
    try:
        f = io.BytesIO()
        torch.onnx.export(model, x, f, dynamo=False, input_names=["input.1"], opset_version=opset,
                          training=torch.onnx.TrainingMode.PRESERVE if preserve_bn else torch.onnx.TrainingMode.EVAL,
                          dynamic_axes={"input.1": {2: "h", 3: "w"}} if dynamic_hw else None)
    finally:
        u._add_onnxscript_fn = saved
    return f.getvalue()


def tiny_iresnet(seed=0, num_features=512):
    return of.randomize_(of.IResNet(layers=(1, 2, 1, 1), widths=(16, 32, 32, 64), num_features=num_features), seed)


def tiny_scrfd(seed=0, score_bias=None, box_bias=None, score_gain=10.0):
    """score_gain spreads the classifier's logits (so that a few anchors stand out above the bias); box_bias: distances
    of every box in strides (large boxes overlap, so NMS keeps few of many candidates)."""
    m = of.randomize_(of.ScrfdNet(stem=(8, 8, 16), stages=(16, 24, 24, 32), blocks=(1, 1, 1, 1), fpn=16, head=16,
                                  stacked=1), seed, score_bias=score_bias)
    with torch.no_grad():
        m.cls.weight.mul_(score_gain)
    if box_bias is not None:
        with torch.no_grad():
            m.reg.bias.fill_(box_bias)
            m.reg.weight.mul_(0.1)
    return m


def write_antelopev2(root, det, rec, det_size=640):
    """<root>/models/antelopev2/{scrfd_10g_bnkps,glintr100}.onnx from two oracle modules."""
    import os
    d = os.path.join(root, "models", "antelopev2")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "scrfd_10g_bnkps.onnx"), "wb") as f:
        f.write(export(det, torch.randn(1, 3, det_size, det_size), dynamic_hw=True))
    with open(os.path.join(d, "glintr100.onnx"), "wb") as f:
        f.write(export(rec, torch.randn(1, 3, 112, 112)))
    return root


def face_image(h, w, seed=0):
    """A BGR uint8 image with a few bright blobs on a textured background."""
    import cv2
    g = np.random.default_rng(seed)
    img = (g.random((h, w, 3)) * 60 + 40).astype(np.uint8)
    for _ in range(3):
        c = (int(g.integers(w // 8, w - w // 8)), int(g.integers(h // 8, h - h // 8)))
        cv2.ellipse(img, c, (w // 10, h // 7), 0, 0, 360, tuple(int(v) for v in g.integers(120, 255, 3)), -1)
    return img
