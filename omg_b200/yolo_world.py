"""YOLO-World on the kernels: the open-vocabulary detector OMG's CLIs run between the stages with the default
`--segment_type yoloworld` (reference inference_lora.py:91-126,173-178,275-283, inference_instantid.py:158-193,341-349):
it finds "man" / "woman" in the decoded stage-1 image and the best box of each word prompts SAM.

Restates ultralytics' WorldModel (yolov8{s,m,l,x}-world v1 with ImagePoolingAttn and ContrastiveHead, -worldv2
without the pooling attention and with BNContrastiveHead), its LetterBox / non_max_suppression / scale_boxes defaults,
roboflow's YOLOWorld surface and supervision's with_nms, from the published behaviour of those packages (none of them is
a dependency here).

The network runs channels-last fp16 with fp32 arithmetic in the kernels:
  - every Conv (Conv2d + BatchNorm(eps 1e-3) + SiLU) is one omg_gemm with the BatchNorm folded and SiLU in the epilogue,
    stride 2 through phase views, writing straight into its slice of the C2f / C2fAttn concat buffer; a backbone
    Bottleneck's shortcut is the GEMM residual; a Concat in front of a 1x1 conv is K-segments over its operands;
  - SPPF's 5 x 5 max-pool is two omg_pool2d(3, 1, 1) (exact for max), the nearest x2 up-sampling omg_channel_op;
  - MaxSigmoidAttnBlock's gating is omg_text_gate; ImagePoolingAttn is omg_adaptive_maxpool, omg_layernorm, omg_gemm
    and omg_attention_small (8 heads of 32 channels, 27 keys);
  - WorldDetect's contrastive scores, DFL, decode, NMS and the rescale to the image are omg_yolo_detect.
Pre-processing (cv2 resize and padding) stays on the host, as in ultralytics.  Class embeddings are CLIP ViT-B/32's
encode_text on PackedClipText (OpenAI's ViT-B-32.pt converted to transformers' CLIPTextModelWithProjection, or an HF
directory).  make_detector / detect_boxes / check_detect_flags are what the CLIs' --detect uses.

Colour order: INPUT_CHANNEL_ORDER names what the first input channel of the network holds.
"""
import math
import os
import pickle
import types

import numpy as np
import torch

from . import _lib as L
from . import ops

# OMG passes an RGB array (load_image_yoloworld = np.asarray of a PIL image) to roboflow's infer.  Restated from
# memory of those packages, unverified here: roboflow's load_image_rgb takes a numpy array for BGR and swaps it to
# "RGB" (so now B, G, R), ultralytics' predictor takes a numpy array for BGR and its preprocess swaps it again
# (im[..., ::-1]), so the network sees R, G, B - the order it was trained in.  infer() takes RGB arrays; preprocess
# feeds them as they are with "RGB" and swaps R and B with "BGR".
INPUT_CHANNEL_ORDER = "RGB"

# ------------------------------------------------------------------------------------- layouts (ultralytics yaml)
SCALES = {"n": (0.33, 0.25, 1024), "s": (0.33, 0.50, 1024), "m": (0.67, 0.75, 768), "l": (1.00, 1.00, 512),
          "x": (1.00, 1.25, 512)}
BACKBONE = [[-1, 1, "Conv", [64, 3, 2]], [-1, 1, "Conv", [128, 3, 2]], [-1, 3, "C2f", [128, True]],
            [-1, 1, "Conv", [256, 3, 2]], [-1, 6, "C2f", [256, True]], [-1, 1, "Conv", [512, 3, 2]],
            [-1, 6, "C2f", [512, True]], [-1, 1, "Conv", [1024, 3, 2]], [-1, 3, "C2f", [1024, True]],
            [-1, 1, "SPPF", [1024, 5]]]
_HEAD_TOP = [[-1, 1, "nn.Upsample", [None, 2, "nearest"]], [[-1, 6], 1, "Concat", [1]],
             [-1, 3, "C2fAttn", [512, 256, 8]], [-1, 1, "nn.Upsample", [None, 2, "nearest"]],
             [[-1, 4], 1, "Concat", [1]], [-1, 3, "C2fAttn", [256, 128, 4]]]
HEAD_V1 = _HEAD_TOP + [[[15, 12, 9], 1, "ImagePoolingAttn", [256]], [15, 1, "Conv", [256, 3, 2]],
                       [[-1, 12], 1, "Concat", [1]], [-1, 3, "C2fAttn", [512, 256, 8]], [-1, 1, "Conv", [512, 3, 2]],
                       [[-1, 9], 1, "Concat", [1]], [-1, 3, "C2fAttn", [1024, 512, 16]],
                       [[15, 19, 22], 1, "WorldDetect", ["nc", 512, False]]]
HEAD_V2 = _HEAD_TOP + [[-1, 1, "Conv", [256, 3, 2]], [[-1, 12], 1, "Concat", [1]], [-1, 3, "C2fAttn", [512, 256, 8]],
                       [-1, 1, "Conv", [512, 3, 2]], [[-1, 9], 1, "Concat", [1]], [-1, 3, "C2fAttn", [1024, 512, 16]],
                       [[15, 18, 21], 1, "WorldDetect", ["nc", 512, True]]]


def layout_yaml(variant, scale):
    """The yolov8-world.yaml (variant 1) / yolov8-worldv2.yaml (variant 2) model dict at one scale."""
    return {"nc": 80, "scales": dict(SCALES), "scale": scale, "backbone": BACKBONE,
            "head": HEAD_V1 if variant == 1 else HEAD_V2}


def make_divisible(x, d=8):
    return int(math.ceil(x / d) * d)


def parse_layout(yaml):
    """ultralytics parse_model's shape arithmetic: one dict per layer with its type, inputs (`f`), repeats and the
    constructor arguments after width / depth / max_channels scaling."""
    nc = yaml.get("nc", 80)
    scale = yaml.get("scale")
    if "scales" in yaml and yaml["scales"]:
        if scale is None:
            scale = next(iter(yaml["scales"]))
        depth, width, max_ch = yaml["scales"][scale]
    else:
        depth, width, max_ch = yaml.get("depth_multiple", 1.0), yaml.get("width_multiple", 1.0), float("inf")
    ch = [3]
    layers = []
    for i, (f, n, m, args) in enumerate(yaml["backbone"] + yaml["head"]):
        m = m.replace("nn.", "")
        n = max(round(n * depth), 1) if n > 1 else n
        spec = {"i": i, "f": f, "type": m, "n": 1}
        if m in ("Conv", "C2f", "SPPF"):
            c1, c2 = ch[f], make_divisible(min(args[0], max_ch) * width, 8)
            spec.update(c1=c1, c2=c2)
            if m == "Conv":
                spec.update(k=args[1], s=args[2] if len(args) > 2 else 1)
            elif m == "C2f":
                spec.update(n=n, shortcut=bool(args[1]) if len(args) > 1 else False)
            else:
                spec.update(k=args[1])
        elif m == "C2fAttn":
            c1, c2 = ch[f], make_divisible(min(args[0], max_ch) * width, 8)
            ec = make_divisible(min(args[1], max_ch // 2) * width, 8)
            nh = int(max(round(min(args[2], max_ch // 2 // 32)) * width, 1)) if args[2] > 1 else args[2]
            spec.update(c1=c1, c2=c2, n=n, ec=ec, nh=nh, gc=512)
        elif m == "Upsample":
            c2 = ch[f]
            spec.update(c2=c2)
        elif m == "Concat":
            c2 = sum(ch[x] for x in f)
            spec.update(c2=c2)
        elif m == "ImagePoolingAttn":
            c2 = None
            spec.update(ec=args[0], ch=[ch[x] for x in f], ct=512, nh=8, k=3)
        elif m == "WorldDetect":
            c2 = None
            spec.update(nc=nc if args[0] == "nc" else args[0], embed=args[1], with_bn=bool(args[2]), ch=[ch[x] for x in f])
        else:
            raise NotImplementedError(f"layer {i}: module {m} is not part of YOLO-World")
        layers.append(spec)
        if i == 0:
            ch = []
        ch.append(c2)
    return layers


def detect_head_channels(ch0, nc=80):
    """(c2, c3) of WorldDetect's box and embedding branches (Detect.__init__ with the yaml's nc)."""
    return max(16, ch0 // 4, 64), max(ch0, min(nc, 100))


def variant_and_scale(sd):
    """(1 | 2, scale) read off a state dict: v1 has ImagePoolingAttn (model.16.query), v2 BNContrastiveHead norms;
    the scale is the stem's width."""
    variant = 1 if any(k.startswith("model.16.query.") for k in sd) else 2
    widths = {make_divisible(min(64, m) * w, 8): s for s, (_, w, m) in SCALES.items()}
    c0 = sd["model.0.conv.weight"].shape[0]
    if c0 not in widths:
        raise ValueError(f"stem width {c0} matches no YOLO-World scale")
    return variant, widths[c0]


# ------------------------------------------------------------------------------------------- checkpoint loading
class _Stub:
    """Stands for any class a checkpoint names: records the constructor arguments and the pickled state, runs nothing."""

    def __init__(self, *args, **kwargs):
        self._args, self._kwargs = args, kwargs

    def __setstate__(self, state):
        self._state = state


_STUBS = {}


def _stub_class(module, name):
    key = (module, name)
    if key not in _STUBS:
        _STUBS[key] = type(name, (_Stub,), {"__module__": "omg_b200.yolo_world._stubs." + module})
    return _STUBS[key]


def _inert(*args, **kwargs):
    return None


def _reconstructor(cls, base, state):
    return cls.__new__(cls) if isinstance(cls, type) and issubclass(cls, _Stub) else _refuse("copyreg", "_reconstructor")


def _refuse(module, name):
    raise pickle.UnpicklingError(f"checkpoint names {module}.{name}, which a weights file has no reason to call")


_SAFE_BUILTINS = {"set", "frozenset", "dict", "list", "tuple", "slice", "range", "complex", "bytearray", "bytes", "int",
                  "float", "bool", "str"}
_SAFE_TORCH = {("torch._utils", "_rebuild_tensor"), ("torch._utils", "_rebuild_tensor_v2"),
               ("torch._utils", "_rebuild_tensor_v3"), ("torch._utils", "_rebuild_parameter"),
               ("torch._utils", "_rebuild_parameter_with_state"), ("torch", "Size"), ("torch", "device"),
               ("collections", "OrderedDict")}
# numbers in training metadata (train_metrics, fitness) pickle as numpy.core.multiarray.scalar(numpy.dtype(...), bytes)
_INERT = {("numpy.core.multiarray", "scalar"), ("numpy._core.multiarray", "scalar")}
_NUMPY_DTYPE = {("numpy", "dtype"), ("numpy.core.multiarray", "dtype"), ("numpy._core.multiarray", "dtype")}


class RestrictedUnpickler(pickle.Unpickler):
    """torch.load's pickle_module.Unpickler for ultralytics checkpoints: torch's tensor / storage rebuild functions,
    dtypes, OrderedDict and plain builtins resolve; any other class-like name (CamelCase) becomes an inert _Stub
    subclass that records its state; any other callable (os.system, builtins.eval, ...) raises UnpicklingError."""

    def find_class(self, module, name):
        if module in ("builtins", "__builtin__") and name in _SAFE_BUILTINS:
            return getattr(__import__("builtins"), name)
        if (module, name) == ("_codecs", "encode"):   # how pickle protocol 2 (torch.save's) writes bytes objects
            import codecs
            return codecs.encode
        if (module, name) in _SAFE_TORCH:
            mod = __import__(module, fromlist=[name])
            return getattr(mod, name)
        if module == "torch" and isinstance(getattr(torch, name, None), torch.dtype):
            return getattr(torch, name)
        if (module, name) == ("copyreg", "_reconstructor"):
            return _reconstructor
        if (module, name) in _INERT:
            return _inert
        if (module, name) in _NUMPY_DTYPE:   # numpy.dtypes.*DType classes are CamelCase and become stubs below
            return _stub_class(module, name)
        if module.split(".")[0] not in ("builtins", "__builtin__") and name[:1].isupper() and name.isidentifier():
            return _stub_class(module, name)
        _refuse(module, name)


restricted_pickle = types.ModuleType("omg_restricted_pickle")
restricted_pickle.Unpickler = RestrictedUnpickler
restricted_pickle.UnpicklingError = pickle.UnpicklingError
restricted_pickle.load = lambda f, **kw: RestrictedUnpickler(f, **kw).load()


def _state(obj):
    s = getattr(obj, "_state", None)
    return s if isinstance(s, dict) else {}


def module_state_dict(obj, prefix=""):
    """Flatten a stub nn.Module tree (its pickled _parameters / _buffers / _modules) into a state dict."""
    st = _state(obj)
    out = {}
    for kind in ("_parameters", "_buffers"):
        for k, v in (st.get(kind) or {}).items():
            if torch.is_tensor(v):
                out[prefix + k] = v.detach()
    for k, m in (st.get("_modules") or {}).items():
        if m is not None:
            out.update(module_state_dict(m, prefix + k + "."))
    return out


def load_checkpoint(path):
    """(state dict fp32, yaml dict or None) of an ultralytics .pt (restricted unpickling, `ema` preferred over `model`),
    a plain torch state dict or a safetensors file."""
    if str(path).endswith(".safetensors"):
        from safetensors.torch import load_file
        return {k: v.float() for k, v in load_file(str(path)).items()}, None
    obj = torch.load(path, map_location="cpu", pickle_module=restricted_pickle, weights_only=False)
    if isinstance(obj, dict) and all(torch.is_tensor(v) for v in obj.values()):
        return {k: v.float() for k, v in obj.items()}, None
    if isinstance(obj, dict):
        model = obj.get("ema") or obj.get("model")
    else:
        model = obj
    if not isinstance(model, _Stub):
        raise ValueError(f"{path}: neither an ultralytics checkpoint nor a state dict")
    yaml = _state(model).get("yaml")
    sd = {k: v.float() for k, v in module_state_dict(model).items() if not k.endswith("num_batches_tracked")}
    return sd, yaml if isinstance(yaml, dict) and "backbone" in yaml else None


# ------------------------------------------------------------------------------------------- pre / post-processing
def letterbox(img, new_shape=640, auto=True, stride=32, pad_value=114):
    """ultralytics LetterBox(new_shape, auto, stride) with scaleup and centring: cv2 INTER_LINEAR resize, constant
    border.  Returns the padded HWC uint8 image."""
    import cv2
    shape = img.shape[:2]
    new_shape = (new_shape, new_shape) if isinstance(new_shape, int) else tuple(new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    dw, dh = dw / 2, dh / 2
    if shape[::-1] != new_unpad:
        img = cv2.resize(img, new_unpad, interpolation=cv2.INTER_LINEAR)
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return cv2.copyMakeBorder(img, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(pad_value,) * 3)


def box_rescale(img1_shape, img0_shape):
    """scale_boxes' (gain, (pad_x, pad_y)) from the letterboxed (h, w) back to the original (h, w)."""
    gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
    pad = (round((img1_shape[1] - img0_shape[1] * gain) / 2 - 0.1), round((img1_shape[0] - img0_shape[0] * gain) / 2 - 0.1))
    return gain, pad


def scale_boxes(img1_shape, boxes, img0_shape):
    """ultralytics scale_boxes + clip_boxes on an [n, 4] xyxy array."""
    gain, pad = box_rescale(img1_shape, img0_shape)
    b = np.array(boxes, dtype=np.float32, copy=True)
    b[:, [0, 2]] -= pad[0]
    b[:, [1, 3]] -= pad[1]
    b[:, :4] /= np.float32(gain)
    b[:, [0, 2]] = b[:, [0, 2]].clip(0, img0_shape[1])
    b[:, [1, 3]] = b[:, [1, 3]].clip(0, img0_shape[0])
    return b


def box_iou_batch(a, b):
    area = lambda x: (x[:, 2] - x[:, 0]) * (x[:, 3] - x[:, 1])  # noqa: E731
    tl = np.maximum(a[:, None, :2], b[:, :2])
    br = np.minimum(a[:, None, 2:], b[:, 2:])
    inter = np.prod(np.clip(br - tl, 0, None), axis=2)
    return inter / (area(a)[:, None] + area(b) - inter)


class Detections:
    """supervision.Detections' fields OMG reads: xyxy [n, 4], confidence [n], class_id [n] (numpy)."""

    def __init__(self, xyxy, confidence, class_id):
        self.xyxy = np.asarray(xyxy, dtype=np.float32).reshape(-1, 4)
        self.confidence = np.asarray(confidence, dtype=np.float32).reshape(-1)
        self.class_id = np.asarray(class_id, dtype=np.int64).reshape(-1)

    def __len__(self):
        return len(self.xyxy)

    def __getitem__(self, idx):
        return Detections(self.xyxy[idx], self.confidence[idx], self.class_id[idx])

    def with_nms(self, threshold=0.5, class_agnostic=False):
        """supervision's box_non_max_suppression: descending confidence, a box removes later ones (of its class unless
        class_agnostic) with IoU > threshold; the survivors keep their original order."""
        if len(self) == 0:
            return self
        order = np.flip(self.confidence.argsort())
        boxes, cats = self.xyxy[order], (np.zeros(len(self)) if class_agnostic else self.class_id[order])
        ious = box_iou_batch(boxes, boxes) - np.eye(len(self))
        keep = np.ones(len(self), dtype=bool)
        for i, (iou, cat) in enumerate(zip(ious, cats)):
            if not keep[i]:
                continue
            keep &= ~((iou > threshold) & (cats == cat))
        return self[keep[order.argsort()]]


class RandomWeights(dict):
    """A state dict drawn on demand for --synthetic runs: PackedYoloWorld(RandomWeights(...), layout_yaml(...)) draws
    each tensor its layout reads.  Weights ~ N(0, 1 / fan_in), norm scales in [0.8, 1.2], running variances in
    [0.75, 1.25], other vectors ~ N(0, 0.1); BNContrastiveHead's logit_scale -1 and every contrastive head's bias
    `cls_bias` (ultralytics initialises it at -10, which leaves no detection over random weights)."""

    def __init__(self, seed=0, cls_bias=0.0):
        super().__init__()
        self.g = torch.Generator().manual_seed(seed)
        self.cls_bias = cls_bias

    def draw(self, key, shape):
        if key in self or key.endswith(".scale"):   # optional parameters stay absent
            return
        if key.endswith("logit_scale"):
            t = torch.full((), -1.0)
        elif ".cv4." in key and key.endswith(".bias") and shape is None:
            t = torch.full((1,), float(self.cls_bias))
        elif key.endswith("dfl.conv.weight"):
            t = torch.arange(16, dtype=torch.float32).view(1, 16, 1, 1)
        elif len(shape) >= 2:
            t = torch.randn(shape, generator=self.g) / math.sqrt(math.prod(shape[1:]))
        elif key.endswith("running_var"):
            t = torch.rand(shape, generator=self.g) * 0.5 + 0.75
        elif key.endswith("weight"):
            t = torch.rand(shape, generator=self.g) * 0.4 + 0.8
        else:
            t = torch.randn(shape, generator=self.g) * 0.1
        self[key] = t


# ------------------------------------------------------------------------------------------------------ executor
def _c8(n):
    return (n + 7) // 8 * 8


class PackedYoloWorld:
    """A WorldModel state dict packed for the kernels (BatchNorm folded, fp16 weights [N, k*k*C] in (ky, kx, c) order,
    the 3-channel input padded to 8).  forward(x, text) runs the network on a letterboxed (1, H, W, 8) fp16 image with
    the L2-normalised class embeddings text fp32 [n, 512] and returns the per-level (box logits, class embeddings)."""

    def __init__(self, sd, yaml=None, device="cuda"):
        self.dev = torch.device(device)
        if yaml is None:
            self.variant, self.scale = variant_and_scale(sd)
            yaml = layout_yaml(self.variant, self.scale)
        else:
            self.scale = yaml.get("scale")
        self.layers = parse_layout(yaml)
        self.variant = 1 if any(s["type"] == "ImagePoolingAttn" for s in self.layers) else 2
        self.sd, self.used = sd, set()
        self.packs = [self._pack_layer(s) for s in self.layers]
        unused = sorted(k for k in sd if k not in self.used and not k.endswith("num_batches_tracked"))
        if unused:
            raise ValueError(f"checkpoint entries the {self.scale}-scale v{self.variant} layout does not use: {unused[:8]}")
        self.sd = None

    # ---------------------------------------------------------------------------------------------------- packing
    def _t(self, key, shape=None):
        if isinstance(self.sd, RandomWeights):
            self.sd.draw(key, shape)
        if key not in self.sd:
            raise KeyError(f"checkpoint has no {key}")
        self.used.add(key)
        t = self.sd[key].double()
        if shape is not None and tuple(t.shape) != tuple(shape):
            raise ValueError(f"{key}: shape {tuple(t.shape)}, the layout expects {tuple(shape)}")
        return t

    def _h(self, t):
        return t.to(self.dev, torch.float16).contiguous()

    def _f(self, t):
        return t.to(self.dev, torch.float32).contiguous()

    def _conv(self, p, c1, c2, k, bn=True, bias=False, cin_pad=None, affine=None):
        """Conv2d [+ BatchNorm folded] [+ a trailing per-channel affine folded] -> {w, bias, k}."""
        w = self._t(p + (".conv.weight" if bn else ".weight"), (c2, c1, k, k))
        b = self._t(p + ".bias", (c2,)) if bias else torch.zeros(c2, dtype=torch.float64)
        if bn:
            g, beta = self._t(p + ".bn.weight", (c2,)), self._t(p + ".bn.bias", (c2,))
            m, v = self._t(p + ".bn.running_mean", (c2,)), self._t(p + ".bn.running_var", (c2,))
            s = g / torch.sqrt(v + 1e-3)
            w, b = w * s[:, None, None, None], beta - m * s
        if affine is not None:
            s, t = affine
            w, b = w * s[:, None, None, None], b * s + t
        cp = cin_pad or c1
        wp = torch.zeros(c2, k, k, cp, dtype=torch.float64)
        wp[..., :c1] = w.permute(0, 2, 3, 1)
        return {"w": self._h(wp.reshape(c2, -1)), "bias": self._h(b), "k": k, "N": c2}

    def _linear(self, p, n_in, n_out):
        return {"w": self._h(self._t(p + ".weight", (n_out, n_in))), "bias": self._h(self._t(p + ".bias", (n_out,)))}

    def _ln(self, p, n):
        return (self._h(self._t(p + ".weight", (n,))), self._h(self._t(p + ".bias", (n,))))

    def _check_c(self, *cs):
        for c in cs:
            if c % 8:
                raise NotImplementedError(f"channel count {c} is not a multiple of 8")

    def _pack_layer(self, s):
        p, t = f"model.{s['i']}", s["type"]
        if t == "Conv":
            self._check_c(s["c2"])
            return self._conv(p, s["c1"], s["c2"], s["k"], cin_pad=_c8(s["c1"]))
        if t in ("C2f", "C2fAttn"):
            c = int(s["c2"] * 0.5)
            self._check_c(c, s["c1"])
            k = {"cv1": self._conv(p + ".cv1", s["c1"], 2 * c, 1),
                 "cv2": self._conv(p + ".cv2", (2 + s["n"] + (t == "C2fAttn")) * c, s["c2"], 1),
                 "m": [(self._conv(f"{p}.m.{j}.cv1", c, c, 3), self._conv(f"{p}.m.{j}.cv2", c, c, 3))
                       for j in range(s["n"])], "c": c}
            if t == "C2fAttn":
                ec, nh = s["ec"], s["nh"]
                a = p + ".attn"
                if c % nh or ec % nh:
                    raise ValueError(f"{p}: {c} / {ec} channels do not split into {nh} heads")
                k["ec"] = self._conv(a + ".ec", c, ec, 1) if c != ec else None
                k["gl"] = self._linear(a + ".gl", s["gc"], ec)
                k["attn_bias"] = self._f(self._t(a + ".bias", (nh,)))
                k["attn_scale"] = self._f(self._t(a + ".scale").reshape(nh)) if a + ".scale" in self.sd else None
                k["proj"] = self._conv(a + ".proj_conv", c, c, 3)
                k["nh"] = nh
            return k
        if t == "SPPF":
            c_ = s["c1"] // 2
            self._check_c(c_)
            return {"cv1": self._conv(p + ".cv1", s["c1"], c_, 1), "cv2": self._conv(p + ".cv2", 4 * c_, s["c2"], 1)}
        if t == "ImagePoolingAttn":
            ec, ct = s["ec"], s["ct"]
            if p + ".scale" in self.sd:
                raise NotImplementedError(f"{p}: ImagePoolingAttn with a learnt scale")
            return {"proj": [self._conv(f"{p}.projections.{j}", c, ec, 1, bn=False, bias=True)
                             for j, c in enumerate(s["ch"])],
                    "q_ln": self._ln(p + ".query.0", ct), "q": self._linear(p + ".query.1", ct, ec),
                    "k_ln": self._ln(p + ".key.0", ec), "k": self._linear(p + ".key.1", ec, ec),
                    "v_ln": self._ln(p + ".value.0", ec), "v": self._linear(p + ".value.1", ec, ec),
                    "o": self._linear(p + ".proj", ec, ct), "ec": ec, "nh": s["nh"], "kk": s["k"]}
        if t == "WorldDetect":
            c2, c3 = detect_head_channels(s["ch"][0])
            E = s["embed"]
            lv = []
            for j, ci in enumerate(s["ch"]):
                q = f"{p}.cv4.{j}"
                aff = None
                if s["with_bn"]:   # BNContrastiveHead's BatchNorm2d(eps 1e-5) folded into cv3's last conv
                    g, beta = self._t(q + ".norm.weight", (E,)), self._t(q + ".norm.bias", (E,))
                    m, v = self._t(q + ".norm.running_mean", (E,)), self._t(q + ".norm.running_var", (E,))
                    sc = g / torch.sqrt(v + 1e-5)
                    aff = (sc, beta - m * sc)
                lv.append({"cv2": [self._conv(f"{p}.cv2.{j}.0", ci, c2, 3), self._conv(f"{p}.cv2.{j}.1", c2, c2, 3),
                                   self._conv(f"{p}.cv2.{j}.2", c2, 64, 1, bn=False, bias=True)],
                           "cv3": [self._conv(f"{p}.cv3.{j}.0", ci, c3, 3), self._conv(f"{p}.cv3.{j}.1", c3, c3, 3),
                                   self._conv(f"{p}.cv3.{j}.2", c3, E, 1, bn=False, bias=True, affine=aff)],
                           "scale": float(math.exp(float(self._t(q + ".logit_scale").reshape(-1)[0]))),
                           "bias": float(self._t(q + ".bias").reshape(-1)[0])})
            self._t(f"{p}.dfl.conv.weight", (1, 16, 1, 1))
            return {"levels": lv, "E": E, "normalize_x": not s["with_bn"]}
        return None

    # ---------------------------------------------------------------------------------------------------- running
    def _run_conv(self, pk, srcs, stride=1, out=None, act=True, residual=None):
        """srcs: list of (B, H, W, Ci) fp16 views concatenated along channels (several only for 1x1 convs)."""
        x = srcs[0]
        B, H, W, _ = x.shape
        k = pk["k"]
        pad = k // 2
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        N = pk["N"]
        if out is None:
            out = torch.empty(B, Ho, Wo, N, dtype=torch.float16, device=self.dev)
        views, segs = [], []
        if k == 1:
            off = 0
            for j, t in enumerate(srcs):
                views.append(ops.view4(t))
                segs.append((j, 0, 0, 0, t.shape[3], off))
                off += t.shape[3]
        else:
            C = x.shape[3]
            vidx = {}
            for ky in range(k):
                for kx in range(k):
                    ry, rx = ky - pad, kx - pad
                    phase, dy, dx = ((0, 0), ry, rx) if stride == 1 else ((ry % 2, rx % 2), ry // 2, rx // 2)
                    if phase[0] >= H or phase[1] >= W:
                        continue
                    if phase not in vidx:
                        vidx[phase] = len(views)
                        views.append(ops.view4(x if stride == 1 else x[:, phase[0]::2, phase[1]::2, :]))
                    segs.append((vidx[phase], dx, dy, 0, C, (ky * k + kx) * C))
        w = pk["w"]
        late = None
        if residual is not None and N % 32:
            residual, late = None, residual
        ops.gemm(views, segs, w, N, w.shape[1], ops.view4(out), bias=pk["bias"], residual=residual,
                 residual_ld=0 if residual is None else residual.stride(2),
                 epilogue=L.EPI_SILU if act else L.EPI_NONE)
        if late is not None:
            ops.channel_op(out, addend=late, out=out)
        return out

    def _c2f(self, s, pk, srcs, guide=None):
        B, H, W, _ = srcs[0].shape
        c, n = pk["c"], s["n"]
        attn = s["type"] == "C2fAttn"
        buf = torch.empty(B, H, W, (2 + n + attn) * c, dtype=torch.float16, device=self.dev)
        self._run_conv(pk["cv1"], srcs, out=buf[..., :2 * c])
        for j, (m1, m2) in enumerate(pk["m"]):
            y = buf[..., (1 + j) * c:(2 + j) * c]
            t = self._run_conv(m1, [y])
            self._run_conv(m2, [t], out=buf[..., (2 + j) * c:(3 + j) * c],
                           residual=y if s.get("shortcut") else None)
        if attn:
            y = buf[..., (1 + n) * c:(2 + n) * c]
            emb = y if pk["ec"] is None else self._run_conv(pk["ec"], [y], act=False)
            dst = buf[..., (2 + n) * c:]
            self._run_conv(pk["proj"], [y], out=dst, act=False)
            ops.text_gate(emb, guide(pk), pk["attn_bias"], pk["nh"], dst, scale=pk["attn_scale"])
        return self._run_conv(pk["cv2"], [buf])

    def _sppf(self, pk, x):
        y0 = self._run_conv(pk["cv1"], [x])
        ys = [y0]
        for _ in range(3):
            ys.append(ops.pool2d(ops.pool2d(ys[-1], 3, 1, 1), 3, 1, 1))
        return self._run_conv(pk["cv2"], ys)

    def _rows_linear(self, x, lin, residual=None):
        return ops.linear(x, lin["w"], bias=lin["bias"], residual=residual)

    def _pool_attn(self, pk, feats, text, n):
        """ImagePoolingAttn: text (B, npad, 512) fp16 -> updated text (the pooled image patches attended by the prompts)."""
        B, npad, ct = text.shape
        ec, kk = pk["ec"], pk["kk"]
        nk = kk * kk * len(feats)
        kv = torch.zeros(B, _c8(nk), ec, dtype=torch.float16, device=self.dev)
        for j, (x, pj) in enumerate(zip(feats, pk["proj"])):
            ops.adaptive_maxpool(self._run_conv(pj, [x], act=False), kk, kv, row0=j * kk * kk)
        kvf = kv.reshape(-1, ec)
        key = self._rows_linear(ops.layernorm(kvf, *pk["k_ln"]), pk["k"]).view(B, -1, ec)
        val = self._rows_linear(ops.layernorm(kvf, *pk["v_ln"]), pk["v"]).view(B, -1, ec)
        tf = text.reshape(-1, ct)
        q = self._rows_linear(ops.layernorm(tf, *pk["q_ln"]), pk["q"]).view(B, npad, ec)
        o = torch.empty(B, npad, ec, dtype=torch.float16, device=self.dev)
        ops.attention_small(q, key, val, o, pk["nh"], ec // pk["nh"], n, nk)
        return self._rows_linear(o.view(-1, ec), pk["o"], residual=tf).view(B, npad, ct)

    @torch.no_grad()
    def forward(self, x, text):
        """x (B, H, W, 8) fp16 letterboxed image (channels 3.. zero), text fp32 [B or 1, n, 512] normalised ->
        (list of per-level (box (B, h, w, 64), emb (B, h, w, E)) fp16, text fp32 [B, n, E] for the head)."""
        B = x.shape[0]
        if text.dim() == 2:
            text = text[None]
        text = text.expand(B, -1, -1)
        n = text.shape[1]
        npad = _c8(max(n, 1))
        txt = torch.zeros(B, npad, text.shape[2], dtype=torch.float16, device=self.dev)
        txt[:, :n] = text
        cur = {"t": txt}

        def guide(pk):
            g = self._rows_linear(cur["t"].reshape(-1, cur["t"].shape[2]), pk["gl"]).view(B, npad, -1)
            return g[:, :n].float().contiguous()

        ys = []
        out = None
        for s, pk in zip(self.layers, self.packs):
            f, t = s["f"], s["type"]
            if s["i"] == 0:
                src = x
            else:
                src = ys[f] if isinstance(f, int) else [ys[j] for j in f]
            if t == "Conv":
                y = self._run_conv(pk, [src], stride=s["s"])
            elif t in ("C2f", "C2fAttn"):
                y = self._c2f(s, pk, src if isinstance(src, list) else [src], guide)
            elif t == "SPPF":
                y = self._sppf(pk, src)
            elif t == "Upsample":
                y = ops.channel_op(None, addend=src, add_scale=2)
            elif t == "Concat":
                y = src   # consumed as K-segments by the next layer's 1x1 cv1
            elif t == "ImagePoolingAttn":
                cur["t"] = self._pool_attn(pk, src, cur["t"], n)
                y = None
            elif t == "WorldDetect":
                out = []
                for xi, lv in zip(src, pk["levels"]):
                    b = xi
                    for q in lv["cv2"][:2]:
                        b = self._run_conv(q, [b])
                    b = self._run_conv(lv["cv2"][2], [b], act=False)
                    e = xi
                    for q in lv["cv3"][:2]:
                        e = self._run_conv(q, [e])
                    e = self._run_conv(lv["cv3"][2], [e], act=False)
                    out.append((b, e))
                y = None
            ys.append(y)
        return out

    def detect(self, x, text, nms, strides=(8, 16, 32)):
        """forward + omg_yolo_detect for image 0 -> (rows [anchors, 6], detections [n, 6]) fp32 device tensors."""
        head = self.packs[-1]
        lv = self.forward(x, text)
        tn = text.reshape(-1, text.shape[-1]).float()
        tn = (tn / tn.norm(dim=-1, keepdim=True).clamp_min(1e-12)).contiguous()
        levels = [(s, b[:1], e[:1], p["scale"], p["bias"]) for s, (b, e), p in zip(strides, lv, head["levels"])]
        return ops.yolo_detect(levels, tn, head["normalize_x"], nms=nms)


# ------------------------------------------------------------------------------------------------ public surface
class YOLOWorld:
    """roboflow inference's YOLOWorld surface on the kernels: YOLOWorld(model_id=..., checkpoint=..., text_encoder=...),
    set_classes(list of words), infer(RGB uint8 image, confidence) -> Detections (descending confidence).

    text_encoder: a callable list[str] -> [n, 512] tensor (CLIP ViT-B/32 encode_text); its rows are L2-normalised here
    as ultralytics' set_classes does."""

    def __init__(self, model_id="yolo_world/l", checkpoint=None, text_encoder=None, device="cuda", state_dict=None,
                 yaml=None):
        self.model_id = model_id
        if state_dict is None:
            if checkpoint is None or not os.path.isfile(checkpoint):
                raise FileNotFoundError(f"YOLO-World checkpoint {checkpoint!r} not found")
            state_dict, ck_yaml = load_checkpoint(checkpoint)
            yaml = yaml or ck_yaml
        self.model = PackedYoloWorld(state_dict, yaml, device)
        self.text_encoder = text_encoder
        self.device = self.model.dev
        self.classes, self.text = None, None
        self.imgsz, self.iou, self.max_det, self.max_wh = 640, 0.7, 300, 7680

    def set_classes(self, classes):
        if self.text_encoder is None:
            raise RuntimeError("YOLOWorld.set_classes needs a text encoder")
        t = torch.as_tensor(self.text_encoder(list(classes))).double()
        self.set_class_embeddings(list(classes), t)

    def set_class_embeddings(self, classes, emb):
        emb = torch.as_tensor(emb).double().reshape(len(classes), -1)
        self.classes = list(classes)
        self.text = (emb / emb.norm(dim=-1, keepdim=True)).to(self.device, torch.float32).contiguous()

    def preprocess(self, image):
        """RGB uint8 HWC -> ((1, h, w, 8) fp16 network input in INPUT_CHANNEL_ORDER, letterboxed (h, w))."""
        img = letterbox(np.ascontiguousarray(image), self.imgsz)
        h, w = img.shape[:2]
        x = np.zeros((1, h, w, 8), dtype=np.float32)
        x[0, ..., :3] = (img if INPUT_CHANNEL_ORDER == "RGB" else img[..., ::-1]).astype(np.float32) / 255.0
        return torch.from_numpy(x).to(self.device, torch.float16), (h, w)

    def infer(self, image, confidence=0.25):
        if self.text is None:
            raise RuntimeError("YOLOWorld.infer before set_classes")
        image = np.asarray(image)
        if image.ndim != 3 or image.shape[2] != 3 or image.dtype != np.uint8:
            raise ValueError("infer takes an RGB uint8 (H, W, 3) image")
        x, shape = self.preprocess(image)
        gain, pad = box_rescale(shape, image.shape[:2])
        nms = {"conf": confidence, "iou": self.iou, "max_wh": self.max_wh, "agnostic": False, "max_det": self.max_det,
               "gain": gain, "pad": pad, "clip": (image.shape[1], image.shape[0])}
        _, det = self.model.detect(x, self.text, nms)
        det = det.cpu().numpy()
        return Detections(det[:, :4], det[:, 4], det[:, 5].astype(np.int64))


def best_box(detector, image, word, confidence=0.1, threshold=0.5):
    """predict_mask's YOLO-World branch (inference_lora.py:109-116): set_classes([word]), infer, supervision's
    with_nms(class_agnostic=True, threshold) and the first box -> (xyxy float array, score), or None."""
    detector.set_classes([word])
    det = detector.infer(image, confidence=confidence).with_nms(threshold=threshold, class_agnostic=True)
    if len(det) == 0:
        return None
    return det.xyxy[0], float(det.confidence[0])


# ------------------------------------------------------------------------------------------ text side (CLIP ViT-B/32)
def clip_text_from_openai(sd):
    """OpenAI CLIP's text tower (token_embedding, positional_embedding, transformer.resblocks.*, ln_final,
    text_projection) -> transformers CLIPTextModelWithProjection (fp32, CPU) with the shapes read off the state dict.
    encode_text = ln_final(x)[first EOT] @ text_projection, which is the projected tower's text_embeds."""
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    sd = {k: v.float() for k, v in sd.items() if not k.startswith("visual.")}
    vocab, width = sd["token_embedding.weight"].shape
    layers = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transformer.resblocks."))
    cfg = CLIPTextConfig(vocab_size=vocab, hidden_size=width, intermediate_size=sd["transformer.resblocks.0.mlp.c_fc.weight"].shape[0],
                         projection_dim=sd["text_projection"].shape[1], num_hidden_layers=layers,
                         num_attention_heads=width // 64, max_position_embeddings=sd["positional_embedding"].shape[0],
                         hidden_act="quick_gelu", layer_norm_eps=1e-5, eos_token_id=vocab - 1)
    out = {"text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
           "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
           "text_model.final_layer_norm.weight": sd["ln_final.weight"],
           "text_model.final_layer_norm.bias": sd["ln_final.bias"],
           "text_projection.weight": sd["text_projection"].t().contiguous()}
    for i in range(layers):
        o, h = f"transformer.resblocks.{i}.", f"text_model.encoder.layers.{i}."
        for n, w in zip("qkv", sd[o + "attn.in_proj_weight"].chunk(3)):
            out[h + f"self_attn.{n}_proj.weight"] = w
        for n, b in zip("qkv", sd[o + "attn.in_proj_bias"].chunk(3)):
            out[h + f"self_attn.{n}_proj.bias"] = b
        for src, dst in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"),
                         ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
            out[h + dst + ".weight"], out[h + dst + ".bias"] = sd[o + src + ".weight"], sd[o + src + ".bias"]
    model = CLIPTextModelWithProjection(cfg)
    missing, unexpected = model.load_state_dict(out, strict=False)
    missing = [k for k in missing if not k.endswith("position_ids")]
    if missing or unexpected:
        raise ValueError(f"CLIP text tower: missing {missing[:4]}, unexpected {unexpected[:4]}")
    return model.eval()


def load_clip_text(path):
    """CLIP ViT-B/32's text tower from OpenAI's ViT-B-32.pt (the TorchScript archive, or its plain state dict) or an HF
    clip-vit-base-patch32 directory -> CLIPTextModelWithProjection (fp32, CPU)."""
    if os.path.isdir(path):
        from transformers import CLIPTextModelWithProjection
        return CLIPTextModelWithProjection.from_pretrained(path, torch_dtype=torch.float32).eval()
    if not os.path.isfile(path):
        raise FileNotFoundError(f"CLIP checkpoint {path!r} not found")
    try:
        sd = torch.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:   # not a TorchScript archive: a plain state dict
        sd = torch.load(path, map_location="cpu", weights_only=True)
    return clip_text_from_openai(sd)


class WordTokenizer:
    """The --synthetic stand-in of CLIP's tokenizer: lower-cased words, each hashed to one id below the BOS (vocab - 2)
    / EOT (vocab - 1) pair, EOT-padded to max_length.  Called like a transformers tokenizer."""

    def __init__(self, vocab=49408):
        self.vocab = vocab

    def _ids(self, text):
        import re
        import zlib
        words = re.findall(r"[a-z0-9]+", text.lower())
        return [self.vocab - 2] + [zlib.crc32(w.encode()) % (self.vocab - 2) for w in words] + [self.vocab - 1]

    def __call__(self, text, padding=None, max_length=77, truncation=False, return_tensors=None):
        batch = [self._ids(t) for t in ([text] if isinstance(text, str) else text)]
        if truncation:
            batch = [b[:max_length - 1] + [b[-1]] if len(b) > max_length else b for b in batch]
        if padding == "max_length":
            batch = [b + [self.vocab - 1] * (max_length - len(b)) for b in batch]
        ids = batch[0] if isinstance(text, str) else batch
        if return_tensors == "pt":
            ids = torch.tensor(batch)
        return _Encoding(input_ids=ids)


class _Encoding(dict):
    def __getattr__(self, name):
        return self[name]


class ClipTextEncoder:
    """YOLOWorld's text encoder: CLIP encode_text of each word on the kernels (PackedClipText), as ultralytics'
    set_classes calls it (the caller's YOLOWorld L2-normalises the rows)."""

    def __init__(self, model, tokenizer, device="cuda"):
        from .text import PackedClipText
        self.tower = PackedClipText(model.to(torch.float16), device)
        self.tokenizer = tokenizer

    def __call__(self, words):
        ids = self.tokenizer(list(words), padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
        out = []
        for i in range(0, len(ids), 8):   # PackedClipText pools at most 8 rows per call
            out.append(self.tower(ids[i:i + 8])[1].float())
        return torch.cat(out)


def synthetic_clip_text(tiny=False, seed=0):
    """A random-init CLIP text tower: ViT-B/32's shapes, or 2 layers of width 128 with --tiny."""
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    torch.manual_seed(seed)
    w, n = (128, 2) if tiny else (512, 12)
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=w, intermediate_size=4 * w, projection_dim=512,
                         num_hidden_layers=n, num_attention_heads=w // 64, max_position_embeddings=77,
                         hidden_act="quick_gelu", layer_norm_eps=1e-5)
    return CLIPTextModelWithProjection(cfg).eval()


# ---------------------------------------------------------------------------------------------------- CLI helpers
DETECT_WORDS = ("man", "woman")


def word_in_prompt(tokenizer, word, prompt):
    """The reference's gate (inference_lora.py:275-283): the word's first token is among the prompt's tokens."""
    return tokenizer(word)["input_ids"][1] in tokenizer(prompt)["input_ids"][1:-1]


def check_detect_flags(detect, segment_type, mask_boxes, sam_boxes, decoded):
    """--detect finds the concepts' boxes with YOLO-World in the decoded stage-1 image."""
    if not detect:
        return
    if segment_type == "GroundingDINO":
        raise SystemExit("--detect runs YOLO-World; the GroundingDINO detector is not built: with --segment_type "
                         "GroundingDINO pass the boxes as --sam_boxes")
    if mask_boxes or sam_boxes:
        raise SystemExit("--detect finds the boxes itself: it excludes --mask_boxes and --sam_boxes")
    if not decoded:
        raise SystemExit("--detect looks at the decoded stage-1 image: pass --decode (with --synthetic: a random-init "
                         "VAE) or, for the LoRA CLI, --vae_fp16_safe")


def make_detector(synthetic, tiny, yoloworld_checkpoint, clip_checkpoint, tokenizer, device="cuda"):
    """YOLOWorld with CLIP ViT-B/32 class embeddings.  --synthetic: random weights (v2, s scale with --tiny, else l)
    whose contrastive bias lets random images give detections, and a random-init text tower."""
    if synthetic:
        det = YOLOWorld(state_dict=RandomWeights(0, cls_bias=0.0), yaml=layout_yaml(2, "s" if tiny else "l"),
                        device=device)
        clip = synthetic_clip_text(tiny)
    else:
        det = YOLOWorld(checkpoint=yoloworld_checkpoint, device=device)
        clip = load_clip_text(clip_checkpoint)
    det.text_encoder = ClipTextEncoder(clip, tokenizer, device)
    return det


def detect_boxes(detector, image, prompt, tokenizer, words=DETECT_WORDS):
    """predict_mask's YOLO-World step for each word present in the prompt: its best box in the decoded stage-1 image
    (None: not in the prompt or not found).  Prints one line per word."""
    image = np.asarray(image.convert("RGB") if hasattr(image, "convert") else image)
    boxes = []
    for w in words:
        r = best_box(detector, image, w) if word_in_prompt(tokenizer, w, prompt) else None
        if r is None:
            print(f"YOLO-World {w!r}: " + ("no detection, concept skipped" if word_in_prompt(tokenizer, w, prompt)
                                          else "not in the prompt, concept skipped"))
            boxes.append(None)
        else:
            box, score = r
            print(f"YOLO-World {w!r}: box {tuple(round(float(v), 1) for v in box)} score {score:.3f}")
            boxes.append(tuple(float(v) for v in box))
    return boxes
