"""Face analysis on the kernels: insightface's FaceAnalysis('antelopev2') surface (an SCRFD detector and an ArcFace
IResNet recogniser, both read from their ONNX files) for the InstantID flow - identity embeddings of the reference
photos and the key-points of the faces in the stage-1 image (reference inference_instantid.py:226-228,353-354,
src/pipelines/instantid_pipeline.py:757-767).

The ONNX graph is packed once (`OnnxNet`): activations are channels-last fp16 (B, H, W, C) with C padded to a multiple
of 8 by zero weight rows / columns; convolutions (k <= 3, stride 1 | 2, symmetric pads, groups 1) run as omg_gemm
K-segments - shifted taps at stride 1, stride-2 phase views at stride 2 - with a following BatchNormalization folded
into the weights, ReLU into the epilogue and an Add whose other operand is already computed into the residual.  A
BatchNormalization that does not follow a conv (IResNet's bn1 sits in front of a zero-padded conv, so it cannot fold
exactly), PReLU, Sigmoid, the FPN's nearest-x2 Resize + Add and the remaining Adds run on omg_channel_op, pooling on
omg_pool2d, and SCRFD's threshold / decode / sort / NMS on omg_scrfd_detect.  Shape arithmetic (Shape, Gather, Concat
of int64, ...) is evaluated on the host from the concrete input shape; Reshape / Transpose / Flatten act on the NCHW
logical view of a channels-last tensor (plumbing).  An op or a conv form outside this set raises NotImplementedError
naming the node: nothing is approximated.

The image steps stay the host cv2 calls insightface makes (resize, blobFromImage, similarity estimate + warpAffine), so
the network inputs match bit for bit.  The landmark (1k3d68, 2d106det) and gender/age models of the pack compute
attributes OMG never reads and are not loaded.  No real antelopev2 file has been run through this executor: the op set
of scrfd_10g_bnkps.onnx / glintr100.onnx is unverified, and an op outside the set above fails loudly at load.
"""
import os

import numpy as np
import torch

from . import _lib as L
from . import onnx as ox
from . import ops


def _c8(n):
    return (n + 7) // 8 * 8


class Act:
    """A channels-last fp16 activation (B, H, W, Cp) whose first C channels are the tensor's; logical shape NCHW, or
    (B, C) for a Gemm's output (flat, stored as H = W = 1)."""

    def __init__(self, t, C, flat=False):
        self.t, self.C, self.flat = t, C, flat

    def logical(self):
        return self.t[:, 0, 0, :self.C] if self.flat else self.t[..., :self.C].permute(0, 3, 1, 2)

    @property
    def shape(self):
        B, H, W, _ = self.t.shape
        return (B, self.C) if self.flat else (B, self.C, H, W)


class _Up2:
    """A nearest-x2 up-sampling not materialised yet: an Add reads it through omg_channel_op's x2 addend."""

    def __init__(self, src):
        self.src = src

    def act(self):
        s = self.src
        return Act(ops.channel_op(None, addend=s.t, add_scale=2), s.C)

    @property
    def shape(self):
        B, C, H, W = self.src.shape
        return (B, C, 2 * H, 2 * W)


_HOST_OPS = {"Shape", "Gather", "Unsqueeze", "Squeeze", "Concat", "Constant", "Cast", "Slice", "Add", "Sub", "Mul",
             "Div", "Floor", "Ceil", "ConstantOfShape", "Range", "Equal", "Where", "Expand", "Reshape", "Identity",
             "Flatten", "Transpose"}
_DEVICE_OPS = {"Conv", "Gemm", "BatchNormalization", "Relu", "PRelu", "Sigmoid", "Add", "Sub", "Mul", "Div", "MaxPool",
               "AveragePool", "Resize", "Upsample", "Reshape", "Transpose", "Flatten", "Concat", "Identity", "Dropout",
               "Shape"}
_ONNX_TO_NP = {1: np.float32, 6: np.int32, 7: np.int64, 9: np.bool_, 10: np.float16, 11: np.float64}


def _s(v):
    return v.decode() if isinstance(v, bytes) else v


class OnnxNet:
    """An ONNX graph of the face models packed for the kernels (see the module docstring).  run(x) takes the network
    input as a channels-last Act and returns the graph outputs as fp32 tensors in logical (ONNX) layout."""

    def __init__(self, model, device="cuda"):
        if isinstance(model, (str, os.PathLike)):
            model = ox.load(model)
        self.model, self.device = model, torch.device(device)
        g = model.graph
        self.nodes = g.nodes
        self.init = dict(g.initializers)
        inits = set(self.init)
        self.input_names = [v.name for v in g.inputs if v.name not in inits]
        self.input_shape = [v.shape for v in g.inputs if v.name not in inits]
        self.output_names = [v.name for v in g.outputs]
        for n in self.nodes:
            if n.op_type == "Constant":
                self.init[n.outputs[0]] = self._constant(n)
            elif n.op_type == "Identity" and n.inputs[0] in self.init:   # the exporter's de-duplicated weights
                self.init[n.outputs[0]] = self.init[n.inputs[0]]
            if n.domain not in ("", "ai.onnx") or (n.op_type not in _HOST_OPS and n.op_type not in _DEVICE_OPS):
                raise NotImplementedError(f"node {n.name!r}: op {n.domain + '.' if n.domain else ''}{n.op_type} is not "
                                          "supported by the face executor")
        self.producer = {o: i for i, n in enumerate(self.nodes) for o in n.outputs}
        self.consumers = {}
        for i, n in enumerate(self.nodes):
            for x in n.inputs:
                self.consumers.setdefault(x, []).append(i)
        self.plan = {}       # node index -> packed op
        self.skip = set()    # nodes folded into an earlier one
        for i, n in enumerate(self.nodes):
            if n.op_type == "Conv":
                self._check_conv(n)
        for i, n in enumerate(self.nodes):
            if i in self.skip:
                continue
            if n.op_type in ("Conv", "Gemm"):
                self.plan[i] = self._pack_gemm(i, n)
                j = self.producer.get(n.inputs[0])
                if n.op_type == "Gemm" and j is not None and self.nodes[j].op_type == "Flatten" and \
                        self.nodes[j].attrs.get("axis", 1) == 1 and self._sole(n.inputs[0]) == i:
                    self.skip.add(j)   # Flatten -> Gemm: the weight's columns are permuted instead
                    self.plan[i]["flat_src"] = self.nodes[j].inputs[0]
            elif n.op_type == "BatchNormalization" and n.inputs[1] in self.init:
                s, t = self._bn(n)
                self.plan[i] = {"scale": self._dev32(s), "shift": self._dev32(t)}
            elif n.op_type == "PRelu":
                self.plan[i] = {"slope": self._dev32(self.init[n.inputs[1]].reshape(-1))}
            elif n.op_type == "Add":
                nxt = self._sole(n.outputs[0])
                if nxt is not None and self.nodes[nxt].op_type == "Relu":
                    self.skip.add(nxt)
                    self.plan[i] = {"out": self.nodes[nxt].outputs[0], "relu": True}

    # ---------------------------------------------------------------------------------------------- load-time packing
    def _constant(self, n):
        if "value" in n.attrs:
            return n.attrs["value"]
        for k, dt in (("value_float", np.float32), ("value_int", np.int64), ("value_floats", np.float32),
                      ("value_ints", np.int64)):
            if k in n.attrs:
                return np.array(n.attrs[k], dtype=dt)
        raise NotImplementedError(f"node {n.name!r}: Constant without a value / value_float(s) / value_int(s)")

    def _sole(self, name):
        """Index of the only consumer of `name`, None if it has several or is a graph output."""
        c = self.consumers.get(name, [])
        return c[0] if len(c) == 1 and name not in self.output_names else None

    def _dev32(self, a):
        return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device=self.device)

    def _bn(self, n):
        g, b, m, v = (self.init[x].astype(np.float64) for x in n.inputs[1:5])
        s = g / np.sqrt(v + float(n.attrs.get("epsilon", 1e-5)))
        return s, b - m * s

    def _check_conv(self, n):
        a = n.attrs
        k = list(a.get("kernel_shape", self.init[n.inputs[1]].shape[2:]))
        pads = list(a.get("pads", [0, 0, 0, 0]))
        strides = list(a.get("strides", [1, 1]))
        what = f"node {n.name!r} (Conv)"
        if _s(a.get("auto_pad", "NOTSET")) not in ("NOTSET", ""):
            raise NotImplementedError(f"{what}: auto_pad is not supported")
        if a.get("group", 1) != 1:
            raise NotImplementedError(f"{what}: groups = {a.get('group')} (only 1)")
        if any(d != 1 for d in a.get("dilations", [1, 1])):
            raise NotImplementedError(f"{what}: dilation is not supported")
        if len(k) != 2 or max(k) > 3:
            raise NotImplementedError(f"{what}: kernel {k} (2-D, k <= 3)")
        if pads[0] != pads[2] or pads[1] != pads[3]:
            raise NotImplementedError(f"{what}: asymmetric pads {pads}")
        if strides[0] != strides[1] or strides[0] not in (1, 2):
            raise NotImplementedError(f"{what}: strides {strides} (1 or 2)")

    def _pack_gemm(self, i, n):
        """Conv / Gemm with a following BatchNormalization folded, then Relu, then an Add whose other operand is
        produced before this node (the residual)."""
        w = self.init[n.inputs[1]].astype(np.float64)
        if n.op_type == "Gemm":
            a = n.attrs
            if a.get("alpha", 1.0) != 1.0 or a.get("beta", 1.0) != 1.0 or a.get("transA", 0):
                raise NotImplementedError(f"node {n.name!r} (Gemm): alpha / beta / transA are not supported")
            if not a.get("transB", 0):
                w = w.T
        b = self.init[n.inputs[2]].astype(np.float64).reshape(-1) if len(n.inputs) > 2 and n.inputs[2] else \
            np.zeros(w.shape[0])
        out, relu, residual = n.outputs[0], False, None
        nxt = self._sole(out)
        if nxt is not None and self.nodes[nxt].op_type == "BatchNormalization" and \
                all(x in self.init for x in self.nodes[nxt].inputs[1:5]):
            s, t = self._bn(self.nodes[nxt])
            w = w * s.reshape(-1, *([1] * (w.ndim - 1)))
            b = b * s + t
            self.skip.add(nxt)
            out = self.nodes[nxt].outputs[0]
            nxt = self._sole(out)
        if nxt is not None and self.nodes[nxt].op_type == "Relu":
            relu = True
            self.skip.add(nxt)
            out = self.nodes[nxt].outputs[0]
            nxt = self._sole(out)
        if nxt is not None and self.nodes[nxt].op_type == "Add":
            other = [x for x in self.nodes[nxt].inputs if x != out]
            if len(other) == 1 and self.producer.get(other[0], -1) < i and other[0] not in self.init:
                residual = other[0]
                self.skip.add(nxt)
                out = self.nodes[nxt].outputs[0]
        N = w.shape[0]
        p = {"N": N, "Np": _c8(N), "w64": w, "bias": None, "relu": relu, "residual": residual, "out": out, "w": {}}
        bp = np.zeros(p["Np"])
        bp[:N] = b
        p["bias"] = torch.as_tensor(bp, dtype=torch.float16, device=self.device)
        if n.op_type == "Conv":
            a = n.attrs
            p["k"] = list(w.shape[2:])
            p["pad"] = list(a.get("pads", [0, 0, 0, 0]))[:2]
            p["stride"] = list(a.get("strides", [1, 1]))[0]
        return p

    def _conv_weight(self, p, Cp):
        if Cp not in p["w"]:
            w = p["w64"]
            N, Cin, kh, kw = w.shape
            wp = np.zeros((p["Np"], kh, kw, Cp))
            wp[:N, :, :, :Cin] = w.transpose(0, 2, 3, 1)
            p["w"][Cp] = torch.as_tensor(wp.reshape(p["Np"], -1), dtype=torch.float16, device=self.device)
        return p["w"][Cp]

    def _fc_weight(self, p, key, C, H, W, Cp):
        """Columns of the Flatten -> Gemm weight in (c, h, w) order re-laid to the activation's (h, w, c-padded)."""
        if key not in p["w"]:
            w = p["w64"]
            N = w.shape[0]
            if w.shape[1] != C * H * W:
                raise ValueError(f"Gemm weight has {w.shape[1]} columns for a flattened {C}x{H}x{W} input")
            wp = np.zeros((p["Np"], H, W, Cp))
            wp[:N, :, :, :C] = w.reshape(N, C, H, W).transpose(0, 2, 3, 1)
            p["w"][key] = torch.as_tensor(wp.reshape(p["Np"], -1), dtype=torch.float16, device=self.device)
        return p["w"][key]

    # ------------------------------------------------------------------------------------------------------ running
    def run(self, *inputs):
        env = self._env = dict(zip(self.input_names, inputs))
        for i, n in enumerate(self.nodes):
            if i in self.skip or n.op_type == "Constant" or n.outputs[0] in self.init:
                continue
            ins = [env[x] if x in env else self.init.get(x) if x else None for x in n.inputs]
            if n.op_type in _HOST_OPS and all(v is None or isinstance(v, np.ndarray) for v in ins):
                env[n.outputs[0]] = self._host(n, ins)
                continue
            p = self.plan.get(i)
            names = [p["out"]] if p is not None and "out" in p else n.outputs
            for name, v in zip(names, self._device(i, n, ins)):
                env[name] = v
        outs = []
        for name in self.output_names:
            v = self._logical(env[name])
            outs.append(v.float() if torch.is_tensor(v) else torch.as_tensor(v))
        self._env = None
        return outs

    def _act(self, v, what):
        if isinstance(v, _Up2):
            return v.act()
        if isinstance(v, Act):
            return v
        raise NotImplementedError(f"{what}: expected a 4-D activation, got {type(v).__name__}")

    def _logical(self, v):
        if isinstance(v, _Up2):
            v = v.act()
        return v.logical() if isinstance(v, Act) else v

    def _residual(self, p, shape, what):
        """The folded Add's other operand as a GEMM residual (contiguous, same padded shape, N % 32 == 0), or as an
        Act that omg_channel_op adds after the GEMM when the epilogue cannot take it."""
        if p["residual"] is None:
            return None, None
        r = self._act(self._env[p["residual"]], what)
        if r.t.is_contiguous() and tuple(r.t.shape) == tuple(shape) and p["Np"] % 32 == 0:
            return r.t, None
        if tuple(r.t.shape) != tuple(shape):
            raise ValueError(f"{what}: residual of shape {tuple(r.shape)} for an output of {tuple(shape)}")
        return None, r

    def _conv(self, p, x, what):
        B, H, W, Cp = x.t.shape
        kh, kw = p["k"]
        ph, pw = p["pad"]
        s = p["stride"]
        Ho, Wo = (H + 2 * ph - kh) // s + 1, (W + 2 * pw - kw) // s + 1
        w = self._conv_weight(p, Cp)
        res, late = self._residual(p, (B, Ho, Wo, p["Np"]), what)
        out = torch.empty(B, Ho, Wo, p["Np"], dtype=torch.float16, device=self.device)
        views, vidx, segs = [], {}, []
        for ky in range(kh):
            for kx in range(kw):
                ry, rx = ky - ph, kx - pw
                phase, dy, dx = ((0, 0), ry, rx) if s == 1 else ((ry % 2, rx % 2), ry // 2, rx // 2)
                if phase[0] >= H or phase[1] >= W:
                    continue   # an input side of 1 pixel leaves the odd phase empty: such a tap reads only padding
                if phase not in vidx:
                    vidx[phase] = len(views)
                    views.append(ops.view4(x.t if s == 1 else x.t[:, phase[0]::2, phase[1]::2, :]))
                segs.append((vidx[phase], dx, dy, 0, Cp, (ky * kw + kx) * Cp))
        ops.gemm(views, segs, w, p["Np"], w.shape[1], ops.view4(out), bias=p["bias"], residual=res,
                 residual_ld=0 if res is None else p["Np"], epilogue=L.EPI_RELU if p["relu"] else L.EPI_NONE)
        if late is not None:
            out = ops.channel_op(out, addend=late.t, out=out)
        return Act(out, p["N"])

    def _gemm(self, p, v, what):
        src = self._env.get(p["flat_src"]) if p.get("flat_src") else None
        if isinstance(src, (Act, _Up2)):   # Flatten -> Gemm: weight columns re-laid to (h, w, c) at first use
            x = self._act(src, what)
            B, H, W, Cp = x.t.shape
            w = self._fc_weight(p, ("hwc", x.C, H, W, Cp), x.C, H, W, Cp)
            xin = x.t.contiguous().reshape(B, H * W * Cp)
        else:
            t = self._logical(src if p.get("flat_src") else v)
            t = t.reshape(t.shape[0], -1).half()
            K = t.shape[1]
            xin = torch.nn.functional.pad(t, (0, _c8(K) - K)).contiguous()
            key = ("plain", K)
            if key not in p["w"]:
                wp = np.zeros((p["Np"], xin.shape[1]))
                wp[:p["N"], :K] = p["w64"]
                p["w"][key] = torch.as_tensor(wp, dtype=torch.float16, device=self.device)
            w = p["w"][key]
        B = xin.shape[0]
        res, late = self._residual(p, (B, 1, 1, p["Np"]), what)
        y = ops.linear(xin, w, bias=p["bias"], epilogue=L.EPI_RELU if p["relu"] else L.EPI_NONE,
                       residual=None if res is None else res.reshape(B, p["Np"]))
        y = y.view(B, 1, 1, p["Np"])
        if late is not None:
            y = ops.channel_op(y, addend=late.t, out=y)
        return Act(y, p["N"], flat=True)

    def _vec(self, c, Cp, what):
        """A constant operand broadcast per channel of an NCHW activation -> fp32 [Cp] (padding channels 0)."""
        c = np.asarray(c, dtype=np.float64)
        if c.size != 1 and (c.ndim < 3 or c.shape[-2:] != (1, 1) or c.size != c.reshape(-1).shape[0]):
            raise NotImplementedError(f"{what}: a constant operand must be a scalar or per channel")
        v = np.zeros(Cp)
        flat = c.reshape(-1)
        v[:] = flat[0] if flat.size == 1 else 0.0
        if flat.size > 1:
            v[:flat.size] = flat
        return self._dev32(v)

    def _binary(self, i, n, ins, what):
        op = n.op_type
        p = self.plan.get(i) or {}
        act = L.CH_ACT_RELU if p.get("relu") else L.CH_ACT_NONE
        a, b = ins[0], ins[1]
        dev = lambda v: isinstance(v, (Act, _Up2))  # noqa: E731
        if dev(a) and dev(b):
            if op != "Add":
                raise NotImplementedError(f"{what}: {op} of two activations")
            if isinstance(a, _Up2) and not isinstance(b, _Up2):
                a, b = b, a
            x = self._act(a, what)
            if isinstance(b, _Up2):
                y = ops.channel_op(x.t, addend=b.src.t, add_scale=2, act=act, act_after_add=True)
            else:
                y = ops.channel_op(x.t, addend=self._act(b, what).t, act=act, act_after_add=True)
            return Act(y, x.C, x.flat)
        if dev(a) and isinstance(b, np.ndarray) or dev(b) and isinstance(a, np.ndarray):
            first = dev(a)
            x, c = (self._act(a, what), b) if first else (self._act(b, what), a)
            Cp = x.t.shape[3]
            if op == "Add":
                scale, shift = None, self._vec(c, Cp, what)
            elif op == "Sub":
                scale, shift = (None, self._vec(-c, Cp, what)) if first else (self._vec(-1.0, Cp, what), self._vec(c, Cp, what))
            elif op == "Mul":
                scale, shift = self._vec(c, Cp, what), None
            elif first:   # Div by a constant
                scale, shift = self._vec(1.0 / np.asarray(c, dtype=np.float64), Cp, what), None
            else:
                raise NotImplementedError(f"{what}: constant / activation")
            return Act(ops.channel_op(x.t, scale=scale, shift=shift, act=act), x.C, x.flat)
        raise NotImplementedError(f"{what}: {op} of a reshaped device tensor")

    def _resize(self, n, ins, what):
        a = n.attrs
        if _s(a.get("mode", "nearest")) != "nearest":
            raise NotImplementedError(f"{what}: mode {_s(a.get('mode'))!r} (nearest only)")
        ctm = _s(a.get("coordinate_transformation_mode", "asymmetric" if n.op_type == "Upsample" else "half_pixel"))
        nm = _s(a.get("nearest_mode", "round_prefer_floor"))
        if n.op_type == "Upsample" or (ctm == "asymmetric" and nm == "floor"):
            pass   # source index floor(dst / 2)
        elif not (ctm in ("half_pixel", "pytorch_half_pixel") and nm in ("round_prefer_floor", "round_prefer_ceil")):
            raise NotImplementedError(f"{what}: coordinate_transformation_mode {ctm!r} / nearest_mode {nm!r}")
        x = self._act(ins[0], what)
        shape = np.array(x.shape)
        if n.op_type == "Upsample":
            scales = ins[1] if len(ins) > 1 and ins[1] is not None else np.array(a.get("scales"))
        else:
            scales = ins[2] if len(ins) > 2 and ins[2] is not None and ins[2].size else None
            if scales is None:
                if len(ins) < 4 or ins[3] is None:
                    raise NotImplementedError(f"{what}: neither scales nor sizes")
                scales = np.asarray(ins[3], dtype=np.float64) / shape
        if [float(s) for s in np.asarray(scales).reshape(-1)] != [1.0, 1.0, 2.0, 2.0]:
            raise NotImplementedError(f"{what}: scales {list(np.asarray(scales).reshape(-1))} (nearest x2 only)")
        return _Up2(x)

    def _device(self, i, n, ins):
        op, a, what = n.op_type, n.attrs, f"node {n.name!r} ({n.op_type})"
        p = self.plan.get(i)
        if op == "Conv":
            return [self._conv(p, self._act(ins[0], what), what)]
        if op == "Gemm":
            return [self._gemm(p, ins[0], what)]
        if op in ("Identity", "Dropout"):
            return [ins[0]]
        if op == "BatchNormalization":
            if p is None:
                raise NotImplementedError(f"{what}: statistics must be initializers")
            x = self._act(ins[0], what)
            Cp = x.t.shape[3]
            return [Act(ops.channel_op(x.t, scale=self._pad32(p["scale"], Cp), shift=self._pad32(p["shift"], Cp)), x.C, x.flat)]
        if op in ("Relu", "Sigmoid", "PRelu"):
            act = {"Relu": L.CH_ACT_RELU, "Sigmoid": L.CH_ACT_SIGMOID, "PRelu": L.CH_ACT_PRELU}[op]
            v = ins[0]
            if isinstance(v, (Act, _Up2)):
                x = self._act(v, what)
                slope = None if p is None else self._pad32(p["slope"], x.t.shape[3])
                return [Act(ops.channel_op(x.t, act=act, slope=slope), x.C, x.flat)]
            if op == "PRelu":
                raise NotImplementedError(f"{what}: PRelu of a reshaped device tensor")
            t = v.contiguous().half()
            flat = t.reshape(1, 1, -1, t.shape[-1] if t.dim() else 1)
            return [ops.channel_op(flat, act=act).reshape(t.shape)]
        if op in ("Add", "Sub", "Mul", "Div"):
            return [self._binary(i, n, ins, what)]
        if op in ("MaxPool", "AveragePool"):
            k, st = list(a["kernel_shape"]), list(a.get("strides", [1, 1]))
            pads = list(a.get("pads", [0, 0, 0, 0]))
            if len(set(k)) != 1 or len(set(st)) != 1 or len(set(pads)) != 1 or \
                    _s(a.get("auto_pad", "NOTSET")) not in ("NOTSET", "") or any(d != 1 for d in a.get("dilations", [1, 1])):
                raise NotImplementedError(f"{what}: square window, equal strides and symmetric pads only")
            x = self._act(ins[0], what)
            y = ops.pool2d(x.t.contiguous(), k[0], st[0], pads[0], bool(a.get("ceil_mode", 0)),
                           bool(a.get("count_include_pad", 0)), op == "MaxPool")
            return [Act(y, x.C)]
        if op in ("Resize", "Upsample"):
            return [self._resize(n, ins, what)]
        if op == "Shape":
            v = ins[0]
            return [np.array(v.shape if isinstance(v, (Act, _Up2)) else tuple(v.shape), dtype=np.int64)]
        # layout plumbing on the logical (NCHW) view
        x = self._logical(ins[0])
        if op == "Transpose":
            return [x.permute(*a.get("perm", list(range(x.dim()))[::-1]))]
        if op == "Reshape":
            shape = [int(d) for d in ins[1]]
            if not a.get("allowzero", 0):
                shape = [x.shape[j] if d == 0 else d for j, d in enumerate(shape)]
            return [x.reshape(shape)]
        if op == "Flatten":
            ax = a.get("axis", 1)
            ax = ax + x.dim() if ax < 0 else ax
            return [x.reshape(int(np.prod(x.shape[:ax])), -1)]
        if op == "Concat":
            return [torch.cat([self._logical(v) for v in ins], dim=a["axis"])]
        raise NotImplementedError(f"{what}: unsupported operands")

    def _pad32(self, v, Cp):
        return v if v.numel() >= Cp else torch.cat([v, torch.zeros(Cp - v.numel(), dtype=v.dtype, device=v.device)])

    def _host(self, n, ins):
        """Shape arithmetic on the host (numpy) - the exporter's Shape / Gather / Unsqueeze / Concat chains."""
        op, a = n.op_type, n.attrs
        x = ins[0] if ins else None
        if op == "Shape":
            return np.array(x.shape, dtype=np.int64)
        if op == "Gather":
            return np.take(x, ins[1], axis=a.get("axis", 0))
        if op in ("Unsqueeze", "Squeeze"):
            axes = list(a["axes"]) if "axes" in a else ([int(v) for v in ins[1]] if len(ins) > 1 and ins[1] is not None else None)
            if op == "Squeeze":
                return np.squeeze(x, axis=tuple(axes) if axes is not None else None)
            for ax in sorted(ax + x.ndim + len(axes) if ax < 0 else ax for ax in axes):
                x = np.expand_dims(x, ax)
            return x
        if op == "Concat":
            return np.concatenate([np.atleast_1d(v) for v in ins], axis=a["axis"])
        if op == "Cast":
            if a["to"] not in _ONNX_TO_NP:
                raise NotImplementedError(f"node {n.name!r} (Cast): to={a['to']}")
            return x.astype(_ONNX_TO_NP[a["to"]])
        if op == "Slice":
            if "starts" in a:
                starts, ends, axes, steps = a["starts"], a["ends"], a.get("axes"), None
            else:
                starts, ends = ins[1], ins[2]
                axes = ins[3] if len(ins) > 3 and ins[3] is not None else None
                steps = ins[4] if len(ins) > 4 and ins[4] is not None else None
            axes = list(range(len(starts))) if axes is None else list(axes)
            sl = [slice(None)] * x.ndim
            for j, ax in enumerate(axes):
                sl[ax] = slice(int(starts[j]), int(max(min(ends[j], 2 ** 62), -2 ** 62)),
                               None if steps is None else int(steps[j]))
            return x[tuple(sl)]
        if op in ("Add", "Sub", "Mul", "Div"):
            y = {"Add": np.add, "Sub": np.subtract, "Mul": np.multiply}.get(op)
            if y is not None:
                return y(x, ins[1]).astype(np.result_type(x, ins[1]))
            if np.issubdtype(x.dtype, np.integer):
                return (x // ins[1]).astype(x.dtype)
            return x / ins[1]
        if op in ("Floor", "Ceil"):
            return (np.floor if op == "Floor" else np.ceil)(x)
        if op == "ConstantOfShape":
            v = a.get("value", np.zeros(1, dtype=np.float32))
            return np.full([int(d) for d in x], v.reshape(-1)[0], dtype=v.dtype)
        if op == "Range":
            return np.arange(x, ins[1], ins[2]).astype(np.result_type(x))
        if op == "Equal":
            return np.equal(x, ins[1])
        if op == "Where":
            return np.where(x, ins[1], ins[2])
        if op == "Expand":
            return x * np.ones([int(d) for d in ins[1]], dtype=x.dtype)
        if op == "Reshape":
            shape = [int(d) for d in ins[1]]
            shape = [x.shape[j] if d == 0 else d for j, d in enumerate(shape)]
            return x.reshape(shape)
        if op == "Identity":
            return x
        if op == "Flatten":
            ax = a.get("axis", 1)
            return x.reshape(int(np.prod(x.shape[:ax])), -1)
        if op == "Transpose":
            return np.transpose(x, a.get("perm"))
        raise NotImplementedError(f"node {n.name!r}: {op} on the host")


def image_to_act(blob, device):
    """NCHW fp32 blob -> channels-last fp16 Act with the channels padded to 8."""
    B, C, H, W = blob.shape
    t = torch.zeros(B, H, W, _c8(C), dtype=torch.float16, device=device)
    t[..., :C] = torch.from_numpy(np.ascontiguousarray(blob.transpose(0, 2, 3, 1))).to(device)
    return Act(t, C)


def _check_finite(what, *ts):
    for t in ts:
        if not bool(torch.isfinite(t).all()):
            raise FloatingPointError(f"{what}: non-finite network output")


# -------------------------------------------------------------------------------------------------- detection
def det_preprocess(img, input_size):
    """SCRFD.detect's input: aspect-preserving cv2 resize pasted at the top left of a zero canvas -> (canvas, det_scale)."""
    import cv2
    im_ratio = float(img.shape[0]) / img.shape[1]
    model_ratio = float(input_size[1]) / input_size[0]
    if im_ratio > model_ratio:
        new_h = input_size[1]
        new_w = int(new_h / im_ratio)
    else:
        new_w = input_size[0]
        new_h = int(new_w * im_ratio)
    det_scale = float(new_h) / img.shape[0]
    canvas = np.zeros((input_size[1], input_size[0], 3), dtype=np.uint8)
    canvas[:new_h, :new_w, :] = cv2.resize(img, (new_w, new_h))
    return canvas, det_scale


class SCRFD:
    """insightface's SCRFD detector on the kernels: detect(img_bgr) -> (det [n, 5] fp32 (box, score), kpss [n, 5, 2])."""

    taskname = "detection"

    def __init__(self, model_file=None, model=None, device="cuda"):
        self.model_file = model_file
        self.net = OnnxNet(model if model is not None else model_file, device)
        self.device = self.net.device
        self.input_mean, self.input_std = 127.5, 128.0
        self.det_thresh, self.nms_thresh = 0.5, 0.4
        self.input_size = None
        shp = self.net.input_shape[0]
        if shp is not None and all(isinstance(d, int) for d in shp[2:]):
            self.input_size = (shp[3], shp[2])
        n_out = len(self.net.output_names)
        if n_out not in (6, 9, 10, 15):
            raise NotImplementedError(f"SCRFD with {n_out} outputs (6, 9, 10 or 15)")
        self.use_kps = n_out in (9, 15)
        self.fmc, self.strides, self.num_anchors = (3, (8, 16, 32), 2) if n_out in (6, 9) else (5, (8, 16, 32, 64, 128), 1)

    def prepare(self, ctx_id=0, det_thresh=None, input_size=None, nms_thresh=None, **kwargs):
        if det_thresh is not None:
            self.det_thresh = det_thresh
        if nms_thresh is not None:
            self.nms_thresh = nms_thresh
        if input_size is not None:
            self.input_size = tuple(input_size)

    def forward_raw(self, det_img):
        """The network's outputs on a prepared canvas (fp32, batch taken from 3-D outputs)."""
        import cv2
        size = tuple(det_img.shape[0:2][::-1])
        blob = cv2.dnn.blobFromImage(det_img, 1.0 / self.input_std, size, (self.input_mean,) * 3, swapRB=True)
        outs = self.net.run(image_to_act(blob, self.device))
        outs = [o[0] if o.dim() == 3 else o for o in outs]
        _check_finite("SCRFD", *outs)
        return outs

    def detect_raw(self, outs, input_h, input_w, det_scale):
        levels = []
        for idx, s in enumerate(self.strides):
            fh, fw = input_h // s, input_w // s
            kp = outs[idx + 2 * self.fmc].contiguous() if self.use_kps else None
            levels.append((s, fh, fw, outs[idx].contiguous(), outs[idx + self.fmc].contiguous(), kp))
        return ops.scrfd_detect(levels, self.num_anchors, self.det_thresh, det_scale, self.nms_thresh)

    def detect(self, img, input_size=None, max_num=0, metric="default"):
        if max_num != 0:
            raise NotImplementedError("SCRFD.detect: max_num selection is not implemented (no OMG caller uses it)")
        input_size = tuple(input_size or self.input_size or (640, 640))
        det_img, det_scale = det_preprocess(img, input_size)
        rows = self.detect_raw(self.forward_raw(det_img), input_size[1], input_size[0], det_scale).cpu().numpy()
        det = rows[:, :5].copy()
        kpss = rows[:, 5:].reshape(-1, 5, 2).copy() if self.use_kps else None
        return det, kpss


# ------------------------------------------------------------------------------------------------ recognition
ARCFACE_DST = np.array([[38.2946, 51.6963], [73.5318, 51.5014], [56.0252, 71.7366], [41.5493, 92.3655],
                        [70.7299, 92.2041]], dtype=np.float32)


def umeyama(src, dst):
    """Least-squares similarity (rotation, uniform scale, translation) taking src to dst (Umeyama 1991), as
    skimage.transform.SimilarityTransform.estimate computes it: the 3 x 3 homogeneous matrix."""
    src, dst = np.asarray(src, dtype=np.float64), np.asarray(dst, dtype=np.float64)
    num, dim = src.shape
    src_mean, dst_mean = src.mean(axis=0), dst.mean(axis=0)
    src_d, dst_d = src - src_mean, dst - dst_mean
    A = dst_d.T @ src_d / num
    d = np.ones((dim,))
    if np.linalg.det(A) < 0:
        d[dim - 1] = -1
    T = np.eye(dim + 1)
    U, S, V = np.linalg.svd(A)
    rank = np.linalg.matrix_rank(A)
    if rank == 0:
        return np.nan * T
    if rank == dim - 1:
        if np.linalg.det(U) * np.linalg.det(V) > 0:
            T[:dim, :dim] = U @ V
        else:
            s = d[dim - 1]
            d[dim - 1] = -1
            T[:dim, :dim] = U @ np.diag(d) @ V
            d[dim - 1] = s
    else:
        T[:dim, :dim] = U @ np.diag(d) @ V
    scale = 1.0 / src_d.var(axis=0).sum() * (S @ d)
    T[:dim, dim] = dst_mean - scale * (T[:dim, :dim] @ src_mean.T)
    T[:dim, :dim] *= scale
    return T


def estimate_norm(lmk, image_size=112):
    assert lmk.shape == (5, 2) and image_size % 112 == 0
    ratio = float(image_size) / 112.0
    return umeyama(lmk, ARCFACE_DST * ratio)[0:2, :]


def norm_crop(img, landmark, image_size=112):
    import cv2
    M = estimate_norm(np.asarray(landmark), image_size)
    return cv2.warpAffine(img, M, (image_size, image_size), borderValue=0.0)


def input_norm_of(model):
    """ArcFaceONNX's input normalisation: (0, 1) when a node named Sub* / _minus* and one named Mul* / _mul* are among
    the graph's first 8 nodes (the normalisation is inside the graph), else (127.5, 127.5)."""
    names = [n.name for n in model.graph.nodes[:8]]
    sub = any(s.startswith(("Sub", "_minus")) for s in names)
    mul = any(s.startswith(("Mul", "_mul")) for s in names)
    return (0.0, 1.0) if sub and mul else (127.5, 127.5)


class ArcFace:
    """insightface's ArcFaceONNX on the kernels: get_feat(aligned crops) -> embeddings (unnormalised)."""

    taskname = "recognition"

    def __init__(self, model_file=None, model=None, device="cuda"):
        self.model_file = model_file
        model = model if model is not None else ox.load(model_file)
        self.net = OnnxNet(model, device)
        self.device = self.net.device
        self.input_mean, self.input_std = input_norm_of(model)
        shp = self.net.input_shape[0]
        self.input_size = (shp[3], shp[2]) if shp is not None and all(isinstance(d, int) for d in shp[2:]) else (112, 112)

    def prepare(self, ctx_id=0, **kwargs):
        pass

    def get_feat(self, imgs):
        import cv2
        if not isinstance(imgs, list):
            imgs = [imgs]
        blob = cv2.dnn.blobFromImages(imgs, 1.0 / self.input_std, self.input_size, (self.input_mean,) * 3, swapRB=True)
        out = self.net.run(image_to_act(blob, self.device))[0]
        _check_finite("ArcFace", out)
        return out.reshape(out.shape[0], -1).cpu().numpy()

    def get(self, img, face):
        face.embedding = self.get_feat(norm_crop(img, face.kps, self.input_size[0]))[0]
        return face.embedding


class Face(dict):
    """insightface.app.common.Face: a dict with attribute access; normed_embedding and embedding_norm derived."""

    def __getattr__(self, name):
        return self.get(name)

    def __setattr__(self, name, value):
        self[name] = value

    @property
    def embedding_norm(self):
        return None if self.embedding is None else float(np.linalg.norm(self.embedding))

    @property
    def normed_embedding(self):
        return None if self.embedding is None else self.embedding / self.embedding_norm


MODEL_FILES = {"detection": "scrfd_10g_bnkps.onnx", "recognition": "glintr100.onnx"}


def antelopev2_files(root, name="antelopev2"):
    """The two model files OMG uses, or None when either is missing."""
    d = os.path.join(os.path.expanduser(root), "models", name)
    files = {k: os.path.join(d, v) for k, v in MODEL_FILES.items()}
    return files if all(os.path.isfile(f) for f in files.values()) else None


class FaceAnalysis:
    """insightface.app.FaceAnalysis('antelopev2') on the kernels: reads <root>/models/<name>/scrfd_10g_bnkps.onnx and
    glintr100.onnx; the pack's landmark and gender/age models are not loaded (OMG reads none of their attributes).
    `providers` is accepted for call compatibility and ignored: everything runs on the CUDA device."""

    def __init__(self, name="antelopev2", root="~/.insightface", providers=None, device="cuda", **kwargs):
        files = antelopev2_files(root, name)
        if files is None:
            raise FileNotFoundError(f"{os.path.join(root, 'models', name)} must hold " + " and ".join(MODEL_FILES.values()))
        self.det_model = SCRFD(files["detection"], device=device)
        self.rec_model = ArcFace(files["recognition"], device=device)
        self.models = {"detection": self.det_model, "recognition": self.rec_model}
        self.det_size = (640, 640)

    def prepare(self, ctx_id, det_thresh=0.5, det_size=(640, 640)):
        self.det_thresh, self.det_size = det_thresh, tuple(det_size)
        self.det_model.prepare(ctx_id, input_size=det_size, det_thresh=det_thresh)
        self.rec_model.prepare(ctx_id)

    def get(self, img, max_num=0):
        """Faces of a BGR uint8 image in the detector's NMS order; every face's crop goes through the recogniser in
        one batch."""
        if max_num != 0:
            raise NotImplementedError("FaceAnalysis.get: max_num selection is not implemented (no OMG caller uses it)")
        bboxes, kpss = self.det_model.detect(img, max_num=0, metric="default")
        if bboxes.shape[0] == 0:
            return []
        faces = [Face(bbox=bboxes[i, 0:4], kps=None if kpss is None else kpss[i], det_score=bboxes[i, 4])
                 for i in range(bboxes.shape[0])]
        if kpss is not None:
            size = self.rec_model.input_size[0]
            emb = self.rec_model.get_feat([norm_crop(img, f.kps, size) for f in faces])
            for f, e in zip(faces, emb):
                f.embedding = e
        return faces
