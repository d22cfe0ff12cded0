"""fp32 torch restatement of ultralytics' WorldModel (YOLO-World v1 / v2) and a float64 numpy restatement of its
post-processing - the reference the kernel path is tested against.  Modules and parameter names follow ultralytics'
state-dict keys (model.{i}.cv1.conv.weight, .attn.gl, .cv4.{k}.logit_scale, ...), so `WorldModel(...).state_dict()`
is also the layout of a synthetic checkpoint.  Written from the published behaviour of ultralytics 8.x, not its source.
The layer arithmetic (parse_model's width / depth scaling) is omg_b200.yolo_world.parse_layout."""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from omg_b200.yolo_world import detect_head_channels, layout_yaml, parse_layout


class Conv(nn.Module):
    def __init__(self, c1, c2, k=1, s=1, act=True):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, k // 2, bias=False)
        self.bn = nn.BatchNorm2d(c2, eps=1e-3, momentum=0.03)
        self.act = nn.SiLU() if act else nn.Identity()

    def forward(self, x):
        return self.act(self.bn(self.conv(x)))


class Bottleneck(nn.Module):
    def __init__(self, c1, c2, shortcut=True):
        super().__init__()
        self.cv1, self.cv2 = Conv(c1, c2, 3), Conv(c2, c2, 3)
        self.add = shortcut and c1 == c2

    def forward(self, x):
        return x + self.cv2(self.cv1(x)) if self.add else self.cv2(self.cv1(x))


class C2f(nn.Module):
    def __init__(self, c1, c2, n=1, shortcut=False):
        super().__init__()
        self.c = int(c2 * 0.5)
        self.cv1 = Conv(c1, 2 * self.c, 1)
        self.cv2 = Conv((2 + n) * self.c, c2, 1)
        self.m = nn.ModuleList(Bottleneck(self.c, self.c, shortcut) for _ in range(n))

    def forward(self, x):
        y = list(self.cv1(x).chunk(2, 1))
        y.extend(m(y[-1]) for m in self.m)
        return self.cv2(torch.cat(y, 1))


class MaxSigmoidAttnBlock(nn.Module):
    def __init__(self, c1, c2, nh=1, ec=128, gc=512, scale=False):
        super().__init__()
        self.nh, self.hc = nh, c2 // nh
        self.ec = Conv(c1, ec, 1, act=False) if c1 != ec else None
        self.gl = nn.Linear(gc, ec)
        self.bias = nn.Parameter(torch.zeros(nh))
        self.proj_conv = Conv(c1, c2, 3, act=False)
        self.scale = nn.Parameter(torch.ones(1, nh, 1, 1)) if scale else 1.0

    def forward(self, x, guide):
        bs, _, h, w = x.shape
        guide = self.gl(guide).view(bs, -1, self.nh, self.hc)
        embed = self.ec(x) if self.ec is not None else x
        embed = embed.view(bs, self.nh, self.hc, h, w)
        aw = torch.einsum("bmchw,bnmc->bmhwn", embed, guide).max(dim=-1)[0]
        aw = aw / (self.hc ** 0.5) + self.bias[None, :, None, None]
        aw = aw.sigmoid() * self.scale
        x = self.proj_conv(x).view(bs, self.nh, -1, h, w)
        return (x * aw.unsqueeze(2)).view(bs, -1, h, w)


class C2fAttn(nn.Module):
    def __init__(self, c1, c2, n=1, ec=128, nh=1, gc=512, shortcut=False):
        super().__init__()
        self.c = int(c2 * 0.5)
        self.cv1 = Conv(c1, 2 * self.c, 1)
        self.cv2 = Conv((3 + n) * self.c, c2, 1)
        self.m = nn.ModuleList(Bottleneck(self.c, self.c, shortcut) for _ in range(n))
        self.attn = MaxSigmoidAttnBlock(self.c, self.c, gc=gc, ec=ec, nh=nh)

    def forward(self, x, guide):
        y = list(self.cv1(x).chunk(2, 1))
        y.extend(m(y[-1]) for m in self.m)
        y.append(self.attn(y[-1], guide))
        return self.cv2(torch.cat(y, 1))


class SPPF(nn.Module):
    def __init__(self, c1, c2, k=5):
        super().__init__()
        c_ = c1 // 2
        self.cv1, self.cv2 = Conv(c1, c_, 1), Conv(c_ * 4, c2, 1)
        self.m = nn.MaxPool2d(k, 1, k // 2)

    def forward(self, x):
        y = [self.cv1(x)]
        y.extend(self.m(y[-1]) for _ in range(3))
        return self.cv2(torch.cat(y, 1))


class ImagePoolingAttn(nn.Module):
    def __init__(self, ec=256, ch=(), ct=512, nh=8, k=3):
        super().__init__()
        self.query = nn.Sequential(nn.LayerNorm(ct), nn.Linear(ct, ec))
        self.key = nn.Sequential(nn.LayerNorm(ec), nn.Linear(ec, ec))
        self.value = nn.Sequential(nn.LayerNorm(ec), nn.Linear(ec, ec))
        self.proj = nn.Linear(ec, ct)
        self.projections = nn.ModuleList(nn.Conv2d(c, ec, 1) for c in ch)
        self.im_pools = nn.ModuleList(nn.AdaptiveMaxPool2d((k, k)) for _ in ch)
        self.ec, self.nh, self.hc, self.k = ec, nh, ec // nh, k

    def forward(self, x, text):
        bs = x[0].shape[0]
        x = [pool(proj(xi)).view(bs, -1, self.k ** 2) for xi, proj, pool in zip(x, self.projections, self.im_pools)]
        x = torch.cat(x, dim=-1).transpose(1, 2)
        q = self.query(text).reshape(bs, -1, self.nh, self.hc)
        k = self.key(x).reshape(bs, -1, self.nh, self.hc)
        v = self.value(x).reshape(bs, -1, self.nh, self.hc)
        aw = F.softmax(torch.einsum("bnmc,bkmc->bmnk", q, k) / self.hc ** 0.5, dim=-1)
        x = torch.einsum("bmnk,bkmc->bnmc", aw, v)
        return self.proj(x.reshape(bs, -1, self.ec)) + text


class ContrastiveHead(nn.Module):
    def __init__(self):
        super().__init__()
        self.bias = nn.Parameter(torch.tensor([-10.0]))
        self.logit_scale = nn.Parameter(torch.ones([]) * torch.tensor(1 / 0.07).log())

    def forward(self, x, w):
        x, w = F.normalize(x, dim=1, p=2), F.normalize(w, dim=-1, p=2)
        return torch.einsum("bchw,bkc->bkhw", x, w) * self.logit_scale.exp() + self.bias


class BNContrastiveHead(nn.Module):
    def __init__(self, embed_dims):
        super().__init__()
        self.norm = nn.BatchNorm2d(embed_dims)
        self.bias = nn.Parameter(torch.tensor([-10.0]))
        self.logit_scale = nn.Parameter(-1.0 * torch.ones([]))

    def forward(self, x, w):
        x, w = self.norm(x), F.normalize(w, dim=-1, p=2)
        return torch.einsum("bchw,bkc->bkhw", x, w) * self.logit_scale.exp() + self.bias


class DFL(nn.Module):
    def __init__(self, c1=16):
        super().__init__()
        self.conv = nn.Conv2d(c1, 1, 1, bias=False).requires_grad_(False)
        self.conv.weight.data[:] = torch.arange(c1, dtype=torch.float).view(1, c1, 1, 1)
        self.c1 = c1

    def forward(self, x):
        b, _, a = x.shape
        return self.conv(x.view(b, 4, self.c1, a).transpose(2, 1).softmax(1)).view(b, 4, a)


def make_anchors(feats, strides, offset=0.5):
    pts, st = [], []
    for f, s in zip(feats, strides):
        h, w = f.shape[2:]
        sx = torch.arange(w, dtype=f.dtype, device=f.device) + offset
        sy = torch.arange(h, dtype=f.dtype, device=f.device) + offset
        sy, sx = torch.meshgrid(sy, sx, indexing="ij")
        pts.append(torch.stack((sx, sy), -1).view(-1, 2))
        st.append(torch.full((h * w, 1), s, dtype=f.dtype, device=f.device))
    return torch.cat(pts), torch.cat(st)


class WorldDetect(nn.Module):
    def __init__(self, nc=80, embed=512, with_bn=False, ch=()):
        super().__init__()
        self.nl, self.reg_max = len(ch), 16
        c2, c3 = detect_head_channels(ch[0], nc)
        self.cv2 = nn.ModuleList(nn.Sequential(Conv(x, c2, 3), Conv(c2, c2, 3), nn.Conv2d(c2, 64, 1)) for x in ch)
        self.cv3 = nn.ModuleList(nn.Sequential(Conv(x, c3, 3), Conv(c3, c3, 3), nn.Conv2d(c3, embed, 1)) for x in ch)
        self.cv4 = nn.ModuleList(BNContrastiveHead(embed) if with_bn else ContrastiveHead() for _ in ch)
        self.dfl = DFL(16)
        self.stride = (8, 16, 32)

    def forward(self, x, text):
        """-> (y [B, 4 + nc, A] = xywh in letterbox pixels and sigmoid scores, raw per-level (box, embedding) maps)."""
        raw = [(self.cv2[i](x[i]), self.cv3[i](x[i])) for i in range(self.nl)]
        cls = [self.cv4[i](raw[i][1], text) for i in range(self.nl)]
        B = x[0].shape[0]
        box = torch.cat([r[0].view(B, 64, -1) for r in raw], 2)
        logits = torch.cat([c.view(B, c.shape[1], -1) for c in cls], 2)
        anchors, strides = make_anchors(x, self.stride)
        d = self.dfl(box)
        lt, rb = d.chunk(2, 1)
        a = anchors.T.unsqueeze(0)
        x1y1, x2y2 = a - lt, a + rb
        dbox = torch.cat(((x1y1 + x2y2) / 2, x2y2 - x1y1), 1) * strides.T
        return torch.cat((dbox, logits.sigmoid()), 1), raw


_MODULES = {"Conv": Conv, "C2f": C2f, "C2fAttn": C2fAttn, "SPPF": SPPF}


class WorldModel(nn.Module):
    def __init__(self, variant=2, scale="l", yaml=None):
        super().__init__()
        self.layers = parse_layout(yaml or layout_yaml(variant, scale))
        mods = []
        for s in self.layers:
            t = s["type"]
            if t == "Conv":
                m = Conv(s["c1"], s["c2"], s["k"], s["s"])
            elif t == "C2f":
                m = C2f(s["c1"], s["c2"], s["n"], s["shortcut"])
            elif t == "C2fAttn":
                m = C2fAttn(s["c1"], s["c2"], s["n"], s["ec"], s["nh"], s["gc"])
            elif t == "SPPF":
                m = SPPF(s["c1"], s["c2"], s["k"])
            elif t == "Upsample":
                m = nn.Upsample(scale_factor=2, mode="nearest")
            elif t == "Concat":
                m = nn.Identity()
            elif t == "ImagePoolingAttn":
                m = ImagePoolingAttn(s["ec"], s["ch"], s["ct"], s["nh"], s["k"])
            else:
                m = WorldDetect(s["nc"], s["embed"], s["with_bn"], s["ch"])
            mods.append(m)
        self.model = nn.ModuleList(mods)

    def forward(self, x, txt_feats):
        """x (B, 3, H, W) in [0, 1], txt_feats (B | 1, n, 512) normalised -> WorldDetect's (y, raw)."""
        txt = txt_feats.expand(x.shape[0], -1, -1)
        ori = txt.clone()
        ys = []
        for s, m in zip(self.layers, self.model):
            f = s["f"]
            if s["i"] > 0 and f != -1:
                x = ys[f] if isinstance(f, int) else [x if j == -1 else ys[j] for j in f]
            if s["type"] == "Concat":
                x = torch.cat(x, 1)
            elif s["type"] == "C2fAttn":
                x = m(x, txt)
            elif s["type"] == "WorldDetect":
                x = m(x, ori)
            elif s["type"] == "ImagePoolingAttn":
                txt = m(x, txt)
            else:
                x = m(x)
            ys.append(x)
        return x


def randomize_(model, seed=0, bias=-10.0):
    """Random weights with random BatchNorm statistics (so folding is exercised); the contrastive heads' bias set to
    `bias` (ultralytics initialises it at -10, which leaves no detection over random weights)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("dfl.conv.weight"):
                continue
            if p.dim() >= 2:
                fan_in = p[0].numel()
                p.copy_(torch.randn(p.shape, generator=g) * (1.0 / math.sqrt(fan_in)))
            else:
                p.copy_(torch.rand(p.shape, generator=g) * 0.4 + 0.8 if "bn" in name or "norm" in name else
                        torch.randn(p.shape, generator=g) * 0.1)
        for name, b in model.named_buffers():
            if name.endswith("running_mean"):
                b.copy_(torch.randn(b.shape, generator=g) * 0.1)
            elif name.endswith("running_var"):
                b.copy_(torch.rand(b.shape, generator=g) * 0.5 + 0.75)
        for m in model.modules():
            if isinstance(m, (ContrastiveHead, BNContrastiveHead)):
                m.bias.fill_(bias)
                if isinstance(m, ContrastiveHead):
                    m.logit_scale.fill_(math.log(1 / 0.07))
    return model.eval()


# -------------------------------------------------------------------------------------- float64 numpy post-processing
def anchor_rows(box, emb, text, strides, cls_scale, cls_bias, normalize_x):
    """omg_yolo_detect pass (a) in float64: per-level box [h, w, 64] and emb [h, w, E] maps -> rows [A, 6]
    (x0, y0, x1, y1, max sigmoid score, first argmax class) in letterbox pixels."""
    t = np.asarray(text, dtype=np.float64)
    out = []
    for b, e, s, sc, bi in zip(box, emb, strides, cls_scale, cls_bias):
        h, w = b.shape[:2]
        b = np.asarray(b, np.float64).reshape(h * w, 4, 16)
        e = np.asarray(e, np.float64).reshape(h * w, -1)
        if normalize_x:
            e = e / np.maximum(np.linalg.norm(e, axis=1, keepdims=True), 1e-12)
        p = 1.0 / (1.0 + np.exp(-(e @ t.T * sc + bi)))
        pb = np.exp(b - b.max(axis=2, keepdims=True))
        d = (pb * np.arange(16)).sum(2) / pb.sum(2)
        gy, gx = np.divmod(np.arange(h * w), w)
        ax, ay = gx + 0.5, gy + 0.5
        x1, y1, x2, y2 = ax - d[:, 0], ay - d[:, 1], ax + d[:, 2], ay + d[:, 3]
        out.append(np.stack([x1 * s, y1 * s, x2 * s, y2 * s, p.max(1), p.argmax(1)], 1))
    return np.concatenate(out)


def nms(boxes, scores, iou_thres):
    """Greedy NMS as torchvision.ops.nms computes it (descending score, ties by lower index; suppress IoU > iou_thres,
    no +1 in the areas) -> kept indices."""
    boxes = np.asarray(boxes, np.float64)
    order = np.lexsort((np.arange(len(scores)), -np.asarray(scores, np.float64)))
    area = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
    supp = np.zeros(len(scores), bool)
    keep = []
    for i in order:
        if supp[i]:
            continue
        keep.append(i)
        xx1 = np.maximum(boxes[i, 0], boxes[:, 0])
        yy1 = np.maximum(boxes[i, 1], boxes[:, 1])
        xx2 = np.minimum(boxes[i, 2], boxes[:, 2])
        yy2 = np.minimum(boxes[i, 3], boxes[:, 3])
        inter = np.clip(xx2 - xx1, 0, None) * np.clip(yy2 - yy1, 0, None)
        iou = inter / (area[i] + area - inter)
        supp |= iou > iou_thres
    return np.array(keep, dtype=np.int64)


def postprocess(rows, conf=0.1, iou=0.7, max_wh=7680, agnostic=False, max_det=300):
    """ultralytics non_max_suppression (single label) on rows [A, 6] -> (kept anchor indices, rows[kept])."""
    rows = np.asarray(rows, np.float64)
    cand = np.nonzero(rows[:, 4] > conf)[0]
    r = rows[cand]
    off = 0.0 if agnostic else r[:, 5:6] * max_wh
    k = nms(r[:, :4] + off, r[:, 4], iou)[:max_det]
    return cand[k], r[k]
