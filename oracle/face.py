"""fp32 oracle of face analysis (insightface FaceAnalysis('antelopev2'), used by the InstantID flow at reference
inference_instantid.py:226-228,353-354 and src/pipelines/instantid_pipeline.py:757-767).

insightface is neither in the reference tree nor installable here, so its behaviour is restated from knowledge of
insightface 0.7.x, not from its source, the way SURVEY section 8c restates diffusers.  This file is the single place to
correct it.  The points most likely to need that: the +1 pixel convention of the NMS areas and overlaps, the
input-normalisation rule of ArcFaceONNX (node names Sub / Mul among the first 8), and the order of the detector outputs
(scores x strides, boxes x strides, key-points x strides).  Ties of equal scores are ordered by ascending anchor index
here (insightface's argsort()[::-1] leaves them in no specified order).

- `IResNet`: insightface's arcface_torch IResNet (IBasicBlock BN-Conv-BN-PReLU-Conv-BN, 1x1 / s2 conv + BN shortcut,
  BN-Flatten-FC-BN1d head); layers (3, 13, 30, 3) is the 100-layer recogniser of glintr100.onnx.
- `ScrfdNet`: an SCRFD-style detector (ResNet-V1e stem, max-pool, avg-down BasicBlock stages, top-down FPN with nearest
  x2, heads shared across strides with a BatchNorm per stride), emitting the nine outputs in insightface's order and
  shapes.  Its default widths follow SCRFD-10G's backbone (stem 28/28/56, stages 56/88/88/224 of 3/4/2/3 blocks).
- numpy restatement of the contract: preprocessing, anchor decode, NMS, Umeyama, norm_crop, get().
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------------------ networks
class IBasicBlock(nn.Module):
    def __init__(self, inplanes, planes, stride=1):
        super().__init__()
        self.bn1 = nn.BatchNorm2d(inplanes, eps=1e-5)
        self.conv1 = nn.Conv2d(inplanes, planes, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes, eps=1e-5)
        self.prelu = nn.PReLU(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes, eps=1e-5)
        self.downsample = None
        if stride != 1 or inplanes != planes:
            self.downsample = nn.Sequential(nn.Conv2d(inplanes, planes, 1, stride, bias=False),
                                            nn.BatchNorm2d(planes, eps=1e-5))

    def forward(self, x):
        identity = x
        out = self.bn3(self.conv2(self.prelu(self.bn2(self.conv1(self.bn1(x))))))
        if self.downsample is not None:
            identity = self.downsample(x)
        return out + identity


class IResNet(nn.Module):
    def __init__(self, layers=(3, 13, 30, 3), widths=(64, 128, 256, 512), num_features=512, input_size=112):
        super().__init__()
        self.conv1 = nn.Conv2d(3, widths[0], 3, 1, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(widths[0], eps=1e-5)
        self.prelu = nn.PReLU(widths[0])
        blocks, cin = [], widths[0]
        for n, w in zip(layers, widths):
            for j in range(n):
                blocks.append(IBasicBlock(cin, w, 2 if j == 0 else 1))
                cin = w
        self.layers = nn.Sequential(*blocks)
        self.bn2 = nn.BatchNorm2d(cin, eps=1e-5)
        fs = input_size // 2 ** len(layers)
        self.fc = nn.Linear(cin * fs * fs, num_features)
        self.features = nn.BatchNorm1d(num_features, eps=1e-5)

    def forward(self, x):
        x = self.layers(self.prelu(self.bn1(self.conv1(x))))
        x = torch.flatten(self.bn2(x), 1)
        return self.features(self.fc(x))


class BasicBlock(nn.Module):
    """ResNet-V1d/e BasicBlock; a strided or widening shortcut is avg-pool (ceil, no pad counted) + 1x1 conv + BN."""

    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, cout, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(cout)
        self.conv2 = nn.Conv2d(cout, cout, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(cout)
        self.down = None
        if stride != 1 or cin != cout:
            pool = [nn.AvgPool2d(stride, stride, ceil_mode=True, count_include_pad=False)] if stride != 1 else []
            self.down = nn.Sequential(*pool, nn.Conv2d(cin, cout, 1, bias=False), nn.BatchNorm2d(cout))

    def forward(self, x):
        out = self.bn2(self.conv2(F.relu(self.bn1(self.conv1(x)))))
        return F.relu(out + (x if self.down is None else self.down(x)))


class ScrfdNet(nn.Module):
    def __init__(self, stem=(28, 28, 56), stages=(56, 88, 88, 224), blocks=(3, 4, 2, 3), fpn=56, head=80,
                 stacked=3, num_anchors=2):
        super().__init__()
        s = [3, *stem]
        self.stem = nn.Sequential(*[m for i in range(3) for m in (
            nn.Conv2d(s[i], s[i + 1], 3, 2 if i == 0 else 1, 1, bias=False), nn.BatchNorm2d(s[i + 1]), nn.ReLU())])
        self.pool = nn.MaxPool2d(3, 2, 1)
        layers, cin = [], stem[-1]
        for i, (c, n) in enumerate(zip(stages, blocks)):
            layers.append(nn.Sequential(*[BasicBlock(cin if j == 0 else c, c, (1 if i == 0 else 2) if j == 0 else 1)
                                          for j in range(n)]))
            cin = c
        self.stages = nn.ModuleList(layers)
        self.lateral = nn.ModuleList([nn.Conv2d(c, fpn, 1) for c in stages[1:]])
        self.fpn = nn.ModuleList([nn.Conv2d(fpn, fpn, 3, 1, 1) for _ in stages[1:]])
        self.head_convs = nn.ModuleList([nn.Conv2d(fpn if i == 0 else head, head, 3, 1, 1) for i in range(stacked)])
        self.head_bns = nn.ModuleList([nn.ModuleList([nn.BatchNorm2d(head) for _ in range(stacked)]) for _ in range(3)])
        self.cls = nn.Conv2d(head, num_anchors, 3, 1, 1)
        self.reg = nn.Conv2d(head, 4 * num_anchors, 3, 1, 1)
        self.kps = nn.Conv2d(head, 10 * num_anchors, 3, 1, 1)

    def forward(self, x):
        x = self.pool(self.stem(x))
        feats = []
        for i, st in enumerate(self.stages):
            x = st(x)
            if i > 0:
                feats.append(x)
        lat = [l(f) for l, f in zip(self.lateral, feats)]
        for i in range(len(lat) - 1, 0, -1):
            lat[i - 1] = lat[i - 1] + F.interpolate(lat[i], scale_factor=2.0, mode="nearest")
        outs = [f(l) for f, l in zip(self.fpn, lat)]
        scores, boxes, kps = [], [], []
        for lvl, y in enumerate(outs):
            for conv, bn in zip(self.head_convs, self.head_bns[lvl]):
                y = F.relu(bn(conv(y)))
            scores.append(self.cls(y).permute(0, 2, 3, 1).reshape(-1, 1).sigmoid())
            boxes.append(self.reg(y).permute(0, 2, 3, 1).reshape(-1, 4))
            kps.append(self.kps(y).permute(0, 2, 3, 1).reshape(-1, 10))
        return (*scores, *boxes, *kps)


def randomize_(model, seed, score_bias=None):
    """Synthetic weights that keep activations O(1) through any depth: He-scaled convs, BatchNorm statistics drawn
    around the batch statistics a unit input would produce (gamma ~ 1, small beta, running var ~ 1), PReLU 0.25.
    score_bias (ScrfdNet): the classifier bias, which sets how many anchors pass the threshold."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                fan = m.weight[0].numel()
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (1.0 / fan) ** 0.5)
                if m.bias is not None:
                    m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.05)
            elif isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
                c = m.num_features
                m.weight.copy_(1.0 + 0.1 * torch.randn(c, generator=g))
                m.bias.copy_(0.05 * torch.randn(c, generator=g))
                m.running_mean.copy_(0.05 * torch.randn(c, generator=g))
                m.running_var.copy_(1.0 + 0.2 * torch.rand(c, generator=g))
            elif isinstance(m, nn.PReLU):
                m.weight.fill_(0.25)
        if isinstance(model, IResNet):   # residual branches: keep the trunk's variance from growing with depth
            for blk in model.layers:
                blk.bn3.weight.mul_(0.3)
        if isinstance(model, ScrfdNet):
            for st in model.stages:
                for blk in st:
                    blk.bn2.weight.mul_(0.3)
            if score_bias is not None:
                model.cls.bias.fill_(score_bias)
            model.reg.bias.fill_(1.0)    # positive distances: boxes of a few strides around each anchor
    return model.eval()


# ------------------------------------------------------------------------------------------- numpy contract
ARCFACE_DST = np.array([[38.2946, 51.6963], [73.5318, 51.5014], [56.0252, 71.7366], [41.5493, 92.3655],
                        [70.7299, 92.2041]], dtype=np.float32)


def det_preprocess(img, input_size=(640, 640)):
    import cv2
    im_ratio = float(img.shape[0]) / img.shape[1]
    if im_ratio > float(input_size[1]) / input_size[0]:
        new_h = input_size[1]
        new_w = int(new_h / im_ratio)
    else:
        new_w = input_size[0]
        new_h = int(new_w * im_ratio)
    det_img = np.zeros((input_size[1], input_size[0], 3), dtype=np.uint8)
    det_img[:new_h, :new_w, :] = cv2.resize(img, (new_w, new_h))
    return det_img, float(new_h) / img.shape[0]


def det_blob(det_img):
    import cv2
    return cv2.dnn.blobFromImage(det_img, 1.0 / 128.0, tuple(det_img.shape[0:2][::-1]), (127.5,) * 3, swapRB=True)


def decode(net_outs, input_h, input_w, det_thresh, strides=(8, 16, 32), num_anchors=2, use_kps=True):
    """SCRFD.forward: per stride, anchors with score >= det_thresh -> (scores, boxes, kpss) concatenated over strides."""
    fmc = len(strides)
    scores_l, boxes_l, kps_l = [], [], []
    for idx, s in enumerate(strides):
        scores = np.asarray(net_outs[idx], dtype=np.float32).reshape(-1)
        bbox = np.asarray(net_outs[idx + fmc], dtype=np.float32).reshape(-1, 4) * np.float32(s)
        h, w = input_h // s, input_w // s
        centers = np.stack(np.mgrid[:h, :w][::-1], axis=-1).astype(np.float32)
        centers = (centers * s).reshape(-1, 2)
        if num_anchors > 1:
            centers = np.stack([centers] * num_anchors, axis=1).reshape(-1, 2)
        pos = np.where(scores >= np.float32(det_thresh))[0]
        b = np.stack([centers[:, 0] - bbox[:, 0], centers[:, 1] - bbox[:, 1],
                      centers[:, 0] + bbox[:, 2], centers[:, 1] + bbox[:, 3]], axis=-1)
        scores_l.append(scores[pos])
        boxes_l.append(b[pos])
        if use_kps:
            k = np.asarray(net_outs[idx + 2 * fmc], dtype=np.float32).reshape(-1, 10) * np.float32(s)
            pts = np.stack([centers[:, i % 2] + k[:, i] for i in range(10)], axis=-1).reshape(-1, 5, 2)
            kps_l.append(pts[pos])
    return scores_l, boxes_l, kps_l


def nms(dets, thresh=0.4):
    """Greedy NMS with the +1 pixel convention; dets [n, 5] already in descending score order."""
    x1, y1, x2, y2 = dets[:, 0], dets[:, 1], dets[:, 2], dets[:, 3]
    one = np.float32(1)
    areas = (x2 - x1 + one) * (y2 - y1 + one)
    order = np.arange(dets.shape[0])
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(i)
        xx1 = np.maximum(x1[i], x1[order[1:]])
        yy1 = np.maximum(y1[i], y1[order[1:]])
        xx2 = np.minimum(x2[i], x2[order[1:]])
        yy2 = np.minimum(y2[i], y2[order[1:]])
        w = np.maximum(np.float32(0), xx2 - xx1 + one)
        h = np.maximum(np.float32(0), yy2 - yy1 + one)
        inter = w * h
        ovr = inter / (areas[i] + areas[order[1:]] - inter)
        order = order[np.where(ovr <= np.float32(thresh))[0] + 1]
    return keep


def detect_from_outputs(net_outs, input_h, input_w, det_scale, det_thresh=0.5, nms_thresh=0.4, **kw):
    """decode + sort + / det_scale + NMS -> (det [n, 5] fp32, kpss [n, 5, 2] fp32)."""
    scores_l, boxes_l, kps_l = decode(net_outs, input_h, input_w, det_thresh, **kw)
    scores = np.concatenate(scores_l).astype(np.float32)
    ds = np.float32(det_scale)
    boxes = (np.concatenate(boxes_l) / ds).astype(np.float32)
    order = np.lexsort((np.arange(scores.size), -scores))   # descending score, ties by anchor index
    pre = np.hstack((boxes, scores[:, None]))[order].astype(np.float32)
    keep = nms(pre, nms_thresh)
    kpss = None
    if kps_l:
        kpss = (np.concatenate(kps_l) / ds).astype(np.float32)[order][keep]
    return pre[keep], kpss


def umeyama(src, dst):
    """skimage's SimilarityTransform.estimate (Umeyama with scale), 3 x 3."""
    src, dst = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    n, dim = src.shape
    sm, dm = src.mean(0), dst.mean(0)
    sd, dd = src - sm, dst - dm
    A = dd.T @ sd / n
    d = np.ones(dim)
    if np.linalg.det(A) < 0:
        d[-1] = -1
    T = np.eye(dim + 1)
    U, S, V = np.linalg.svd(A)
    rank = np.linalg.matrix_rank(A)
    if rank == 0:
        return np.nan * T
    if rank == dim - 1 and np.linalg.det(U) * np.linalg.det(V) > 0:
        T[:dim, :dim] = U @ V
    else:
        dd_ = d.copy()
        if rank == dim - 1:
            dd_[-1] = -1
        T[:dim, :dim] = U @ np.diag(dd_) @ V
    scale = 1.0 / sd.var(0).sum() * (S @ d)
    T[:dim, dim] = dm - scale * (T[:dim, :dim] @ sm)
    T[:dim, :dim] *= scale
    return T


def norm_crop(img, kps, image_size=112):
    import cv2
    M = umeyama(kps, ARCFACE_DST * (image_size / 112.0))[:2]
    return cv2.warpAffine(img, M, (image_size, image_size), borderValue=0.0)


def rec_blob(crops, mean=127.5, std=127.5, size=112):
    import cv2
    return cv2.dnn.blobFromImages(crops, 1.0 / std, (size, size), (mean,) * 3, swapRB=True)


@torch.no_grad()
def get(img, det_net, rec_net, det_thresh=0.5, det_size=(640, 640), rec_mean=127.5, rec_std=127.5):
    """FaceAnalysis.get with the fp32 torch modules: list of dicts (bbox, kps, det_score, embedding)."""
    det_img, det_scale = det_preprocess(img, det_size)
    outs = [o.numpy() for o in det_net(torch.from_numpy(det_blob(det_img)))]
    det, kpss = detect_from_outputs(outs, det_size[1], det_size[0], det_scale, det_thresh)
    faces = [dict(bbox=det[i, :4], kps=kpss[i], det_score=det[i, 4]) for i in range(det.shape[0])]
    for f in faces:
        blob = rec_blob([norm_crop(img, f["kps"])], rec_mean, rec_std)
        f["embedding"] = rec_net(torch.from_numpy(blob))[0].numpy()
    return faces
