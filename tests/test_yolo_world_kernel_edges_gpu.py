"""Kernel edges of the YOLO-World kernels (omg_text_gate, omg_adaptive_maxpool, omg_yolo_detect) through the C ABI, with
the conventions of test_face_sam_kernel_edges_gpu.py:

* omg_text_gate and pass (a) of omg_yolo_detect are bounded per element against float64 references computed from the
  same fp16 / fp32 values the kernels read,  |out - ref| <= 4 u |ref| + k u rms(ref);
* pass (b) of omg_yolo_detect (threshold, sort, NMS, rescale) is compared bit for bit with a float32 restatement of
  ultralytics' non_max_suppression / torchvision's nms / scale_boxes (`nms_float32` below) run on the kernel's own rows;
* outputs sit in NaN guard buffers that must stay intact, operands in NaN-poisoned windows (wider rows, extra pixel
  rows), per-head / per-class vectors in NaN-padded buffers;
* every case runs twice and must be bit-identical (candidate compaction in pass (b) uses atomicAdd).
`pytest -s` prints the k each case needs.  omg_adaptive_maxpool's cases are parameters of
test_yolo_world_gpu.py::test_adaptive_maxpool_matches_torch (compared bit for bit with torch)."""
import ctypes as C
import math
import os
import sys
import zlib

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_face_sam_kernel_edges_gpu import Rows, _nan_vec  # noqa: E402
from test_kernel_edges_gpu import PAD, Guard, check, same_bits, twice  # noqa: E402

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24

# Per-element k, with the worst value the family's cases need on an NVIDIA H100 80GB HBM3 at a 700 W power limit beside
# it (a value <= 0 means every element is already within 4 u |ref|).
K_GATE = 1.0          # measured 0.00 (every head split, prompt count, layout and saturated gates)
K_ANCHOR_BOX = 12.0   # measured 7.91 (3 levels, E = 512, normalize_x = 0); 3.75 on the executor's head maps
K_ANCHOR_SCORE = 48.0  # measured <= 0 in the cases here; 33.3 on the v2 x-scale executor's head maps
                       # (test_yolo_world_gpu.py: 512-channel dot products of un-normalised embeddings)

SMEM_LIMIT = 232448    # opt-in shared memory per block on sm_90


@pytest.fixture(scope="module")
def lib():
    from omg_b200 import _lib
    return _lib.load()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _call(rc, lib, what):
    assert rc == 0, f"{what}: {lib.omg_last_error().decode()}"


def _window(rows, cols, ld, extra_rows=3, dtype=torch.float16):
    """[rows, cols] operand with a row stride of ld inside a NaN buffer with `extra_rows` more rows."""
    return Rows(rows + extra_rows, cols, ld, dtype=dtype).out[:rows]


# ------------------------------------------------------------------------------------------------------- text_gate
def _gate_grid():
    for hc in (16, 32, 64):
        for nh in (1, 2, 3, 6, 8, 9, 10, 200):
            P = 256 // nh
            # nh = 200: P = 1 pixel per block, 56 idle threads; the guide of 2 prompts fits at every hc
            yield f"hc{hc}-nh{nh}", (hc, nh, 2 if nh == 200 else 7, 2, 2 * P + 1, hc * nh, "strided", nh % 2 == 0, 0)


# name -> (hc, nh, n prompts, B, HW, C2, layout, scale given, saturated gates (0: no, 1: +-100 logits))
GATE_CASES = dict(_gate_grid())
GATE_CASES.update({
    "C2-8-per-head-nh3": (32, 3, 5, 2, 100, 24, "strided", True, 0),
    "C2-40-per-head-nh3": (32, 3, 5, 2, 100, 120, "strided", False, 0),
    "C2-40-per-head-hc16-nh10": (16, 10, 4, 2, 60, 400, "strided", True, 0),
    "n1": (32, 8, 1, 2, 70, 256, "strided", True, 0),
    "n2": (32, 8, 2, 2, 70, 256, "strided", False, 0),
    "n80": (32, 8, 80, 2, 70, 256, "strided", True, 0),
    "n226-smem-limit": (32, 8, 226, 2, 70, 256, "strided", True, 0),   # (226 * 256 + 256) * 4 B = 232 448 B
    "HW1-B3": (32, 8, 4, 3, 1, 256, "strided", True, 0),
    "HW-P-1-B3": (32, 8, 4, 3, 31, 256, "strided", False, 0),
    "HW-P-B3": (32, 8, 4, 3, 32, 256, "strided", True, 0),
    "HW-P+1-B3": (32, 8, 4, 3, 33, 256, "strided", False, 0),
    "HW6400-B3": (32, 8, 80, 3, 6400, 256, "strided", True, 0),
    "nh3-HW-P-1": (32, 3, 4, 3, 84, 96, "strided", True, 0),
    "nh3-HW-P+1": (32, 3, 4, 3, 86, 96, "strided", False, 0),
    "inplace-concat-nh4": (32, 4, 6, 2, 150, 128, "inplace", False, 0),
    "inplace-concat-nh3-scale": (32, 3, 6, 2, 150, 96, "inplace", True, 0),
    "inplace-concat-hc64-nh6": (64, 6, 3, 3, 50, 384, "inplace", True, 0),
    "saturated-scale": (32, 8, 5, 2, 70, 256, "strided", True, 1),
    "saturated-no-scale": (16, 6, 5, 2, 70, 96, "strided", False, 1),
})


def gate_reference(embed, guide, bias, scale, nh, p):
    """float64 MaxSigmoidAttnBlock gating: embed [B * HW, Ce], guide [B, n, Ce], p [B * HW, C2]."""
    B, n, Ce = guide.shape
    hc, C2 = Ce // nh, p.shape[1]
    e = embed.double().view(B, -1, nh, hc)
    a = torch.einsum("bpmc,bnmc->bpmn", e, guide.double().view(B, n, nh, hc)).amax(-1) / math.sqrt(hc)
    gate = torch.sigmoid(a + bias.double())
    if scale is not None:
        gate = gate * scale.double()
    return (p.double().view(B, -1, nh, C2 // nh) * gate[..., None]).view(-1, C2)


@pytest.mark.parametrize("case", list(GATE_CASES))
def test_text_gate_heads_prompts_and_layouts(lib, case):
    hc, nh, n, B, HW, C2, layout, with_scale, saturate = GATE_CASES[case]
    Ce, M = hc * nh, B * HW
    assert (n * Ce + (256 // nh) * nh) * 4 <= SMEM_LIMIT
    g = _gen(zlib.crc32(case.encode()))
    embed = (torch.randn(M, Ce, generator=g, device="cuda") * (0.05 if saturate else 1.0)).half()
    guide = torch.randn(B, n, Ce, generator=g, device="cuda")    # a different guide per image
    if saturate:   # logits of about +-100: gates of exactly scale[h] and exactly 0
        bias = torch.tensor([100.0, -100.0], device="cuda").repeat(nh)[:nh]
    else:
        bias = torch.randn(nh, generator=g, device="cuda")
    scale = 0.5 + torch.rand(nh, generator=g, device="cuda") if with_scale else None
    p = (torch.randn(M, C2, generator=g, device="cuda") * 2).half()
    guide_p, bias_p = _nan_vec(guide.reshape(-1)), _nan_vec(bias)
    scale_p = None if scale is None else _nan_vec(scale)
    ref = gate_reference(embed, guide, bias, scale, nh, p)
    what = f"text_gate {case}"

    def launch(e_ptr, ld_e, p_ptr, ld_p, o_ptr, ld_o):
        _call(lib.omg_text_gate(e_ptr, ld_e, Ce, guide_p.data_ptr(), n, bias_p.data_ptr(),
                                None if scale_p is None else scale_p.data_ptr(), nh, p_ptr, ld_p, o_ptr, ld_o, C2, B, HW,
                                _stream()), lib, what)
        torch.cuda.synchronize()

    if layout == "inplace":
        # C2fAttn's concat buffer [.. | .. | y (the embedding, ec = None) | proj_conv's output, gated in place]
        assert Ce == C2
        base = (torch.randn(M, 4 * C2, generator=g, device="cuda")).half()
        base[:, 2 * C2:3 * C2] = embed
        base[:, 3 * C2:] = p

        def run():
            buf = base.clone()
            launch(buf[:, 2 * C2:].data_ptr(), 4 * C2, buf[:, 3 * C2:].data_ptr(), 4 * C2, buf[:, 3 * C2:].data_ptr(),
                   4 * C2)
            assert same_bits(buf[:, :3 * C2], base[:, :3 * C2]), f"{what}: another slice of the concat buffer changed"
            return [buf[:, 3 * C2:].clone()]
    else:
        e_in = _window(M, Ce, Ce + 24)
        e_in.copy_(embed)
        p_in = _window(M, C2, C2 + 8)
        p_in.copy_(p)
        p_before = p_in.clone()

        def run():
            out = Guard((M, C2))
            launch(e_in.data_ptr(), e_in.stride(0), p_in.data_ptr(), p_in.stride(0), out.out.data_ptr(),
                   out.out.stride(0))
            assert out.intact(), f"{what}: write outside the output rows"
            assert same_bits(p_in, p_before), f"{what}: p changed by an out-of-place call"
            return [out.out.clone()]

    out, = twice(run)
    check(out, ref, K_GATE, what=what)
    if saturate:
        grp = C2 // nh
        on = (bias > 0).repeat_interleave(grp)
        full = (p.float() * (1.0 if scale is None else scale.repeat_interleave(grp))).half()
        assert torch.equal(out[:, on], full[:, on]), f"{what}: a saturated gate is not exactly scale[h]"
        assert (out[:, ~on] == 0).all(), f"{what}: a gate of logit -100 is not exactly 0"


# ----------------------------------------------------------------------------------------------- yolo_detect pass (a)
def _level_operands(dist_or_logits, emb, box_ld, emb_ld):
    """Box logits [A, 64] and embeddings [A, E] in NaN-poisoned windows (wider rows, extra anchor rows)."""
    A, E = emb.shape
    box = _window(A, 64, box_ld)
    box.copy_(dist_or_logits)
    e = _window(A, E, emb_ld)
    e.copy_(emb)
    return box, e


def yolo_desc(levels, text, normalize_x):
    """levels: [(stride, fh, fw, box [A, 64], emb [A, E], cls_scale, cls_bias)]; text: fp32 [nc, E] device view
    (in a NaN-padded buffer)."""
    from omg_b200 import _lib as L
    d = L.YoloDesc()
    d.n_levels, d.nc, d.E, d.normalize_x = len(levels), text.shape[0], text.shape[1], int(bool(normalize_x))
    for i, (s, fh, fw, box, emb, sc, bi) in enumerate(levels):
        d.box[i], d.emb[i], d.box_ld[i], d.emb_ld[i] = box.data_ptr(), emb.data_ptr(), box.stride(0), emb.stride(0)
        d.cls_scale[i], d.cls_bias[i] = sc, bi
        d.stride[i], d.fh[i], d.fw[i] = s, fh, fw
    d.text = text.data_ptr()
    return d


def _rows_only(lib, d, T, what):
    rows = Guard((T, 6), dtype=torch.float32, flat=True)
    d.rows, d.out, d.count = rows.out.data_ptr(), None, None
    _call(lib.omg_yolo_detect(C.byref(d), _stream()), lib, what)
    torch.cuda.synchronize()
    assert rows.intact(), f"{what}: write outside the rows"
    return rows.out.clone()


# name -> (levels [(stride, fh, fw, cls_scale, cls_bias)], E, nc, normalize_x, box_ld, emb_ld - E)
ANCHOR_CASES = {
    "1level-7x13-E32-nc3": ([(8, 7, 13, 8.0, -1.0)], 32, 3, True, 72, 8),
    "4levels-nonsquare-E40-nc80": ([(8, 7, 13, 8.0, -1.0), (16, 1, 40, 6.0, 0.5), (32, 40, 1, 9.0, -0.5),
                                    (64, 1, 1, 5.0, 1.0)], 40, 80, True, 80, 16),
    "3levels-letterbox-E512-nc80": ([(8, 24, 40, 9.0, -1.0), (16, 12, 20, 7.0, -0.5), (32, 6, 10, 5.0, 0.0)], 512, 80,
                                    True, 72, 8),
    "3levels-letterbox-E512-nc80-bn": ([(8, 24, 40, 3.0, -1.0), (16, 12, 20, 2.0, 0.5), (32, 6, 10, 4.0, -0.5)], 512, 80,
                                       False, 72, 24),
    "2levels-E1024-nc1024": ([(8, 6, 10, 8.0, -1.0), (16, 3, 5, 6.0, 0.0)], 1024, 1024, True, 64 + 8, 8),
    "2levels-E32-nc1": ([(16, 5, 9, 3.0, -1.0), (32, 3, 5, 2.0, 1.0)], 32, 1, False, 128, 32),
    # the middle level saturates: every logit in [21, 29], so every fp32 sigmoid is 1.0 and the class is the first
    "3levels-saturated-E64-nc7": ([(8, 8, 12, 8.0, -1.0), (16, 4, 6, 4.0, 25.0), (32, 2, 3, 9.0, 0.5)], 64, 7, True,
                                  72, 8),
}


def _anchor_inputs(case):
    levels, E, nc, normalize, box_ld, emb_pad = ANCHOR_CASES[case]
    g = torch.Generator().manual_seed(zlib.crc32(case.encode()))
    text = torch.nn.functional.normalize(torch.randn(nc, E, generator=g), dim=-1)
    tie = (1, nc - 1) if nc >= 3 else None
    if tie:   # identical text rows: their scores tie exactly, and the lower class must win
        text[tie[1]] = text[tie[0]]
    out = []
    for li, (s, fh, fw, sc, bi) in enumerate(levels):
        A = fh * fw
        logits = torch.randn(A, 64, generator=g) * 3.0
        cls = torch.randint(0, nc, (A,), generator=g)
        if tie:
            cls[::5] = tie[0]
        # every embedding leans towards one class's text row, so the largest score is clear of the rest
        emb = (torch.randn(A, E, generator=g) + 2 * math.sqrt(E) * text[cls]) / math.sqrt(E)
        emb[0] = 0.0        # an all-zero embedding row: F.normalize's clamp, score sigmoid(cls_bias), class 0
        emb[-1] = 0.0
        out.append((s, fh, fw, logits.half().cuda(), emb.half().cuda(), sc, bi))
    return out, text.cuda(), normalize, box_ld, emb_pad, tie


def _logits64(emb, text, sc, bi, normalize):
    e = emb.double()
    if normalize:
        e = e / e.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return e @ text.double().T * sc + bi


@pytest.mark.parametrize("case", list(ANCHOR_CASES))
def test_yolo_anchor_rows_levels_grids_and_classes(lib, case):
    from omg_b200 import ops
    from oracle import yolo_world as O
    levels, text, normalize, box_ld, emb_pad, tie = _anchor_inputs(case)
    E, nc = text.shape[1], text.shape[0]
    T = sum(fh * fw for _, fh, fw, *_ in levels)
    ops_levels, abi_levels = [], []
    for s, fh, fw, logits, emb, sc, bi in levels:
        box, e = _level_operands(logits, emb, box_ld, E + emb_pad)
        abi_levels.append((s, fh, fw, box, e, sc, bi))
        ops_levels.append((s, box.as_strided((1, fh, fw, 64), (fh * fw * box_ld, fw * box_ld, box_ld, 1)),
                           e.as_strided((1, fh, fw, E), (fh * fw * (E + emb_pad), fw * (E + emb_pad), E + emb_pad, 1)),
                           sc, bi))
    text_p = _nan_vec(text.reshape(-1)).view(nc, E)
    d = yolo_desc(abi_levels, text_p, normalize)
    rows, = twice(lambda: [_rows_only(lib, d, T, case)])
    # the Python wrapper (which fills fh / fw from the tensors' shapes) launches the same thing
    rows_ops, _ = ops.yolo_detect(ops_levels, text.contiguous(), normalize)
    assert same_bits(rows_ops, rows), f"{case}: ops.yolo_detect differs from the C-ABI call"

    strides = [lv[0] for lv in levels]
    ref = torch.from_numpy(O.anchor_rows([lv[3].cpu().numpy().reshape(lv[1], lv[2], 64) for lv in levels],
                                         [lv[4].cpu().numpy().reshape(lv[1], lv[2], E) for lv in levels],
                                         text.cpu().numpy(), strides, [lv[5] for lv in levels],
                                         [lv[6] for lv in levels], normalize)).cuda()
    check(rows[:, :4], ref[:, :4], K_ANCHOR_BOX, u=U32, what=f"anchor boxes {case}")
    check(rows[:, 4], ref[:, 4], K_ANCHOR_SCORE, u=U32, what=f"anchor scores {case}")
    # classes: the first class of the float64 maximum wherever the runner-up is more than 1e-6 below it
    logit = torch.cat([_logits64(lv[4], text, lv[5], lv[6], normalize) for lv in levels])
    if tie:
        logit[:, tie[1]] = logit[:, tie[0]]   # identical text rows: identical logits, whatever the GEMM's order
    p = torch.sigmoid(logit)
    pmax = p.max(1, keepdim=True).values
    tied = p == pmax
    first = tied.int().argmax(1)
    runner_up = p.masked_fill(tied, -1.0).max(1).values
    sure = (pmax[:, 0] - runner_up) > 1e-6
    cls = rows[:, 5].long()
    assert torch.equal(cls[sure], first[sure]), f"{case}: class differs from the float64 argmax"
    n_tied = int((sure & (tied.sum(1) > 1)).sum())
    assert n_tied > 0 or nc == 1, f"{case}: no exact tie was exercised"
    sat = (logit >= 20).all(1)
    assert torch.equal(cls[sat], torch.zeros_like(cls[sat])), f"{case}: a saturated row's class is not the first"
    assert not ((logit > 10) & (logit < 20)).any(), f"{case}: a logit between 10 and 20 blurs the saturated set"
    print(f"[anchors] {case}: {T} anchors, {int(sure.sum())} with a clear class ({n_tied} exact ties), "
          f"{int(sat.sum())} saturated")


# ----------------------------------------------------------------------------------------------- yolo_detect pass (b)
def nms_float32(rows, conf, iou, max_wh=7680.0, agnostic=False, max_det=300, gain=1.0, pad=(0.0, 0.0),
                clip=(4096.0, 4096.0)):
    """ultralytics non_max_suppression (single label per anchor) with torchvision's nms, then scale_boxes / clip_boxes,
    restated in float32 in the kernel's order of operations: candidates score > conf, sorted by (-score, anchor index),
    boxes offset by cls * max_wh, IoU = inter / ((a_p + a_q) - inter), suppression when IoU > iou, the first max_det
    kept, then min(max((x - pad) / gain, 0), clip).  rows [T, 6] float32 -> (kept anchor indices, output rows)."""
    f = np.float32
    r = np.asarray(rows, np.float32)
    cand = np.nonzero(r[:, 4] > f(conf))[0]
    order = cand[np.lexsort((cand, -r[cand, 4]))]
    off = np.zeros(len(order), np.float32) if agnostic else r[order, 5] * f(max_wh)
    b = r[order, :4] + off[:, None]
    area = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    supp = np.zeros(len(order), bool)
    keep = []
    with np.errstate(invalid="ignore", divide="ignore"):
        for i in range(len(order)):
            if len(keep) >= max_det:
                break
            if supp[i]:
                continue
            keep.append(i)
            q = b[i + 1:]
            w = np.maximum(f(0), np.minimum(b[i, 2], q[:, 2]) - np.maximum(b[i, 0], q[:, 0]))
            h = np.maximum(f(0), np.minimum(b[i, 3], q[:, 3]) - np.maximum(b[i, 1], q[:, 1]))
            inter = w * h
            supp[i + 1:] |= inter / ((area[i] + area[i + 1:]) - inter) > f(iou)   # NaN (0 / 0) never suppresses
    kept = order[np.asarray(keep, np.int64)]
    out = r[kept].copy()
    lo = np.array([pad[0], pad[1], pad[0], pad[1]], np.float32)
    hi = np.array([clip[0], clip[1], clip[0], clip[1]], np.float32)
    out[:, :4] = np.minimum(np.maximum((out[:, :4] - lo) / f(gain), f(0)), hi)
    return kept, out


def run_detect(lib, d, T, nms, what):
    """Both passes into guarded rows / out; rows at or past the count must stay untouched.  -> (rows, out[:count])."""
    max_out = nms["max_det"] + 4
    rows = Guard((T, 6), dtype=torch.float32, flat=True)
    out = Guard((max_out, 6), dtype=torch.float32, flat=True)
    count = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    d.rows, d.out, d.max_out, d.count = rows.out.data_ptr(), out.out.data_ptr(), max_out, count.data_ptr()
    d.conf, d.iou, d.max_wh = nms["conf"], nms["iou"], nms.get("max_wh", 7680.0)
    d.agnostic, d.max_det = int(nms.get("agnostic", False)), nms["max_det"]
    d.gain, (d.pad_x, d.pad_y), (d.clip_w, d.clip_h) = nms.get("gain", 1.0), nms.get("pad", (0.0, 0.0)), \
        nms.get("clip", (4096.0, 4096.0))
    _call(lib.omg_yolo_detect(C.byref(d), _stream()), lib, what)
    torch.cuda.synchronize()
    n = int(count.item())
    assert rows.intact() and out.intact(), f"{what}: write outside rows / out"
    assert 0 <= n <= nms["max_det"], f"{what}: count {n}"
    assert same_bits(out.out[n:], out.before[PAD + 6 * n:PAD + 6 * max_out].view(-1, 6)), \
        f"{what}: rows at or past the count were written"
    return rows.out.clone(), out.out[:n].clone()


class Scene:
    """Exact geometry: one-hot DFL logits (the chosen bin 0, every other bin -inf) make every distance an integer and
    every corner a multiple of stride / 2; scores from normalize_x = 0 and unit-basis text rows, so the score of class k
    is sigmoid(emb[k] * cls_scale + cls_bias) and equal embedding values give equal scores."""

    def __init__(self, grids, E=32, nc=2, low=-8.0):
        self.grids, self.E, self.nc = grids, E, nc     # grids: [(stride, fh, fw)]
        self.dist = [torch.zeros(fh * fw, 4, dtype=torch.long) for _, fh, fw in grids]
        self.emb = [torch.full((fh * fw, E), low) for _, fh, fw in grids]
        self.logits = [None] * len(grids)     # random DFL logits instead of one-hot, where set

    def anchor(self, level, x, y, dist, cls, value):
        a = y * self.grids[level][2] + x
        self.dist[level][a] = torch.tensor(dist)
        self.emb[level][a, cls] = value

    def levels(self):
        out = []
        for i, (s, fh, fw) in enumerate(self.grids):
            A = fh * fw
            if self.logits[i] is None:
                b = torch.full((A, 4, 16), float("-inf"))
                b.scatter_(2, self.dist[i].view(A, 4, 1), 0.0)
                b = b.view(A, 64)
            else:
                b = self.logits[i]
            box, e = _level_operands(b.half().cuda(), self.emb[i].half().cuda(), 72, self.E + 8)
            out.append((s, fh, fw, box, e, 1.0, 0.0))
        text = torch.eye(self.nc, self.E, device="cuda")
        return out, _nan_vec(text.reshape(-1)).view(self.nc, self.E)


def _scene_iou_half(iou):
    # stride 8: cell (0, 0), l = t = 0, r = b = 2 -> [4, 20]^2; cell (1, 0), l = 1, t = 0, r = b = 1 -> [4, 20] x [4, 12]:
    # intersection 128, union 256, IoU exactly 0.5
    s = Scene([(8, 4, 4)])
    s.anchor(0, 0, 0, (0, 0, 2, 2), 0, 3.0)
    s.anchor(0, 1, 0, (1, 0, 1, 1), 0, 2.0)
    return s, {"conf": 0.25, "iou": iou, "max_det": 300}, [0, 1] if iou >= 0.5 else [0]


def _scene_iou_zero():
    s = Scene([(8, 4, 4)])
    s.anchor(0, 0, 0, (0, 0, 2, 2), 0, 3.0)     # [4, 20]^2
    s.anchor(0, 2, 0, (0, 0, 2, 2), 0, 2.0)     # [20, 36] x [4, 20]: shares an edge, intersection 0: kept
    s.anchor(0, 1, 1, (0, 0, 1, 1), 0, 1.5)     # [12, 20]^2 inside the first: suppressed
    s.anchor(0, 2, 2, (0, 0, 1, 1), 0, 1.0)     # [20, 28]^2: touches the first at a corner, the second along y = 20
    return s, {"conf": 0.25, "iou": 0.0, "max_det": 300}, [0, 2, 10]


def _random_values(A, g, lo=-2.0, hi=2.0):
    return (torch.rand(A, generator=g) * (hi - lo) + lo).half().float()


def _scene_zero_area(max_det=300, conf=0.25, saturated=False):
    # every distance 0: points, IoU 0 / 0 = NaN between any two, so nothing is ever suppressed
    s = Scene([(8, 3, 4), (16, 2, 2)])
    g = torch.Generator().manual_seed(7)
    for lv, e in enumerate(s.emb):
        e[:, 0] = _random_values(len(e), g)
        if saturated:
            e[::3, 1] = 30.0    # sigmoid(30) is 1.0 in fp32
    scores = torch.sigmoid(torch.cat([e[:, :2].max(1).values for e in s.emb]).double())
    want = [int(a) for a in np.lexsort((np.arange(len(scores)), -scores.numpy())) if scores[a] > conf][:max_det]
    return s, {"conf": conf, "iou": 0.7, "max_det": max_det}, want


def _scene_ties_across_levels():
    # every score equal; boxes [x + 0.5, x + 1.5] * stride touch their neighbours and overlap other levels' with IoU
    # 0.25 at most: the first max_det anchors by index, in that order
    s = Scene([(8, 6, 5), (16, 3, 3), (32, 2, 2)])
    for d, e in zip(s.dist, s.emb):
        d[:] = torch.tensor([0, 0, 1, 1])
        e[:, 0] = 1.0
    return s, {"conf": 0.25, "iou": 0.7, "max_det": 20}, list(range(20))


def _scene_two_classes(agnostic):
    s = Scene([(8, 3, 3)])
    s.anchor(0, 0, 0, (0, 0, 2, 2), 0, 2.0)     # [4, 20]^2, class 0
    s.anchor(0, 1, 0, (1, 0, 1, 2), 1, 1.0)     # [4, 20]^2 as well, class 1
    return s, {"conf": 0.25, "iou": 0.7, "max_det": 300, "agnostic": agnostic}, [0] if agnostic else [0, 1]


def _scene_offsets_round():
    # stride 1, random DFL logits, classes 1000..1023 winning: cls * 7680 is about 7.7e6, where fp32 rounds the offset
    # coordinates to 0.5 or 1
    s = Scene([(1, 24, 32)], E=1024, nc=1024, low=-6.0)
    g = torch.Generator().manual_seed(11)
    s.logits[0] = torch.randn(24 * 32, 64, generator=g) * 3.0
    s.emb[0][:, 1000:] = torch.rand(24 * 32, 24, generator=g) * 3.0
    return s, {"conf": 0.25, "iou": 0.45, "max_det": 300}, None


def _scene_rescale():
    # letterbox 160 x 240 of a 233 x 380 image: gain 0.6, pad (6, 10); random integer distances, and two boxes of
    # distance 15 in the corners that cross both clip edges
    s = Scene([(8, 20, 30)], nc=3)
    g = torch.Generator().manual_seed(3)
    s.dist[0] = torch.randint(0, 16, (600, 4), generator=g)
    s.emb[0][:, :3] = _random_values(600 * 3, g).view(600, 3)
    s.anchor(0, 0, 0, (15, 15, 15, 15), 0, 6.0)
    s.anchor(0, 29, 19, (15, 15, 15, 15), 1, 6.0)
    return s, {"conf": 0.3, "iou": 0.7, "max_det": 300, "gain": 0.6, "pad": (6.0, 10.0), "clip": (380.0, 233.0)}, None


def _scene_anchor_cap():
    # 100^2 + 80^2 + 40 x 35 = 17 800 anchors, every one a candidate, all tied, all points: the first 300 by index
    s = Scene([(8, 100, 100), (16, 80, 80), (32, 40, 35)])
    for e in s.emb:
        e[:, 0] = 1.0
    return s, {"conf": 0.25, "iou": 0.7, "max_det": 300}, list(range(300))


SCENES = {
    "iou-exactly-0.5": lambda: _scene_iou_half(0.5),
    "iou-0.4999": lambda: _scene_iou_half(0.4999),
    "iou-0-touching-kept": _scene_iou_zero,
    "zero-area-nan-iou": _scene_zero_area,
    "ties-across-levels": _scene_ties_across_levels,
    "two-classes-identical-boxes": lambda: _scene_two_classes(False),
    "two-classes-identical-boxes-agnostic": lambda: _scene_two_classes(True),
    "stride1-nc1024-offsets-round": _scene_offsets_round,
    "max-det-0": lambda: _scene_zero_area(max_det=0),
    "max-det-1": lambda: _scene_zero_area(max_det=1),
    "conf-1-no-candidates": lambda: _scene_zero_area(conf=1.0, saturated=True),
    "rescale-gain-0.6-clipped": _scene_rescale,
    "anchor-cap-17800": _scene_anchor_cap,
    "conf-equals-an-anchor-score": None,
}


@pytest.mark.parametrize("scene", list(SCENES))
def test_yolo_nms_matches_float32_restatement_bit_for_bit(lib, scene):
    if scene == "conf-equals-an-anchor-score":
        s, nms, want = _scene_zero_area()
    else:
        s, nms, want = SCENES[scene]()
    levels, text = s.levels()
    T = sum(fh * fw for _, fh, fw in s.grids)
    d = yolo_desc(levels, text, False)
    if scene == "conf-equals-an-anchor-score":
        # conf read back as the fp32 score of one anchor (pass (a) alone): that anchor is not a candidate
        r = _rows_only(lib, d, T, scene).cpu().numpy()
        g = int(np.argsort(r[:, 4])[len(r) // 2])
        nms["conf"] = float(r[g, 4])
        want = [a for a in want if r[a, 4] > r[g, 4]]
        assert g not in want and len(want) == int((r[:, 4] > r[g, 4]).sum()) > 0
    rows, out = twice(lambda: list(run_detect(lib, d, T, nms, scene)))
    kept, ref = nms_float32(rows.cpu().numpy(), **nms)
    out = out.cpu().numpy()
    print(f"[nms] {scene}: {T} anchors, {int((rows[:, 4].cpu().numpy() > np.float32(nms['conf'])).sum())} candidates, "
          f"{len(out)} kept")
    if want is not None:
        assert kept.tolist() == want, f"{scene}: the restatement keeps {kept.tolist()}, the scene implies {want}"
    assert out.shape == ref.shape, f"{scene}: count {len(out)}, restatement {len(ref)}"
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), f"{scene}: rows differ from the restatement"
    if scene == "rescale-gain-0.6-clipped":
        assert (out[:, :2] == 0).any(0).all() and out[:, 2].max() == 380.0 and out[:, 3].max() == 233.0
    if scene == "stride1-nc1024-offsets-round":
        assert len(out) > 20 and out[:, 5].min() >= 1000


# ------------------------------------------------------------------------------------------------------ launch plan
def test_yolo_world_kernels_replay_from_a_launch_plan(lib):
    """One call of each of the three entry points recorded in a plan, omg_yolo_detect with both passes: the plan holds
    three calls, and four kernels launch (omg_yolo_detect is one call but two launches, pass (a) then pass (b)), both
    while recording and on replay.  A replay into cleared outputs gives the same bits."""
    from omg_b200 import ops
    g = _gen(21)
    B, HW, nh, hc = 2, 40, 4, 32
    Ce = nh * hc
    embed = torch.randn(B * HW, Ce, generator=g, device="cuda").half()
    p = torch.randn(B * HW, Ce, generator=g, device="cuda").half()
    guide = torch.randn(B, 3, Ce, generator=g, device="cuda")
    bias = torch.randn(nh, generator=g, device="cuda")
    gate_out = torch.empty_like(p)
    x = torch.randn(B, 7, 11, 64, generator=g, device="cuda").half()
    kv = torch.empty(B, 16, 64, dtype=torch.float16, device="cuda")
    s, nms, _ = _scene_iou_zero()
    levels, text = s.levels()
    d = yolo_desc(levels, text, False)
    rows = torch.empty(16, 6, device="cuda")
    det = torch.empty(8, 6, device="cuda")
    count = torch.empty(1, dtype=torch.int32, device="cuda")
    d.rows, d.out, d.max_out, d.count = rows.data_ptr(), det.data_ptr(), 8, count.data_ptr()
    d.conf, d.iou, d.max_wh, d.max_det, d.gain, d.clip_w, d.clip_h = 0.25, 0.0, 7680.0, 8, 1.0, 4096.0, 4096.0
    outputs = [gate_out, kv, rows, det, count]

    def calls():
        st = _stream()
        _call(lib.omg_text_gate(embed.data_ptr(), Ce, Ce, guide.data_ptr(), 3, bias.data_ptr(), None, nh, p.data_ptr(),
                                Ce, gate_out.data_ptr(), Ce, Ce, B, HW, st), lib, "omg_text_gate")
        _call(lib.omg_adaptive_maxpool(x.data_ptr(), 64, B, 7, 11, 64, 3, kv.data_ptr(), 16 * 64, 64, 4, st), lib,
              "omg_adaptive_maxpool")
        _call(lib.omg_yolo_detect(C.byref(d), st), lib, "omg_yolo_detect")

    for t in outputs:
        t.zero_()
    plan = ops.LaunchPlan()
    n0 = lib.omg_launch_count()
    with plan:
        calls()
    assert lib.omg_launch_count() - n0 == 4 and len(plan) == 3
    torch.cuda.synchronize()
    first = [t.clone() for t in outputs]
    assert int(count.item()) == 3
    for t in outputs:
        t.zero_()
    n0 = lib.omg_launch_count()
    plan.run()
    torch.cuda.synchronize()
    assert lib.omg_launch_count() - n0 == 4
    for a, b in zip(outputs, first):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
