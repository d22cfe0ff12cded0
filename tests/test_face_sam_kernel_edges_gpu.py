"""Kernel edges of the face-analysis kernels (omg_channel_op, omg_pool2d, omg_scrfd_detect) and of the SAM mask kernels
(omg_sam_mask_head, omg_sam_postprocess) through the C ABI, against float64 references computed on the GPU from the same
fp16 / fp32 values the kernels read (helpers of test_kernel_edges_gpu.py):

* every element is bounded,  |out - ref| <= 4 u |ref| + k u rms(ref)  (u = 2^-11 for fp16 outputs, 2^-24 for fp32);
* outputs sit in NaN guard buffers that must stay intact, operands in NaN-poisoned windows, per-channel vectors in
  NaN-padded buffers, so a read or write outside the operand shows up;
* every case runs twice and must be bit-identical.  `pytest -s` prints the k each case needs.

omg_scrfd_detect is compared exactly with the numpy restatement of SCRFD.detect (oracle/face.py)."""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_edges_gpu import PAD, Guard, check, same_bits, twice  # noqa: E402

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
NAN = float("nan")

# Per-element k, with the worst value the family's cases need on an NVIDIA H100 80GB HBM3 at a 700 W power limit beside
# it (a value <= 0 means every element is already within 4 u |ref|).
K_CHANNEL = 1.0      # measured 0.00 (every layout, activation and addend)
K_POOL_AVG = 1.0     # measured 0.00 (average pooling; max pooling is compared bit for bit)
K_MASK_HEAD = 64.0   # measured 42.0 (M = 2, |mean| / sigma = 32)
K_POSTPROCESS = 4096.0  # measured 1967 (1024 x 768 crop -> 333 x 517: the fp32 source index of an inexact scale,
                        # as PyTorch computes it for fp32 tensors)


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


class Rows(Guard):
    """`rows` x `cols` window with a row stride of `ld` elements, starting `off` elements into a NaN buffer (NaN columns
    between the rows, PAD NaN elements after the last).  off = PAD keeps the window 16 B aligned, PAD + 1 does not.
    Guard.intact() checks everything outside the window."""

    def __init__(self, rows, cols, ld, off=PAD, dtype=torch.float16):
        self.buf = torch.full((off + rows * ld + PAD,), NAN, dtype=dtype, device="cuda")
        self.out = self.buf.as_strided((rows, cols), (ld, 1), off)
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        self.inside.as_strided((rows, cols), (ld, 1), off).fill_(True)
        self.before = self.buf.clone()


def _nan_vec(v):
    """fp32 [C] as the middle of a NaN buffer of C + 8: a read past either end is NaN."""
    buf = torch.full((v.numel() + 8,), NAN, dtype=torch.float32, device="cuda")
    buf[4:4 + v.numel()].copy_(v)
    return buf[4:4 + v.numel()]


# ------------------------------------------------------------------------------------------------------- channel_op
ACTS = {"none": 0, "relu": 1, "prelu": 2, "sigmoid": 3}

# name -> (B, H, W, C, ldx, ldy, ld_add, x offset, y offset, addend offset, in place, x NULL)
LAYOUTS = {
    "vector": (2, 4, 6, 64, 64, 64, 64, PAD, PAD, PAD, False, False),
    "scalar_ldx20": (2, 4, 6, 16, 20, 16, 16, PAD, PAD, PAD, False, False),
    "scalar_x_off2": (2, 4, 6, 64, 64, 64, 64, PAD + 1, PAD, PAD, False, False),
    "scalar_y_off2": (2, 4, 6, 64, 64, 64, 64, PAD, PAD + 1, PAD, False, False),
    "scalar_add_off2": (2, 4, 6, 64, 64, 64, 64, PAD, PAD, PAD + 1, False, False),
    "C12": (2, 4, 6, 12, 12, 12, 12, PAD, PAD, PAD, False, False),
    "score_map": (1, 1, 12800, 1, 1, 1, 1, PAD, PAD, PAD, False, False),
    "inplace_vector": (2, 4, 6, 64, 64, 64, 64, PAD, PAD, PAD, True, False),
    "inplace_scalar": (2, 4, 6, 16, 20, 20, 16, PAD, PAD, PAD, True, False),
    "x_null_up2": (3, 4, 6, 64, 0, 64, 80, PAD, PAD, PAD, False, True),
}


def _channel_cases():
    for lay, spec in LAYOUTS.items():
        for act in ACTS:
            if lay == "score_map" and act != "sigmoid":
                continue
            for after in (0, 1):
                for add_scale in (0, 1, 2):
                    if (lay == "score_map" and add_scale == 2) or (spec[11] and add_scale != 2):
                        continue
                    yield pytest.param(lay, act, after, add_scale, id=f"{lay}-{act}-after{after}-add{add_scale}")


def _channel_ref(x, scale, shift, slope, a, act, after):
    v = (x.double() if x is not None else torch.zeros_like(a, dtype=torch.float64)) * scale.double() + shift.double()
    f = {"none": lambda z: z, "relu": lambda z: z.clamp_min(0), "sigmoid": torch.sigmoid,
         "prelu": lambda z: torch.where(z >= 0, z, z * slope.double())}[act]
    return f(v + a) if after else f(v) + a


@pytest.mark.parametrize("layout,act,after,add_scale", list(_channel_cases()))
def test_channel_op_layouts(lib, layout, act, after, add_scale):
    B, H, W, Cc, ldx, ldy, ld_add, ox, oy, oa, inplace, x_null = LAYOUTS[layout]
    g = _gen(zlib.crc32(f"{layout}-{act}-{after}-{add_scale}".encode()))
    P = B * H * W
    if act == "sigmoid":   # inputs up to |v| = 30, where __expf and the division must still round right
        x = ((torch.rand(P, Cc, generator=g, device="cuda") * 2 - 1) * 30).half()
        scale = 0.5 + 0.5 * torch.rand(Cc, generator=g, device="cuda")
    else:
        x = (torch.randn(P, Cc, generator=g, device="cuda") * 3).half()
        scale = torch.randn(Cc, generator=g, device="cuda")
    shift = torch.randn(Cc, generator=g, device="cuda")
    slope = torch.tensor([-0.5, 0.0, 1.5, 0.25, -2.0, 3.0], device="cuda").repeat(Cc)[:Cc]   # negative, zero and > 1
    scale_p, shift_p, slope_p = _nan_vec(scale), _nan_vec(shift), _nan_vec(slope)
    Ha, Wa = (H // add_scale, W // add_scale) if add_scale else (H, W)
    addend = (torch.randn(B * Ha * Wa, Cc, generator=g, device="cuda") * 2).half() if add_scale else None
    if add_scale:
        a_in = Rows(B * Ha * Wa, Cc, ld_add, oa).out
        a_in.copy_(addend)
        a4 = addend.double().view(B, Ha, 1, Wa, 1, Cc).expand(B, Ha, add_scale, Wa, add_scale, Cc).reshape(P, Cc)
    else:
        a_in, a4 = None, torch.zeros(P, Cc, dtype=torch.float64, device="cuda")
    x_in = None
    if not x_null and not inplace:
        x_in = Rows(P, Cc, ldx, ox).out
        x_in.copy_(x)
    ref = _channel_ref(None if x_null else x, scale, shift, slope, a4, act, after)

    def run():
        out = Rows(P, Cc, ldy, oy)
        if x_null:
            xp, lx = None, 0
        elif inplace:   # y == x, as face.py runs its post-GEMM adds
            out.out.copy_(x)
            xp, lx = out.out.data_ptr(), ldx
        else:
            xp, lx = x_in.data_ptr(), ldx
        rc = lib.omg_channel_op(xp, lx, out.out.data_ptr(), ldy, scale_p.data_ptr(), shift_p.data_ptr(),
                                slope_p.data_ptr(), None if a_in is None else a_in.data_ptr(), ld_add if add_scale else 0,
                                add_scale, B, H, W, Cc, ACTS[act], after, _stream())
        _call(rc, lib, "omg_channel_op")
        torch.cuda.synchronize()
        assert out.intact(), "write outside the output rows"
        return [out.out.clone()]

    out, = twice(run)
    check(out, ref, K_CHANNEL, what=f"channel_op {layout} {act} after={after} add={add_scale}")


# ----------------------------------------------------------------------------------------------------------- pool2d
POOL_SIZES = [(1, 1), (2, 3), (5, 4), (7, 7)]
POOL_C = [8, 24, 520]


def _pool_cases():
    for k in (1, 2, 3):
        for stride in (1, 2):
            for pad in (0, 1):
                if 2 * pad > k:
                    continue
                for ceil in (0, 1):
                    for mode in ("max", "avg", "avg_cip"):
                        yield pytest.param(k, stride, pad, ceil, mode, id=f"k{k}-s{stride}-p{pad}-ceil{ceil}-{mode}")


@pytest.mark.parametrize("k,stride,pad,ceil,mode", list(_pool_cases()))
def test_pool2d_windows(lib, k, stride, pad, ceil, mode):
    """Every image size and channel count for one window configuration: windows clipped on both sides, the ceil-mode
    rule that drops a last window starting in the right pad, max over all-negative windows (the first half of the
    channels are negative everywhere), and the divisor with and without the padding."""
    from omg_b200 import ops
    is_max, cip = mode == "max", mode == "avg_cip"
    worst = 0.0
    for (H, W) in POOL_SIZES:
        for Cc in POOL_C:
            B = 3
            what = f"pool2d k{k} s{stride} p{pad} ceil{ceil} {mode} {H}x{W} C={Cc}"
            g = _gen(H * 1000 + W * 100 + Cc + k)
            x = torch.randn(B, H, W, Cc, generator=g, device="cuda")
            x[..., :Cc // 2] = -x[..., :Cc // 2].abs() - 0.01
            x = x.half()
            n = x.numel()
            xbuf = torch.full((PAD + n + PAD,), NAN, dtype=torch.float16, device="cuda")
            x_in = xbuf[PAD:PAD + n].view(B, H, W, Cc)
            x_in.copy_(x)
            Ho, Wo = ops.pool2d_out_size(H, k, stride, pad, ceil), ops.pool2d_out_size(W, k, stride, pad, ceil)
            if H + 2 * pad < k or W + 2 * pad < k:
                out = Guard((B, max(Ho, 1), max(Wo, 1), Cc), flat=True)
                n0 = lib.omg_launch_count()
                rc = lib.omg_pool2d(x_in.data_ptr(), out.out.data_ptr(), B, H, W, Cc, k, stride, pad, ceil, int(cip),
                                    int(is_max), _stream())
                assert rc == 1 and "larger than the padded input" in lib.omg_last_error().decode(), what
                assert lib.omg_launch_count() == n0 and out.intact(), what
                continue
            xd = x.double().permute(0, 3, 1, 2)
            if is_max:
                ref = F.max_pool2d(xd, k, stride, pad, ceil_mode=bool(ceil))
            else:
                ref = F.avg_pool2d(xd, k, stride, pad, ceil_mode=bool(ceil), count_include_pad=cip)
            ref = ref.permute(0, 2, 3, 1)
            assert ref.shape == (B, Ho, Wo, Cc), what

            def run():
                out = Guard((B, Ho, Wo, Cc), flat=True)
                _call(lib.omg_pool2d(x_in.data_ptr(), out.out.data_ptr(), B, H, W, Cc, k, stride, pad, ceil, int(cip),
                                     int(is_max), _stream()), lib, what)
                torch.cuda.synchronize()
                assert out.intact(), f"{what}: write outside the output"
                return [out.out.clone()]

            out, = twice(run)
            if is_max:
                assert same_bits(out, ref.half()), f"{what}: max pooling differs from the float64 reference"
            else:
                check(out, ref, K_POOL_AVG, what=what)


# ----------------------------------------------------------------------------------------------------- scrfd_detect
def _heads(seed, grids, A, use_kps, all_above=False):
    g = np.random.default_rng(seed)
    s, b, kp = [], [], []
    for fh, fw in grids:
        n = fh * fw * A
        s.append((0.5 + g.random((n, 1)) * 0.5 if all_above else g.random((n, 1))).astype(np.float32))
        b.append((g.random((n, 4)) * 3 + 0.2).astype(np.float32))
        kp.append((g.normal(size=(n, 10)) * 2).astype(np.float32))
    return s + b + (kp if use_kps else [])


def _scrfd_desc(outs, strides, grids, A, use_kps, det_thresh, nms_thresh, det_scale):
    from omg_b200 import _lib as L
    nl = len(strides)
    dev = [torch.from_numpy(o).cuda() for o in outs]
    d = L.ScrfdDesc()
    d.n_levels, d.num_anchors = nl, A
    for i, (s, (fh, fw)) in enumerate(zip(strides, grids)):
        d.scores[i], d.boxes[i] = dev[i].data_ptr(), dev[nl + i].data_ptr()
        d.kps[i] = dev[2 * nl + i].data_ptr() if use_kps else None
        d.stride[i], d.fh[i], d.fw[i] = s, fh, fw
    d.det_thresh, d.nms_thresh, d.det_scale = det_thresh, nms_thresh, det_scale
    return d, dev


SCRFD_CASES = {
    # name: (input H, W, strides, num_anchors, key-points, nms_thresh, every score above the threshold)
    "480x640_5levels_A1": (480, 640, (8, 16, 32, 64, 128), 1, True, 0.4, False),
    "240x320_5levels_A4": (240, 320, (8, 16, 32, 64, 128), 4, True, 0.4, False),
    "480x640_A2_no_kps": (480, 640, (8, 16, 32), 2, False, 0.4, False),
    "680x640_A2_17800_anchors": (680, 640, (8, 16, 32), 2, True, 0.4, True),
    "480x640_A2_ties_nms0": (480, 640, (8, 16, 32), 2, True, 0.0, False),
    "64x96_1level_A1": (64, 96, (8,), 1, True, 0.4, False),
}


@pytest.mark.parametrize("case", list(SCRFD_CASES))
def test_scrfd_detect_grids_anchors_and_levels(lib, case):
    from oracle import face as of
    H, W, strides, A, use_kps, nms, all_above = SCRFD_CASES[case]
    grids = [(H // s, W // s) for s in strides]
    T = sum(fh * fw * A for fh, fw in grids)
    if case.endswith("17800_anchors"):
        assert T == 17800
    outs = _heads(len(case), grids, A, use_kps, all_above)
    if "ties" in case:   # equal scores on anchors of different levels (and within one): ties go to the lower index
        for lvl, idx in ((0, 7), (1, 3), (2, 0), (0, 100), (2, 11)):
            outs[lvl][idx] = 0.875
    det_thresh, det_scale = 0.5, 0.75
    det, kpss = of.detect_from_outputs(outs, H, W, det_scale, det_thresh, nms, strides=strides, num_anchors=A,
                                       use_kps=use_kps)
    d, keep_alive = _scrfd_desc(outs, strides, grids, A, use_kps, det_thresh, nms, det_scale)

    def run():
        out = Guard((T, 15), dtype=torch.float32, flat=True)
        count = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        d.out, d.max_out, d.count = out.out.data_ptr(), T, count.data_ptr()
        _call(lib.omg_scrfd_detect(C.byref(d), _stream()), lib, case)
        torch.cuda.synchronize()
        n = int(count.item())
        assert out.intact(), "write outside the output rows"
        assert 0 <= n <= T and same_bits(out.out[n:], out.before[PAD + 15 * n:PAD + 15 * T].view(T - n, 15)), \
            "rows at or past count were written"
        return [out.out[:n].clone()]

    rows, = twice(run)
    rows = rows.cpu().numpy()
    print(f"[scrfd] {case}: {T} anchors, {rows.shape[0]} faces")
    assert rows.shape[0] == det.shape[0] > 0
    np.testing.assert_array_equal(rows[:, :5], det)
    if use_kps:
        np.testing.assert_array_equal(rows[:, 5:], kpss.reshape(-1, 10))
    else:
        assert not rows[:, 5:].any(), "key-point columns without key-points must be 0"


def test_scrfd_detect_rejects_more_anchors_than_shared_memory_holds(lib):
    strides, A = (8, 16, 32, 64, 128), 4
    grids = [(480 // s, 640 // s) for s in strides]
    outs = _heads(0, grids, A, True)
    d, keep_alive = _scrfd_desc(outs, strides, grids, A, True, 0.5, 0.4, 1.0)
    out = Guard((17800, 15), dtype=torch.float32, flat=True)
    count = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    d.out, d.max_out, d.count = out.out.data_ptr(), 17800, count.data_ptr()
    n0 = lib.omg_launch_count()
    assert lib.omg_scrfd_detect(C.byref(d), _stream()) == 1
    assert "exceed the 17800" in lib.omg_last_error().decode()
    assert lib.omg_launch_count() == n0 and out.intact() and int(count.item()) == -1


# ---------------------------------------------------------------------------------------------------- sam_mask_head
def _mask_head_case(B, M, seed, mean_over_sigma=0.0):
    g = _gen(seed)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")  # noqa: E731
    if mean_over_sigma:   # rows of |mean| / sigma = 32: the LayerNorm must not lose the variance to cancellation
        sign = torch.where(r(B, 64, 64, 2, 2, 1) >= 0, 1.0, -1.0)
        up1 = (sign * mean_over_sigma * 0.25 + 0.25 * r(B, 64, 64, 2, 2, 64)).half()
    else:
        up1 = (r(B, 64, 64, 2, 2, 64) * 1.5 + 0.3).half()
    lw, lb = 1 + 0.2 * r(64), 0.2 * r(64)
    w2, b2 = r(2, 2, 64, 32) / 8, 0.1 * r(32)
    hyper = r(B, M, 32).half()
    return up1, lw, lb, w2, b2, hyper


def mask_head_reference(up1, lw, lb, w2, b2, hyper, eps=1e-6):
    """float64: LayerNorm2d, erf-GELU, ConvTranspose2d(64 -> 32, k2, s2) as an einsum, GELU, hypernetwork product."""
    B = up1.shape[0]
    x = up1.double().permute(0, 1, 3, 2, 4, 5).reshape(B, 128, 128, 64)          # (b, 2y + dy, 2x + dx, c)
    mu = x.mean(-1, keepdim=True)
    var = (x - mu).pow(2).mean(-1, keepdim=True)
    v = F.gelu((x - mu) / torch.sqrt(var + eps) * lw.double() + lb.double())
    u = torch.einsum("byxc,eqco->byexqo", v, w2.double()).reshape(B, 256, 256, 32) + b2.double()
    u = F.gelu(u)
    return torch.einsum("bmo,bpqo->bmpq", hyper.double(), u)


@pytest.mark.parametrize("M,mean_over_sigma", [(1, 0.0), (2, 0.0), (4, 0.0), (2, 32.0)])
def test_sam_mask_head_against_float64(lib, M, mean_over_sigma):
    B = 2
    up1, lw, lb, w2, b2, hyper = _mask_head_case(B, M, seed=M + int(mean_over_sigma), mean_over_sigma=mean_over_sigma)
    ref = mask_head_reference(up1, lw, lb, w2, b2, hyper)
    wide = torch.full((B, 4, 48), NAN, dtype=torch.float16, device="cuda")   # hyper_ms = 48, rows past M are NaN
    h_in = wide[:, :M, 8:40]
    h_in.copy_(hyper)
    w2buf = torch.full((w2.numel() + 8,), NAN, device="cuda")
    w2buf[:w2.numel()].copy_(w2.reshape(-1))
    up1buf = torch.full((up1.numel() + PAD,), NAN, dtype=torch.float16, device="cuda")
    up1buf[:up1.numel()].copy_(up1.reshape(-1))
    vecs = [_nan_vec(lw), _nan_vec(lb), _nan_vec(b2)]
    ptrs = (up1buf.data_ptr(), vecs[0].data_ptr(), vecs[1].data_ptr(), w2buf.data_ptr(), vecs[2].data_ptr(),
            h_in.data_ptr())

    def run():
        out = Guard((B, M, 256, 256), dtype=torch.float32, flat=True)
        _call(lib.omg_sam_mask_head(*ptrs, h_in.stride(0), h_in.stride(1), B, M, 1e-6, out.out.data_ptr(), _stream()),
              lib, "omg_sam_mask_head")
        torch.cuda.synchronize()
        assert out.intact(), "write outside the output"
        return [out.out.clone()]

    out, = twice(run)
    check(out, ref, K_MASK_HEAD, u=U32, what=f"sam_mask_head M={M} |mean|/sigma={mean_over_sigma}")


# -------------------------------------------------------------------------------------------------- sam_postprocess
POST_CASES = [(256, 1024, 1024, 768, 333, 517), (64, 64, 64, 40, 7, 5), (256, 1024, 1024, 1024, 1, 1),
              (128, 512, 300, 512, 600, 1024)]


def postprocess_reference(low, mid, h_in, w_in, H, W):
    x = F.interpolate(low.double()[None], (mid, mid), mode="bilinear", align_corners=False)[..., :h_in, :w_in]
    return F.interpolate(x, (H, W), mode="bilinear", align_corners=False)[0]


class ByteGuard:
    """uint8 output [n] inside a buffer of 0xA5 bytes, PAD on each side (the kernel writes 0 | 1 only)."""

    def __init__(self, n):
        self.buf = torch.full((n + 2 * PAD,), 0xA5, dtype=torch.uint8, device="cuda")
        self.out = self.buf[PAD:PAD + n]

    def intact(self):
        return bool((self.buf[:PAD] == 0xA5).all() and (self.buf[-PAD:] == 0xA5).all())


@pytest.mark.parametrize("threshold", [0.0, 0.7])
@pytest.mark.parametrize("low,mid,h_in,w_in,H,W", POST_CASES)
def test_sam_postprocess_against_float64(lib, low, mid, h_in, w_in, H, W, threshold):
    BM = 5
    lowres = torch.randn(BM, low, low, generator=_gen(low + H), device="cuda") * 3
    lr = torch.full((lowres.numel() + PAD,), NAN, device="cuda")
    lr[:lowres.numel()].copy_(lowres.reshape(-1))
    ref = postprocess_reference(lowres, mid, h_in, w_in, H, W)
    what = f"sam_postprocess low {low} mid {mid} in {h_in}x{w_in} -> {H}x{W} thr {threshold}"

    def call(want_mask, want_logits):
        m = ByteGuard(BM * H * W) if want_mask else None
        lg = Guard((BM, H, W), dtype=torch.float32, flat=True) if want_logits else None
        _call(lib.omg_sam_postprocess(lr.data_ptr(), BM, low, mid, h_in, w_in, H, W, threshold,
                                      None if m is None else m.out.data_ptr(), None if lg is None else lg.out.data_ptr(),
                                      _stream()), lib, what)
        torch.cuda.synchronize()
        assert (m is None or m.intact()) and (lg is None or lg.intact()), f"{what}: write outside the output"
        return m, lg

    def run():
        m, lg = call(True, True)
        return [m.out.view(BM, H, W).to(torch.int16), lg.out.clone()]   # (twice compares 2- and 4-byte elements)

    mask, logits = twice(run)
    assert torch.equal(call(True, False)[0].out.view(BM, H, W).to(torch.int16), mask), \
        "mask-only call differs from the mask of the two-output call"
    assert same_bits(call(False, True)[1].out, logits), "logits-only call differs from the two-output call"
    assert int(mask.min()) >= 0 and int(mask.max()) <= 1
    assert torch.equal(mask.bool(), logits > threshold), "mask is not logits > threshold"
    check(logits, ref, K_POSTPROCESS, u=U32, what=what)
    r = ref.reshape(-1)
    band = 4 * U32 * r.abs() + K_POSTPROCESS * U32 * r.pow(2).mean().sqrt()
    clear = (r - threshold).abs() > band
    assert torch.equal(mask.reshape(-1).bool()[clear], (r > threshold)[clear]), \
        f"{what}: mask differs outside the rounding band"


# ------------------------------------------------------------------------------------------------------ launch plan
def test_face_and_sam_kernels_replay_from_a_launch_plan(lib):
    """One call of each of the five entry points recorded in a plan: five launches while recording, and a replay into
    cleared outputs gives the same bits."""
    from omg_b200 import ops
    g = _gen(5)
    x = torch.randn(2, 6, 8, 16, generator=g, device="cuda").half()
    scale, shift = torch.rand(16, generator=g, device="cuda") + 0.5, torch.randn(16, generator=g, device="cuda")
    ch_out = torch.empty_like(x)
    pool_out = torch.empty(2, ops.pool2d_out_size(6, 3, 2, 1, True), ops.pool2d_out_size(8, 3, 2, 1, True), 16,
                           dtype=torch.float16, device="cuda")
    strides, grids = (8, 16), [(4, 6), (2, 3)]
    outs = _heads(9, grids, 2, True)
    T = sum(fh * fw * 2 for fh, fw in grids)
    d, keep_alive = _scrfd_desc(outs, strides, grids, 2, True, 0.5, 0.4, 1.0)
    det_out = torch.zeros(T, 15, device="cuda")   # rows past the count are never written
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    d.out, d.max_out, d.count = det_out.data_ptr(), T, count.data_ptr()
    up1, lw, lb, w2, b2, hyper = _mask_head_case(1, 2, seed=3)
    w2 = w2.contiguous()
    low_out = torch.empty(1, 2, 256, 256, device="cuda")
    mask = torch.empty(2, 100, 150, dtype=torch.uint8, device="cuda")
    logits = torch.empty(2, 100, 150, device="cuda")
    outputs = [ch_out, pool_out, det_out, count, low_out, mask, logits]

    def calls():
        s = _stream()
        _call(lib.omg_channel_op(x.data_ptr(), 16, ch_out.data_ptr(), 16, scale.data_ptr(), shift.data_ptr(), None,
                                 None, 0, 0, 2, 6, 8, 16, 1, 0, s), lib, "omg_channel_op")
        _call(lib.omg_pool2d(x.data_ptr(), pool_out.data_ptr(), 2, 6, 8, 16, 3, 2, 1, 1, 0, 1, s), lib, "omg_pool2d")
        _call(lib.omg_scrfd_detect(C.byref(d), s), lib, "omg_scrfd_detect")
        _call(lib.omg_sam_mask_head(up1.data_ptr(), lw.data_ptr(), lb.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                                    hyper.data_ptr(), hyper.stride(0), hyper.stride(1), 1, 2, 1e-6, low_out.data_ptr(), s),
              lib, "omg_sam_mask_head")
        _call(lib.omg_sam_postprocess(low_out.data_ptr(), 2, 256, 1024, 700, 1024, 100, 150, 0.0, mask.data_ptr(),
                                      logits.data_ptr(), s), lib, "omg_sam_postprocess")

    plan = ops.LaunchPlan()
    n0 = lib.omg_launch_count()
    with plan:
        calls()
    assert lib.omg_launch_count() - n0 == 5 and len(plan) == 5
    torch.cuda.synchronize()
    first = [t.clone() for t in outputs]
    assert int(count.item()) > 0
    for t in outputs:
        t.zero_()
    plan.run()
    torch.cuda.synchronize()
    for a, b in zip(outputs, first):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
