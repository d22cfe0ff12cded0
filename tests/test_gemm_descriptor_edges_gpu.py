"""Edges of the GEMM descriptors the executors compose from several A views and K-segments, against float64 references
computed on the GPU from the same fp16 operands the kernel read (per-element bound, guarded outputs and two bit-identical
runs, as in test_kernel_edges_gpu.py):

* stride-2 phase views: ops.conv3x3_s2 (UNet down-samplers, the SAM encoder's tanh-GELU convs) at outputs of 1 to 131
  columns, and face.OnnxNet's stride-2 convs (k 1 / 2 / 3, pad 0 / 1) on odd inputs, where the four phases differ in size;
* several A views in one accumulator: the maximum of 4 views and 12 segments by hand, the ResBlock shortcut
  concatenation and `extra` K-segments in the middle of the weight;
* un-merged LoRA: a `b_idx = 1` segment against w2 at summed ranks with tails and several K blocks, with every epilogue
  the ABI allows beside it, and the whole tiny UNet at ranks that are not multiples of 8;
* one launch of each family recorded in a launch plan and replayed.

Inputs of the spatial cases sit in a NaN ring (`ringed`): a phase view or shifted tap that reads outside its view
without TMA zero-fill turns into NaN in the result.  Bounds are K_GEMM and, for fp32 twins, K_F32; on an NVIDIA H100 80GB
HBM3 at a 700 W power limit the fp16 cases needed k <= 0.16 and the fp32 twins k <= 21.4 (r_tot = 136).
"""
import pytest
import torch
import torch.nn.functional as F

from test_kernel_edges_gpu import K_F32, K_GEMM, PAD, Guard, check, poisoned, rnd, same_bits, twice  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


@pytest.fixture(scope="module")
def L():
    from omg_b200 import _lib
    return _lib


def ringed(t, ring=2):
    """t [B, H, W, C] (C % 8 == 0) as a window of a NaN buffer [B, H + 2 ring, W + 2 ring, C + PAD]: every image sits
    inside `ring` NaN pixels on each side, and every pixel has NaN channels past C."""
    B, H, W, C = t.shape
    buf = torch.full((B, H + 2 * ring, W + 2 * ring, C + PAD), float("nan"), dtype=t.dtype, device="cuda")
    v = buf[:, ring:ring + H, ring:ring + W, :C]
    v.copy_(t)
    return v


def nan_rows(t):
    """A contiguous weight matrix t [N, K] followed by PAD NaN rows (rows past N must never be read)."""
    buf = torch.full((t.shape[0] + PAD, t.shape[1]), float("nan"), dtype=t.dtype, device="cuda")
    buf[:t.shape[0]].copy_(t)
    return buf[:t.shape[0]]


def nchw(t):
    return t.double().permute(0, 3, 1, 2)


def shifted(x, dx, dy):
    """x [B, H, W, C] read at (h + dy, w + dx), zero outside the image (|dx|, |dy| <= 2)."""
    B, H, W, _ = x.shape
    p = F.pad(x.permute(0, 3, 1, 2), (2, 2, 2, 2))
    return p[:, :, 2 + dy:2 + dy + H, 2 + dx:2 + dx + W].permute(0, 2, 3, 1)


def colstats_match(part, out):
    od, tot = out.double(), part.sum(1).double()
    assert ((tot[..., 0] - od.sum((1, 2))).abs() <= 1e-4 * od.abs().sum((1, 2))).all()
    assert ((tot[..., 1] - (od * od).sum((1, 2))).abs() <= 1e-4 * (od * od).sum((1, 2))).all()


# ------------------------------------------------------------------------------------------------ stride-2 phase views
S2_SIZES = [(2, 2), (2, 10), (10, 2), (6, 14), (18, 262)]   # outputs 1x1, 1x5, 5x1, 3x7 and 9x131 (two tiles per row)


def _s2_case(ops, L, H, W, Cin, N, epi="NONE", planes=False, seed=0):
    B = 3
    G = 2 if planes else 1
    x = ringed(rnd(B, H, W, Cin, seed=seed + 1))
    wt = rnd(G * N, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=seed + 2)
    w = nan_rows(ops.pack_conv3x3_weight(wt))
    bias = rnd(N, seed=seed + 3)
    Ho, Wo = H // 2, W // 2
    e = getattr(L, "EPI_" + epi)

    def run():
        g = Guard((B, Ho, Wo, N))
        part = torch.full((B, ops.colstats_blocks(Wo, Ho), N, 2), float("nan"), device="cuda")
        ops.conv3x3_s2(x, w, bias=bias, out=g.out, block_n=320 if N == 320 else 0, colstats=part, epilogue=e,
                       row_groups=[1, 3] if planes else None)
        torch.cuda.synchronize()
        assert g.intact(), "write outside the output window"
        return [g.out.clone(), part]

    out, part = twice(run)
    colstats_match(part, out)
    what = f"conv3x3_s2 {H}x{W} Cin={Cin} N={N} {epi}" + (" planes" if planes else "")
    for gi, (i0, i1) in enumerate([(0, 1), (1, 3)] if planes else [(0, B)]):
        ref = F.conv2d(nchw(x[i0:i1]), wt[gi * N:(gi + 1) * N].double(), bias.double(), stride=2, padding=1)
        if epi == "GELU_TANH":
            ref = F.gelu(ref, approximate="tanh")
        check(out[i0:i1].permute(0, 3, 1, 2), ref, K_GEMM, what=what + (f" stream {gi}" if planes else ""))


@pytest.mark.parametrize("Cin,N", [(40, 96), (128, 320)])
@pytest.mark.parametrize("H,W", S2_SIZES)
def test_conv3x3_s2_phase_views(ops, L, H, W, Cin, N):
    """Cin 40: a K tail in every phase segment; N 320 with block_n 320.  Bias and column statistics."""
    _s2_case(ops, L, H, W, Cin, N)


@pytest.mark.parametrize("H,W", S2_SIZES)
def test_conv3x3_s2_gelu_tanh(ops, L, H, W):
    """The SAM encoder's stride-2 ConvLayers (BN folded, tanh-GELU) run through ops.conv3x3_s2's epilogue argument."""
    _s2_case(ops, L, H, W, 40, 96, epi="GELU_TANH", seed=5)


@pytest.mark.parametrize("H,W", [(6, 14), (18, 262)])
def test_conv3x3_s2_weight_planes(ops, L, H, W):
    """row_groups=[1, 3]: image 0 uses weight plane 0, images 1 and 2 plane 1 (per-stream LoCon down-sampler)."""
    _s2_case(ops, L, H, W, 40, 96, planes=True, seed=9)


# ----------------------------------------------------------------------------------- face.OnnxNet stride-2 convs, odd H / W
class _ConvNet(torch.nn.Module):
    """One stride-2 Conv, optionally followed by BatchNorm + ReLU (folded into the GEMM by the executor)."""

    def __init__(self, cin, n, k, pad, bn):
        super().__init__()
        self.conv = torch.nn.Conv2d(cin, n, k, stride=2, padding=pad)
        self.bn = torch.nn.BatchNorm2d(n) if bn else None

    def forward(self, x):
        y = self.conv(x)
        return torch.relu(self.bn(y)) if self.bn is not None else y


class _AddNet(torch.nn.Module):
    """y = Conv k3 s2 p1 (x); out = Conv k1 s2 p0 (x) + y.  The Add folds into the second conv: as its epilogue residual
    when the padded width Np % 32 == 0, else through omg_channel_op after the GEMM.  y is a graph output too."""

    def __init__(self, cin, n):
        super().__init__()
        self.a = torch.nn.Conv2d(cin, n, 3, stride=2, padding=1)
        self.b = torch.nn.Conv2d(cin, n, 1, stride=2, padding=0)

    def forward(self, x):
        y = self.a(x)
        return self.b(x) + y, y


def _face_net(kind, cin, n, bn, seed):
    torch.manual_seed(seed)
    if kind == "add":
        m = _AddNet(cin, n)
        with torch.no_grad():
            m.a.weight.mul_(0.25)   # keeps y small beside the sum, so the late path's two roundings stay within 4 u |ref|
    else:
        k, pad = {"k3p1": (3, 1), "k1p0": (1, 0), "k3p0": (3, 0), "k2p0": (2, 0)}[kind]
        m = _ConvNet(cin, n, k, pad, bn)
        if bn:
            with torch.no_grad():
                m.bn.weight.uniform_(0.5, 1.5)
                m.bn.bias.uniform_(-0.3, 0.3)
                m.bn.running_mean.uniform_(-0.2, 0.2)
                m.bn.running_var.uniform_(0.5, 2.0)
    return m.eval()


FACE = [("k3p1", 3, 24, True), ("k3p1", 20, 20, False), ("k1p0", 12, 24, False), ("k3p0", 20, 24, True),
        ("k3p0", 3, 20, False), ("k2p0", 3, 24, False), ("k2p0", 12, 20, True), ("add", 12, 32, False),
        ("add", 20, 20, False)]


FACE_CASES = [(kind, cin, n, bn, H, W) for kind, cin, n, bn in FACE
              for H, W in [(7, 9), (5, 5), (3, 3)] + ([(1, 1)] if kind in ("k3p1", "k1p0", "add") else [])]


@pytest.mark.parametrize("kind,cin,n,bn,H,W", FACE_CASES,
                         ids=[f"{k}-cin{c}-n{n}{'-bn' if b else ''}-{h}x{w}" for k, c, n, b, h, w in FACE_CASES])
def test_face_conv_stride2_odd_inputs(kind, cin, n, bn, H, W):
    """Per element against float64 convs on the executor's own packed fp16 weights and bias (the padded input channels
    and output columns included); relative L2 against the unfused module in float64 (BatchNorm folding)."""
    from omg_b200 import face as ff
    from util_face import export
    m = _face_net(kind, cin, n, bn, seed=cin + n)
    net = ff.OnnxNet(ff.ox.loads(export(m, torch.randn(1, cin, 7, 9), dynamic_hw=True)))
    B, Cp = 2, (cin + 7) // 8 * 8
    x0 = rnd(B, H, W, Cp, seed=H * 16 + W)
    x0[..., cin:] = 0
    x = ringed(x0)
    outs = twice(lambda: [o.clone() for o in net.run(ff.Act(x, cin))])
    with torch.no_grad():
        ref_m = m.double().cuda()(nchw(x0)[:, :cin])
    ref_m = ref_m if isinstance(ref_m, tuple) else (ref_m,)
    assert [tuple(o.shape) for o in outs] == [tuple(r.shape) for r in ref_m]
    convs = [net.plan[i] for i, nd in enumerate(net.nodes) if nd.op_type == "Conv"]
    what = f"face {kind} Cin={cin} N={n} {H}x{W}"
    for p, o in zip(convs, outs[::-1] if kind == "add" else outs):   # add: convs (y, sum), outputs (sum, y)
        w = p["w"][Cp].double()
        kh, kw = p["k"]
        wc = w.view(p["Np"], kh, kw, Cp).permute(0, 3, 1, 2)
        ref = F.conv2d(nchw(x0), wc, p["bias"].double(), stride=2, padding=p["pad"][0])[:, :n]
        if p["relu"]:
            ref = ref.clamp_min(0)
        if p["residual"] is not None:
            ref = ref + outs[1].double()
        check(o, ref, K_GEMM, what=what + (" (+ residual)" if p["residual"] is not None else ""))
    for o, r in zip(outs, ref_m):
        rl = ((o.double() - r).norm() / r.norm()).item()
        assert rl < 2e-3, f"{what}: relative L2 {rl:.3e} against the unfused module"


# ------------------------------------------------------------------------------------- several A views, K-segments by hand
def _multi_view_desc(ops, seed=0):
    """n_a = 4, n_segs = 12: the 8 off-centre taps of a dilation-2 3x3 conv on view 0 (72 channels: a K tail), 1x1
    segments on view 1 (8 channels) and view 2 (40), and the channel window [64, 192) and the tail [192, 200) of view 3.
    b_k0 descends along the segment list.  Returns (run(out), reference)."""
    B, H, W, N = 2, 5, 13, 96
    chans = [72, 8, 40, 200]
    xs = [rnd(B, H, W, c, seed=seed + 1 + i) for i, c in enumerate(chans)]
    views = [ringed(x) for x in xs]
    spec = [(0, dx, dy, 0, 72) for dy in (-2, 0, 2) for dx in (-2, 0, 2) if (dx, dy) != (0, 0)]
    spec += [(1, 0, 0, 0, 8), (2, 0, 0, 0, 40), (3, 0, 0, 64, 128), (3, 0, 0, 192, 8)]
    Ktot = sum(s[4] for s in spec)
    segs, k = [], Ktot
    for a, dx, dy, c0, kl in spec:
        k -= kl
        segs.append((a, dx, dy, c0, kl, k))
    w = nan_rows(rnd(N, Ktot, scale=Ktot ** -0.5, seed=seed + 7))
    bias = rnd(N, seed=seed + 8)
    ref = bias.double().expand(B, H, W, N).clone()
    for a, dx, dy, c0, kl, k0 in segs:
        ref += shifted(xs[a].double()[..., c0:c0 + kl], dx, dy) @ w[:, k0:k0 + kl].double().t()
    # view 0's part is a dilation-2 conv without its centre tap
    w0 = torch.zeros(N, 72, 3, 3, dtype=torch.float64, device="cuda")
    for a, dx, dy, c0, kl, k0 in segs[:8]:
        w0[:, :, dy // 2 + 1, dx // 2 + 1] = w[:, k0:k0 + kl].double()
    part0 = sum(shifted(xs[0].double(), dx, dy) @ w[:, k0:k0 + kl].double().t() for _, dx, dy, _, kl, k0 in segs[:8])
    assert torch.allclose(part0.permute(0, 3, 1, 2), F.conv2d(nchw(xs[0]), w0, dilation=2, padding=2))

    def run(out):
        ops.gemm([ops.view4(v) for v in views], segs, w, N, Ktot, ops.view4(out), bias=bias)

    return run, ref


def test_four_views_twelve_segments(ops):
    run_desc, ref = _multi_view_desc(ops)

    def run():
        g = Guard(tuple(ref.shape))
        run_desc(g.out)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    check(out, ref, K_GEMM, what="4 views / 12 segments, b_k0 descending")


@pytest.mark.parametrize("W", [5, 96, 130])
def test_conv3x3_two_shortcut_views(ops, W):
    """ResBlock shortcut concatenation: 9 taps of a 40-channel input plus 1x1 segments of a 40- and a 24-channel view,
    their weight columns out of order (24-channel block first); rowvec and residual."""
    B, H, Cin, N = 2, 3, 40, 96
    x = ringed(rnd(B, H, W, Cin, seed=1))
    s1, s2 = ringed(rnd(B, H, W, 40, seed=2)), ringed(rnd(B, H, W, 24, seed=3))
    wt = rnd(N, Cin, 3, 3, scale=(9 * Cin + 64) ** -0.5, seed=4)
    w1, w2 = rnd(N, 40, scale=0.1, seed=5), rnd(N, 24, scale=0.1, seed=6)
    w = nan_rows(torch.cat([ops.pack_conv3x3_weight(wt), w2, w1], dim=1))
    bias, temb, res = rnd(N, seed=7), rnd(B, N, seed=8), rnd(B, H, W, N, seed=9)

    def run():
        g = Guard((B, H, W, N))
        ops.conv3x3(x, w, bias=bias, rowvec=temb, residual=res, out=g.out, shortcut=[(s1, 9 * Cin + 24), (s2, 9 * Cin)])
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    ref = F.conv2d(nchw(x), wt.double(), bias.double(), padding=1) + nchw(s1.double() @ w1.double().t()) \
        + nchw(s2.double() @ w2.double().t()) + temb.double()[:, :, None, None] + nchw(res)
    check(out.permute(0, 3, 1, 2), ref, K_GEMM, what=f"conv3x3 + 2 shortcut views W={W}")


def test_linear_extra_segments_mid_weight(ops):
    """`extra` K-segments whose weight columns sit in the middle of w, not right after x's: x [0, 72), t2 [72, 80),
    t1 [120, 160); columns [80, 120) and [160, 168) belong to no segment."""
    M, N = 300, 160
    x, t1, t2 = poisoned(rnd(M, 72, seed=1)), poisoned(rnd(M, 40, seed=2)), poisoned(rnd(M, 8, seed=3))
    w = nan_rows(rnd(N, 168, scale=120 ** -0.5, seed=4))
    b, r = rnd(N, seed=5), poisoned(rnd(M, N, seed=6))

    def run():
        g = Guard((M, N))
        ops.linear(x, w, bias=b, residual=r, out=g.out, extra=[(t1, 120), (t2, 72)])
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    wd = w.double()
    ref = x.double() @ wd[:, :72].t() + t1.double() @ wd[:, 120:160].t() + t2.double() @ wd[:, 72:80].t() \
        + b.double() + r.double()
    check(out, ref, K_GEMM, what="linear extra segments mid-weight")


# ------------------------------------------------------------------------------------------------- un-merged LoRA segments
LORA_MODES = ["bias", "residual", "geglu", "row_stats", "fp32_twins", "ln_2_groups", "ln_3_groups"]


def _lora_case(ops, L, r_tot, mode, seed=0):
    """out = epi(x W^T + t B2^T ...) with t [M, r_tot] a column window of a NaN-bordered buffer, block-diagonal the way
    UNetRunner._lin writes it: the rows of stream g are non-zero only in stream g's columns (8 per rank unit, dealt
    round-robin; a stream may have none).  Streams end at 128-row boundaries, the last one inside a tile."""
    ln = mode.startswith("ln")
    G = 3 if mode == "ln_3_groups" else 2
    ends = [128 * (g + 1) for g in range(G - 1)] + [128 * (G - 1) + 168]
    starts = [0] + ends[:-1]
    M, K, N = ends[-1], 200, 320
    units = r_tot // 8
    widths = [8 * (units // G + (1 if g < units % G else 0)) for g in range(G)]
    t0 = torch.zeros(M, r_tot, dtype=torch.float16, device="cuda")
    c = 0
    for g in range(G):
        t0[starts[g]:ends[g], c:c + widths[g]] = rnd(ends[g] - starts[g], widths[g], scale=0.5, seed=seed + 10 + g)
        c += widths[g]
    t = poisoned(t0)
    x = poisoned(rnd(M, K, seed=seed + 1) + (0.5 if ln else 0.0))
    wu, bu = rnd(N, K, scale=K ** -0.5, seed=seed + 2), rnd(N, seed=seed + 3)
    b2u = rnd(N, r_tot, scale=r_tot ** -0.5, seed=seed + 4)
    h = x.double() @ wu.double().t() + t0.double() @ b2u.double().t()
    kw, flat = {}, False
    if mode == "geglu":
        wp, bp = ops.pack_geglu_weight(wu, bu)
        w, b2, kw["bias"], kw["epilogue"] = nan_rows(wp), nan_rows(ops.pack_geglu_weight(b2u)[0]), bp, L.EPI_GEGLU
        hb = h + bu.double()
        ref = hb[:, :N // 2] * F.gelu(hb[:, N // 2:])
    else:
        w, b2 = nan_rows(wu), nan_rows(b2u)
        ref = h + bu.double()
        kw["bias"] = bu
    if mode == "residual":
        kw["residual"] = poisoned(rnd(M, N, seed=seed + 5))
        ref = ref + kw["residual"].double()
    if mode == "row_stats":
        flat = True
        parts = ops.gemm_plan(N, L.EPI_NONE, M)[1]
    if mode == "fp32_twins":
        flat = True
        r32 = torch.randn(M, N, generator=torch.Generator(device="cuda").manual_seed(seed + 6), device="cuda")
        ref = ref + r32.double()
    if ln:
        flat = True
        del kw["bias"]
        xd = x.double()
        stats = torch.stack([xd.sum(1), (xd * xd).sum(1)], dim=-1)[None].float().contiguous()
        c1 = (wu.float().sum(1)[None] + 0.1 * rnd(G, N, seed=seed + 7).float()).contiguous()
        c2 = rnd(G, N, seed=seed + 8).float().contiguous()
        kw["ln"] = (stats, 1, M, 0, K, 1e-5, c1.view(-1), c2.view(-1), ends)
        mean = xd.mean(1, keepdim=True)
        rstd = (xd.var(1, unbiased=False, keepdim=True) + 1e-5).rsqrt()
        rows = torch.cat([torch.full((e - s,), g, device="cuda") for g, (s, e) in enumerate(zip(starts, ends))]).long()
        ref = rstd * (h - mean * c1.double()[rows]) + c2.double()[rows]
    n_out = N // 2 if mode == "geglu" else N

    def run(out=None, out32=None, stats_out=None):
        ops.linear(x, w, out=out, lora=(t, b2), stats_out=stats_out, out_f32=out32,
                   residual_f32=r32 if mode == "fp32_twins" else None, **kw)

    def guarded():
        g = Guard((M, n_out), flat=flat)
        g32 = Guard((M, n_out), dtype=torch.float32, flat=True) if mode == "fp32_twins" else None
        st = torch.full((parts, M, 2), float("nan"), device="cuda") if mode == "row_stats" else None
        run(g.out, None if g32 is None else g32.out, st)
        torch.cuda.synchronize()
        assert g.intact() and (g32 is None or g32.intact())
        return [g.out.clone()] + ([g32.out.clone()] if g32 is not None else []) + ([st] if st is not None else [])

    return guarded, run, ref, n_out


@pytest.mark.parametrize("mode", LORA_MODES)
@pytest.mark.parametrize("r_tot", [8, 24, 40, 64, 72, 136])
def test_unmerged_lora_segment(ops, L, r_tot, mode):
    """r_tot 8 .. 136: K tails of the w2 segment and up to 3 K blocks; bias, residual, GEGLU (pack_geglu_weight of B2),
    row statistics, fp32 twins, and the folded LayerNorm with per-stream c1 / c2 planes (2 and 3 streams)."""
    guarded, _, ref, _ = _lora_case(ops, L, r_tot, mode)
    res = twice(guarded)
    what = f"un-merged LoRA r_tot={r_tot} {mode}"
    if mode == "fp32_twins":
        check(res[1], ref, K_F32, rel_l2=1e-5, u=2.0 ** -24, what=what + " out_f32")
        assert same_bits(res[0], res[1].half())
        return
    check(res[0], ref, K_GEMM, what=what)
    if mode == "row_stats":
        st = res[1].sum(0).double()
        assert ((st[:, 0] - ref.sum(1)).abs() <= 1e-4 * ref.abs().sum(1)).all()
        assert ((st[:, 1] - (ref * ref).sum(1)).abs() <= 1e-4 * (ref * ref).sum(1)).all()


# ------------------------------------------------------------------------------------ executor: LoRA at any summed rank
@pytest.fixture(scope="module")
def unet_env():
    from omg_b200.config import UNetConfig
    from omg_b200.unet import PackedUNet
    from util_models import weights
    cfg = UNetConfig.tiny()
    sd = weights(cfg, 0)
    return {"cfg": cfg, "sd": sd, "model": PackedUNet(cfg, sd)}


RANK_SETS = [(4,), (2,), (6,), (4, 8)]


@pytest.mark.parametrize("ranks", RANK_SETS, ids=["+".join(map(str, r)) for r in RANK_SETS])
def test_concept_unet_lora_any_rank(unet_env, ranks):
    """The tiny UNet with LoRA sets whose summed ranks are not multiples of 8 (attn1.qkv: 3 r, attn2.kv: 2 r), in both
    merge modes, against the fp32 oracle with the tolerance of test_unet_gpu.py."""
    from omg_b200.unet import PackedUNet, UNetRunner
    from oracle import unet as ou
    from test_unet_gpu import TOL, _inputs
    from util_models import from_nhwc, lora, ocfg, oracle_lora, rel, to_nhwc8
    cfg, sd = unet_env["cfg"], unet_env["sd"]
    B, H, W = 2, 32, 32
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 7)
    adapters = [(lora(cfg, 11 + i, rank=r), wgt) for i, (r, wgt) in enumerate(zip(ranks, (0.7, 0.5)))]
    model = PackedUNet(cfg, sd)
    model.add_lora_set("c", adapters, 0.8)
    ref = ou.unet_forward(ou.Ctx(sd, ocfg(cfg), lora=oracle_lora(adapters, 0.8)), x, 250.0, ctx, pooled, tid)
    base = ou.unet_forward(ou.Ctx(sd, ocfg(cfg)), x, 250.0, ctx, pooled, tid)
    for merged in (True, False):
        r = UNetRunner(model, B, H, W, lora_key="c", use_graphs=False)
        r.merge_lora = merged
        r.set_conditioning([250.0], ctx, pooled, tid)
        r.sample_in.copy_(to_nhwc8(x))
        out = from_nhwc(r.forward(0))
        e = rel(out, ref)
        print(f"lora ranks {ranks} {'merged' if merged else 'unmerged'}: rel err {e:.3e}, lora effect {rel(ref, base):.3e}")
        assert e < TOL and rel(ref, base) > 5 * e


def test_two_lora_streams_one_launch(unet_env):
    """Two streams with LoRA sets of rank 4 and 6 in one runner: in the un-merged mode each stream's t block has
    columns of its own (and set_context's attn2.kv takes this path in both modes)."""
    from omg_b200.unet import PackedUNet, RowGroup, UNetRunner
    from oracle import unet as ou
    from test_unet_gpu import TOL, _inputs
    from util_models import from_nhwc, lora, ocfg, oracle_lora, rel, to_nhwc8
    cfg, sd = unet_env["cfg"], unet_env["sd"]
    B, H, W = 4, 32, 32
    x, ctx, pooled, tid = _inputs(cfg, B, H, W, 8)
    sets = {"a": [(lora(cfg, 21, rank=4), 0.9)], "b": [(lora(cfg, 22, rank=6), 0.6)]}
    model = PackedUNet(cfg, sd)
    for k, ad in sets.items():
        model.add_lora_set(k, ad, 1.0)
    refs = [ou.unet_forward(ou.Ctx(sd, ocfg(cfg), lora=oracle_lora(sets[k], 1.0)), x[i0:i1], 300.0, ctx[i0:i1],
                            pooled[i0:i1], tid[i0:i1]) for k, (i0, i1) in (("a", (0, 2)), ("b", (2, 4)))]
    for merged in (True, False):
        r = UNetRunner(model, B, H, W, use_graphs=False, groups=[RowGroup(0, 2, "a"), RowGroup(2, 4, "b")])
        r.merge_lora = merged
        r.set_conditioning([300.0], [(ctx[:2], "a", False), (ctx[2:], "b", False)], pooled, tid)
        r.sample_in.copy_(to_nhwc8(x))
        out = from_nhwc(r.forward(0))
        for (k, (i0, i1)), ref in zip((("a", (0, 2)), ("b", (2, 4))), refs):
            e = rel(out[i0:i1], ref)
            print(f"two streams, stream {k} {'merged' if merged else 'unmerged'}: rel err {e:.3e}")
            assert e < TOL


# --------------------------------------------------------------------------------------------------- launch-plan replays
def test_plan_replays_one_descriptor_per_family(ops, L):
    """A phase-view conv, the 4-view / 12-segment GEMM and an un-merged LoRA GEMM recorded in one omg_plan and replayed
    from C: bit-identical to the recorded launches."""
    B, H, W, Cin, N = 3, 18, 262, 40, 96
    x = ringed(rnd(B, H, W, Cin, seed=1))
    w_s2, b_s2 = rnd(N, 9 * Cin, scale=(9 * Cin) ** -0.5, seed=2), rnd(N, seed=3)
    mv_run, mv_ref = _multi_view_desc(ops, seed=20)
    _, lora_run, _, n_out = _lora_case(ops, L, 72, "residual", seed=30)
    outs = [torch.empty(B, H // 2, W // 2, N, dtype=torch.float16, device="cuda"),
            torch.empty(tuple(mv_ref.shape), dtype=torch.float16, device="cuda"),
            torch.empty(296, n_out, dtype=torch.float16, device="cuda")]

    def launch():
        ops.conv3x3_s2(x, w_s2, bias=b_s2, out=outs[0], epilogue=L.EPI_GELU_TANH)
        mv_run(outs[1])
        lora_run(outs[2])

    plan = ops.LaunchPlan()
    with plan:
        launch()
    assert len(plan) == 3
    torch.cuda.synchronize()
    recorded = [o.clone() for o in outs]
    for o in outs:
        o.fill_(float("nan"))
    plan.run()
    torch.cuda.synchronize()
    for a, b in zip(recorded, outs):
        assert torch.isfinite(a.float()).all() and same_bits(a, b)
