"""Kernel edges through the C ABI: tile tails, descriptor features without another kernel-level test, guarded outputs and
NaN-poisoned neighbours, against float64 references computed on the GPU from the same fp16 inputs the kernel saw.

* `check` bounds every element, not only the relative L2 norm:  |out - ref| <= 4 u |ref| + k u rms(ref)  with u the unit
  roundoff of the stored type (2^-11 for fp16, so 4 u = 2^-9), plus "no NaN / inf".  k is set per kernel family below.
* `Guard` places an output inside a larger NaN-filled buffer (rows before and after, columns on both sides, hence a larger
  batch stride for 3-D / 4-D outputs); after the call everything outside the output must be bit-identical.
* `poisoned` places an operand inside a NaN-filled buffer (wider rows, extra token rows past the logical end), so a read
  outside the operand shows up as NaN in the result.
Both stay inside memory the test owns: a stray access changes values, it cannot fault.  Every case runs twice and must
be bit-identical (no kernel uses atomics).  `pytest -s` prints the k each case needs.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

PAD = 8  # elements; a multiple of 8 keeps the kernels' 16 B row alignment

# Per-element k of each kernel family, with the worst value the family's cases need on an NVIDIA H100 80GB HBM3 at a
# 400 W power limit (a value <= 0 means every element is already within 4 u |ref|).
K_GEMM = 1.0      # measured 0.00 (GEMM, convs, weight planes)
K_F32 = 32.0      # fp32 results, u = 2^-24: measured 17.4 (out_f32, 320-wide tiles), 7.7 (fuse_step latents);
                  # the same Euler step through solver_step needs 1.9 (H100 80GB HBM3 at 700 W)
K_ATTN = 4.0      # measured 1.6 (16 items, n_kv = 77)
K_NORM = 1.0      # measured 0.23 (GroupNorm from omg_colstats at |mean| / sigma = 32)
K_ELEM = 1.0      # measured 0.00
K_VISION = 1.0    # measured 0.00


def check(out, ref, k, rel_l2=2e-3, u=2.0 ** -11, what=""):
    o, r = out.double(), ref.double()
    assert torch.isfinite(o).all(), f"{what}: non-finite output"
    rms = r.pow(2).mean().sqrt().clamp_min(1e-30)
    err = (o - r).abs()
    need = ((err - 4 * u * r.abs()) / (u * rms)).max().item()
    rl = ((o - r).norm() / r.norm().clamp_min(1e-30)).item()
    print(f"[check] {what}: rel_l2 {rl:.3e}, k needed {need:.2f} (bound {k})")
    assert rl <= rel_l2, f"{what}: relative L2 {rl:.3e} > {rel_l2}"
    assert need <= k, f"{what}: per-element error needs k = {need:.2f} > {k}"


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


class Guard:
    """Output view of `shape` inside a NaN-filled buffer.  window: PAD rows before and 2 PAD after along dim -2 and PAD
    columns on both sides (3-D / 4-D: a larger batch / row stride); flat: contiguous, PAD elements before and after."""

    def __init__(self, shape, dtype=torch.float16, flat=False):
        if flat:
            n = math.prod(shape)
            self.buf = torch.full((n + 2 * PAD,), float("nan"), dtype=dtype, device="cuda")
            idx = (slice(PAD, PAD + n),)
            self.out = self.buf[idx[0]].view(shape)
        else:
            full = list(shape)
            full[-2] += 3 * PAD
            full[-1] += 2 * PAD
            self.buf = torch.full(full, float("nan"), dtype=dtype, device="cuda")
            idx = (slice(None),) * (len(shape) - 2) + (slice(PAD, PAD + shape[-2]), slice(PAD, PAD + shape[-1]))
            self.out = self.buf[idx]
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        self.inside[idx] = True
        self.before = self.buf.clone()

    def intact(self):
        return bool(((_bits(self.buf) == _bits(self.before)) | self.inside).all())


def poisoned(t, rows=0):
    """t [..., T, C] as a window of a NaN buffer [..., T + rows, C + 2 PAD] (columns [PAD, PAD + C), rows [0, T))."""
    full = list(t.shape)
    full[-2] += rows
    full[-1] += 2 * PAD
    buf = torch.full(full, float("nan"), dtype=t.dtype, device="cuda")
    v = buf[..., :t.shape[-2], PAD:PAD + t.shape[-1]]
    v.copy_(t)
    return v


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


def twice(run):
    """run() -> list of output tensors; a second run must reproduce them bit for bit."""
    a, b = run(), run()
    for x, y in zip(a, b):
        assert same_bits(x, y), "second run differs"
    return a


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


@pytest.fixture(scope="module")
def L():
    from omg_b200 import _lib
    return _lib


# ---------------------------------------------------------------------------------------------------------------- GEMM
# family -> (block_n, cta_pair, N with a partial last n-tile; 320 needs N % 320 == 0)
FAMILIES = {"64": (64, 1, 224), "128": (128, 1, 352), "160": (160, 1, 224), "160-tall": (160, 3, 224),
            "256": (256, 1, 288), "320": (320, 1, 640)}


def _epi_ref(v, epi, L):
    if epi == L.EPI_SILU:
        return v * torch.sigmoid(v)
    if epi == L.EPI_QUICK_GELU:
        return v * torch.sigmoid(1.702 * v)
    if epi == L.EPI_GELU:
        return F.gelu(v)
    if epi == L.EPI_GELU_TANH:
        return F.gelu(v, approximate="tanh")
    if epi == L.EPI_RELU:
        return v.clamp_min(0)
    return v


def _linear_case(ops, M, N, K, bn, cta_pair, epi=0, seed=0):
    """A = channel window of NaN-poisoned rows (the K tail ends at the view's last channel, so TMA must zero-fill it);
    weight rows past N, bias entries past N and residual columns around the window are NaN; output in a guarded window."""
    x = poisoned(rnd(M, K, seed=seed + 1))
    wbuf = torch.full((N + PAD, K), float("nan"), dtype=torch.float16, device="cuda")
    w = wbuf[:N]
    w.copy_(rnd(N, K, scale=K ** -0.5, seed=seed + 2))
    bbuf = torch.full((N + PAD,), float("nan"), dtype=torch.float16, device="cuda")
    b = bbuf[:N]
    b.copy_(rnd(N, seed=seed + 3))
    r = poisoned(rnd(M, N, seed=seed + 4))

    def run():
        g = Guard((M, N))
        ops.linear(x, w, bias=b, residual=r, out=g.out, epilogue=epi, block_n=bn, cta_pair=cta_pair)
        torch.cuda.synchronize()
        assert g.intact(), "write outside the output window"
        return [g.out.clone()]

    out, = twice(run)
    from omg_b200 import _lib as L
    ref = _epi_ref(x.double() @ w.double().t() + b.double(), epi, L) + r.double()
    return out, ref


@pytest.mark.parametrize("K", [8, 40, 200, 1000])
@pytest.mark.parametrize("M", [1, 127, 129, 383])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_gemm_tile_families_with_tails(ops, family, M, K):
    bn, cta_pair, N = FAMILIES[family]
    out, ref = _linear_case(ops, M, N, K, bn, cta_pair)
    check(out, ref, K_GEMM, what=f"gemm {family} M={M} N={N} K={K}")
    if cta_pair == 3:  # tall tiles compute exactly what single 128-row tiles compute
        single, _ = _linear_case(ops, M, N, K, bn, 1)
        assert same_bits(out, single)


@pytest.mark.parametrize("family", ["64", "160-tall", "256", "320"])
@pytest.mark.parametrize("epi", ["NONE", "SILU", "QUICK_GELU", "GELU", "GELU_TANH", "RELU"])
def test_gemm_epilogues_with_bias_and_residual(ops, L, epi, family):
    bn, cta_pair, N = FAMILIES[family]
    out, ref = _linear_case(ops, 383, N, 200, bn, cta_pair, epi=getattr(L, "EPI_" + epi), seed=10)
    check(out, ref, K_GEMM, what=f"gemm {epi} {family}")


def test_gemm_geglu_partial_last_tile(ops, L):
    M, N, K = 129, 576, 200                     # 576 = 2 x 256 + 64: the GEGLU tile (256) has a tail
    x = poisoned(rnd(M, K, seed=1))
    w, b = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)   # interleaved (value_j, gate_j) rows

    def run():
        g = Guard((M, N // 2))
        ops.linear(x, w, bias=b, out=g.out, epilogue=L.EPI_GEGLU)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    h = x.double() @ w.double().t() + b.double()
    check(out, h[:, 0::2] * F.gelu(h[:, 1::2]), K_GEMM, what="gemm GEGLU N=576")


def _group_sizes(groups, align):
    sizes = [align * (1 + i % 3) for i in range(groups)]
    sizes[-1] += 40                              # the last stream ends inside a tile
    ends, e = [], 0
    for s in sizes:
        e += s
        ends.append(e)
    return ends


@pytest.mark.parametrize("ln", [False, True], ids=["plain", "folded_ln"])
@pytest.mark.parametrize("align", [128, 256])
@pytest.mark.parametrize("groups", [2, 3, 8])
def test_gemm_per_stream_weight_planes(ops, groups, align, ln):
    """w_group_planes + col_group_end (merged-LoRA grouped forwards): rows of stream g multiply with weight plane g, and
    with the folded LayerNorm also use c1 / c2 plane g.  Boundaries on multiples of 128 but not 256 make tall tiles
    inapplicable (both m-tiles of a tall tile must belong to one stream); on multiples of 256 tall tiles run.  Either
    way the result is bit-equal to single 128-row tiles."""
    ends = _group_sizes(groups, align)
    M, N, K = ends[-1], 320, 200
    starts = [0] + ends[:-1]
    x = poisoned(rnd(M, K, seed=1) + (0.5 if ln else 0.0))
    wbuf = torch.full((groups * N + PAD, K), float("nan"), dtype=torch.float16, device="cuda")
    w = wbuf[:groups * N]
    w.copy_(rnd(groups * N, K, scale=K ** -0.5, seed=2))
    b = rnd(N, seed=3)
    kw = {}
    if ln:
        xd = x.double()
        stats = torch.stack([xd.sum(1), (xd * xd).sum(1)], dim=-1)[None].float().contiguous()   # one partial plane
        c1 = w.float().view(groups, N, K).sum(-1).contiguous()
        c2 = rnd(groups, N, seed=4).float().contiguous()
        kw["ln"] = (stats, 1, M, 0, K, 1e-5, c1.view(-1), c2.view(-1), ends)
    else:
        kw["bias"] = b

    def run(cta_pair):
        g = Guard((M, N), flat=ln)   # the folded LayerNorm indexes its statistics by pixel: contiguous output
        ops.linear(x, w, out=g.out, block_n=160, cta_pair=cta_pair, row_groups=ends, **kw)
        torch.cuda.synchronize()
        assert g.intact()
        return g.out.clone()

    out = run(3)
    assert same_bits(out, run(3))
    assert same_bits(out, run(1))
    for gi, (r0, r1) in enumerate(zip(starts, ends)):
        xg, wg = x[r0:r1].double(), w[gi * N:(gi + 1) * N].double()
        if ln:
            mean = xg.mean(1, keepdim=True)
            rstd = (xg.var(1, unbiased=False, keepdim=True) + 1e-5).rsqrt()
            ref = rstd * (xg @ wg.t() - mean * c1[gi].double()) + c2[gi].double()
        else:
            ref = xg @ wg.t() + b.double()
        check(out[r0:r1], ref, K_GEMM, what=f"weight planes {groups} groups / {align}, stream {gi}")


@pytest.mark.parametrize("mode", ["alone", "in_place", "with_statistics"])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_gemm_fp32_trunk_twins(ops, family, mode):
    """residual_f32 / out_f32: the addend comes from the fp32 trunk and the unrounded result is stored as fp32; the fp16
    output is that stored value rounded (bit-equal to out_f32.half()).  In place as the UNet runs it (residual_f32 is
    out_f32), and together with GroupNorm column statistics and LayerNorm row statistics out of the same epilogue."""
    bn, cta_pair, N = FAMILIES[family]
    M, K = 383, 200
    x = poisoned(rnd(M, K, seed=1))
    w, b = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    r32 = torch.randn(M, N, generator=torch.Generator(device="cuda").manual_seed(4), device="cuda")
    ref = x.double() @ w.double().t() + b.double() + r32.double()
    parts = (4 if bn == 320 else 2) * ((N + bn - 1) // bn)

    def run():
        g = Guard((M, N), flat=True)
        g32 = Guard((M, N), dtype=torch.float32, flat=True)
        if mode == "in_place":
            g32.out.copy_(r32)
            g32.before = g32.buf.clone()
        kw = {}
        if mode == "with_statistics":
            kw["colstats"] = torch.full((1, ops.colstats_blocks(M, 1), N, 2), float("nan"), device="cuda")
            kw["stats_out"] = torch.full((parts, M, 2), float("nan"), device="cuda")
        ops.linear(x, w, bias=b, out=g.out, block_n=bn, cta_pair=cta_pair,
                   residual_f32=g32.out if mode == "in_place" else r32, out_f32=g32.out, **kw)
        torch.cuda.synchronize()
        assert g.intact() and g32.intact()
        return [g.out.clone(), g32.out.clone()] + [kw[k] for k in ("colstats", "stats_out") if k in kw]

    res = twice(run)
    out, o32 = res[0], res[1]
    check(o32, ref, K_F32, rel_l2=1e-5, u=2.0 ** -24, what=f"out_f32 {family} {mode}")
    assert same_bits(out, o32.half())
    if mode == "with_statistics":
        cs, st = res[2].sum(1)[0].double(), res[3].sum(0).double()
        od, fd = out.double(), o32.double()
        assert ((cs[:, 0] - od.sum(0)).abs() <= 1e-4 * od.abs().sum(0)).all()
        assert ((cs[:, 1] - (od * od).sum(0)).abs() <= 1e-4 * (od * od).sum(0)).all()
        assert ((st[:, 0] - fd.sum(1)).abs() <= 1e-4 * fd.abs().sum(1)).all()
        assert ((st[:, 1] - (fd * fd).sum(1)).abs() <= 1e-4 * (fd * fd).sum(1)).all()


@pytest.mark.parametrize("W,H", [(1, 9), (3, 7), (5, 5), (96, 3), (130, 3)])
def test_conv3x3_narrow_and_odd_widths(ops, W, H):
    """Pixel tiles of 1, 4 and 8 columns, a 128 x 1 tile a quarter empty (W = 96) and two tiles per row (W = 130), odd H,
    three images; 40-channel K segments (tails) of a NaN-poisoned input; rowvec, residual and column statistics."""
    B, Cin, N = 3, 40, 96
    x = poisoned(rnd(B, H, W, Cin, seed=1))
    wt = rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    bias, temb, res = rnd(N, seed=3), rnd(B, N, seed=4), rnd(B, H, W, N, seed=5)

    def run():
        g = Guard((B, H, W, N))
        part = torch.full((B, ops.colstats_blocks(W, H), N, 2), float("nan"), device="cuda")
        ops.conv3x3(x, ops.pack_conv3x3_weight(wt), bias=bias, rowvec=temb, residual=res, out=g.out, colstats=part)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone(), part]

    out, part = twice(run)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), bias.double(), padding=1) \
        + temb.double()[:, :, None, None] + res.double().permute(0, 3, 1, 2)
    check(out.permute(0, 3, 1, 2), ref, K_GEMM, what=f"conv W={W} H={H}")
    od, tot = out.double(), part.sum(1).double()
    assert ((tot[..., 0] - od.sum((1, 2))).abs() <= 1e-4 * od.abs().sum((1, 2))).all()
    assert ((tot[..., 1] - (od * od).sum((1, 2))).abs() <= 1e-4 * (od * od).sum((1, 2))).all()


def test_upsample_conv_odd_sizes(ops):
    B, H, W, Cin, N = 2, 5, 7, 40, 64
    x = rnd(B, H, W, Cin, seed=1)
    wt, bias = rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2), rnd(N, seed=3)

    def run():
        g = Guard((B, 2 * H, 2 * W, N))
        part = torch.full((B, 4 * ops.colstats_blocks(W, H), N, 2), float("nan"), device="cuda")
        ops.upsample2x_conv3x3(x, ops.pack_conv3x3_weight(wt), bias=bias, out=g.out, colstats=part)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone(), part]

    out, part = twice(run)
    ref = F.conv2d(F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest"), wt.double(),
                   bias.double(), padding=1)
    check(out.permute(0, 3, 1, 2), ref, K_GEMM, what="upsample conv 5 x 7")
    od, tot = out.double(), part.sum(1).double()
    assert ((tot[..., 0] - od.sum((1, 2))).abs() <= 1e-4 * od.abs().sum((1, 2))).all()


# ----------------------------------------------------------------------------------------------------------- attention
def _attn_ref(q, k, v, items, heads, D, n_q, n_kv, scale, causal=False):
    """fp64 softmax(scale Q K^T) V per item (out_b, q_b, k_b, v_b) -> {out_b: [n_q, heads * D]}."""
    res = {}
    for ob, qb, kb, vb in items:
        qh = q[qb, :n_q].double().view(n_q, heads, D).transpose(0, 1)
        kh = k[kb, :n_kv].double().view(n_kv, heads, D).transpose(0, 1)
        vh = v[vb, :n_kv].double().view(n_kv, heads, D).transpose(0, 1)
        s = qh @ kh.transpose(-1, -2) * scale
        if causal:
            s = s.masked_fill(torch.ones(n_q, n_kv, dtype=torch.bool, device="cuda").triu(1), float("-inf"))
        res[ob] = (torch.softmax(s, -1) @ vh).transpose(0, 1).reshape(n_q, heads * D)
    return res


def _attn_case(ops, n_q, n_kv, heads, items, n_src, scale=0.125, causal=False, gain=1.0, out_weight=None, seed=0,
               D=64):
    """Q / K / V are head windows (col0 = PAD) of NaN-poisoned rows, with NaN token rows past n_q / n_kv in every batch
    slab; out is a guarded window (rows past n_q reached through out_bs)."""
    Cc = heads * D
    q = poisoned(rnd(n_src, n_q, Cc, scale=gain, seed=seed + 1), rows=16)
    k = poisoned(rnd(n_src, n_kv, Cc, scale=gain, seed=seed + 2), rows=16)
    v = poisoned(rnd(n_src, n_kv, Cc, seed=seed + 3), rows=16)
    n_out = max(it[0] for it in items) + 1
    base = rnd(n_out, n_q, Cc, seed=seed + 4)

    def run():
        g = Guard((n_out, n_q, Cc))
        if out_weight is not None:
            g.out.copy_(base)
            g.before = g.buf.clone()
        qb, kb, vb, obuf = q._base, k._base, v._base, g.buf[:, PAD:]   # out rows start at the window's first row
        if D == 64:
            ops.attention(qb, kb, vb, obuf, heads, n_q, n_kv, items, q_col0=PAD, k_col0=PAD, v_col0=PAD, out_col0=PAD,
                          scale=scale, causal=causal, out_weight=1.0 if out_weight is None else out_weight,
                          accumulate=out_weight is not None)
        else:
            ops.attention_small(qb, kb, vb, obuf, heads, D, n_q, n_kv, q_col0=PAD, k_col0=PAD, v_col0=PAD,
                                out_col0=PAD, scale=scale, items=items)
        torch.cuda.synchronize()
        assert g.intact(), "write outside the output window"
        return [g.out.clone()]

    out, = twice(run)
    ref = _attn_ref(q, k, v, items, heads, D, n_q, n_kv, scale, causal)
    for ob, r in ref.items():
        if out_weight is not None:
            r = base[ob].double() + out_weight * r
        check(out[ob], r, K_ATTN, what=f"attention n_q={n_q} n_kv={n_kv} heads={heads} D={D} out row {ob}")


@pytest.mark.parametrize("scale", [0.125, 0.3])
@pytest.mark.parametrize("heads", [1, 3])
@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 77, 127, 128])
def test_attention_causal(ops, n, heads, scale):
    _attn_case(ops, n, n, heads, [(0, 1, 0, 1), (1, 0, 1, 0)], 2, scale=scale, causal=True, seed=n)


def test_attention_sixteen_items_repeated_and_permuted_sources(ops):
    g = torch.Generator().manual_seed(5)
    src = torch.randint(0, 5, (16, 3), generator=g).tolist()
    outs = torch.randperm(16, generator=g).tolist()
    items = [(o, s[0], s[1], s[2]) for o, s in zip(outs, src)]
    _attn_case(ops, 130, 77, 2, items, 5, seed=1)


@pytest.mark.parametrize("n_q", [1, 129])
def test_attention_single_key(ops, n_q):
    _attn_case(ops, n_q, 1, 2, [(0, 0, 0, 0), (1, 1, 0, 1)], 2, seed=2)


def test_attention_logits_spanning_60(ops):
    """q, k ~ 4.5 N(0, 1): scaled logits reach about +-60, so the running maximum jumps between key blocks."""
    _attn_case(ops, 200, 300, 2, [(0, 0, 0, 0)], 1, gain=4.5, seed=3)


@pytest.mark.parametrize("out_weight", [0.0, -0.5])
def test_attention_accumulate(ops, out_weight):
    _attn_case(ops, 150, 90, 3, [(0, 0, 1, 1), (1, 1, 0, 0)], 2, out_weight=out_weight, seed=4)


@pytest.mark.parametrize("D", [16, 32])
@pytest.mark.parametrize("n_q,n_kv", [(200, 5), (130, 63), (64, 64), (1, 65), (64, 65), (1, 127), (64, 128), (64, 129),
                                      (1, 4097), (64, 4097)])
def test_attention_small_edges(ops, D, n_q, n_kv):
    """Shared-memory path (n_kv <= 64) and split-key path (n_kv > 64, n_q <= 64) around the 64-key and 128-key chunk
    boundaries; head windows of NaN-poisoned rows, NaN rows past n_kv, guarded output."""
    _attn_case(ops, n_q, n_kv, 2, [(0, 1, 1, 0), (1, 0, 0, 1)], 2, scale=D ** -0.5, seed=n_kv, D=D)


@pytest.mark.parametrize("n_items,n_kv", [(17, 129), (33, 129), (33, 40)])
def test_attention_small_many_items_share_one_workspace(ops, n_items, n_kv):
    g = torch.Generator().manual_seed(n_items)
    src = torch.randint(0, 3, (n_items, 3), generator=g).tolist()
    items = [(i, s[0], s[1], s[2]) for i, s in enumerate(src)]
    _attn_case(ops, 20, n_kv, 2, items, 3, scale=32 ** -0.5, seed=7, D=32)


# --------------------------------------------------------------------------------------------------------------- norms
def _gn_ref(x, gamma, beta, eps, silu):
    B, HW, C = x.shape
    xd = x.double().view(B, HW, 32, C // 32)
    mean = xd.mean((1, 3), keepdim=True)
    var = xd.var((1, 3), unbiased=False, keepdim=True)
    y = ((xd - mean) / (var + eps).sqrt()).view(B, HW, C) * gamma.double() + beta.double()
    return F.silu(y) if silu else y


def _gn_both(ops, x1, x2, gamma, beta, eps, silu):
    """(statistics-pass GroupNorm, GroupNorm from omg_colstats partials), each into a guarded contiguous output."""
    B, HW = x1.shape[:2]
    C = x1.shape[2] + (0 if x2 is None else x2.shape[2])
    g1, g2 = Guard((B, HW, C), flat=True), Guard((B, HW, C), flat=True)
    ops.groupnorm(x1, gamma, beta, eps, silu, x2=x2, out=g1.out)
    p1 = ops.colstats(x1)
    p2 = None if x2 is None else ops.colstats(x2)
    ops.groupnorm_apply(x1, p1, gamma, beta, eps, silu, x2=x2, part2=p2, out=g2.out)
    torch.cuda.synchronize()
    assert g1.intact() and g2.intact()
    return [g1.out.clone(), g2.out.clone()]


@pytest.mark.parametrize("silu", [0, 1])
@pytest.mark.parametrize("C1,C2", [(32, 0), (2560, 0), (40, 56)])
@pytest.mark.parametrize("HW", [1, 7, 77, 4127])
def test_groupnorm_edges(ops, HW, C1, C2, silu):
    """HW % 32 != 0 (partial 32-row column-statistics blocks), one pixel, 1 and 80 channels per group, and 96 channels
    split 40 | 56 so that a group of 3 channels straddles the two sources."""
    B = 2
    x1 = rnd(B, HW, C1, seed=1) + 0.3
    x2 = rnd(B, HW, C2, scale=2.0, seed=2) if C2 else None
    C = C1 + C2
    gamma, beta = rnd(C, seed=3) * 0.2 + 1, rnd(C, seed=4) * 0.2
    a, b = twice(lambda: _gn_both(ops, x1, x2, gamma, beta, 1e-6, silu))
    x = x1 if x2 is None else torch.cat([x1, x2], -1)
    ref = _gn_ref(x, gamma, beta, 1e-6, silu)
    check(a, ref, K_NORM, what=f"groupnorm HW={HW} C={C1}|{C2}")
    check(b, ref, K_NORM, what=f"groupnorm_apply HW={HW} C={C1}|{C2}")


def test_groupnorm_does_not_depend_on_batch_position(ops):
    B, HW, C = 4, 77, 320
    x = rnd(B, HW, C, seed=1) * 2 + 0.5
    gamma, beta = rnd(C, seed=2) + 1, rnd(C, seed=3)
    full = _gn_both(ops, x, None, gamma, beta, 1e-5, 1)
    rolled = _gn_both(ops, x.roll(1, 0).contiguous(), None, gamma, beta, 1e-5, 1)
    for i in range(B):
        alone = _gn_both(ops, x[i:i + 1].contiguous(), None, gamma, beta, 1e-5, 1)
        for f, r, a in zip(full, rolled, alone):
            assert same_bits(f[i], a[0]) and same_bits(f[i], r[(i + 1) % B])


@pytest.mark.parametrize("rows", [1, 9])
@pytest.mark.parametrize("C", [8, 768, 776, 1280, 1288, 2048, 2560])
def test_layernorm_register_tile_boundaries(ops, C, rows):
    """C / 8 = 96 | 97 and 160 | 161 cross the kernel's register-tile instantiations (3, 5, 10 vectors per lane)."""
    x = rnd(rows, C, seed=C) * 3 + 1
    gamma, beta = rnd(C, seed=2) + 1, rnd(C, seed=3)

    def run():
        g = Guard((rows, C), flat=True)
        ops.layernorm(x, gamma, beta, out=g.out)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    ref = F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-5)
    check(out, ref, K_NORM, what=f"layernorm C={C} rows={rows}")


# ---------------------------------------------------------------------------------------- one-pass statistics (E[x^2] - mean^2)
def _offset(shape, ratio, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return ratio * (torch.randint(0, 2, shape, generator=g, device="cuda").float() * 2 - 1)


@pytest.mark.parametrize("ratio", [8, 32])
def test_groupnorm_one_pass_statistics_with_large_mean(ops, ratio):
    """Every group offset by +-ratio standard deviations: the GroupNorm partials (statistics pass, omg_colstats, and the
    GEMM epilogue's column statistics) compute the variance as E[x^2] - mean^2 in fp32, whose cancellation error grows
    with (|mean| / sigma)^2.  Measured on an H100 80GB HBM3 at 400 W (relative L2, k needed), statistics pass /
    omg_colstats / GEMM column statistics: ratio 8: 2.08e-4, 0.01 / 2.08e-4, 0.02 / 2.08e-4, 0.01;  ratio 32: 2.15e-4,
    0.11 / 2.32e-4, 0.23 / 2.17e-4, 0.10.  All three paths hold the standard bound at 32."""
    B, HW, C = 1, 1024, 640
    off = _offset((B, 1, 32, 1), ratio, 1).expand(B, HW, 32, C // 32).reshape(B, HW, C)
    x = (torch.randn(B, HW, C, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda") + off).half()
    gamma, beta = rnd(C, seed=3) * 0.2 + 1, rnd(C, seed=4) * 0.2
    a, b = _gn_both(ops, x, None, gamma, beta, 1e-5, 0)
    ref = _gn_ref(x, gamma, beta, 1e-5, 0)
    check(a, ref, K_NORM, what=f"groupnorm |mean|/sigma={ratio}")
    check(b, ref, K_NORM, what=f"groupnorm from omg_colstats |mean|/sigma={ratio}")
    # producer GEMM: its bias puts every output group at +-ratio sigma; column statistics out of the epilogue
    K = 256
    xin, w = rnd(HW, K, seed=5), rnd(C, K, scale=K ** -0.5, seed=6)
    bias = _offset((32, 1), ratio, 7).expand(32, C // 32).reshape(C).half()
    y = torch.empty(HW, C, dtype=torch.float16, device="cuda")
    part = torch.full((1, ops.colstats_blocks(HW, 1), C, 2), float("nan"), device="cuda")
    ops.linear(xin, w, bias=bias, out=y, colstats=part)
    g = Guard((1, HW, C), flat=True)
    ops.groupnorm_apply(y.view(1, HW, C), part, gamma, beta, 1e-5, 0, out=g.out)
    torch.cuda.synchronize()
    check(g.out, _gn_ref(y.view(1, HW, C), gamma, beta, 1e-5, 0), K_NORM,
          what=f"groupnorm from GEMM column statistics |mean|/sigma={ratio}")


@pytest.mark.parametrize("ratio", [8, 32])
def test_folded_layernorm_one_pass_statistics_with_large_mean(ops, L, ratio):
    """Rows of the residual stream offset by +-ratio standard deviations: the producer GEMM's row statistics and the
    consumer's folded LayerNorm (E[x^2] - mean^2 in fp32).  Measured on an H100 80GB HBM3 at 400 W: ratio 8: relative
    L2 2.13e-4, k 0.75;  ratio 32: relative L2 3.16e-4, k 3.2.  The relative L2 bound holds at both; the per-element
    error grows with the ratio, so each ratio has its own k (about twice the measured value)."""
    M, C, N = 512, 1280, 640
    o, wo = rnd(M, C, scale=0.5, seed=1), rnd(C, C, scale=C ** -0.5, seed=2)
    noise = torch.randn(M, C, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda")
    sigma = (o.double() @ wo.double().t() + noise.double()).std(1, keepdim=True).float()
    h0 = (noise + _offset((M, 1), ratio, 4) * sigma).half()
    parts = ops.gemm_plan(C, L.EPI_NONE, M)[1]
    stats = torch.full((parts, M, 2), float("nan"), device="cuda")
    h = h0.clone()
    ops.linear(o, wo, residual=h, out=h, stats_out=stats)
    gam, bet = rnd(C, seed=5) * 0.2 + 1, rnd(C, seed=6) * 0.3
    w, b = rnd(N, C, scale=C ** -0.5, seed=7), rnd(N, seed=8)
    wl = (w.float() * gam.float()[None, :]).half()
    c1 = wl.float().sum(1).contiguous()
    c2 = (w.double() @ bet.double() + b.double()).float().contiguous()
    out = ops.linear(h, wl, ln=(stats, parts, M, 0, C, 1e-5, c1, c2, [M]))
    hd = h.double()
    xn = (hd - hd.mean(1, keepdim=True)) / (hd.var(1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    check(out, xn @ wl.double().t() + c2.double(), {8: 1.5, 32: 6.0}[ratio],
          what=f"folded LayerNorm |mean|/sigma={ratio}")


# -------------------------------------------------------------------------------------------------------- element-wise
@pytest.mark.parametrize("in_place", [False, True])
@pytest.mark.parametrize("alpha", [0.0, -1.5, 0.8])
@pytest.mark.parametrize("n", [8, 2056, 2 ** 20 + 8])
def test_axpy(ops, n, alpha, in_place):
    a, b = rnd(n, seed=1), rnd(n, seed=2)
    alpha32 = torch.tensor(alpha, dtype=torch.float32).item()

    def run():
        g = Guard((n,), flat=True)
        g.out.copy_(a)
        g.before = g.buf.clone()
        ops.axpy(g.out if in_place else a, b, alpha, out=g.out)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    ref = a.double() + alpha32 * b.double()
    if alpha == 0.0:
        assert same_bits(out, a)
    else:
        check(out, ref, K_ELEM, what=f"axpy n={n} alpha={alpha}")


@pytest.mark.parametrize("C", [8, 200, 2048])
@pytest.mark.parametrize("Lk", [1, 77, 93])
def test_ctx_mix(ops, Lk, C):
    B = 3
    ctx = rnd(B, Lk, C, seed=1)
    g = torch.Generator(device="cuda").manual_seed(2)
    coef = torch.randn(Lk, Lk, generator=g, device="cuda")
    coef[torch.rand(Lk, Lk, generator=g, device="cuda") < 0.4] = 0.0        # exact zeros and negatives

    def run():
        gd = Guard((B, Lk, C), flat=True)
        ops.ctx_mix(ctx, coef, out=gd.out)
        torch.cuda.synchronize()
        assert gd.intact()
        return [gd.out.clone()]

    out, = twice(run)
    check(out, torch.einsum("wn,bnc->bwc", coef.double(), ctx.double()), K_ELEM, what=f"ctx_mix L={Lk} C={C}")


@pytest.mark.parametrize("kernel", ["fuse", "solver"])
@pytest.mark.parametrize("next_inputs", ["both", "main_only", "concept_only"])
@pytest.mark.parametrize("HW", [1, 129, 4097])
def test_fuse_step_eight_concepts(ops, HW, next_inputs, kernel):
    """8 concepts: overlapping masks, two concepts without a mask (skipped), a 0.5-valued stripe (outside the mask, as in
    the reference's `mask == 1` selection); NaN in channels 4..7 of every noise row must reach no output; the fp16
    latent copy is the fp32 state rounded; a NULL next-input pointer leaves its buffer untouched.  The same Euler step
    runs through omg_fuse_step and through omg_solver_step with Euler's coefficients (no history, no noise)."""
    from omg_b200.scheduler import StepCoeffs
    gen = torch.Generator(device="cuda").manual_seed(HW)

    def noise(rows):
        t = torch.full((rows, HW, 8), float("nan"), dtype=torch.float16, device="cuda")
        t[..., :4] = torch.randn(rows, HW, 4, generator=gen, device="cuda").half()
        return t

    nm = noise(4)
    ncs = [noise(2) for _ in range(8)]
    masks = []
    for k in range(8):
        if k in (2, 5):
            masks.append(None)
            continue
        m = (torch.rand(HW, generator=gen, device="cuda") < 0.35).float()
        if k == 1:
            m[::3] = 0.5
        masks.append(m.contiguous())
    lat0 = torch.randn(2, HW, 4, generator=gen, device="cuda") * 10
    sig, sign, gs = 5.0, 4.2, 7.5

    def run():
        lat = Guard((2, HW, 4), dtype=torch.float32, flat=True)
        lat.out.copy_(lat0)
        lat.before = lat.buf.clone()
        l16 = Guard((2, HW, 4), flat=True)
        nxt, nxc = Guard((4, HW, 8), flat=True), Guard((2, HW, 8), flat=True)
        nxt_p = nxt.out if next_inputs != "concept_only" else None
        nxc_p = nxc.out if next_inputs != "main_only" else None
        if kernel == "fuse":
            ops.fuse_step(nm, ncs, masks, gs, sig, sign, lat.out, nxt_p, nxc_p, latents_f16=l16.out)
        else:
            k = StepCoeffs(1.0, -sig, sign / sig, 1.0 - sign / sig, 0.0, 0.0, 1.0 / math.sqrt(sign * sign + 1))
            ops.solver_step(nm, ncs, masks, gs, k, lat.out, nxt_p, nxc_p, l16.out)
        torch.cuda.synchronize()
        assert lat.intact() and l16.intact() and nxt.intact() and nxc.intact()
        return [lat.out.clone(), l16.out.clone(), nxt.out.clone(), nxc.out.clone()]

    lat, l16, nxt, nxc = twice(run)
    n = nm[..., :4].double()
    sel = [(masks[k] == 1.0).double()[:, None] if masks[k] is not None else None for k in range(8)]
    U = torch.zeros(HW, 1, dtype=torch.float64, device="cuda")
    for s in sel:
        if s is not None:
            U = torch.maximum(U, s)
    new = [n[1] * (1 - U), n[3] * (1 - U)]
    for k, s in enumerate(sel):
        if s is not None:
            new[0] = new[0] + s * ncs[k][0, :, :4].double()
            new[1] = new[1] + s * ncs[k][1, :, :4].double()
    eps = torch.stack([n[0] + gs * (n[2] - n[0]), new[0] + gs * (new[1] - new[0])])
    ref = lat0.double() + eps * (sign - sig)
    check(lat, ref, K_F32, rel_l2=1e-6, u=2.0 ** -24, what=f"{kernel}_step latents HW={HW}")
    assert same_bits(l16, lat.half())
    sc = ref / math.sqrt(sign * sign + 1)
    if next_inputs != "concept_only":
        check(nxt[..., :4], torch.cat([sc, sc]), K_ELEM, what=f"{kernel}_step next_main_in HW={HW}")
        assert (_bits(nxt[..., 4:]) == 0).all()
    else:
        assert torch.isnan(nxt).all()
    if next_inputs != "main_only":
        check(nxc[..., :4], torch.stack([sc[1], sc[1]]), K_ELEM, what=f"{kernel}_step next_concept_in HW={HW}")
        assert (_bits(nxc[..., 4:]) == 0).all()
    else:
        assert torch.isnan(nxc).all()


# -------------------------------------------------------------------------------------------------------------- vision
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("ksize,stride", [(3, 1), (5, 1), (3, 2), (5, 2)])
@pytest.mark.parametrize("H,W", [(21, 17), (1, 1), (2, 3)])
def test_dwconv(ops, H, W, ksize, stride, act):
    B, C = 2, 48
    x = poisoned(rnd(B, H, W, C, seed=1))
    w, bias = rnd(ksize * ksize, C, scale=0.3, seed=2), rnd(C, seed=3)
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride

    def run():
        g = Guard((B, Ho, Wo, C), flat=True)
        ops.dwconv(x, w, bias, out=g.out, ksize=ksize, stride=stride, act=act)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().t().reshape(C, 1, ksize, ksize), bias.double(),
                   stride=stride, padding=ksize // 2, groups=C)
    if act:
        ref = F.gelu(ref, approximate="tanh")
    check(out.permute(0, 3, 1, 2), ref, K_VISION, what=f"dwconv {H}x{W} k={ksize} s={stride}")


def test_group1x1_pixel_tail(ops):
    P, C = 100, 96                                   # 100 pixels: the last 64-pixel block is partial
    x = poisoned(rnd(P, C, seed=1))
    w = rnd(C, 32, scale=32 ** -0.5, seed=2)

    def run():
        g = Guard((P, C))
        ops.group1x1(x, w, g.out)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    xg = x.double().view(P, C // 32, 32)
    ref = torch.einsum("goi,pgi->pgo", w.double().view(C // 32, 32, 32), xg).reshape(P, C)
    check(out, ref, K_VISION, what="group1x1")


@pytest.mark.parametrize("N", [1, 63, 65])
def test_relu_linear_attention(ops, N):
    B, D = 2, 32
    qkv = rnd(B, N, 3 * D, seed=N) + 0.3

    def run():
        g = Guard((B, N, D), flat=True)
        ops.relu_linear_attention(qkv, 1, dim=D, out=g.out)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    q, k, v = qkv.double().split(D, -1)
    q, k = q.clamp_min(0), k.clamp_min(0)
    kv = k.transpose(1, 2) @ torch.cat([v, torch.ones_like(v[..., :1])], -1)
    o = q @ kv
    check(out, o[..., :D] / (o[..., D:] + 1e-15), K_VISION, what=f"relu linear attention N={N}")


@pytest.mark.parametrize("H,W,Ho,Wo", [(7, 5, 13, 4), (16, 12, 16, 12), (5, 4, 23, 17), (20, 30, 9, 11)])
def test_resize_bicubic(ops, H, W, Ho, Wo):
    B, C = 2, 16
    x = rnd(B, H, W, C, seed=1)

    def run():
        g = Guard((B, Ho, Wo, C), flat=True)
        ops.resize_bicubic(x, Ho, Wo, out=g.out)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    ref = F.interpolate(x.double().permute(0, 3, 1, 2), size=(Ho, Wo), mode="bicubic", align_corners=False)
    check(out.permute(0, 3, 1, 2), ref, K_VISION, what=f"bicubic {H}x{W} -> {Ho}x{Wo}")
    if (H, W) == (Ho, Wo):
        assert same_bits(out, x)
