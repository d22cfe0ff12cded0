"""Ping-pong GEMM schedule: units of 128 rows x 64 / 128 / 160 columns dealt alternately to the two consumer warpgroups.

* Per-CTA unit counts of 0, 1, odd and even (launches of 1, 131, 132, 263, 264 and 265 units on a 132-SM H100) with units
  of 1, 3 and 7 K blocks, so the shared-memory ring wraps inside one unit and across the other warpgroup's unit.
* A logical tile wider than a unit (block_n 256 / 320, and the former tall 256 x 160 tile) is bit-equal to the tiles of
  the unit's width, with every epilogue feature: bias, rowvec, residual, fp32 twins, activations, row-statistics
  producer -> folded-LayerNorm consumer, column statistics and per-stream weight planes.
* Three dependent GEMMs captured in a CUDA graph (programmatic dependent launch between them) equal eager launches.
Operands are NaN-poisoned windows and outputs guarded windows, as in test_kernel_edges_gpu.py.
"""
import pytest
import torch

from test_kernel_edges_gpu import K_GEMM, Guard, check, poisoned, rnd, same_bits, twice  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


@pytest.fixture(scope="module")
def L():
    from omg_b200 import _lib
    return _lib


@pytest.mark.parametrize("k_blocks", [1, 3, 7])
@pytest.mark.parametrize("units", [1, 131, 132, 263, 264, 265])
@pytest.mark.parametrize("bn", [64, 160])
def test_unit_counts_and_ring_wrap(ops, bn, units, k_blocks):
    N, K = bn, 64 * k_blocks
    M = 128 * (units - 1) + 77                    # the last unit's m-tile is partial
    x = poisoned(rnd(M, K, seed=units))
    w, b, r = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3), poisoned(rnd(M, N, seed=4))

    def run():
        g = Guard((M, N))
        ops.linear(x, w, bias=b, residual=r, out=g.out, block_n=bn)
        torch.cuda.synchronize()
        assert g.intact(), "write outside the output window"
        return [g.out.clone()]

    out, = twice(run)
    check(out, x.double() @ w.double().t() + b.double() + r.double(), K_GEMM, what=f"{units} units of {bn} x {K}")


# logical tile -> the unit-wide tile it must reproduce bit for bit: (block_n, cta_pair) pairs and an N with a partial
# last logical tile (320 needs N % 320 == 0)
WIDE = {"256": ((256, 1), (128, 1), 416), "320": ((320, 1), (160, 1), 640), "tall": ((160, 3), (160, 1), 416)}


@pytest.mark.parametrize("epi", ["NONE", "SILU", "GELU"])
@pytest.mark.parametrize("wide", list(WIDE))
def test_wide_tile_equals_units_linear(ops, L, wide, epi):
    """bias + residual, or fp32 twins with column and row statistics, with activations"""
    (bw, cw), (bu, cu), N = WIDE[wide]
    M, K = 641, 264
    x = poisoned(rnd(M, K, seed=1))
    w, b, r = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3), poisoned(rnd(M, N, seed=4))
    r32 = torch.randn(M, N, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    epilogue = getattr(L, "EPI_" + epi)

    def run(bn, cta_pair, twins):
        g = Guard((M, N), flat=twins)
        if not twins:
            ops.linear(x, w, bias=b, residual=r, out=g.out, epilogue=epilogue, block_n=bn, cta_pair=cta_pair)
            torch.cuda.synchronize()
            assert g.intact()
            return [g.out.clone()]
        parts = (4 if bn == 320 else 2) * ((N + bn - 1) // bn)
        g32 = Guard((M, N), dtype=torch.float32, flat=True)
        cs = torch.full((1, ops.colstats_blocks(M, 1), N, 2), float("nan"), device="cuda")
        st = torch.full((parts, M, 2), float("nan"), device="cuda")
        ops.linear(x, w, bias=b, out=g.out, epilogue=epilogue, block_n=bn, cta_pair=cta_pair, residual_f32=r32,
                   out_f32=g32.out, colstats=cs, stats_out=st)
        torch.cuda.synchronize()
        assert g.intact() and g32.intact()
        return [g.out.clone(), g32.out.clone(), cs, st]

    for twins in (False, True):
        a, u = twice(lambda: run(bw, cw, twins)), run(bu, cu, twins)
        for t, v in zip(a[:3], u[:3]):
            assert same_bits(t, v)
        if twins:  # row statistics: the same partials; a 256-wide tile has one plane per 128-wide unit
            sa, su = a[3], u[3]
            if bw == 256:
                assert same_bits(sa, su[0::2]) and bool((su[1::2] == 0).all())
            else:
                assert same_bits(sa, su)


@pytest.mark.parametrize("wide", list(WIDE))
def test_wide_tile_equals_units_conv_rowvec_colstats(ops, wide):
    (bw, cw), (bu, cu), N = WIDE[wide]
    B, H, W, Cin = 3, 12, 20, 40                   # 40 channels: every tap segment has a K tail
    x = poisoned(rnd(B, H, W, Cin, seed=1))
    wt = rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    bias, temb, res = rnd(N, seed=3), rnd(B, N, seed=4), rnd(B, H, W, N, seed=5)

    def run(bn, cta_pair):
        g = Guard((B, H, W, N))
        cs = torch.full((B, ops.colstats_blocks(W, H), N, 2), float("nan"), device="cuda")
        ops.conv3x3(x, ops.pack_conv3x3_weight(wt), bias=bias, rowvec=temb, residual=res, out=g.out, block_n=bn,
                    cta_pair=cta_pair, colstats=cs)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone(), cs]

    a, u = twice(lambda: run(bw, cw)), run(bu, cu)
    assert same_bits(a[0], u[0]) and same_bits(a[1], u[1])
    ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), bias.double(), padding=1) \
        + temb.double()[:, :, None, None] + res.double().permute(0, 3, 1, 2)
    check(a[0].permute(0, 3, 1, 2), ref, K_GEMM, what=f"conv {wide}")


@pytest.mark.parametrize("wide", list(WIDE))
def test_wide_tile_row_statistics_into_folded_layernorm(ops, wide):
    """A row-statistics producer of either width feeds a folded-LayerNorm consumer; the consumer's output is bit-equal."""
    (bw, cw), (bu, cu), N = WIDE[wide]
    M, K, N2 = 383, 200, 192
    x = poisoned(rnd(M, K, seed=1))
    w, b = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    w2 = rnd(N2, N, scale=N ** -0.5, seed=4)
    c1 = w2.float().sum(-1).contiguous()
    c2 = rnd(N2, seed=5).float().contiguous()

    def run(bn, cta_pair):
        parts = (4 if bn == 320 else 2) * ((N + bn - 1) // bn)
        h = torch.empty(M, N, dtype=torch.float16, device="cuda")
        st = torch.full((parts, M, 2), float("nan"), device="cuda")
        ops.linear(x, w, bias=b, out=h, block_n=bn, cta_pair=cta_pair, stats_out=st)
        g = Guard((M, N2), flat=True)
        ops.linear(h, w2, out=g.out, ln=(st, parts, M, 0, N, 1e-5, c1, c2, [M]))
        torch.cuda.synchronize()
        assert g.intact()
        return [h, g.out.clone()]

    a, u = twice(lambda: run(bw, cw)), run(bu, cu)
    assert same_bits(a[0], u[0]) and same_bits(a[1], u[1])
    hd = a[0].double()
    mean, var = hd.mean(1, keepdim=True), hd.var(1, unbiased=False, keepdim=True)
    ref = (var + 1e-5).rsqrt() * (hd @ w2.double().t() - mean * c1.double()) + c2.double()
    check(a[1], ref, K_GEMM, what=f"folded LayerNorm after a {wide} producer")


@pytest.mark.parametrize("wide", list(WIDE))
def test_wide_tile_weight_planes(ops, wide):
    """Per-stream weight planes with row groups on multiples of 128 (not 256): each unit picks its own plane."""
    (bw, cw), (bu, cu), N = WIDE[wide]
    ends = [128, 384, 640, 1000]
    M, K = ends[-1], 200
    x = poisoned(rnd(M, K, seed=1))
    w = rnd(len(ends) * N, K, scale=K ** -0.5, seed=2)
    b = rnd(N, seed=3)

    def run(bn, cta_pair):
        g = Guard((M, N))
        ops.linear(x, w, bias=b, out=g.out, block_n=bn, cta_pair=cta_pair, row_groups=ends)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(lambda: run(bw, cw))
    assert same_bits(out, run(bu, cu)[0])
    for gi, (r0, r1) in enumerate(zip([0] + ends[:-1], ends)):
        ref = x[r0:r1].double() @ w[gi * N:(gi + 1) * N].double().t() + b.double()
        check(out[r0:r1], ref, K_GEMM, what=f"{wide} weight plane {gi}")


@pytest.mark.parametrize("N", [576, 704])
def test_geglu_partial_last_unit(ops, L, N):
    """GEGLU runs on 160-wide units: N = 576 ends in a unit of 96 valid columns, N = 704 in one of 64."""
    M, K = 300, 136
    x = poisoned(rnd(M, K, seed=1))
    w, b = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)

    def run():
        g = Guard((M, N // 2))
        ops.linear(x, w, bias=b, out=g.out, epilogue=L.EPI_GEGLU)
        torch.cuda.synchronize()
        assert g.intact()
        return [g.out.clone()]

    out, = twice(run)
    h = x.double() @ w.double().t() + b.double()
    check(out, h[:, 0::2] * torch.nn.functional.gelu(h[:, 1::2]), K_GEMM, what=f"GEGLU N={N}")


def test_dependent_chain_in_cuda_graph(ops):
    """y1 = x W1^T, y2 = y1 W2^T + y1[:, :N2], y3 = silu(y2 W3^T): each GEMM reads the previous one's output, launched
    with programmatic dependent launch; a captured graph replayed on new input equals eager launches bit for bit."""
    M, K, N1, N2, N3 = 4100, 320, 640, 256, 320
    x = rnd(M, K, seed=1)
    w1, w2, w3 = rnd(N1, K, scale=K ** -0.5, seed=2), rnd(N2, N1, scale=N1 ** -0.5, seed=3), rnd(N3, N2, scale=N2 ** -0.5, seed=4)
    from omg_b200 import _lib as L
    y1 = torch.empty(M, N1, dtype=torch.float16, device="cuda")
    y2 = torch.empty(M, N2, dtype=torch.float16, device="cuda")
    y3 = torch.empty(M, N3, dtype=torch.float16, device="cuda")

    def chain():
        ops.linear(x, w1, out=y1, block_n=256)
        ops.linear(y1, w2, residual=y1[:, :N2], out=y2, block_n=128)
        ops.linear(y2, w3, out=y3, epilogue=L.EPI_SILU, block_n=320)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()  # warm-up: module load and function attributes outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        chain()
    x.copy_(rnd(M, K, seed=9))
    graph.replay()
    torch.cuda.synchronize()
    got = [t.clone() for t in (y1, y2, y3)]
    for t in (y1, y2, y3):
        t.fill_(float("nan"))
    chain()
    torch.cuda.synchronize()
    for a, b in zip(got, (y1, y2, y3)):
        assert same_bits(a, b)
    r1 = (x.double() @ w1.double().t()).half().double()
    check(y1, r1, K_GEMM, what="chain y1")
