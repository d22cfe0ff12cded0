"""Residual staged in shared memory by TMA (fp16 GEMMs without activations or fp32 twins) against the epilogue's global
loads, bit for bit.

The staged path runs whenever the residual's base is 16 B aligned.  A copy of the same residual whose base sits 8 B off
that alignment cannot be described by a tensor map, so the same launch on it runs the register path: that is the
reference every case is compared with.  Cases run in place (out = residual) as the UNet's transformer blocks and
ResBlocks do, with row statistics out:
* unit widths 64 / 128 / 160 and block_n 256 / 320, with N tails and a partial last m-tile;
* conv grids with W not a power of two and an odd batch (pixels outside the image in every tile row), time-embedding
  row vector and GroupNorm column statistics;
* per-CTA unit counts of 0, 1, odd and even (launches of 1, 131, 132, 263, 264, 265 units on a 132-SM H100);
* per-stream weight planes (the residual's columns carry no plane offset);
* three GEMMs, each adding the previous one's output, with programmatic dependent launch in a CUDA graph.
"""
import os
import subprocess
import sys

import pytest
import torch

from test_kernel_edges_gpu import K_GEMM, check, poisoned, rnd, same_bits, twice  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


def off16(t):
    """A contiguous copy of t in a NaN buffer, its base 8 B past a 16 B boundary (no tensor map can describe it)."""
    buf = torch.full((t.numel() + 8,), float("nan"), dtype=t.dtype, device=t.device)
    v = buf[4:4 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 8
    return v


def aligned(t):
    v = torch.empty_like(t, memory_format=torch.contiguous_format)
    v.copy_(t)
    assert v.data_ptr() % 16 == 0
    return v


# block_n -> N with a partial last unit (320 needs N % 320 == 0)
WIDTHS = {64: 224, 128: 352, 160: 224, 256: 288, 320: 640}


@pytest.mark.parametrize("bn", list(WIDTHS))
def test_inplace_linear_row_statistics(ops, bn):
    N = WIDTHS[bn]
    M, K = 641, 264
    x = poisoned(rnd(M, K, seed=1))
    w, b, r = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3), rnd(M, N, seed=4)
    parts = (4 if bn == 320 else 2) * ((N + bn - 1) // bn)

    def run(h):
        st = torch.full((parts, M, 2), float("nan"), device="cuda")
        ops.linear(x, w, bias=b, residual=h, out=h, block_n=bn, stats_out=st)
        torch.cuda.synchronize()
        return [h.clone(), st]

    staged = twice(lambda: run(aligned(r)))
    reg = run(off16(r))
    for a, u in zip(staged, reg):
        assert same_bits(a, u)
    check(staged[0], x.double() @ w.double().t() + b.double() + r.double(), K_GEMM, what=f"in-place residual bn={bn}")


@pytest.mark.parametrize("bn", list(WIDTHS))
def test_inplace_conv_grid_rowvec_colstats(ops, bn):
    N = WIDTHS[bn]
    B, H, W, Cin = 3, 12, 20, 40                   # 20 wide: 32 x 4 tiles, 12 columns of every tile row off the image
    x = poisoned(rnd(B, H, W, Cin, seed=1))
    wt = rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    wp = ops.pack_conv3x3_weight(wt)
    bias, temb, res = rnd(N, seed=3), rnd(B, N, seed=4), rnd(B, H, W, N, seed=5)

    def run(h):
        cs = torch.full((B, ops.colstats_blocks(W, H), N, 2), float("nan"), device="cuda")
        ops.conv3x3(x, wp, bias=bias, rowvec=temb, residual=h, out=h, block_n=bn, colstats=cs)
        torch.cuda.synchronize()
        return [h.clone(), cs]

    staged = twice(lambda: run(aligned(res)))
    reg = run(off16(res))
    for a, u in zip(staged, reg):
        assert same_bits(a, u)
    ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), bias.double(), padding=1) \
        + temb.double()[:, :, None, None] + res.double().permute(0, 3, 1, 2)
    check(staged[0].permute(0, 3, 1, 2), ref, K_GEMM, what=f"in-place conv residual bn={bn}")


@pytest.mark.parametrize("k_blocks", [1, 3])
@pytest.mark.parametrize("units", [1, 131, 132, 263, 264, 265])
@pytest.mark.parametrize("bn", [64, 160])
def test_unit_counts(ops, bn, units, k_blocks):
    N, K = bn, 64 * k_blocks
    M = 128 * (units - 1) + 77
    x = poisoned(rnd(M, K, seed=units))
    w, b, r = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3), rnd(M, N, seed=4)

    def run(h):
        st = torch.full((2, M, 2), float("nan"), device="cuda")
        ops.linear(x, w, bias=b, residual=h, out=h, block_n=bn, stats_out=st)
        torch.cuda.synchronize()
        return [h.clone(), st]

    staged = run(aligned(r))
    reg = run(off16(r))
    for a, u in zip(staged, reg):
        assert same_bits(a, u)
    check(staged[0], x.double() @ w.double().t() + b.double() + r.double(), K_GEMM, what=f"{units} units of {bn} x {K}")


@pytest.mark.parametrize("bn", [64, 160, 320])
def test_weight_planes(ops, bn):
    """Two streams with weight planes of their own; the residual is read at the output's columns."""
    N = 640 if bn == 320 else 320
    ends = [384, 1000]
    M, K = ends[-1], 200
    x = poisoned(rnd(M, K, seed=1))
    w = rnd(len(ends) * N, K, scale=K ** -0.5, seed=2)
    b, r = rnd(N, seed=3), rnd(M, N, seed=4)

    def run(h):
        ops.linear(x, w, bias=b, residual=h, out=h, block_n=bn, row_groups=ends)
        torch.cuda.synchronize()
        return [h.clone()]

    staged, = run(aligned(r))
    assert same_bits(staged, run(off16(r))[0])
    for gi, (r0, r1) in enumerate(zip([0] + ends[:-1], ends)):
        ref = x[r0:r1].double() @ w[gi * N:(gi + 1) * N].double().t() + b.double() + r[r0:r1].double()
        check(staged[r0:r1], ref, K_GEMM, what=f"weight plane {gi}, bn={bn}")


_CHAIN = r"""
import sys
import torch
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
from omg_b200 import ops
from test_kernel_edges_gpu import rnd, same_bits
from test_gemm_residual_smem_gpu import aligned, off16

M, N = 4100, 640
x = rnd(M, N, seed=1)
ws = [rnd(N, N, scale=N ** -0.5, seed=2 + i) for i in range(3)]
bns = (160, 128, 320)


def chain(ys):
    # y0 <- x W0^T + y0 (in place), y_i = x W_i^T + y_(i-1): each GEMM adds the previous one's output
    ops.linear(x, ws[0], residual=ys[0], out=ys[0], block_n=bns[0])
    for i in (1, 2):
        ops.linear(x, ws[i], residual=ys[i - 1], out=ys[i], block_n=bns[i])


def fresh(make):
    return [make(rnd(M, N, seed=10 + i)) for i in range(3)]


s = torch.cuda.Stream()
ys = fresh(aligned)
s.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(s):
    chain(ys)  # warm-up: module load and function attributes outside the capture
torch.cuda.current_stream().wait_stream(s)
torch.cuda.synchronize()
graph = torch.cuda.CUDAGraph()
with torch.cuda.graph(graph):
    chain(ys)
init = fresh(lambda t: t)
for y, t in zip(ys, init):
    y.copy_(t)
graph.replay()
torch.cuda.synchronize()
eager = fresh(aligned)
chain(eager)
reg = fresh(off16)
chain(reg)
torch.cuda.synchronize()
for a, b, c in zip(ys, eager, reg):
    assert same_bits(a, b), "graph replay differs from eager launches"
    assert same_bits(a, c), "staged residual differs from the register path"
ref = init[0].double()
for w in ws:
    ref = ref + x.double() @ w.double().t()
rel = ((ys[2].double() - ref).norm() / ref.norm()).item()
assert rel < 2e-3, rel
print("chain ok", rel)
"""


def test_dependent_chain_in_cuda_graph():
    """Each GEMM's residual is the previous one's output, launched with programmatic dependent launch (OMG_PDL=1, read
    once per process, hence a process of its own): the staged residual must be read after the previous kernel's
    writes.  Graph replay, eager launches and the register path agree bit for bit."""
    env = dict(os.environ, OMG_PDL="1")
    p = subprocess.run([sys.executable, "-c", _CHAIN, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
