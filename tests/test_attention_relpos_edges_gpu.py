"""Kernel edges of omg_attention_relpos (SAM ViT attention with decomposed relative-position bias) through the C ABI,
against the float64 restatement of segment_anything's Attention / window_partition (relpos_reference of
test_sam_vit_gpu.py) computed on the GPU one head at a time from the same fp16 values the kernel reads.

The kernel's geometry comes from the window and the grid: a CTA holds byq = min(128 / Ww, Wh) window rows of queries,
a key block byk = min(64 / Ww, Wh) window rows, and the query / key slots past Ww * byq and Ww * byk are dead.  Padded
keys are zero in shared memory and carry scale q.k_bias in their logit and v_bias in the output (weighted by their
probability mass).  The cases below run every regime of that geometry: windows of 1 to 64 (byk from 64 down to 1, key
blocks with and without dead slots), windows larger than the grid, windowed grids larger than SAM's 64 x 64, degenerate
global grids, the ViT-B/L/H head layouts, logits dominated by the rel-pos bias or by the padded keys, scales other than
head_dim^-0.5, and head windows inside wider rows.

* every element is bounded,  |out - ref| <= 4 u |ref| + k u rms(ref)  (u = 2^-11), with one k for the whole file;
* qkv is read from a NaN-poisoned buffer with extra token rows per image (batch stride != H W ld), the tables and
  k_bias / v_bias from NaN-padded buffers, and the output sits in a NaN guard buffer that must stay intact;
* every case runs twice and must be bit-identical.  `pytest -s` prints the k each case needs."""
import functools
import os
import sys
import zlib

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_edges_gpu import Guard, check, poisoned, same_bits, twice  # noqa: E402
from test_sam_vit_gpu import _nan_rows, make_case, relpos_reference  # noqa: E402

pytestmark = pytest.mark.gpu

# Per-element k, with the worst value the cases need on an NVIDIA H100 80GB HBM3 at a 700 W power limit beside it.
K_RELPOS_EDGE = 7.0   # measured 3.46 (head_dim 80, 64 x 64 grid in one window of 64)
LOG2E = 1.4426950408889634


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


def _seed(what):
    return zlib.crc32(what.encode())


def reference(qkv, H, W, heads, hd, th, tw, window, bias, scale=None):
    """relpos_reference one head at a time: a global 64 x 64 score tensor is 128 MiB per head and image in float64."""
    C = heads * hd

    def head(t, h):  # q, k, v columns of head h out of [..., 3C]
        return torch.cat([t[..., s * C + h * hd:s * C + (h + 1) * hd] for s in range(3)], -1)

    return torch.cat([relpos_reference(head(qkv, h), H, W, 1, hd, th, tw, window, head(bias, h), scale)
                      for h in range(heads)], -1)


def _extra_rows(t, rows=16):
    """t [B, T, ld] as the first T rows per image of a NaN buffer [B, T + rows, ld]: the row stride stays ld."""
    buf = torch.full((t.shape[0], t.shape[1] + rows, t.shape[2]), float("nan"), dtype=t.dtype, device="cuda")
    v = buf[:, :t.shape[1]]
    v.copy_(t)
    return v


def run_edge(ops, B, H, W, heads, hd, window, what, case=None, scale=None, table_scale=0.15, wide_rows=True):
    """One guarded, twice-run, checked case; returns (out, ref, call) with call(out=...) launching it again.
    wide_rows: qkv rows are NaN-padded on both sides (ld = 3C + 16); otherwise ld = 3C and only token rows are added."""
    if case is None:
        case = make_case(B, H, W, heads, hd, window, seed=_seed(what), table_scale=table_scale)
    qkv, bias, th, tw = case
    C = heads * hd
    ref = reference(qkv, H, W, heads, hd, th, tw, window, bias, scale)
    q_in = poisoned(qkv, rows=16) if wide_rows else _extra_rows(qkv)
    assert q_in.stride(0) != H * W * q_in.stride(1)
    th_in, tw_in = _nan_rows(th), _nan_rows(tw)
    kb, vb = _nan_rows(bias[C:2 * C].contiguous()), _nan_rows(bias[2 * C:].contiguous())
    call = functools.partial(ops.attention_relpos, q_in, H, W, heads, hd, th_in, tw_in, window=window, k_bias=kb,
                             v_bias=vb, scale=scale)

    def run():
        g = Guard((B, H * W, C))
        call(out=g.out)
        assert g.intact(), f"{what}: write outside the output"
        return [g.out.clone()]

    out, = twice(run)
    check(out, ref, K_RELPOS_EDGE, what=what)
    return out, ref, call


# ------------------------------------------------------------------------------------------------------ window sweep
SWEEP_WINDOWS = [1, 2, 7, 8, 14, 16, 31, 32, 33, 40, 63, 64]
# one odd grid per window, padded by a different amount on each axis (window 1 pads nothing)
ODD_GRID = {w: (37, 45) for w in SWEEP_WINDOWS}
ODD_GRID.update({2: (37, 46), 8: (37, 46)})


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("window", SWEEP_WINDOWS)
@pytest.mark.parametrize("grid", ["64x64", "odd"])
def test_window_sweep(ops, hd, window, grid):
    """byk = min(64 / Ww, Wh) window rows per key block: the whole window in one block up to window 8 (window 1: one
    token per group), 4 and 2 rows at 14 - 32, one row at 33 - 64 (64 - Ww dead key slots); powers of two fill the query
    and key tiles exactly.  On 64 x 64, windows 7, 14, 31, 33, 40 and 63 pad the grid (63: three of the four groups are
    mostly padding); on the odd grid every window but 1 pads both axes."""
    H, W = (64, 64) if grid == "64x64" else ODD_GRID[window]
    run_edge(ops, 2, H, W, 2, hd, window, what=f"hd {hd} {H}x{W} window {window}")


# ---------------------------------------------------------------------------------------------- window >= the grid
def _padded_keys_dominate(case, heads, hd, scale):
    """Add a common direction u (|u| = 4) to every query of a head and make k_bias = a u with scale a |u|^2 = 6: a padded
    key's logit is 6 +- 1.5 against about 0 +- 2 for a real key, so the padded keys hold nearly all the probability mass
    and the output is close to v_bias."""
    qkv, bias, th, tw = case
    C = heads * hd
    g = torch.Generator(device="cuda").manual_seed(11)
    u = torch.randn(heads, hd, generator=g, device="cuda")
    u = (4.0 * u / u.norm(dim=1, keepdim=True)).reshape(C)
    qkv = qkv.clone()
    qkv[..., :C] = (qkv[..., :C].float() + u).half()
    bias = bias.clone()
    bias[C:2 * C] = (6.0 / (16.0 * scale) * u).half()
    return qkv, bias, th, tw


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("H,W,window", [(5, 9, 14), (20, 20, 40)])
@pytest.mark.parametrize("padded_keys", ["random", "dominant"])
def test_window_larger_than_the_grid(ops, hd, H, W, window, padded_keys):
    """One group per image that is more than half padding (151 of 196, 1200 of 1600 keys), so scale q.k_bias and the
    padded probability mass lp weigh heavily; 'dominant' makes the padded keys carry the maximum (lp ~ l)."""
    heads, B = 2, 2
    what = f"hd {hd} {H}x{W} window {window} padded keys {padded_keys}"
    case = make_case(B, H, W, heads, hd, window, seed=_seed(what))
    if padded_keys == "dominant":
        case = _padded_keys_dominate(case, heads, hd, hd ** -0.5)
    _, ref, _ = run_edge(ops, B, H, W, heads, hd, window, what=what, case=case)
    if padded_keys == "dominant":
        vb = case[1][2 * heads * hd:].double()
        assert ((ref - vb).norm() / ref.norm()).item() < 0.1, "the padded keys do not dominate"


# ------------------------------------------------------------------------------------ windowed grids beyond 64 x 64
@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("H,W,window", [(100, 37, 14), (130, 9, 64)])
def test_windowed_grid_larger_than_sam(ops, hd, H, W, window):
    """8 x 3 groups of 14 (padding 12 / 5) and 3 x 1 groups of 64 (padding 62 / 55): group origins up to 128 rows down
    the grid, padding on the last row and column of groups only."""
    run_edge(ops, 2, H, W, 2, hd, window, what=f"hd {hd} {H}x{W} window {window}")


# ------------------------------------------------------------------------------------------- degenerate global grids
@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("B,H,W", [(2, 1, 1), (2, 1, 64), (2, 64, 1), (2, 1, 33), (2, 47, 33), (3, 64, 64)])
def test_global_degenerate_grids(ops, hd, B, H, W):
    """Tables of one row (1 x W, H x 1), a single column of 64 tokens in one query tile and one key block, a 47 x 33
    grid of 33-wide key blocks, and three images with batch strides of the padded buffers."""
    run_edge(ops, B, H, W, 3, hd, 0, what=f"hd {hd} B={B} global {H}x{W}")


# ------------------------------------------------------------------------------------------- real ViT head layouts
@pytest.mark.parametrize("window", [0, 14])
@pytest.mark.parametrize("kind,heads,hd", [("vit_b", 12, 64), ("vit_l", 16, 64), ("vit_h", 16, 80)])
def test_vit_head_layouts(ops, kind, heads, hd, window):
    """The qkv Linear's output of ViT-B / L / H as it is (ld 2304 / 3072 / 3840, head offsets up to 15 x 80 + 2 x 1280)
    for a global and a window-14 block, two images."""
    run_edge(ops, 2, 64, 64, heads, hd, window, what=f"{kind} window {window} ld {3 * heads * hd}", wide_rows=False)


# --------------------------------------------------------------------------------------------- bias-dominated logits
@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("window", [0, 14])
def test_bias_dominated_logits(ops, hd, window):
    """Tables large enough that q.R reaches about +-30 in the log2 domain, so the running maximum of a query row moves
    between key blocks because of bias_h + bias_w alone."""
    what = f"hd {hd} 64x64 window {window} bias-dominated"
    case = make_case(2, 64, 64, 2, hd, window, seed=_seed(what), table_scale=4.6 / hd ** 0.5)
    qkv, _, th, tw = case
    q = qkv[..., :hd].double()                                 # head 0
    peak = max((q @ t.double().t()).abs().max().item() for t in (th, tw)) * LOG2E
    assert peak > 20, f"q.R reaches only {peak:.1f} in the log2 domain"
    run_edge(ops, 2, 64, 64, 2, hd, window, what=f"{what} (|q.R| log2 e up to {peak:.0f})", case=case)


# --------------------------------------------------------------------------------------------------------- scale
@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("scale", [0.3, 0.02])
def test_scale_other_than_head_dim(ops, hd, scale):
    """The softmax scale multiplies q.k and q.k_bias, never the rel-pos terms; padded 37 x 45 grid in windows of 14."""
    run_edge(ops, 2, 37, 45, 2, hd, 14, what=f"hd {hd} 37x45 window 14 scale {scale}", scale=scale)


# ------------------------------------------------------------------------------------------------- head isolation
@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("H,W,window", [(30, 17, 7), (47, 33, 0)])
def test_heads_inside_a_wider_row(ops, hd, H, W, window):
    """Heads 1 - 4 of a six-head qkv row, written at out_col0 = hd of a six-head NaN output row: no column outside
    [hd, 5 hd) and no row past the grid may change.  k_bias / v_bias are the four heads' slices of NaN-padded vectors."""
    B, heads, launched = 2, 6, 4
    what = f"hd {hd} {H}x{W} window {window} heads 1-4 of 6"
    qkv, bias, th, tw = make_case(B, H, W, heads, hd, window, seed=_seed(what))
    C = heads * hd
    ref = reference(qkv, H, W, heads, hd, th, tw, window, bias)[..., hd:(1 + launched) * hd]
    q_in = poisoned(qkv, rows=16)
    th_in, tw_in = _nan_rows(th), _nan_rows(tw)
    kb = _nan_rows(bias[C + hd:C + (1 + launched) * hd].contiguous())
    vb = _nan_rows(bias[2 * C + hd:2 * C + (1 + launched) * hd].contiguous())

    def run():
        buf = torch.full((B, H * W + 8, C), float("nan"), dtype=torch.float16, device="cuda")
        out = buf[:, :H * W]
        ops.attention_relpos(q_in, H, W, launched, hd, th_in, tw_in, window=window, k_bias=kb, v_bias=vb, out=out,
                             q_col0=hd, k_col0=C + hd, v_col0=2 * C + hd, out_col0=hd)
        outside = torch.cat([buf[:, :, :hd], buf[:, :, (1 + launched) * hd:]], -1)
        assert outside.isnan().all() and buf[:, H * W:].isnan().all(), f"{what}: write outside heads 1 - 4"
        return [out[..., hd:(1 + launched) * hd].clone()]

    out, = twice(run)
    check(out, ref, K_RELPOS_EDGE, what=what)


# ------------------------------------------------------------------------------------------------ launch-plan replay
@pytest.mark.parametrize("B,H,W,heads,hd,window", [(2, 37, 45, 2, 80, 33), (2, 130, 9, 2, 64, 64),
                                                    (2, 64, 64, 16, 80, 14)])
def test_launch_plan_replays_the_same_bits(ops, B, H, W, heads, hd, window):
    """A recorded plan of one launch writes exactly the eager launch's bits, and nothing outside the output."""
    what = f"plan hd {hd} {H}x{W} window {window} heads {heads}"
    out, _, call = run_edge(ops, B, H, W, heads, hd, window, what=what)
    g = Guard((B, H * W, heads * hd))
    plan = ops.LaunchPlan()
    with plan:
        call(out=g.out)
    assert len(plan) == 1
    g.out.fill_(float("nan"))
    plan.run()
    torch.cuda.synchronize()
    assert same_bits(g.out, out), f"{what}: replay differs from the eager launch"
    assert g.intact(), f"{what}: replay wrote outside the output"
