"""omg_attention_relpos (SAM ViT attention with decomposed relative-position bias) through the C ABI against a float64
restatement of segment_anything's Attention / window_partition (oracle/sam_vit.py) computed on the GPU from the same fp16
qkv, tables and biases the kernel reads.  Every case runs twice and must be bit-identical; outputs sit in NaN guard
buffers and operands in NaN-poisoned ones (helpers of test_kernel_edges_gpu.py)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_edges_gpu import Guard, check, poisoned, same_bits, twice  # noqa: E402

pytestmark = pytest.mark.gpu

# Per-element k (|out - ref| <= 4 u |ref| + k u rms(ref), u = 2^-11), worst value measured on an NVIDIA H100 80GB HBM3 at
# a 400 W power limit beside it.
K_RELPOS = 4.0    # measured 2.44 (B = 2, head_dim 80, global 64 x 64)


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


def _rnd(shape, scale, g):
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


def _nan_rows(t, extra=8):
    """t [n, ...] as the first rows of a NaN buffer with `extra` more rows (tables) / elements (bias vectors)."""
    buf = torch.full((t.shape[0] + extra,) + tuple(t.shape[1:]), float("nan"), dtype=t.dtype, device="cuda")
    buf[extra // 2:extra // 2 + t.shape[0]].copy_(t)
    return buf[extra // 2:extra // 2 + t.shape[0]]


def relpos_reference(qkv, H, W, heads, hd, th, tw, window, bias, scale=None):
    """float64 (B, H*W, C): segment_anything Attention after qkv, with window_partition's padding made of qkv(0) = bias
    (scale None: head_dim^-0.5)."""
    from oracle.sam_vit import attention_core, window_unpartition
    B, C = qkv.shape[0], heads * hd
    x = qkv.double().view(B, H, W, 3 * C)
    if window:
        Hp, Wp = -(-H // window) * window, -(-W // window) * window
        full = bias.double().view(1, 1, 1, 3 * C).expand(B, Hp, Wp, 3 * C).clone()
        full[:, :H, :W] = x
        wins = full.view(B, Hp // window, window, Wp // window, window, 3 * C).permute(0, 1, 3, 2, 4, 5)
        y = attention_core(wins.reshape(-1, window, window, 3 * C), heads, th.double(), tw.double(), scale)
        y = window_unpartition(y, window, (Hp, Wp), (H, W))
    else:
        y = attention_core(x, heads, th.double(), tw.double(), scale)
    return y.reshape(B, H * W, C)


def make_case(B, H, W, heads, hd, window, seed=0, table_scale=0.15):
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = heads * hd
    S_h, S_w = (window, window) if window else (H, W)
    qkv = _rnd((B, H * W, 3 * C), 1.0, g)
    bias = _rnd((3 * C,), 1.0, g)
    th, tw = _rnd((2 * S_h - 1, hd), table_scale, g), _rnd((2 * S_w - 1, hd), table_scale, g)
    return qkv, bias, th, tw


def run_case(ops, B, H, W, heads, hd, window, seed=0, what=""):
    qkv, bias, th, tw = make_case(B, H, W, heads, hd, window, seed)
    C = heads * hd
    ref = relpos_reference(qkv, H, W, heads, hd, th, tw, window, bias)
    q_in = poisoned(qkv, rows=16)
    th_in, tw_in = _nan_rows(th), _nan_rows(tw)
    kb, vb = _nan_rows(bias[C:2 * C].contiguous()), _nan_rows(bias[2 * C:].contiguous())

    def run():
        g = Guard((B, H * W, C))
        ops.attention_relpos(q_in, H, W, heads, hd, th_in, tw_in, window=window, k_bias=kb, v_bias=vb, out=g.out)
        assert g.intact(), f"{what}: write outside the output"
        return [g.out.clone()]

    out, = twice(run)
    check(out, ref, K_RELPOS, what=what)
    return out


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("window", [0, 14])
def test_relpos_sam_grid(ops, hd, window):
    """The 64 x 64 SAM token grid: global attention (tables of 127 rows), and 14 x 14 windows (padding 6 on both axes)."""
    run_case(ops, 1, 64, 64, 2, hd, window, seed=hd + window, what=f"hd {hd} window {window}")


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("H,W,window", [(20, 31, 14), (9, 13, 5), (9, 13, 0), (3, 64, 0), (14, 14, 14), (30, 17, 7)])
def test_relpos_small_grids_padded_unevenly(ops, hd, H, W, window):
    """Padding 8 / 11, 1 / 2 and 5 / 4 on the two axes; global grids narrower and shorter than a key block."""
    run_case(ops, 1, H, W, 3, hd, window, seed=H * W + window, what=f"hd {hd} {H}x{W} window {window}")


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("window", [0, 14])
def test_relpos_batch_position_does_not_change_bits(ops, hd, window):
    H = W = 64 if window == 0 else 40
    out = run_case(ops, 2, H, W, 2, hd, window, seed=7, what=f"B=2 hd {hd} window {window}")
    qkv, bias, th, tw = make_case(2, H, W, 2, hd, window, seed=7)
    C = 2 * hd
    kb, vb = bias[C:2 * C].contiguous(), bias[2 * C:].contiguous()
    swapped = ops.attention_relpos(qkv.flip(0).contiguous(), H, W, 2, hd, th, tw, window=window, k_bias=kb, v_bias=vb)
    single = ops.attention_relpos(qkv[1:].contiguous(), H, W, 2, hd, th, tw, window=window, k_bias=kb, v_bias=vb)
    assert same_bits(swapped.flip(0), out)
    assert same_bits(single[0], out[1])


def test_relpos_column_offsets_and_launch_plan(ops):
    """q / k / v windows at non-default columns of a wider row, out at a column offset; one launch per call, and a
    recorded plan replays the same bits."""
    from omg_b200 import _lib as L
    H, W, heads, hd, window = 20, 20, 2, 80, 14
    qkv, bias, th, tw = make_case(1, H, W, heads, hd, window, seed=3)
    C = heads * hd
    ref = relpos_reference(qkv, H, W, heads, hd, th, tw, window, bias)
    wide = torch.zeros(1, H * W, 3 * C + 32, dtype=torch.float16, device="cuda")
    wide[..., 8:8 + C] = qkv[..., 2 * C:]              # v first, then q, then k
    wide[..., 16 + C:16 + 2 * C] = qkv[..., :C]
    wide[..., 24 + 2 * C:24 + 3 * C] = qkv[..., C:2 * C]
    out = torch.full((1, H * W, C + 16), float("nan"), dtype=torch.float16, device="cuda")
    kw = dict(window=window, k_bias=bias[C:2 * C].contiguous(), v_bias=bias[2 * C:].contiguous(), out=out,
              q_col0=16 + C, k_col0=24 + 2 * C, v_col0=8, out_col0=16)
    n0 = L.launch_count()
    ops.attention_relpos(wide, H, W, heads, hd, th, tw, **kw)
    assert L.launch_count() - n0 == 1
    check(out[..., 16:], ref, K_RELPOS, what="column offsets")
    first = out[..., 16:].clone()
    plan = ops.LaunchPlan()
    with plan:
        ops.attention_relpos(wide, H, W, heads, hd, th, tw, **kw)
    assert len(plan) == 1
    out.fill_(0)
    plan.run()
    torch.cuda.synchronize()
    assert same_bits(out[..., 16:], first)
    assert torch.equal(out[..., :16], torch.zeros_like(out[..., :16]))   # columns before out_col0 are not written
