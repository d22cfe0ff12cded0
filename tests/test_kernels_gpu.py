"""GPU parity of each hand-written kernel (through the C ABI) against a plain fp32 torch restatement of the same
op on the same fp16 inputs.  Tolerances: relative L2 <= 2e-3 (fp16 storage of the result, fp32 accumulation)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel(a, b):
    a = a.float()
    b = b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


@pytest.fixture(scope="module")
def ops():
    from omg_b200 import ops
    return ops


@pytest.mark.parametrize("M,N,K,bn", [(256, 256, 128, 0), (4096, 1280, 1280, 0), (1000, 640, 320, 0),
                                      (308, 2560, 2048, 0), (4, 1280, 2816, 0), (512, 320, 960, 160),
                                      (512, 320, 960, 64), (2048, 1920, 640, 128), (2048, 1280, 640, 256),
                                      (4096, 1280, 1280, 320), (512, 640, 1024, 320), (300, 320, 640, 320),
                                      (2176, 960, 192, 320)])
def test_linear(ops, M, N, K, bn):
    x, w, b = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    r = rnd(M, N, seed=4)
    out = ops.linear(x, w, bias=b, residual=r, block_n=bn)
    ref = x.float() @ w.float().t() + b.float() + r.float()
    torch.cuda.synchronize()
    assert rel(out, ref) < 2e-3


def test_linear_silu_and_lora(ops):
    M, N, K, R = 1024, 640, 640, 32
    x, w = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2)
    a, bw = rnd(R, K, scale=K ** -0.5, seed=3), rnd(N, R, scale=0.1 * R ** -0.5, seed=4)
    t = ops.linear(x, a)  # t = A x   [M, R]
    wcat = torch.cat([w, 0.8 * bw], dim=1).contiguous()  # [N, K + R]
    out = ops.linear(x, wcat, extra=[(t, K)])
    ref = x.float() @ w.float().t() + (t.float() @ (0.8 * bw).float().t())
    assert rel(out, ref) < 2e-3
    out2 = ops.linear(x, w, epilogue=2)
    assert rel(out2, F.silu(x.float() @ w.float().t())) < 2e-3


def test_geglu(ops):
    M, C = 1024, 640
    x = rnd(M, C, seed=1)
    w, b = rnd(8 * C, C, scale=C ** -0.5, seed=2), rnd(8 * C, seed=3)
    wi, bi = ops.pack_geglu_weight(w, b)
    out = ops.linear(x, wi, bias=bi, epilogue=1)
    h = x.float() @ w.float().t() + b.float()
    ref = h[:, :4 * C] * F.gelu(h[:, 4 * C:])
    assert out.shape == (M, 4 * C)
    assert rel(out, ref) < 2e-3


@pytest.mark.parametrize("B,H,W,Cin,N", [(2, 32, 32, 128, 256), (1, 64, 64, 320, 320), (2, 16, 16, 640, 1280),
                                         (1, 128, 128, 64, 128), (1, 24, 40, 64, 64)])
def test_conv3x3(ops, B, H, W, Cin, N):
    x = rnd(B, H, W, Cin, seed=1)
    w = rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    b = rnd(N, seed=3)
    temb = rnd(B, N, seed=4)
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(w), bias=b, rowvec=temb)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b.float(), padding=1) + temb.float()[:, :, None, None]
    assert rel(out.permute(0, 3, 1, 2), ref) < 2e-3


def test_conv3x3_shortcut_residual(ops):
    B, H, W, C1, C2, N = 2, 32, 32, 128, 64, 256
    h = rnd(B, H, W, N, seed=1)
    xa, xb = rnd(B, H, W, C1, seed=2), rnd(B, H, W, C2, seed=3)
    w = rnd(N, N, 3, 3, scale=(9 * N) ** -0.5, seed=4)
    ws = rnd(N, C1 + C2, scale=(C1 + C2) ** -0.5, seed=5)
    b = rnd(N, seed=6)
    wcat = torch.cat([ops.pack_conv3x3_weight(w), ws], dim=1).contiguous()
    out = ops.conv3x3(h, wcat, bias=b, shortcut=[(xa, 9 * N), (xb, 9 * N + C1)])
    x = torch.cat([xa, xb], dim=3).float().permute(0, 3, 1, 2)
    ref = F.conv2d(h.float().permute(0, 3, 1, 2), w.float(), b.float(), padding=1) + \
        F.conv2d(x, ws.float()[:, :, None, None])
    assert rel(out.permute(0, 3, 1, 2), ref) < 2e-3
    # identity shortcut as residual
    r = rnd(B, H, W, N, seed=7)
    out2 = ops.conv3x3(h, ops.pack_conv3x3_weight(w), bias=b, residual=r)
    ref2 = F.conv2d(h.float().permute(0, 3, 1, 2), w.float(), b.float(), padding=1) + r.float().permute(0, 3, 1, 2)
    assert rel(out2.permute(0, 3, 1, 2), ref2) < 2e-3


def test_conv_small_channels(ops):
    # conv_in (4 -> 320, stored as 8 channels) and conv_out (320 -> 4, stored as 8)
    B, H, W = 2, 32, 32
    x = torch.zeros(B, H, W, 8, device="cuda", dtype=torch.float16)
    x[..., :4] = rnd(B, H, W, 4, seed=1)
    w = rnd(320, 4, 3, 3, scale=36 ** -0.5, seed=2)
    w8 = torch.zeros(320, 8, 3, 3, device="cuda", dtype=torch.float16)
    w8[:, :4] = w
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(w8))
    ref = F.conv2d(x[..., :4].float().permute(0, 3, 1, 2), w.float(), padding=1)
    assert rel(out.permute(0, 3, 1, 2), ref) < 2e-3
    y = rnd(B, H, W, 320, seed=3)
    wo = rnd(4, 320, 3, 3, scale=2880 ** -0.5, seed=4)
    wo8 = torch.zeros(8, 320, 3, 3, device="cuda", dtype=torch.float16)
    wo8[:4] = wo
    out = ops.conv3x3(y, ops.pack_conv3x3_weight(wo8))
    ref = F.conv2d(y.float().permute(0, 3, 1, 2), wo.float(), padding=1)
    assert rel(out[..., :4].permute(0, 3, 1, 2), ref) < 2e-3
    assert out[..., 4:].abs().max().item() == 0.0


@pytest.mark.parametrize("B,H,W,C", [(2, 32, 32, 128), (1, 64, 64, 320)])
def test_conv_down_up(ops, B, H, W, C):
    x = rnd(B, H, W, C, seed=1)
    w = rnd(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=2)
    b = rnd(C, seed=3)
    wp = ops.pack_conv3x3_weight(w)
    xn = x.float().permute(0, 3, 1, 2)
    out = ops.conv3x3_s2(x, wp, bias=b)
    ref = F.conv2d(xn, w.float(), b.float(), stride=2, padding=1)
    assert rel(out.permute(0, 3, 1, 2), ref) < 2e-3
    out = ops.upsample2x_conv3x3(x, wp, bias=b)
    ref = F.conv2d(F.interpolate(xn, scale_factor=2.0, mode="nearest"), w.float(), b.float(), padding=1)
    assert rel(out.permute(0, 3, 1, 2), ref) < 2e-3


def _attn_ref(q, k, v, heads, scale):
    B, Nq, Cc = q.shape
    d = Cc // heads
    qh = q.float().view(B, Nq, heads, d).transpose(1, 2)
    kh = k.float().view(B, -1, heads, d).transpose(1, 2)
    vh = v.float().view(B, -1, heads, d).transpose(1, 2)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1)
    return (p @ vh).transpose(1, 2).reshape(B, Nq, Cc)


@pytest.mark.parametrize("B,N,heads", [(2, 1024, 10), (1, 4096, 5), (2, 256, 20), (1, 384, 2)])
def test_self_attention(ops, B, N, heads):
    Cc = heads * 64
    qkv = rnd(B, N, 3 * Cc, seed=1)
    out = torch.empty(B, N, Cc, device="cuda", dtype=torch.float16)
    items = [(b, b, b, b) for b in range(B)]
    ops.attention(qkv, qkv, qkv, out, heads, N, N, items, q_col0=0, k_col0=Cc, v_col0=2 * Cc)
    ref = _attn_ref(qkv[..., :Cc], qkv[..., Cc:2 * Cc], qkv[..., 2 * Cc:], heads, 0.125)
    assert rel(out, ref) < 2e-3


@pytest.mark.parametrize("n_q,n_kv,gain", [(256, 200, 1.0), (130, 321, 1.0), (512, 640, 2.5), (128, 129, 2.5),
                                            (384, 1024, 3.0), (121, 121, 1.0), (200, 57, 1.0), (64, 63, 2.5)])
def test_attention_block_edges(ops, n_q, n_kv, gain):
    """Self-attention kernel edges: odd block counts, a partial last block, n_q != n_kv, and score ranges large enough
    that the lazy O rescale fires; with and without `accumulate`."""
    heads = 3
    Cc = heads * 64
    q = rnd(2, n_q, Cc, seed=11) * gain
    kv = rnd(2, n_kv, 2 * Cc, seed=12)
    kv[..., :Cc] *= gain
    out = torch.empty(2, n_q, Cc, device="cuda", dtype=torch.float16)
    items = [(0, 1, 1, 0), (1, 0, 0, 1)]  # out row 0 <- Q,K of row 1 with V of row 0, and vice versa
    ops.attention(q, kv, kv, out, heads, n_q, n_kv, items, k_col0=0, v_col0=Cc)
    ref = _attn_ref(q[[1, 0]], kv[[1, 0]][..., :Cc], kv[..., Cc:], heads, 0.125)
    assert rel(out, ref) < 2e-3
    base = rnd(2, n_q, Cc, seed=13)
    out2 = base.clone()
    ops.attention(q, kv, kv, out2, heads, n_q, n_kv, items, k_col0=0, v_col0=Cc, out_weight=0.5, accumulate=True)
    assert rel(out2, base.float() + 0.5 * ref) < 2e-3


@pytest.mark.parametrize("B,n_q,n_kv,heads", [(4, 1024, 77, 20), (2, 4096, 77, 10), (2, 200, 16, 3), (1, 128, 128, 7),
                                              (2, 300, 100, 5), (1, 64, 5, 1), (8, 1024, 77, 20), (2, 256, 57, 3),
                                              (1, 130, 121, 2), (1, 100, 59, 1)])
def test_cross_attention_head_group_kernel(ops, B, n_q, n_kv, heads):
    """Cross-attention kernel (one key block, a CTA walks a group of heads): text keys (77), IP tokens (16), padded key
    counts, ragged query tiles, head counts with a tail group; remapped rows and the accumulate / out_weight term."""
    Cc = heads * 64
    q = rnd(B, n_q, Cc, seed=21)
    kv = rnd(B + 1, n_kv, 2 * Cc, seed=22)
    out = torch.empty(B, n_q, Cc, device="cuda", dtype=torch.float16)
    items = [(b, (b + 1) % B, b + 1, b) for b in range(B)]
    ops.attention(q, kv, kv, out, heads, n_q, n_kv, items, k_col0=0, v_col0=Cc)
    qi = [(b + 1) % B for b in range(B)]
    ref = _attn_ref(q[qi], kv[[b + 1 for b in range(B)]][..., :Cc], kv[:B][..., Cc:], heads, 0.125)
    assert rel(out, ref) < 2e-3
    base = rnd(B, n_q, Cc, seed=23)
    out2 = base.clone()
    ops.attention(q, kv, kv, out2, heads, n_q, n_kv, items, k_col0=0, v_col0=Cc, out_weight=0.8, accumulate=True)
    assert rel(out2, base.float() + 0.8 * ref) < 2e-3


@pytest.mark.parametrize("B,N,n_kv,heads", [(4, 1024, 1024, 20), (2, 2048, 320, 8), (3, 640, 200, 5), (1, 4096, 4096, 3)])
def test_self_attention_persistent_many_tiles(ops, B, N, n_kv, heads):
    """The persistent self-attention kernel: 2 x #SM CTAs walk several tiles each as one stream of KV blocks (barrier
    phases run across tile boundaries, Q double-buffered, O handed back through o_free): more tiles than CTAs, odd block
    counts per tile, a partial last block, remapped batch rows and the accumulate term."""
    Cc = heads * 64
    q = rnd(B, N, Cc, seed=41) * 1.5
    kv = rnd(B, n_kv, 2 * Cc, seed=42)
    kv[..., :Cc] *= 1.5
    out = torch.empty(B, N, Cc, device="cuda", dtype=torch.float16)
    items = [(b, (b + 1) % B, (b + 1) % B, b) for b in range(B)]
    ops.attention(q, kv, kv, out, heads, N, n_kv, items, k_col0=0, v_col0=Cc)
    idx = [(b + 1) % B for b in range(B)]
    ref = _attn_ref(q[idx], kv[idx][..., :Cc], kv[..., Cc:], heads, 0.125)
    assert rel(out, ref) < 2e-3
    base = rnd(B, N, Cc, seed=43)
    out2 = base.clone()
    ops.attention(q, kv, kv, out2, heads, N, n_kv, items, k_col0=0, v_col0=Cc, out_weight=0.7, accumulate=True)
    assert rel(out2, base.float() + 0.7 * ref) < 2e-3


def test_attention_p2p_remap_and_cross(ops):
    B, N, heads, Lk = 4, 1024, 10, 77
    Cc = heads * 64
    qkv = rnd(B, N, 3 * Cc, seed=1)
    out = torch.empty(B, N, Cc, device="cuda", dtype=torch.float16)
    # rows (u0,u1,c0,c1): c1 takes Q,K from c0 and V from itself (replace_self_attention)
    items = [(0, 0, 0, 0), (1, 1, 1, 1), (2, 2, 2, 2), (3, 2, 2, 3)]
    ops.attention(qkv, qkv, qkv, out, heads, N, N, items, q_col0=0, k_col0=Cc, v_col0=2 * Cc)
    q, k, v = qkv[..., :Cc], qkv[..., Cc:2 * Cc], qkv[..., 2 * Cc:]
    ref = _attn_ref(q[[0, 1, 2, 2]], k[[0, 1, 2, 2]], v, heads, 0.125)
    assert rel(out, ref) < 2e-3
    # cross attention: 77 text keys + 16 image keys, decoupled: txt + 0.8 * ip
    qx = rnd(B, N, Cc, seed=2)
    kv = rnd(B, Lk, 2 * Cc, seed=3)
    kvip = rnd(B, 16, 2 * Cc, seed=4)
    it = [(b, b, b, b) for b in range(B)]
    ops.attention(qx, kv, kv, out, heads, N, Lk, it, k_col0=0, v_col0=Cc)
    ref_t = _attn_ref(qx, kv[..., :Cc], kv[..., Cc:], heads, 0.125)
    assert rel(out, ref_t) < 2e-3
    ops.attention(qx, kvip, kvip, out, heads, N, 16, it, k_col0=0, v_col0=Cc, out_weight=0.8, accumulate=True)
    ref_ip = _attn_ref(qx, kvip[..., :Cc], kvip[..., Cc:], heads, 0.125)
    assert rel(out, ref_t + 0.8 * ref_ip) < 2e-3


@pytest.mark.parametrize("B,HW,C1,C2,silu", [(2, 1024, 320, 0, 1), (2, 4096, 640, 320, 1), (1, 256, 1280, 1280, 1),
                                             (3, 1024, 640, 0, 0)])
def test_groupnorm(ops, B, HW, C1, C2, silu):
    x1 = rnd(B, HW, C1, seed=1) + 0.5
    x2 = rnd(B, HW, C2, scale=2.0, seed=2) if C2 else None
    Cc = C1 + C2
    g, b = rnd(Cc, seed=3) + 1, rnd(Cc, seed=4)
    out = ops.groupnorm(x1, g, b, 1e-5, silu, x2=x2)
    x = x1 if x2 is None else torch.cat([x1, x2], dim=2)
    ref = F.group_norm(x.float().transpose(1, 2), 32, g.float(), b.float(), 1e-5).transpose(1, 2)
    if silu:
        ref = F.silu(ref)
    assert rel(out, ref) < 2e-3


@pytest.mark.parametrize("rows,C", [(4096, 640), (1000, 1280), (77, 2048)])
def test_layernorm(ops, rows, C):
    x = rnd(rows, C, seed=1) * 3 + 1
    g, b = rnd(C, seed=2) + 1, rnd(C, seed=3)
    out = ops.layernorm(x, g, b)
    ref = F.layer_norm(x.float(), (C,), g.float(), b.float(), 1e-5)
    assert rel(out, ref) < 2e-3


def test_fuse_step(ops):
    H = W = 64
    HW = H * W
    g = torch.Generator(device="cuda").manual_seed(0)
    nm = torch.zeros(4, HW, 8, device="cuda", dtype=torch.float16)
    nm[..., :4] = torch.randn(4, HW, 4, generator=g, device="cuda").half()
    ncs, masks = [], []
    for k in range(2):
        n = torch.zeros(2, HW, 8, device="cuda", dtype=torch.float16)
        n[..., :4] = torch.randn(2, HW, 4, generator=g, device="cuda").half()
        ncs.append(n)
        m = torch.zeros(H, W, device="cuda")
        m[8:40, 4 + 20 * k:36 + 20 * k] = 1.0  # overlapping rectangles
        masks.append(m.reshape(-1).contiguous())
    lat = torch.randn(2, HW, 4, generator=g, device="cuda") * 10
    lat0 = lat.clone()
    nxt = torch.empty(4, HW, 8, device="cuda", dtype=torch.float16)
    nxc = torch.empty(2, HW, 8, device="cuda", dtype=torch.float16)
    sig, sign, gs = 5.0, 4.2, 7.5
    ops.fuse_step(nm, ncs, masks, gs, sig, sign, lat, nxt, nxc)
    # restatement of lora_pipeline.py:568-615
    noise = nm[..., :4].float()
    U = ((masks[0] == 1) | (masks[1] == 1)).float()[None, :, None]
    edit = torch.stack([noise[1], noise[3]])
    new = edit * (1 - U)
    for k in range(2):
        new = new + ncs[k][..., :4].float() * masks[k][None, :, None]
    noise = noise.clone()
    noise[1], noise[3] = new[0], new[1]
    eps = noise[:2] + gs * (noise[2:] - noise[:2])
    ref = lat0 + eps * (sign - sig)
    assert rel(lat, ref) < 1e-6
    sc = ref / math.sqrt(sign * sign + 1)
    assert rel(nxt[..., :4], torch.cat([sc, sc])) < 1e-3
    assert rel(nxc[..., :4], torch.stack([sc[1], sc[1]])) < 1e-3
    assert nxt[..., 4:].abs().max().item() == 0


def test_ctx_mix(ops):
    ctx = rnd(2, 77, 2048, seed=1)
    coef = torch.rand(77, 77, device="cuda")
    out = ops.ctx_mix(ctx, coef)
    ref = torch.einsum("wn,bnc->bwc", coef, ctx.float())
    assert rel(out, ref) < 2e-3


@pytest.mark.parametrize("M,C,N,geglu", [(4096, 1280, 3840, False), (2048, 640, 640, False), (1024, 640, 5120, True),
                                         (300, 320, 320, False)])
def test_layernorm_folded_into_gemm_pair(ops, M, C, N, geglu):
    """producer GEMM (residual add) emits row statistics; consumer GEMM applies LayerNorm in its epilogue."""
    from omg_b200 import _lib as L
    o, wo, bo = rnd(M, C, seed=1), rnd(C, C, scale=C ** -0.5, seed=2), rnd(C, seed=3)
    h0 = rnd(M, C, seed=4) * 2 + 0.7                        # residual stream with a non-zero mean
    gam, bet = rnd(C, seed=5) * 0.2 + 1, rnd(C, seed=6) * 0.3
    w, b = rnd(N, C, scale=C ** -0.5, seed=7), rnd(N, seed=8)
    parts = ops.gemm_plan(C, L.EPI_NONE, M)[1]
    stats = torch.zeros(parts, M, 2, device="cuda")
    h = h0.clone()
    ops.linear(o, wo, bias=bo, residual=h, out=h, stats_out=stats)
    href = o.float() @ wo.float().t() + bo.float() + h0.float()
    assert rel(h, href) < 2e-3
    s = stats.sum(0)
    assert torch.allclose(s[:, 0], href.sum(1), rtol=2e-3, atol=2e-2)
    if geglu:
        w, b = ops.pack_geglu_weight(w, b)
    wl = (w.float() * gam.float()[None, :]).half()
    c1 = wl.float().sum(1).contiguous()
    c2 = (w.float() @ bet.float() + b.float()).contiguous()
    out = ops.linear(h, wl, epilogue=1 if geglu else 0, ln=(stats, parts, M, 0, C, 1e-5, c1, c2, [M]))
    x = F.layer_norm(h.float(), (C,), gam.float(), bet.float(), 1e-5)
    y = x @ w.float().t() + b.float()
    if geglu:
        y = y[:, 0::2] * F.gelu(y[:, 1::2])
    assert rel(out, y) < 3e-3


@pytest.mark.parametrize("M,N,K", [(4096, 1280, 1280), (2176, 640, 512), (384, 320, 128), (8192, 1280, 5120)])
def test_linear_tall_tiles(ops, M, N, K):
    """256 x 160 tiles in one CTA (two 128-row sub-tiles share each weight tile); odd m-tile counts included."""
    x, w, b = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    r = rnd(M, N, seed=4)
    out = ops.linear(x, w, bias=b, residual=r, block_n=160, cta_pair=3)
    ref = x.float() @ w.float().t() + b.float() + r.float()
    assert rel(out, ref) < 2e-3
    assert torch.equal(out, ops.linear(x, w, bias=b, residual=r, block_n=160, cta_pair=1))


def test_tall_tiles_conv_rowvec_and_stats(ops):
    from omg_b200 import _lib as L
    B, H, W, Cin, Nc = 3, 16, 16, 128, 320          # 256 pixels per image: the two sub-tiles of a tall tile differ in image
    xi = rnd(B, H, W, Cin, seed=7)
    wc = rnd(Nc, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=8)
    bc, temb = rnd(Nc, seed=9), rnd(B, Nc, seed=10)
    out = ops.conv3x3(xi, ops.pack_conv3x3_weight(wc), bias=bc, rowvec=temb, block_n=160, cta_pair=3)
    ref = F.conv2d(xi.float().permute(0, 3, 1, 2), wc.float(), bc.float(), padding=1) + temb.float()[:, :, None, None]
    assert rel(out.permute(0, 3, 1, 2), ref) < 2e-3
    # row statistics emitted by a tall-tile producer feed a folded LayerNorm
    M, C, N = 1024, 320, 640
    o, wo = rnd(M, C, seed=1), rnd(C, C, scale=C ** -0.5, seed=2)
    h0 = rnd(M, C, seed=4) + 0.5
    parts = ops.gemm_plan(C, L.EPI_NONE, M)[1]
    stats = torch.zeros(parts, M, 2, device="cuda")
    h = h0.clone()
    ops.linear(o, wo, residual=h, out=h, stats_out=stats, block_n=160, cta_pair=3)
    href = o.float() @ wo.float().t() + h0.float()
    s = stats.sum(0)
    assert torch.allclose(s[:, 0], href.sum(1), rtol=2e-3, atol=2e-2)
    assert torch.allclose(s[:, 1], (href * href).sum(1), rtol=3e-3, atol=2e-2)


def test_fuse_step_matches_the_reference_fusion_statements(ops):
    """omg_fuse_step against tests/golden/fusion.pt: the output of the reference's own fusion + guidance statements
    (lora_pipeline.py:568-612, executed from the method's AST): one concept without a mask (skipped), two overlapping
    masks, a non-binary stripe in one mask.  The Euler update on top is x + eps * (sigma_next - sigma)."""
    import os
    from omg_b200.pipelines import _binary_latent_mask
    d = torch.load(os.path.join(os.path.dirname(__file__), "golden", "fusion.pt"))
    n_in = d["noise_pred_in"]
    h, w = n_in.shape[2], n_in.shape[3]
    HW = h * w

    def nhwc8(x):
        t = torch.zeros(x.shape[0], HW, 8, device="cuda", dtype=torch.float16)
        t[..., :4] = x.permute(0, 2, 3, 1).reshape(x.shape[0], HW, 4).half().cuda()
        return t

    active = [k for k, m in enumerate(d["masks"]) if m is not None]
    assert active == [0, 2]
    nm = nhwc8(n_in)
    ncs = [nhwc8(d["region_noise"][k]) for k in active]
    masks = [_binary_latent_mask(d["masks"][k], h, w, "cuda") for k in active]
    lat0 = (torch.randn(2, HW, 4, generator=torch.Generator().manual_seed(1)) * 10).cuda()
    lat = lat0.clone()
    nxt = torch.empty(4, HW, 8, device="cuda", dtype=torch.float16)
    nxc = torch.empty(2, HW, 8, device="cuda", dtype=torch.float16)
    sig, sign = 5.0, 4.2
    ops.fuse_step(nm, ncs, masks, d["guidance_scale"], sig, sign, lat, nxt, nxc)
    eps = d["noise_after_cfg"].permute(0, 2, 3, 1).reshape(2, HW, 4).cuda()
    ref = lat0 + eps * (sign - sig)
    assert rel(lat, ref) < 1e-5


def _gn_ref(x, gamma, beta, eps, silu):
    y = F.group_norm(x.float().permute(0, 3, 1, 2), 32, gamma.float(), beta.float(), eps)
    return F.silu(y) if silu else y


@pytest.mark.parametrize("B,H,W,C1,C2", [(2, 32, 32, 640, 320), (3, 16, 16, 320, 0), (1, 8, 8, 1280, 1280), (2, 4, 4, 64, 32)])
def test_groupnorm_from_producer_column_statistics(ops, B, H, W, C1, C2):
    """GroupNorm whose statistics come out of the producing conv / GEMM epilogues (per-channel partials of the
    fp16-rounded outputs): convs with tall, single and partial tiles, the group boundaries of the concatenation
    straddling the two sources (640 | 320 -> 30 channels per group), against torch.group_norm of the stored tensors."""
    cin = 64
    x = rnd(B, H, W, cin, seed=1)
    w1 = rnd(C1, cin, 3, 3, scale=(9 * cin) ** -0.5, seed=2)
    y1 = torch.empty(B, H, W, C1, device="cuda", dtype=torch.float16)
    p1 = torch.full((B, ops.colstats_blocks(W, H), C1, 2), float("nan"), device="cuda")
    ops.conv3x3(x, ops.pack_conv3x3_weight(w1), bias=rnd(C1, seed=3), out=y1, colstats=p1)
    tot = p1.sum(1)
    assert torch.allclose(tot[..., 0], y1.float().sum((1, 2)), rtol=1e-3, atol=5e-2)
    assert torch.allclose(tot[..., 1], (y1.float() ** 2).sum((1, 2)), rtol=1e-3, atol=5e-2)
    # the stand-alone statistics kernel produces the same totals (and, for full tiles, the same blocks)
    p1b = ops.colstats(y1)
    assert torch.allclose(p1b.sum(1), tot, rtol=1e-4, atol=1e-2)
    y2 = p2 = None
    if C2:
        w2 = rnd(C2, cin, scale=cin ** -0.5, seed=4)
        y2 = torch.empty(B, H, W, C2, device="cuda", dtype=torch.float16)
        if (H * W) % 128 == 0:  # token-major producer (Transformer2DModel.proj_out): [B*HW, C] GEMM, per-image partials
            p2 = torch.full((B, ops.colstats_blocks(H * W, 1), C2, 2), float("nan"), device="cuda")
            ops.linear(x.view(-1, cin), w2, out=y2.view(-1, C2), residual=rnd(B * H * W, C2, seed=5), colstats=p2)
        else:
            ops.linear(x.view(-1, cin), w2, out=y2.view(-1, C2))
            p2 = ops.colstats(y2)
    C = C1 + C2
    gamma, beta = rnd(C, seed=6) * 0.2 + 1.0, rnd(C, seed=7) * 0.2
    for silu in (0, 1):
        out = ops.groupnorm_apply(y1, p1, gamma, beta, 1e-5, silu, x2=y2, part2=p2)
        xin = y1 if y2 is None else torch.cat([y1, y2], dim=-1)
        ref = _gn_ref(xin, gamma, beta, 1e-5, silu)
        assert rel(out.permute(0, 3, 1, 2), ref) < 2e-3
        old = ops.groupnorm(y1, gamma, beta, 1e-5, silu, x2=y2)   # statistics-pass variant: same result
        assert rel(out, old.float()) < 1e-3


def test_column_statistics_of_down_and_up_convs(ops):
    B, H, W, C = 2, 16, 16, 128
    x = rnd(B, H, W, C, seed=1)
    wd = ops.pack_conv3x3_weight(rnd(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=2))
    d = torch.empty(B, H // 2, W // 2, C, device="cuda", dtype=torch.float16)
    pd = torch.full((B, ops.colstats_blocks(W // 2, H // 2), C, 2), float("nan"), device="cuda")
    ops.conv3x3_s2(x, wd, bias=rnd(C, seed=3), out=d, colstats=pd)
    assert torch.allclose(pd.sum(1)[..., 0], d.float().sum((1, 2)), rtol=1e-3, atol=5e-2)
    assert torch.allclose(pd.sum(1)[..., 1], (d.float() ** 2).sum((1, 2)), rtol=1e-3, atol=5e-2)
    u = torch.empty(B, 2 * H, 2 * W, C, device="cuda", dtype=torch.float16)
    pu = torch.full((B, 4 * ops.colstats_blocks(W, H), C, 2), float("nan"), device="cuda")
    ops.upsample2x_conv3x3(x, wd, bias=rnd(C, seed=4), out=u, colstats=pu)
    assert torch.allclose(pu.sum(1)[..., 0], u.float().sum((1, 2)), rtol=1e-3, atol=5e-2)
    assert torch.allclose(pu.sum(1)[..., 1], (u.float() ** 2).sum((1, 2)), rtol=1e-3, atol=5e-2)


def test_pair320_tiles_conv_residual_stats_and_lora(ops):
    """128 x 320 tiles (two N = 160 wgmmas per K step, one 320-column accumulator): a conv with time-embedding
    row vector and residual, GroupNorm column statistics and LayerNorm row statistics out of the same epilogue, an
    un-merged LoRA K-segment against the second weight matrix."""
    from omg_b200 import _lib as L
    B, H, W, Cin, N = 3, 16, 16, 128, 640
    x = rnd(B, H, W, Cin, seed=1)
    w = rnd(N, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    bias, temb, res = rnd(N, seed=3), rnd(B, N, seed=4), rnd(B, H, W, N, seed=5)
    part = torch.full((B, ops.colstats_blocks(W, H), N, 2), float("nan"), device="cuda")
    out = ops.conv3x3(x, ops.pack_conv3x3_weight(w), bias=bias, rowvec=temb, residual=res, block_n=320, colstats=part)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias.float(), padding=1) + temb.float()[:, :, None, None] \
        + res.float().permute(0, 3, 1, 2)
    assert rel(out.permute(0, 3, 1, 2), ref) < 2e-3
    assert torch.allclose(part.sum(1)[..., 0], out.float().sum((1, 2)), rtol=1e-3, atol=5e-2)
    # row statistics (LayerNorm fold producer) + LoRA segment, default tile choice
    M, C = 1024, 640
    o, wo = rnd(M, C, seed=6), rnd(C, C, scale=C ** -0.5, seed=7)
    t, b2 = rnd(M, 32, seed=8), rnd(C, 32, scale=0.1, seed=9)
    h0 = rnd(M, C, seed=10)
    parts = ops.gemm_plan(C, L.EPI_NONE, M)[1]
    stats = torch.full((parts, M, 2), float("nan"), device="cuda")
    h = h0.clone()
    ops.linear(o, wo, residual=h, out=h, stats_out=stats, lora=(t, b2))
    href = o.float() @ wo.float().t() + t.float() @ b2.float().t() + h0.float()
    assert rel(h, href) < 2e-3
    sm = stats.sum(0)
    assert torch.allclose(sm[:, 0], href.sum(1), rtol=2e-3, atol=3e-2)
    assert torch.allclose(sm[:, 1], (href * href).sum(1), rtol=3e-3, atol=3e-2)
